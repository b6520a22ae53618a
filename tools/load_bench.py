"""Loading a safetensors file onto the GPU with and without verification: mxd_tree_load_file against what a user does
today.

Workloads, written to /dev/shm (so every row reads the same page-cache-resident bytes) from data generated on the GPU:
  llama  the Llama-3-8B layout in fp16 (tests/checkpoint_fixtures.llama_shapes): 291 tensors, about 16 GB
  moe    an MoE-shaped file: 32 layers x 42 experts x 3 projections of 512 x 1024 fp16 = 4,032 tensors of 1 MiB, about
         4.2 GB; it exposes the per-copy submit cost of one H2D copy per tensor piece
The files are written tensor by tensor in safetensors_layout's format (the tensor order safetensors.torch.save_file
uses), so the host never holds the whole state dict.

Rows, in GB/s of file bytes (host clock around calls that return after the device work is done):
  a  Engine.tree_digest_file: the same pinned-ring staging, hashing only
  b  checkpoint.load_safetensors: file -> one CUDA tensor per entry, tree digest of the bytes that landed there
  c  safetensors.torch.load_file(device="cuda:0"), then checkpoint.tree_digest_safetensors: verified loading today
  d  safetensors.torch.load_file(device="cuda:0") alone, no verification
Rows b and c must give row a's root.  Every row is warmed up once; then 3 repeats, rows alternated, best kept.
Targets (llama): b >= 0.9 a and b > c.  The moe numbers are reported, not gated.

    python tools/load_bench.py [--layouts llama,moe] [--dir /dev/shm] [--out result.json]
"""
import argparse
import json
import math
import os
import shutil
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import modelx_b200  # noqa: E402
from modelx_b200.checkpoint import load_safetensors, safetensors_layout, tree_digest_safetensors  # noqa: E402
from tests.checkpoint_fixtures import llama_shapes  # noqa: E402

SEED = 0x6D6F64656C78
REPEATS = 3


def smi(field):
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={field}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or out.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unavailable ({e})"


def moe_shapes(layers=32, experts=42):
    return [(f"model.layers.{i}.mlp.experts.{e}.{w}.weight", (512, 1024))
            for i in range(layers) for e in range(experts) for w in ("w1", "w2", "w3")]


def write_file(eng, path, shapes):
    """A safetensors file of fp16 tensors filled by dev_gen_fill, written one tensor at a time."""
    metas = {name: torch.empty(shape, dtype=torch.float16, device="meta") for name, shape in shapes}
    header, order = safetensors_layout(metas, {"format": "pt"})
    index = {name: i for i, (name, _) in enumerate(shapes)}
    st = torch.cuda.current_stream().cuda_stream
    with open(path, "wb") as f:
        f.write(header)
        for name in order:
            t = torch.empty(metas[name].shape, dtype=torch.float16, device="cuda")
            eng.dev_gen_fill(0, t.data_ptr(), 0, t.numel() * 2, SEED + index[name], st)
            f.write(t.reshape(-1).view(torch.uint8).cpu().numpy().tobytes())
    return header


def run_layout(eng, name, shapes, directory):
    import safetensors.torch as st
    path = os.path.join(directory, f"load_bench_{name}.safetensors")
    need = sum(2 * math.prod(shape) for _, shape in shapes) + (64 << 20)
    if shutil.disk_usage(directory).free < need:
        raise SystemExit(f"{directory} has {shutil.disk_usage(directory).free / 1e9:.1f} GB free, {name} needs {need / 1e9:.1f} GB")
    try:
        header = write_file(eng, path, shapes)
        size = os.path.getsize(path)
        roots = {}

        def row_a():
            roots["a"] = eng.tree_digest_file(path)[1]

        def row_b():
            tensors, _, roots["b"], _ = load_safetensors(eng, path, "cuda:0")
            del tensors

        def row_c():
            tensors = st.load_file(path, device="cuda:0")
            roots["c"] = tree_digest_safetensors(eng, header, tensors)[1]
            del tensors

        def row_d():
            tensors = st.load_file(path, device="cuda:0")
            torch.cuda.synchronize()
            del tensors

        rows = {"a": row_a, "b": row_b, "c": row_c, "d": row_d}
        for fn in rows.values():
            fn()
        assert roots["b"] == roots["a"] and roots["c"] == roots["a"], "roots differ between rows"
        rates = {k: [] for k in rows}
        for _ in range(REPEATS):
            for key, fn in rows.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                rates[key].append(size / (time.perf_counter() - t0) / 1e9)
                assert key == "d" or roots[key] == roots["a"], f"row {key}: root differs from row a"
        return dict(layout=name, tensors=len(shapes), bytes=size, root=modelx_b200.digest_string(roots["a"]),
                    rates_gbps={k: [round(r, 2) for r in v] for k, v in rates.items()})
    finally:
        if os.path.exists(path):
            os.unlink(path)
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--layouts", default="llama,moe")
    ap.add_argument("--dir", default="/dev/shm")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "load_bench measures on a CUDA device; there is nothing to measure without one"
    torch.cuda.set_device(0)
    card = dict(name=smi("name"), power_limit=smi("power.limit"), sm_clock=smi("clocks.sm"),
                max_sm_clock=smi("clocks.max.sm"), usable_cpus=len(os.sched_getaffinity(0)))
    print("card:", json.dumps(card))
    layouts = {"llama": llama_shapes(), "moe": moe_shapes()}
    results = []
    with modelx_b200.Engine(devices=[0]) as eng:
        for name in args.layouts.split(","):
            r = run_layout(eng, name, layouts[name], args.dir)
            best = {k: max(v) for k, v in r["rates_gbps"].items()}
            if name == "llama":
                r["targets"] = {"b >= 0.9 a": best["b"] >= 0.9 * best["a"], "b > c": best["b"] > best["c"]}
            print(f"--- {name}: {r['bytes'] / 1e9:.2f} GB, {r['tensors']} tensors, root {r['root']}")
            for k, v in r["rates_gbps"].items():
                print(f"  {k}  " + "  ".join(f"{x:6.2f}" for x in v) + f"   GB/s   ({max(v) / best['a']:.3f} x a)")
            if "targets" in r:
                print("  targets:", json.dumps(r["targets"]))
            results.append(r)
    line = dict(card=card, results=results)
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
