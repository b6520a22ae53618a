"""Tree digest of a safetensors checkpoint resident in HBM: mxd_dev_tree_digest_extents against the contiguous path.

Workload: a synthetic Llama-3-8B-shaped fp16 state dict (291 tensors, about 16 GB, filled by dev_gen_fill), and the
same structure scaled to about 32 GB (a contiguous copy for the baseline still fits in 80 GB).  Rows, in GB/s of blob:
  a  mxd_dev_tree_digest on one contiguous 16-byte-aligned buffer of the same size (the reference rate)
  b  the extents path with that buffer as one extent
  c  the safetensors layout (header + 291 tensors as extents), header length = 0 mod 16
  d  the same with the header length = 8 mod 16
  e  an odd-length int8 tensor in front of the others: every later tensor byte sits at an odd offset in its leaf
  f  copy-then-digest: D2D gather of header + tensors into one buffer, then mxd_dev_tree_digest
  g  mxd_dev_tree_digest on a contiguous buffer at an address = 8 mod 16
Rows a, b, c, f and g hash the same bytes and must give the same root; d and e are checked against a gathered copy of
their own bytes.  CUDA events, 3 warm-up and 5 timed steps per row, rows alternated over 3 repeats.

    python tools/extents_bench.py [--scales 16,32] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import modelx_b200  # noqa: E402
from tests.checkpoint_fixtures import header_in_order, llama_shapes  # noqa: E402

TP = (8 << 20, 16 << 10, 8)
SEED = 0x6D6F64656C78
SCALES = {16: dict(), 32: dict(layers=68)}          # layers=68: about 31.8 GB
WARMUP, STEPS, REPEATS = 3, 5, 3


def smi(field):
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={field}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or out.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unavailable ({e})"


def run_scale(eng, gb):
    st = torch.cuda.current_stream()
    sp = st.cuda_stream
    shapes = llama_shapes(**SCALES[gb])
    tensors = {}
    for i, (name, shape) in enumerate(shapes):
        t = torch.empty(shape, dtype=torch.float16, device="cuda")
        eng.dev_gen_fill(0, t.data_ptr(), 0, t.numel() * 2, SEED + i, sp)
        tensors[name] = t
    odd = torch.empty(4097 + 7, dtype=torch.int8, device="cuda")
    eng.dev_gen_fill(0, odd.data_ptr(), 0, odd.numel() // 8 * 8, SEED - 1, sp)
    tensors["odd.int8"] = odd[:4097]
    names = [n for n, _ in shapes]

    def spec(order):
        return [(n, "I8" if tensors[n].dtype == torch.int8 else "F16", tuple(tensors[n].shape),
                 tensors[n].numel() * tensors[n].element_size()) for n in order]

    layouts = {}
    for key, order, mod16 in (("c", names, 0), ("d", names, 8), ("e", ["odd.int8"] + names, 8)):
        header = header_in_order(spec(order), mod16)
        d_header = torch.frombuffer(bytearray(header), dtype=torch.uint8).to("cuda")
        ext = [(d_header.data_ptr(), len(header))] + [(tensors[n].data_ptr(), tensors[n].numel() * tensors[n].element_size())
                                                      for n in order]
        views = [d_header] + [tensors[n].reshape(-1).view(torch.uint8) for n in order]
        layouts[key] = dict(ext=ext, views=views, size=sum(n for _, n in ext), mod16=len(header) % 16)
    size = layouts["c"]["size"]
    assert layouts["e"]["size"] == max(lay["size"] for lay in layouts.values())
    buf = torch.empty(layouts["e"]["size"] + 16, dtype=torch.uint8, device="cuda")
    nch = -(-layouts["e"]["size"] // TP[0])
    out = torch.empty(nch * 32 + 32, dtype=torch.uint8, device="cuda")
    d_chunks, d_root = out.data_ptr(), out.data_ptr() + nch * 32

    def gather(lay, off):
        pos = off
        for v in lay["views"]:
            buf[pos:pos + v.numel()].copy_(v)
            pos += v.numel()

    def contiguous(off, n):
        eng.dev_tree_digest(0, buf.data_ptr() + off, n, TP, d_chunks, d_root, sp)

    def extents(ext):
        eng.dev_tree_digest_extents(0, ext, TP, d_chunks, d_root, sp)

    def result(n):
        torch.cuda.synchronize()
        k = -(-n // TP[0])
        return out[:k * 32].cpu().numpy().tobytes(), out[nch * 32:].cpu().numpy().tobytes()

    # ---- roots: every row against a gathered copy of the bytes it hashes --------------------------------------------
    roots = {}
    for key in ("c", "d", "e"):
        lay = layouts[key]
        gather(lay, 0)
        contiguous(0, lay["size"])
        want = result(lay["size"])
        extents(lay["ext"])
        assert result(lay["size"]) == want, f"row {key}: extents path differs from the gathered copy"
        roots[key] = want[1].hex()
    gather(layouts["c"], 8)
    contiguous(8, size)
    assert result(size)[1].hex() == roots["c"], "row g differs"
    gather(layouts["c"], 0)
    contiguous(0, size)
    assert result(size)[1].hex() == roots["c"], "row a differs"
    extents([(buf.data_ptr(), size)])
    assert result(size)[1].hex() == roots["c"], "row b differs"
    gather(layouts["c"], 0)
    contiguous(0, size)
    assert result(size)[1].hex() == roots["c"], "row f differs"

    rows = {
        "a": (size, lambda: contiguous(0, size)),
        "b": (size, lambda: extents([(buf.data_ptr(), size)])),
        "c": (size, lambda: extents(layouts["c"]["ext"])),
        "d": (layouts["d"]["size"], lambda: extents(layouts["d"]["ext"])),
        "e": (layouts["e"]["size"], lambda: extents(layouts["e"]["ext"])),
        "f": (size, lambda: (gather(layouts["c"], 0), contiguous(0, size))),
        "g": (size, lambda: contiguous(8, size)),
    }
    rates = {k: [] for k in rows}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(REPEATS):
        for key, (n, fn) in rows.items():
            for _ in range(WARMUP):
                fn()
            e0.record(st)
            for _ in range(STEPS):
                fn()
            e1.record(st)
            e1.synchronize()
            rates[key].append(STEPS * n / (e0.elapsed_time(e1) * 1e-3) / 1e9)
    res = dict(scale_gb=gb, tensors=len(shapes), bytes=size, header_mod16={k: v["mod16"] for k, v in layouts.items()},
               root_c=roots["c"], rates_gbps={k: [round(r, 1) for r in v] for k, v in rates.items()})
    del tensors, buf, out, layouts
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--scales", default="16,32")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "extents_bench measures on a CUDA device; there is nothing to measure without one"
    torch.cuda.set_device(0)
    card = dict(name=smi("name"), power_limit=smi("power.limit"), sm_clock=smi("clocks.sm"),
                max_sm_clock=smi("clocks.max.sm"))
    print("card:", json.dumps(card))
    results = []
    with modelx_b200.Engine(devices=[0]) as eng:
        for gb in (int(s) for s in args.scales.split(",")):
            r = run_scale(eng, gb)
            best = {k: max(v) for k, v in r["rates_gbps"].items()}
            a = best["a"]
            r["targets"] = {
                "c >= 0.9 a": best["c"] >= 0.9 * a, "d >= 0.9 a": best["d"] >= 0.9 * a, "e >= 0.8 a": best["e"] >= 0.8 * a,
                "b,c,d,e > f": all(best[k] > best["f"] for k in "bcde"),
            }
            print(f"--- {gb} GB: {r['bytes'] / 1e9:.2f} GB, {r['tensors']} tensors, header mod 16 {r['header_mod16']}")
            for k, v in r["rates_gbps"].items():
                print(f"  {k}  " + "  ".join(f"{x:7.1f}" for x in v) + f"   GB/s   ({max(v) / a:.3f} x a)")
            print("  targets:", json.dumps(r["targets"]))
            results.append(r)
    line = dict(card=card, results=results)
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(line, f, indent=1)


if __name__ == "__main__":
    main()
