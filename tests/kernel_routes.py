"""Kernel battery: every SHA-256 and tree-leaf kernel across its launch contract, compared bit for bit with hashlib.

One route per process, because the tuning knobs that select a kernel are read once, when the library loads:

    python -m tests.kernel_routes --route lanes --backend cuda

The worker sets the route's knobs itself (and clears any other MXD_TUNE_* knob) before it loads the library, runs the
battery, prints one JSON result line and exits non-zero on the first mismatch, naming the case.  On the CUDA backend the
battery runs under torch.profiler and the set of kernels that ran must be the one the route promises.  ``--backend
mock`` runs the same cases against the CPU test double (tests/mock_build.py) with numpy buffers standing in for device
memory: a rehearsal of the harness itself (case generation, canaries, neighbour flips), without the kernel check.

Not collected by pytest; tests/test_gpu_kernels.py runs it.
"""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import random
import re
import sys
import tempfile
import time

import numpy as np

PAIR = "k_sha256_chains_pair"
LANES12 = "k_sha256_lanes<12,64>"
LEAVES = "k_tree_leaves<false>"
LEAVES_FUSED = "k_tree_leaves<true>"
DEFAULT_SHA = frozenset({PAIR, "k_sha256_chains_coop<0>", LANES12})

_SMALL_OFF = {"MXD_TUNE_PAIR": "0", "MXD_TUNE_COOP": "0"}
_COOP = {"MXD_TUNE_PAIR": "0", "MXD_TUNE_COOP": "1000000000"}

# name -> (knobs, kernels the battery must run).  For the sha256 routes the set is every k_sha256_* kernel that ran;
# for the leaves routes it is every k_tree_leaves kernel (their tree levels above the leaves use the default dispatch).
# The fused routes also run k_tree_leaves<false>: fan-out 3 divides no power of 64, so nothing can be fused.
ROUTES = {
    "default": ({}, None),
    "pair": ({"MXD_TUNE_PAIR": "1000000000"}, {PAIR}),
    "coop0": (dict(_COOP), {"k_sha256_chains_coop<0>"}),
    "coop1": (dict(_COOP, MXD_TUNE_CHAIN="1"), {"k_sha256_chains_coop<1>"}),
    "coop2": (dict(_COOP, MXD_TUNE_CHAIN="2"), {"k_sha256_chains_coop<2>"}),
    "lanes": (dict(_SMALL_OFF), {LANES12}),
    "lanes_minb8": (dict(_SMALL_OFF, MXD_TUNE_MINB="8"), {"k_sha256_lanes<16,64>"}),
    "lanes_minb4": (dict(_SMALL_OFF, MXD_TUNE_MINB="4"), {"k_sha256_lanes<8,64>"}),
    "lanes_cta32": (dict(_SMALL_OFF, MXD_TUNE_CTA="32"), {"k_sha256_lanes<24,32>"}),
    "leaves_sched": ({"MXD_TUNE_LEAF_SCHED": "2"}, {LEAVES}),
    "leaves_fused": ({"MXD_TUNE_FUSE": "1"}, {LEAVES, LEAVES_FUSED}),
    "leaves_fused_sched": ({"MXD_TUNE_FUSE": "1", "MXD_TUNE_LEAF_SCHED": "2"}, {LEAVES, LEAVES_FUSED}),
}
LEAF_ROUTES = ("leaves_sched", "leaves_fused", "leaves_fused_sched")
BIG_STREAM_ROUTES = ("pair", "coop0", "lanes")   # the other variants share the length code of these three

LENGTHS = list(range(131)) + [64 * k + r for k in (1, 2, 3, 7, 16, 17) for r in (0, 1, 55, 56, 57, 63)] + [65_549, 1_048_631]
OFFSETS = list(range(16)) + [17, 4095]
BATCH_SIZES = (1, 15, 16, 17, 31, 32, 33, 63, 64, 65)
SEGS = (32, 64, 100, 256, 16_384, 16_392)
TAILS = (0, 1, 55, 56, 57, 63)
SEED = 0x6D6F64656C78

GUARD = np.array([(0xA5 ^ (7 * i)) & 0xFF for i in range(64)], dtype=np.uint8)
UNSET = 0x5A        # pre-fill of every digest slot; 32 bytes of it are not a digest anyone will meet


class Mismatch(Exception):
    def __init__(self, case, detail):
        super().__init__(f"{case}: {detail}")
        self.case = case


def sha(b) -> bytes:
    return hashlib.sha256(bytes(b)).digest()


def _align(x: int, a: int) -> int:
    return (x + a - 1) // a * a


# ---- memory the kernels read and write: torch tensors on the GPU, or numpy arrays for the test double -----------------
class _CudaBuf:
    def __init__(self, torch, n):
        self.torch = torch
        self.t = torch.empty(n + 256, dtype=torch.uint8, device="cuda")
        self.o = (-self.t.data_ptr()) % 256
        self.ptr = self.t.data_ptr() + self.o      # 256-byte aligned

    def put(self, off, arr):
        if len(arr):
            self.t[self.o + off:self.o + off + len(arr)].copy_(self.torch.from_numpy(np.ascontiguousarray(arr, dtype=np.uint8)))

    def get(self, off, n) -> bytes:
        return self.t[self.o + off:self.o + off + n].cpu().numpy().tobytes()


class _HostBuf:
    def __init__(self, n):
        self.a = np.zeros(n + 256, dtype=np.uint8)
        self.o = (-self.a.ctypes.data) % 256
        self.ptr = self.a.ctypes.data + self.o

    def put(self, off, arr):
        self.a[self.o + off:self.o + off + len(arr)] = arr

    def get(self, off, n) -> bytes:
        return self.a[self.o + off:self.o + off + n].tobytes()


class Out:
    """An output region with GUARD bytes on both sides, pre-filled with UNSET.  ptr = region start (lead bytes past a
    256-byte boundary, so 16-byte aligned for the default lead)."""

    def __init__(self, bat, nbytes, lead=64):
        self.n, self.lead = nbytes, lead
        self.buf = bat.alloc(lead + nbytes + 64)
        self.buf.put(0, np.concatenate([np.resize(GUARD, lead), np.full(nbytes, UNSET, np.uint8), GUARD]))
        self.ptr = self.buf.ptr + lead

    def take(self, case, slot=32) -> bytes:
        raw = self.buf.get(0, self.lead + self.n + 64)
        if raw[:self.lead] != np.resize(GUARD, self.lead).tobytes():
            raise Mismatch(case, "bytes before the output were written")
        if raw[-64:] != GUARD.tobytes():
            raise Mismatch(case, "bytes after the output were written")
        body = raw[self.lead:self.lead + self.n]
        if slot:
            for i in range(0, self.n, slot):
                if body[i:i + slot] == bytes([UNSET]) * slot:
                    raise Mismatch(case, f"output slot {i // slot} was not written")
        return body


def kernel_label(name: str):
    """'void mxd::(anonymous namespace)::k_sha256_lanes<12, 64>(mxd::MsgJob)' (or its mangled form) -> 'k_sha256_lanes<12,64>'"""
    m = re.search(r"(k_sha256_lanes|k_sha256_chains_coop|k_sha256_chains_pair|k_tree_leaves)", name)
    if not m:
        return None
    base, rest = m.group(1), name[m.end():]
    args = []
    if rest.startswith("<"):
        args = [a.strip() for a in rest[1:rest.index(">")].split(",")]
    elif rest.startswith("I"):                                  # Itanium mangling: ILi12ELi64EE, ILb0EE
        args = re.findall(r"L[ib](\d+)E", rest[:rest.find("EE") + 2])
    if base == "k_tree_leaves":
        args = ["true" if a in ("true", "1", "(bool)1") else "false" for a in args]
    return base + (f"<{','.join(args)}>" if args else "")


class Battery:
    def __init__(self, route, backend):
        self.route, self.backend = route, backend
        self.cases = 0
        self.kernels = set()
        self.big_stream_seconds = None
        import modelx_b200
        from tests.oracle_lib import Oracle
        self.orc = Oracle()
        if backend == "cuda":
            import torch
            assert torch.cuda.is_available(), "the cuda backend needs a CUDA device"
            self.torch = torch
            torch.cuda.set_device(0)
            self.sms = torch.cuda.get_device_properties(0).multi_processor_count
            lib = None
        else:
            from tests import mock_build
            self.torch = None
            self.sms = 132                               # sizes only: the test double has no SMs
            lib = mock_build.build()
        self.eng = modelx_b200.Engine(devices=[0], ring_bytes=4 << 20, lib_path=lib)
        self.rng = np.random.default_rng(1234)

    # -- plumbing -------------------------------------------------------------------------------------------------------
    def alloc(self, n):
        return _CudaBuf(self.torch, n) if self.torch else _HostBuf(n)

    def sync(self):
        if self.torch:
            self.torch.cuda.synchronize()

    def bytes_(self, n) -> np.ndarray:
        return self.rng.integers(0, 256, size=n, dtype=np.uint8)

    def expect(self, case, got, want, lengths=None):
        self.cases += 1
        if got != want:
            if isinstance(got, list):
                bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
                detail = f"{len(bad)} of {len(want)} digests differ, first at index {bad[0] if bad else len(got)}"
                if lengths:
                    detail += f"; lengths of the first that differ: {[lengths[i] for i in bad[:24]]}"
                raise Mismatch(case, detail)
            raise Mismatch(case, "result differs from the reference")

    def profiled(self, fn):
        """Run fn under torch.profiler (CUDA activity only) -> labels of the digest kernels it launched, in launch order."""
        if not self.torch:
            fn()
            return None
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            self.torch.ones(1, device="cuda").add_(1)      # the session is tracing before the first digest kernel
            fn()
            self.sync()
        evs = sorted((e for e in prof.events() if kernel_label(e.name)), key=lambda e: e.time_range.start)
        if not evs:
            raise Mismatch("profiler", "the profiler recorded no digest kernel at all: which kernel ran is unverified")
        return [kernel_label(e.name) for e in evs]

    # -- spans: dev_sha256_batch with the span array in device memory ------------------------------------------------
    def spans(self, case, specs):
        """specs[i]: (length, start offset from a 256-aligned address) | None ({NULL, 0}) | ("same", j) (span j again).
        Messages are laid out with >= 16 bytes between them, so the 16 bytes on each side can be flipped."""
        n = len(specs)
        starts, pos = [], 256
        for s in specs:
            if s is None or s[0] == "same":
                starts.append(None)
                continue
            ln, off = s
            st = _align(pos + 16, 256) + off
            starts.append(st)
            pos = st + ln
        total = pos + 16 + 64
        data = self.bytes_(total)
        buf = self.alloc(total)
        buf.put(0, data)
        table = np.zeros((n, 2), dtype=np.uint64)
        want = []
        for i, s in enumerate(specs):
            if s is None:
                want.append(sha(b""))
            elif s[0] == "same":
                table[i] = table[s[1]]
                want.append(want[s[1]])
            else:
                table[i] = (buf.ptr + starts[i], s[0])
                want.append(sha(data[starts[i]:starts[i] + s[0]]))
        d_spans = self.alloc(16 * n)
        d_spans.put(0, table.view(np.uint8).reshape(-1))

        def run(tag):
            out = Out(self, 32 * n)
            self.eng.dev_sha256_batch(0, d_spans.ptr, n, out.ptr)
            self.sync()
            body = out.take(f"{case} {tag}")
            self.expect(f"{case} {tag}", [body[32 * i:32 * i + 32] for i in range(n)], want,
                        [0 if sp is None else sp[0] if sp[0] != "same" else specs[sp[1]][0] for sp in specs])
        run("")
        flipped = data.copy()                     # every message's neighbours change, the messages do not
        for i, s in enumerate(specs):
            if starts[i] is not None:
                flipped[starts[i] - 16:starts[i]] ^= 0xFF
                flipped[starts[i] + s[0]:starts[i] + s[0] + 16] ^= 0x3C
        buf.put(0, flipped)
        run("neighbours flipped")

    def span_cases(self):
        for off in OFFSETS:
            self.spans(f"spans lengths 0..1048631 at offset {off}", [(ln, off) for ln in LENGTHS])
        for n in BATCH_SIZES:
            for name, specs in self.compositions(n):
                self.spans(f"spans n={n} {name}", specs)

    @staticmethod
    def compositions(n):
        yield "one length", [(64 * 3 + 57, 0)] * n
        for at in sorted({0, 15, 16, 31, 32, n - 1}):
            if at < n:
                yield f"long message at lane {at}", [(64 * 40 + 59 if i == at else (13 * i) % 120, 0) for i in range(n)]
        for lo in (5, 6):      # aligned; the fewest full blocks in a group is odd / even (the pair producer's hot loop)
            yield f"fewest full blocks {lo}", [(64 * (lo + (7 * i) % 4) + TAILS[i % 6], 0) for i in range(n)]
        yield "aligned plus one unaligned", [(64 * 24 + (5 * i) % 64, 3 if i == n // 2 else 0) for i in range(n)]
        yield "null span", [None if i == n // 2 else (100 + i, i % 16) for i in range(n)]
        if n > 1:
            yield "two spans with one pointer", [("same", 0) if i == n - 1 else (64 * 9 + 57 + i, i % 3) for i in range(n)]

    # -- segments: dev_sha256_segments ---------------------------------------------------------------------------------
    def segment_cases(self):
        for seg in SEGS:
            for nbytes in sorted({0, 1, seg - 1, seg, seg + 1, 37 * seg + 13}):
                for off in (0, 1, 3, 8):
                    self.segments(f"segments seg={seg} nbytes={nbytes} offset={off}", seg, nbytes, off)
        out = Out(self, 32)                       # NULL data is fine for an empty message
        self.eng.dev_sha256_segments(0, 0, 0, 64, out.ptr)
        self.sync()
        self.expect("segments NULL data, 0 bytes", out.take("segments NULL data"), sha(b""))

    def segments(self, case, seg, nbytes, off):
        total = 256 + off + nbytes + 16 + 64
        data = self.bytes_(total)
        buf = self.alloc(total)
        start = 256 + off
        nseg = max(1, -(-nbytes // seg))
        want = [sha(data[start + i * seg:start + min((i + 1) * seg, nbytes)]) for i in range(nseg)]
        for tag in ("", "neighbours flipped"):
            if tag:
                data[start - 16:start] ^= 0xFF
                data[start + nbytes:start + nbytes + 16] ^= 0x3C
            buf.put(0, data)
            out = Out(self, 32 * nseg)
            self.eng.dev_sha256_segments(0, buf.ptr + start, nbytes, seg, out.ptr)
            self.sync()
            body = out.take(f"{case} {tag}")
            self.expect(f"{case} {tag}", [body[32 * i:32 * i + 32] for i in range(nseg)], want)

    # -- chained state: the incremental hasher (one message per launch) --------------------------------------------------
    def hasher_cases(self):
        pool = self.bytes_(12 << 20)
        h = self.eng.hasher()
        ref = hashlib.sha256()
        self.expect("hasher empty", h.sum(), ref.digest())
        at = 0
        for n in (1, 63, 64, 65, (4 << 20) - 1, 4 << 20, (4 << 20) + 1, 3, 64, (4 << 20) + 1):
            piece = pool[at:at + n].tobytes()
            at = (at + 4099) % (8 << 20)
            h.write(piece)
            ref.update(piece)
            self.expect(f"hasher after {h.written()} bytes", h.sum(), ref.digest())
            self.expect(f"hasher second sum after {h.written()} bytes", h.sum(), ref.digest())
        h.reset()
        ref = hashlib.sha256()
        self.expect("hasher after reset", h.sum(), ref.digest())
        for n in ((4 << 20) + 1, 65):
            piece = pool[n:2 * n].tobytes()
            h.write(piece)
            ref.update(piece)
        self.expect("hasher continued after reset", h.sum(), ref.digest())
        if self.route in BIG_STREAM_ROUTES:
            # 2^29 + 77 bytes: the bit length (prefix + len) * 8 needs the high word in chained mode
            t0 = time.time()
            h.reset()
            ref = hashlib.sha256()
            total, k = (1 << 29) + 77, 0
            while h.written() < total:
                n = min((3 << 20) + 5 + 64 * (k % 7), total - h.written())
                piece = pool[(k * 4099) % (8 << 20):][:n].tobytes()
                h.write(piece)
                ref.update(piece)
                k += 1
            self.expect("hasher one stream of 536870989 bytes", h.sum(), ref.digest())
            self.big_stream_seconds = round(time.time() - t0, 2)
        h.close()

    # -- the digest service (descriptor mode: kFresh, kSkip, oidx != m) on a small ring -----------------------------------
    def service_cases(self):
        rng = random.Random(7)
        pool = self.bytes_(7 << 20).tobytes()
        sizes = [0 if i % 97 == 0 else rng.randrange(1, 3000) for i in range(5000)]
        for i, s in ((17, 3 << 20), (2500, (5 << 20) + 3), (4999, (2 << 20) + 61)):
            sizes[i] = s
        msgs = [pool[(i * 4099) % (len(pool) - s):][:s] for i, s in enumerate(sizes)]
        self.expect("service 5000 ragged host messages", self.eng.sha256_batch(msgs), [sha(m) for m in msgs])
        with tempfile.TemporaryDirectory() as d:
            data = pool[:5_000_013]
            p = os.path.join(d, "parts.bin")
            with open(p, "wb") as f:
                f.write(data)
            parts = [(0, 3_000_000), (1_000_000, 3_000_007), (5, 0), (4_000_000, 1_000_013), (0, len(data)), (4_999_999, 14)]
            self.expect("service overlapping file parts", self.eng.sha256_file_parts(p, parts),
                        [sha(data[o:o + n]) for o, n in parts])
            fsizes = [0, 1, 63, 64, 65, 4095, 100_000, 3 << 20, (6 << 20) + 5, 777, 56, 57, (1 << 20) + 1, 12_345,
                      2 << 20, 9, 300_000, (4 << 20) - 3, 128, 1000]
            failing = 8
            jobs, want, seen = [], [], {}
            for i, s in enumerate(fsizes):
                body = pool[i * 1000:i * 1000 + s]
                q = os.path.join(d, f"job{i}.bin")
                with open(q, "wb") as f:
                    f.write(body)
                job = {"path": q}
                if i % 3 == 1:
                    job["ranges"] = [(0, s), (s // 3, s - s // 3), (0, s // 2)]
                if i == failing:
                    calls = []

                    def sink(offset, b, calls=calls):
                        calls.append(offset)
                        if len(calls) == 2:
                            raise IOError("the sink refuses its second piece")
                    job["sink"] = sink
                elif i % 4 == 2:
                    seen[i] = {}
                    job["sink"] = lambda offset, b, got=seen[i]: got.__setitem__(offset, b)
                jobs.append(job)
                want.append([sha(body[o:o + n]) for o, n in job.get("ranges", [(0, s)])])
            res = self.eng.sha256_file_jobs(jobs)
            self.cases += 1
            if res[failing]["status"] != -4:
                raise Mismatch("service file jobs", f"the job whose sink failed reports {res[failing]['status']}, not -4")
            for i, r in enumerate(res):
                if i == failing:
                    continue
                if r["status"] != 0 or r["size"] != fsizes[i]:
                    raise Mismatch("service file jobs", f"job {i}: status {r['status']} size {r['size']}")
                self.expect(f"service file job {i} next to a failed one", r["digests"][:len(want[i])], want[i])
                if i in seen:
                    got = b"".join(seen[i][o] for o in sorted(seen[i]))
                    self.expect(f"service file job {i} sink bytes", got, pool[i * 1000:i * 1000 + fsizes[i]])

    # -- k_compare and k_gen_fill ------------------------------------------------------------------------------------------
    def compare_gen_cases(self):
        for n in (1, 255, 256, 257, 1000):
            got = self.bytes_(32 * n)
            d_got = self.alloc(32 * n)
            d_got.put(0, got)
            for tag, at, byte, bit in (("equal", None, 0, 0), ("bit flipped in byte 0", n // 3, 0, 0x01),
                                       ("bit flipped in byte 31", n - 1, 31, 0x80)):
                want = got.copy()
                exp = [1] * n
                if at is not None:
                    want[32 * at + byte] ^= bit
                    exp[at] = 0
                d_want = self.alloc(32 * n)
                d_want.put(0, want)
                out = Out(self, n)
                self.eng.dev_compare(0, d_got.ptr, d_want.ptr, n, out.ptr)
                self.sync()
                self.expect(f"compare n={n} {tag}", list(out.take(f"compare n={n} {tag}", slot=1)), exp)
        n = 64 * self.sms * 256 * 8 + 8 * 13           # more words than the capped grid has threads: the grid-stride loop
        for off in (0, 8, 8 * 123_457):
            out = Out(self, n, lead=72)                # 8-byte aligned, not 16
            self.eng.dev_gen_fill(0, out.ptr, off, n, SEED)
            self.sync()
            self.expect(f"gen_fill offset={off} n={n}", out.take(f"gen_fill offset={off}", slot=None), self.orc.gen(off, n, SEED))

    # -- trees: dev_tree_digest, dev_tree_chunks + dev_tree_finish -------------------------------------------------------
    TREES = [  # (size, chunk, leaf, fanout); leaf counts mostly not multiples of 64
        (0, 64 * 2 ** 7, 64, 2), (1, 64 * 2 ** 6, 64, 2), (64 * 1001 + 17, 64 * 2 ** 7, 64, 2), (64 * 1001 + 17, 64 * 2 ** 6, 64, 2),
        (0, 64 * 27, 64, 3), (100_003, 64 * 27, 64, 3), (1, 64 * 3, 64, 3),
        (64 * 700 + 63, 64 * 4 ** 3, 64, 4), (64 * 700 + 63, 64 * 4 ** 4, 64, 4), (1, 64 * 4, 64, 4),
        (0, 64 * 64, 64, 8), (64 * 517 + 56, 64 * 8 ** 2, 64, 8), (300_001, 64 * 8 ** 3, 64, 8),
        (64 * 99 + 60, 1024 * 8, 1024, 8), (1_000_003, 1024 * 64, 1024, 8),
        (1, 64 * 64, 64, 64), (64 * 130 + 1, 64 * 64, 64, 64), ((1 << 20) + 7, 128 * 64 * 64, 128, 64),
        (100_000, 128, 64, 2),     # 782 chunks: the levels above them start with a wide launch and a ragged last group
    ]

    def tree(self, case, data_host, size, chunk, leaf, fanout, off, buf=None):
        tp = (chunk, leaf, fanout)
        nch = max(1, -(-size // chunk))
        want_chunks, _, want_root = self.orc.tree_digest(data_host[off:off + size].tobytes(), chunk, leaf, fanout)
        want_chunks = b"".join(want_chunks)
        if buf is None:
            buf = self.alloc(len(data_host))
            buf.put(0, data_host)
        ptr = buf.ptr + off
        d_chunks, d_root = Out(self, 32 * nch), Out(self, 32)
        self.eng.dev_tree_digest(0, ptr, size, tp, d_chunks.ptr, d_root.ptr)
        self.sync()
        self.expect(f"{case} tree_digest chunks", d_chunks.take(case), want_chunks)
        self.expect(f"{case} tree_digest root", d_root.take(case), want_root)
        d_root = Out(self, 32)
        self.eng.dev_tree_digest(0, ptr, size, tp, 0, d_root.ptr)
        self.sync()
        self.expect(f"{case} tree_digest root without a chunk list", d_root.take(case), want_root)
        d_chunks, d_root = Out(self, 32 * nch), Out(self, 32)
        self.eng.dev_tree_chunks(0, ptr, size, tp, d_chunks.ptr)
        self.sync()
        got_chunks = d_chunks.take(case)
        self.expect(f"{case} tree_chunks", got_chunks, want_chunks)
        self.eng.dev_tree_finish(0, d_chunks.ptr, nch, size, tp, d_root.ptr)
        self.sync()
        self.expect(f"{case} tree_finish", d_root.take(case), self.orc.tree_finish(want_chunks, size, leaf, fanout))

    def tree_cases(self):
        for size, chunk, leaf, fanout in self.TREES:
            for off in (0, 5):
                data = self.bytes_(256 + size + 64)
                case = f"tree size={size} chunk={chunk} leaf={leaf} fanout={fanout} offset={off}"
                self.tree(case, data, size, chunk, leaf, fanout, 256 + off)
                buf = self.alloc(len(data))
                data[256 + off - 16:256 + off] ^= 0xFF
                data[256 + off + size:256 + off + size + 16] ^= 0x3C
                buf.put(0, data)
                self.tree(case + " neighbours flipped", data, size, chunk, leaf, fanout, 256 + off, buf)

    def big_leaf_case(self):
        """64-byte leaves, at least 2 * SMs * 32 units of 64 leaves: more than twice the resident CTAs at any occupancy,
        so MXD_TUNE_LEAF_SCHED=2 takes the persistent schedule (a launch and its sweep)."""
        size = 2 * self.sms * 32 * 64 * 64 + 64 * 37 + 29
        tp = (64 * 8 ** 3, 64, 8)
        fill = _align(size, 8)
        buf = self.alloc(fill)
        self.eng.dev_gen_fill(0, buf.ptr, 0, fill, SEED + 1)
        host = np.frombuffer(self.orc.gen(0, fill, SEED + 1), dtype=np.uint8)
        self.tree(f"tree of {size} bytes in 64-byte leaves", host, size, *tp, 0, buf)
        out = Out(self, 32 * -(-size // tp[0]))
        before = self.eng.stats()["kernel_launches"]
        labels = self.profiled(lambda: self.eng.dev_tree_chunks(0, buf.ptr, size, tp, out.ptr))
        return self.eng.stats()["kernel_launches"] - before, labels

    # -- which kernel runs where a route does not force one ----------------------------------------------------------
    def default_boundaries(self):
        pair_max = 2 * 16 * self.sms
        got = []
        for n, want in ((pair_max, PAIR), (pair_max + 1, "k_sha256_chains_coop<0>"),
                        (32_768, "k_sha256_chains_coop<0>"), (32_769, LANES12)):
            data = self.bytes_(n)
            buf = self.alloc(n)
            buf.put(0, data)
            out = Out(self, 32 * n)
            labels = self.profiled(lambda: self.eng.dev_sha256_segments(0, buf.ptr, n, 1, out.ptr))
            self.sync()
            body = out.take(f"default dispatch n={n}")
            self.expect(f"default dispatch n={n}", [body[32 * i:32 * i + 32] for i in range(n)], [sha(data[i:i + 1]) for i in range(n)])
            if labels is not None and labels != [want]:
                raise Mismatch(f"default dispatch n={n}", f"ran {labels}, expected [{want}]")
            got.append(labels)
        return got

    # -- the route ---------------------------------------------------------------------------------------------------
    def run(self):
        promised = ROUTES[self.route][1]
        if self.route in LEAF_ROUTES:
            battery = [self.tree_cases]
        else:
            battery = [self.span_cases, self.segment_cases, self.hasher_cases, self.service_cases, self.compare_gen_cases,
                       self.tree_cases]
        labels = self.profiled(lambda: [step() for step in battery])
        if labels is not None:
            self.kernels = set(labels)
            leaves = {k for k in self.kernels if k.startswith("k_tree_leaves")}
            shas = self.kernels - leaves
            if self.route in LEAF_ROUTES:
                if leaves != promised or not shas <= DEFAULT_SHA:
                    raise Mismatch("kernel check", f"ran {sorted(self.kernels)}, route promises {sorted(promised)}")
            elif promised is None:
                if leaves or not shas <= DEFAULT_SHA:
                    raise Mismatch("kernel check", f"ran {sorted(self.kernels)} under the default dispatch")
            elif self.kernels != promised:
                raise Mismatch("kernel check", f"ran {sorted(self.kernels)}, route promises {sorted(promised)}")
        if self.route == "default":
            self.default_boundaries()
        if self.route in LEAF_ROUTES:
            # leaves: a persistent launch and its sweep under MXD_TUNE_LEAF_SCHED=2, else one launch; then one launch per
            # tree level between the highest fused level and the chunk list (level 3: 8^3 leaves per chunk)
            launches, labels = self.big_leaf_case()
            fused = 2 if "MXD_TUNE_FUSE" in ROUTES[self.route][0] else 0
            want = (2 if "MXD_TUNE_LEAF_SCHED" in ROUTES[self.route][0] else 1) + 3 - fused
            if launches != want:
                raise Mismatch("persistent leaf schedule", f"{launches} launches for one tree_chunks call, expected {want}")
            if labels is not None and not {k for k in labels if k.startswith("k_tree_leaves")} <= promised:
                raise Mismatch("persistent leaf schedule", f"ran {labels}")


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--route", required=True, choices=sorted(ROUTES))
    ap.add_argument("--backend", default="cuda", choices=("cuda", "mock"))
    args = ap.parse_args(argv)
    for k in [k for k in os.environ if k.startswith("MXD_TUNE_")]:
        del os.environ[k]
    os.environ.update(ROUTES[args.route][0])              # before the library is loaded: knobs are read once
    t0 = time.time()
    res = {"route": args.route, "backend": args.backend}
    try:
        b = Battery(args.route, args.backend)
        b.run()
    except Mismatch as e:
        res.update(ok=False, case=e.case, error=str(e))
        print(json.dumps(res), flush=True)
        return 1
    res.update(ok=True, cases=b.cases, kernels=sorted(b.kernels), seconds=round(time.time() - t0, 1),
               big_stream_seconds=b.big_stream_seconds,
               torch_peak_bytes=b.torch.cuda.max_memory_allocated() if b.torch else None)
    b.eng.close()
    print(json.dumps(res), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
