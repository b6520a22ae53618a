"""mxd_tree_load_file -- a file copied through the pinned ring straight into device spans, tree-digested from the bytes
that landed there -- and modelx_b200.checkpoint.load_safetensors / Client.load_safetensors on top of it.

Every load is checked three ways: the destination bytes equal the file, the root and chunk digests equal
mxd_tree_digest_file of the file and the CPU oracle, and the bytes around every destination are untouched.  The host
logic runs on the CPU test double (`-m "not gpu"`) and on the H100 (`-m gpu`, k_tree_leaves_extents)."""
import ctypes as C
import json
import os
import random

import numpy as np
import pytest

import modelx_b200
from modelx_b200 import _native as N
from tests.checkpoint_fixtures import SMALL, llama_shapes
from tests.test_gpu_parity import TREE_CASES

SEED = 0x6D6F64656C78
RING = 4 << 20                 # four 1 MiB slots: small files cross several
SLOT = RING // 4
GUARD = 0xEE
TP = (8 << 20, 16 << 10, 8)


class DevMem:
    """Device memory that the library's pointer checks classify as device memory of device 0: torch on the GPU, the
    test double's own allocator (mockcuda::alloc(size, kind 2 = device, ordinal), exported with C++ linkage) on the
    CPU."""

    def __init__(self, backend):
        self.torch, self.blocks = None, []
        if backend is None:
            import torch
            assert torch.cuda.is_available(), "the cuda backend needs a CUDA device"
            torch.cuda.set_device(0)
            self.torch = torch
        else:
            lib = C.CDLL(backend)
            self._alloc, self._free = lib._ZN8mockcuda5allocEmii, lib._ZN8mockcuda7releaseEPv
            self._alloc.restype, self._alloc.argtypes = C.c_void_p, [C.c_size_t, C.c_int, C.c_int]
            self._free.restype, self._free.argtypes = None, [C.c_void_p]

    def alloc(self, n):
        """-> base address of n bytes filled with GUARD"""
        if self.torch:
            t = self.torch.full((n,), GUARD, dtype=self.torch.uint8, device="cuda")
            self.blocks.append(t)
            return t.data_ptr()
        p = self._alloc(n, 2, 0)
        assert p
        C.memset(p, GUARD, n)
        self.blocks.append(p)
        return p

    def get(self, ptr, n) -> bytes:
        if self.torch:
            for t in self.blocks:
                if t.data_ptr() <= ptr and ptr + n <= t.data_ptr() + t.numel():
                    o = ptr - t.data_ptr()
                    return t[o:o + n].cpu().numpy().tobytes()
            raise AssertionError("not in a block")
        return C.string_at(ptr, n)

    def release(self):
        if not self.torch:
            for p in self.blocks:
                self._free(p)
        self.blocks = []


@pytest.fixture
def dev(backend):
    m = DevMem(backend)
    yield m
    m.release()


@pytest.fixture
def eng(backend):
    e = modelx_b200.Engine(devices=[0], ring_bytes=RING, lib_path=backend)
    yield e
    e.close()


def _align(x, a):
    return (x + a - 1) // a * a


def lay_out(dev, lengths, offs):
    """One allocation holding a span of lengths[i] bytes at offset offs[i] from a 256-byte boundary for every i, with
    guard bytes between and around them.  -> (spans [(ptr, len)], base, total bytes of the allocation)"""
    starts, pos = [], 0
    for n, o in zip(lengths, offs):
        st = _align(pos + 64, 256) + o
        starts.append(st)
        pos = st + n
    total = pos + 64
    base = dev.alloc(total)
    return [(base + st, n) for st, n in zip(starts, lengths)], base, total


def expect_bytes(spans, base, total, data):
    """What the allocation must hold after a load of `data` into `spans`."""
    want = bytearray([GUARD]) * total
    pos = 0
    for p, n in spans:
        want[p - base:p - base + n] = data[pos:pos + n]
        pos += n
    assert pos == len(data)
    return bytes(want)


def write(tmp_path, data, name="blob.bin"):
    path = str(tmp_path / name)
    with open(path, "wb") as f:
        f.write(data)
    return path


def check_load(eng, dev, oracle, tmp_path, data, lengths, offs=None, tp=TP):
    """Load `data` (as a file) into spans of `lengths` and check bytes, digests and guards."""
    offs = offs if offs is not None else [0] * len(lengths)
    path = write(tmp_path, data)
    spans, base, total = lay_out(dev, lengths, offs)
    got = eng.tree_load_file(0, path, spans, *tp)
    assert dev.get(base, total) == expect_bytes(spans, base, total, data)
    want_chunks, _, want_root = oracle.tree_digest(np.frombuffer(data, np.uint8) if data else b"", *tp)
    assert got == (want_chunks, want_root, len(data))
    assert got == eng.tree_digest_file(path, *tp)
    return got


def cuts_to_lengths(size, cuts):
    bounds = [0] + sorted(c for c in set(cuts) if 0 < c < size) + [size]
    return [b - a for a, b in zip(bounds, bounds[1:])]


def blob(oracle, n, seed=7):
    return oracle.gen(seed, n, SEED) if n else b""


# ---- sizes and tree parameters ---------------------------------------------------------------------------------------
def test_empty_and_one_byte_files(eng, dev, oracle, tmp_path):
    check_load(eng, dev, oracle, tmp_path, b"", [])
    check_load(eng, dev, oracle, tmp_path, b"", [0, 0])
    check_load(eng, dev, oracle, tmp_path, b"\x5c", [1])
    check_load(eng, dev, oracle, tmp_path, b"\x5c", [0, 1, 0], [3, 7, 0])


@pytest.mark.parametrize("size,chunk,leaf,fanout", TREE_CASES)
def test_tree_cases(eng, dev, oracle, tmp_path, size, chunk, leaf, fanout):
    rng = random.Random(size * 31 + fanout)
    data = blob(oracle, size)
    lengths = cuts_to_lengths(size, rng.sample(range(size + 1), min(size + 1, 12))) if size else [0]
    check_load(eng, dev, oracle, tmp_path, data, lengths, [rng.randrange(16) for _ in lengths], (chunk, leaf, fanout))


@pytest.mark.parametrize("off", range(16))
def test_destinations_at_every_address_offset(eng, dev, oracle, tmp_path, off):
    rng = random.Random(200 + off)
    lengths = [5000, 64, 1, (1 << 20) + 3, 63, 3 * (16 << 10) + 17, 777]
    data = bytes(rng.randbytes(sum(lengths)))
    tp = (1 << 18, 1 << 12, 4)
    check_load(eng, dev, oracle, tmp_path, data, lengths, [off] * len(lengths), tp)
    check_load(eng, dev, oracle, tmp_path, data, lengths, [(off + 5 * i) % 16 for i in range(len(lengths))], tp)


def test_span_boundaries_at_leaf_and_slot_boundaries(eng, dev, oracle, tmp_path):
    leaf = TP[1]
    size = 3 * SLOT + 5 * leaf + 123
    data = blob(oracle, size, 8)
    for d in (-1, 0, 1):
        cuts = [k * leaf + d for k in (1, 2, 7, 64, 65, 130)] + [k * SLOT + d for k in (1, 2, 3)]
        check_load(eng, dev, oracle, tmp_path, data, cuts_to_lengths(size, cuts), [(3 * k + d) % 16 for k in range(len(cuts) + 1)])


def test_one_leaf_of_150_tiny_spans(eng, dev, oracle, tmp_path):
    rng = random.Random(9)
    tiny = [rng.randrange(1, 9) for _ in range(150)]                  # < 1 leaf in all, across a slot boundary
    lengths = [SLOT - 300] + tiny + [2 * SLOT + 4321]
    data = bytes(rng.randbytes(sum(lengths)))
    check_load(eng, dev, oracle, tmp_path, data, lengths, [rng.randrange(16) for _ in lengths])
    check_load(eng, dev, oracle, tmp_path, data, lengths, [rng.randrange(16) for _ in lengths], (256, 64, 2))


def test_empty_spans_mixed_in(eng, dev, oracle, tmp_path):
    rng = random.Random(10)
    lengths = [0, 70_000, 0, 0, SLOT, 1, 0, 33_333, 0]
    data = bytes(rng.randbytes(sum(lengths)))
    check_load(eng, dev, oracle, tmp_path, data, lengths, [rng.randrange(16) for _ in lengths])


# ---- accounting ------------------------------------------------------------------------------------------------------
def test_read_once_accounting_and_one_launch_per_slot(eng, dev, oracle, tmp_path):
    size = 3 * SLOT + 1000
    data = blob(oracle, size, 11)
    path = write(tmp_path, data)
    spans, base, total = lay_out(dev, cuts_to_lengths(size, [100, SLOT - 1, 2 * SLOT + 7]), [0, 3, 9, 12])
    eng.prof_read()
    eng.prof_enable(True)
    eng.trace_enable(True)
    s0 = eng.stats()
    got = eng.tree_load_file(0, path, spans, *TP)
    s1 = eng.stats()
    eng.prof_enable(False)
    eng.trace_enable(False)
    prof = eng.prof_read()
    csv = str(tmp_path / "trace.csv")
    eng.trace_dump(csv)
    for key in ("src_bytes_read", "h2d_bytes"):
        assert s1[key] - s0[key] == size, key
    assert got[1] == eng.tree_digest_file(path, *TP)[1]
    s2 = eng.stats()
    assert s1["bytes_hashed"] - s0["bytes_hashed"] == s2["bytes_hashed"] - s1["bytes_hashed"]   # leaves + levels, as for the file
    slots = -(-size // SLOT)
    assert prof["launches"] == slots and prof["bytes"] == size
    with open(csv) as f:
        rows = f.read().strip().split("\n")[1:]
    assert len(rows) == slots and sum(int(r.split(",")[2]) for r in rows) == size
    assert dev.get(base, total) == expect_bytes(spans, base, total, data)


# ---- argument rejection: before any destination byte is written or any file byte read --------------------------------
class Outs:
    """Pre-filled outputs of one raw mxd_tree_load_file call."""

    def __init__(self, nch=4):
        self.nch = nch
        self.chunks = (C.c_uint8 * (32 * nch))(*([0x5A] * (32 * nch)))
        self.root = (C.c_uint8 * 32)(*([0x5A] * 32))
        self.got, self.size = C.c_uint64(0xABCD), C.c_uint64(0xABCD)

    def untouched(self):
        return bytes(self.chunks) == b"\x5a" * (32 * self.nch) and bytes(self.root) == b"\x5a" * 32 and \
            self.got.value == 0xABCD and self.size.value == 0xABCD


def raw_call(eng, spans, path, o, handle=None, dev=0, tp=N.TreeParams(*TP, 0), n=None, use_none=False, root=True,
             cap=None):
    n = len(spans) if n is None else n
    arr = None if use_none else (N.Span * max(len(spans), 1))(*[N.Span(p, ln) for p, ln in spans])
    return eng._lib.mxd_tree_load_file(eng.handle if handle is None else handle, dev,
                                       path.encode() if path is not None else None, arr, n,
                                       C.byref(tp) if tp is not None else None, o.chunks, o.nch if cap is None else cap,
                                       C.byref(o.got), C.byref(o.size), o.root if root else None)


def test_rejects_bad_arguments(eng, dev, oracle, tmp_path):
    size = 2 * SLOT + 5000                                          # 1 chunk of 8 MiB
    data = blob(oracle, size, 12)
    path = write(tmp_path, data)
    spans, base, total = lay_out(dev, [1000, size - 1000], [0, 5])
    (p0, n0), (p1, n1) = spans
    host = np.zeros(size + 64, np.uint8)
    bad_tp = N.TreeParams(TP[0] + 64, TP[1], TP[2], 0)
    cases = {
        "NULL handle": dict(handle=C.c_void_p(0)),
        "device index past the engine's devices": dict(dev=eng.device_count()),
        "negative device index": dict(dev=-1),
        "NULL path": dict(path=None),
        "NULL root": dict(root=False),
        "bad tree parameters": dict(tp=bad_tp),
        "reserved != 0": dict(tp=N.TreeParams(*TP, 1)),
        "n > 0 with a NULL span array": dict(spans=[], n=2, use_none=True),
        "NULL span with a nonzero length": dict(spans=[(p0, n0), (0, 5), (p1, n1 - 5)]),
        "total length overflows": dict(spans=[(p0, 1 << 63), (p1, 1 << 63), (p1, size)]),
        "host memory as a destination": dict(spans=[(p0, n0), (host.ctypes.data, n1)]),
        "overlapping destinations": dict(spans=[(p0, n0), (p0 + n0 - 1, n1)]),
        "the same destination twice": dict(spans=[(p1, n0), (p1, n1)]),
        "total one byte short": dict(spans=[(p0, n0), (p1, n1 - 1)]),
        "total one byte long": dict(spans=[(p0, n0), (p1, n1 + 1)]),
        "chunk_digests below the chunk count": dict(cap=0),
    }
    s0 = eng.stats()
    for what, kw in cases.items():
        o = Outs()
        args = dict(spans=spans, path=path)
        args.update(kw)
        assert raw_call(eng, o=o, **args) == N.MXD_ERR_INVALID, what
        assert o.untouched(), what
    s1 = eng.stats()
    assert dev.get(base, total) == b"\xee" * total                  # no destination byte written
    for key in ("src_bytes_read", "h2d_bytes", "bytes_hashed", "kernel_launches"):
        assert s1[key] == s0[key], key
    with pytest.raises(modelx_b200.MxdError) as ei:
        eng.tree_load_file(0, path, [(p0, n0), (p1, n1 - 1)], *TP)
    assert ei.value.status == N.MXD_ERR_INVALID and "the file has" in ei.value.detail
    o = Outs()
    assert raw_call(eng, spans, path, o) == N.MXD_OK                # the same arguments, corrected, work
    assert bytes(o.root) == oracle.tree_digest(np.frombuffer(data, np.uint8), *TP)[2] and o.size.value == size


def test_missing_file_directory_and_canceled_operation(eng, dev, oracle, tmp_path):
    data = blob(oracle, 5000, 13)
    path = write(tmp_path, data)
    spans, base, total = lay_out(dev, [5000], [0])
    for what, p in (("missing", str(tmp_path / "nope.bin")), ("directory", str(tmp_path))):
        o = Outs()
        assert raw_call(eng, spans, p, o) == N.MXD_ERR_IO, what
        assert o.untouched(), what
    with pytest.raises(modelx_b200.MxdError) as ei:
        eng.tree_load_file(0, str(tmp_path / "nope.bin"), spans, *TP)
    assert ei.value.status == N.MXD_ERR_IO
    with eng.op() as op:
        op.cancel()
        s0 = eng.stats()
        o = Outs()
        assert raw_call(op, spans, path, o) == N.MXD_ERR_CANCELED
        assert o.untouched() and eng.stats()["src_bytes_read"] == s0["src_bytes_read"]
    assert dev.get(base, total) == b"\xee" * total


# ---- checkpoint.load_safetensors: input checks on the host (no device needed) ---------------------------------------
def test_load_safetensors_rejects_bad_files(mock_lib, tmp_path):
    import struct
    from modelx_b200.checkpoint import MAX_HEADER_BYTES, load_safetensors
    eng = modelx_b200.Engine(devices=[0], lib_path=mock_lib)
    try:
        text = json.dumps({"a": {"dtype": "U8", "shape": [3], "data_offsets": [0, 3]}}).encode()
        text += b" " * (-len(text) % 8)
        good = struct.pack("<Q", len(text)) + text + b"xyz"
        cases = [
            ("shorter than", b"\x01\x02"),
            ("over the", struct.pack("<Q", MAX_HEADER_BYTES + 8) + b"{}"),
            ("safetensors header", struct.pack("<Q", len(text) + 8) + text),
            ("the file has", good + b"!"),
            ("the file has", good[:-1]),
        ]
        for msg, raw in cases:
            p = write(tmp_path, raw, "bad.safetensors")
            with pytest.raises(ValueError, match=msg):
                load_safetensors(eng, p, "cpu")
        p = write(tmp_path, good, "good.safetensors")
        with pytest.raises(ValueError, match="not a CUDA device"):
            load_safetensors(eng, p, "cpu")
        for bad in (b"\x00" * 31, "sha256:xyz", 5):
            with pytest.raises(ValueError):
                load_safetensors(eng, p, "cpu", expect=bad)
    finally:
        eng.close()


def test_client_requires_a_tree_identity(mock_lib, tmp_path):
    from modelx_b200 import client
    from modelx_b200.client import _tree_identity
    eng = modelx_b200.Engine(devices=[0], lib_path=mock_lib)
    try:
        d = tmp_path / "model"
        d.mkdir()
        (d / "modelx.yaml").write_bytes(b"framework: pytorch\nmodelFiles: []\n")
        (d / "w.safetensors").write_bytes(os.urandom(3000))
        reg = client.LocalRegistry(str(tmp_path / "reg"), eng)
        cl = client.Client(eng)
        cl.push(reg, "library/m", "v1", str(d))                      # whole-file SHA-256 identity only
        with pytest.raises(ValueError, match="--tree"):
            cl.load_safetensors(reg, "library/m", "v1", "w.safetensors")
        with pytest.raises(ValueError, match="no blob named"):
            cl.load_safetensors(reg, "library/m", "v1", "other.safetensors")
        cl.push_tree(reg, "library/m", "v2", str(d))
        desc = [b for b in json.loads(reg.get_manifest_json("library/m", "v2"))["blobs"] if b["name"] == "w.safetensors"][0]
        assert _tree_identity(desc) == (desc["digest"], dict(chunk=8 << 20, leaf=16 << 10, fanout=8))
        m = json.loads(cl.push_digest_json(str(d), with_tree=True))
        desc = [b for b in m["blobs"] if b["name"] == "w.safetensors"][0]
        root = desc["annotations"]["modelx.tree.v1"].split(";")[0]
        assert _tree_identity(desc) == (root, dict(chunk=8 << 20, leaf=16 << 10, fanout=8))
        assert root == modelx_b200.digest_string(eng.tree_digest_file(str(d / "w.safetensors"))[1])
    finally:
        eng.close()


# ---- GPU only ----------------------------------------------------------------------------------------------------------
def _torch():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.cuda.set_device(0)
    return torch


@pytest.fixture(scope="module")
def small_file(tmp_path_factory):
    """About 1 GB saved by safetensors.torch.save_file: the SMALL Llama layout, an odd-length int8 tensor and a
    zero-element tensor."""
    torch = _torch()
    st = pytest.importorskip("safetensors.torch")
    g = torch.Generator(device="cuda").manual_seed(SEED)
    tensors = {n: torch.randn(s, dtype=torch.float16, device="cuda", generator=g) for n, s in llama_shapes(**SMALL)}
    tensors["odd.int8"] = torch.randint(-128, 128, (4097,), dtype=torch.int8, device="cuda", generator=g)
    tensors["empty.bf16"] = torch.empty(0, 7, dtype=torch.bfloat16, device="cuda")
    path = str(tmp_path_factory.mktemp("load") / "model.safetensors")
    st.save_file({k: v.cpu() for k, v in tensors.items()}, path, metadata={"format": "pt"})
    del tensors
    return path


@pytest.mark.gpu
def test_load_safetensors_equals_load_file(engine, small_file):
    torch = _torch()
    st = pytest.importorskip("safetensors.torch")
    from modelx_b200.checkpoint import parse_safetensors_header, tree_digest_safetensors
    tensors, chunks, root, size = load_safetensors_(engine, small_file)
    want = st.load_file(small_file, device="cuda:0")
    with open(small_file, "rb") as f:
        n = int.from_bytes(f.read(8), "little")
        header = n.to_bytes(8, "little") + f.read(n)
    entries, _ = parse_safetensors_header(header)
    assert list(tensors) == list(entries) and sorted(tensors) == sorted(want)
    for name, t in tensors.items():
        assert t.device == torch.device("cuda", 0) and t.dtype == want[name].dtype and t.shape == want[name].shape, name
        assert torch.equal(t, want[name]), name
    storages = sorted((t.untyped_storage().data_ptr(), t.untyped_storage().nbytes()) for t in tensors.values() if t.numel())
    assert all(a + n <= b for (a, n), (b, _) in zip(storages, storages[1:]))   # separate allocations
    assert size == os.path.getsize(small_file) > 0.9e9
    assert (chunks, root, size) == engine.tree_digest_file(small_file)
    assert (chunks, root, size) == tree_digest_safetensors(engine, header, tensors)
    assert load_safetensors_(engine, small_file, expect=modelx_b200.digest_string(root))[2] == root
    assert load_safetensors_(engine, small_file, expect=root)[2] == root


def load_safetensors_(engine, path, **kw):
    from modelx_b200.checkpoint import load_safetensors
    return load_safetensors(engine, path, **kw)


@pytest.mark.gpu
def test_flipped_byte_raises_digest_mismatch(engine, small_file, tmp_path):
    _torch()
    from modelx_b200.checkpoint import DigestMismatch
    chunks, root, size = engine.tree_digest_file(small_file)
    bad = str(tmp_path / "bad.safetensors")
    with open(small_file, "rb") as f, open(bad, "wb") as g:
        raw = bytearray(f.read())
        pos = len(raw) // 3 + 12345                                 # inside a tensor: the header is a few KB
        raw[pos] ^= 0x40
        g.write(raw)
    with pytest.raises(DigestMismatch) as ei:
        load_safetensors_(engine, bad, expect=root)
    e = ei.value
    assert e.expected == root and e.root != root and e.size == size
    assert [k for k in range(len(chunks)) if chunks[k] != e.chunk_digests[k]] == [pos // TP[0]]


@pytest.mark.gpu
def test_memory_reused_from_a_queued_kernel(engine, small_file):
    """A tensor that a long kernel still writes on the current stream is freed; the loaded tensors reuse its memory.
    load_safetensors synchronises the stream first, so the fill cannot land on the loaded weights."""
    torch = _torch()
    st = pytest.importorskip("safetensors.torch")
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    big = torch.empty(os.path.getsize(small_file) + (64 << 20), dtype=torch.uint8, device="cuda")
    lo, hi = big.data_ptr(), big.data_ptr() + big.numel()
    torch.cuda._sleep(2_000_000_000)                                # about a second of GPU time queued ahead of the fill
    big.fill_(0x77)
    del big
    tensors, *_ = load_safetensors_(engine, small_file)
    torch.cuda.synchronize()
    assert any(lo <= t.data_ptr() < hi for t in tensors.values() if t.numel()), "the allocator did not reuse the block"
    want = st.load_file(small_file, device="cuda:0")
    for name, t in tensors.items():
        assert torch.equal(t, want[name]), name


@pytest.mark.gpu
def test_client_load_safetensors(engine, small_file, tmp_path):
    torch = _torch()
    st = pytest.importorskip("safetensors.torch")
    from modelx_b200 import client
    from modelx_b200.checkpoint import DigestMismatch
    d = tmp_path / "model"
    d.mkdir()
    (d / "modelx.yaml").write_bytes(b"framework: pytorch\nmodelFiles: []\n")
    with open(small_file, "rb") as f:
        (d / "model.safetensors").write_bytes(f.read())
    reg = client.LocalRegistry(str(tmp_path / "reg"), engine)
    cl = client.Client(engine)
    rep = cl.push_tree(reg, "library/m", "v1", str(d))
    want = st.load_file(small_file, device="cuda:0")
    got = cl.load_safetensors(reg, "library/m", "v1", "model.safetensors")
    assert sorted(got) == sorted(want)
    for name, t in got.items():
        assert torch.equal(t, want[name]), name
    # whole-file keyed with a tree annotation (push --tree of the digest phase): the same blob under its SHA-256
    m = cl.push_digest_json(str(d), with_tree=True)
    desc = [b for b in json.loads(m)["blobs"] if b["name"] == "model.safetensors"][0]
    reg.put_blob("library/w", desc["digest"], str(d / "model.safetensors"))
    reg.put_manifest("library/w", "v1", m)
    got = cl.load_safetensors(reg, "library/w", "v1", "model.safetensors")
    for name, t in got.items():
        assert torch.equal(t, want[name]), name
    del got
    # a corrupted store blob
    dg = [b for b in rep["blobs"] if b["name"] == "model.safetensors"][0]["digest"]
    stored = tmp_path / "reg" / client.blob_digest_path("library/m", dg)
    with open(stored, "r+b") as f:
        f.seek(os.path.getsize(stored) // 2)
        b = f.read(1)
        f.seek(-1, 1)
        f.write(bytes([b[0] ^ 1]))
    with pytest.raises(DigestMismatch):
        cl.load_safetensors(reg, "library/m", "v1", "model.safetensors")
    cl.push(reg, "library/p", "v1", str(d))
    with pytest.raises(ValueError, match="--tree"):
        cl.load_safetensors(reg, "library/p", "v1", "model.safetensors")
