"""mxd_dev_tree_digest_extents -- the tree digest of a blob scattered over device buffers -- and modelx_b200.checkpoint,
which digests a safetensors checkpoint straight from its tensors.

Every result is compared with the CPU oracle's tree digest of the concatenated bytes.  The host logic runs on the CPU
test double (`-m "not gpu"`, numpy buffers) and on the H100 (`-m gpu`, torch buffers, k_tree_leaves_extents)."""
import ctypes as C
import random

import numpy as np
import pytest

import modelx_b200
from modelx_b200 import _native as N
from tests.checkpoint_fixtures import SMALL, header_in_order, llama_shapes
from tests.kernel_routes import UNSET, Out, _CudaBuf, _HostBuf, kernel_label
from tests.test_gpu_parity import TREE_CASES

EMPTY_ROOT = "fb9af61a9a239006147620a656344630ac38f49a0203a41630345e5ed2363195"   # docs/TREE_FORMAT.md
EMPTY_CHUNK = "75d7682c8b5955557b2ef33654f31512b9b3edd17f74b5bf422ccabbd7537e1a"  # tests/golden/tree_golden.json
SEED = 0x6D6F64656C78


class Arena:
    """Buffers the kernels read and write: torch tensors on the GPU, numpy arrays for the test double."""

    def __init__(self, backend):
        self.torch = None
        if backend is None:
            import torch
            assert torch.cuda.is_available(), "the cuda backend needs a CUDA device"
            torch.cuda.set_device(0)
            self.torch = torch

    def alloc(self, n):
        return _CudaBuf(self.torch, n) if self.torch else _HostBuf(n)

    def sync(self):
        if self.torch:
            self.torch.cuda.synchronize()


@pytest.fixture
def arena(backend):
    return Arena(backend)


def _align(x, a):
    return (x + a - 1) // a * a


def lay_out(arena, pieces):
    """pieces[i]: (bytes as uint8 array, start offset from a 256-aligned address) or ("same", j): extent j again.
    -> (extents [(ptr, len)], the concatenated bytes, keepalive)."""
    starts, pos = [], 256
    for p in pieces:
        if isinstance(p[0], str):
            starts.append(None)
            continue
        st = _align(pos + 16, 256) + p[1]
        starts.append(st)
        pos = st + len(p[0])
    buf = arena.alloc(pos + 64)
    buf.put(0, np.full(pos + 64, 0xEE, np.uint8))       # bytes between extents are not part of the blob
    extents, parts = [], []
    for p, st in zip(pieces, starts):
        if st is None:
            extents.append(extents[p[1]])
            parts.append(parts[p[1]])
            continue
        buf.put(st, p[0])
        extents.append((buf.ptr + st, len(p[0])))
        parts.append(p[0])
    data = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
    return extents, data, buf


def digest_extents(eng, arena, extents, chunk, leaf, fanout, with_chunks=True):
    """dev_tree_digest_extents into guarded, pre-filled outputs -> (chunk digests list or None, root)."""
    size = sum(n for _, n in extents)
    nch = max(1, -(-size // chunk))
    o_chunks = Out(arena, nch * 32) if with_chunks else None
    o_root = Out(arena, 32)
    eng.dev_tree_digest_extents(0, extents, (chunk, leaf, fanout), o_chunks.ptr if with_chunks else 0, o_root.ptr)
    arena.sync()
    root = o_root.take("root")
    if not with_chunks:
        return None, root
    raw = o_chunks.take("chunks")
    return [raw[32 * i:32 * i + 32] for i in range(nch)], root


def check(eng, arena, oracle, pieces, chunk, leaf, fanout):
    extents, data, keep = lay_out(arena, pieces)
    got = digest_extents(eng, arena, extents, chunk, leaf, fanout)
    want_chunks, _, want_root = oracle.tree_digest(np.ascontiguousarray(data), chunk, leaf, fanout)
    assert got == (want_chunks, want_root)
    return got


def rand_bytes(rng, n):
    return np.frombuffer(rng.randbytes(n), np.uint8) if n else np.zeros(0, np.uint8)


# ---- the empty blob ------------------------------------------------------------------------------------------------
def test_empty_blob(any_engine, arena, oracle):
    buf = arena.alloc(64)
    for extents in ([], [(0, 0)], [(buf.ptr, 0), (0, 0), (buf.ptr + 3, 0)]):
        chunks, root = digest_extents(any_engine, arena, extents, 8 << 20, 16 << 10, 8)
        assert root.hex() == EMPTY_ROOT and [c.hex() for c in chunks] == [EMPTY_CHUNK]
    want_chunks, _, want_root = oracle.tree_digest(b"", 8 << 20, 16 << 10, 8)
    assert (chunks, root) == (want_chunks, want_root)


# ---- one extent: the same as mxd_dev_tree_digest, launch for launch ------------------------------------------------
@pytest.mark.parametrize("size,off", [(1, 0), (1000, 3), (16384, 8), (100_003, 5), ((1 << 20) + 77, 12)])
def test_single_extent_equals_dev_tree_digest(any_engine, arena, oracle, size, off):
    rng = random.Random(size)
    tp = (1 << 16, 1024, 8)
    extents, data, keep = lay_out(arena, [(rand_bytes(rng, size), off)])
    s0 = any_engine.stats()
    got = digest_extents(any_engine, arena, extents, *tp)
    s1 = any_engine.stats()
    nch = len(got[0])
    o_chunks, o_root = Out(arena, nch * 32), Out(arena, 32)
    any_engine.dev_tree_digest(0, extents[0][0], size, tp, o_chunks.ptr, o_root.ptr)
    arena.sync()
    s2 = any_engine.stats()
    raw = o_chunks.take("chunks")
    assert got == ([raw[32 * i:32 * i + 32] for i in range(nch)], o_root.take("root"))
    want_chunks, _, want_root = oracle.tree_digest(data, *tp)
    assert got == (want_chunks, want_root)
    for key in ("kernel_launches", "bytes_hashed"):
        assert s1[key] - s0[key] == s2[key] - s1[key], key


# ---- lengths and start addresses -----------------------------------------------------------------------------------
LEAF, FANOUT = 1024, 4
CHUNK = LEAF * FANOUT * FANOUT


@pytest.mark.parametrize("off", range(16))
def test_lengths_at_every_offset(any_engine, arena, oracle, off):
    rng = random.Random(100 + off)
    lengths = [0, 1, 3, 8, 63, 64, 65, LEAF - 1, LEAF, LEAF + 1, CHUNK - 1, CHUNK, CHUNK + 1] + \
        [rng.randrange(1, 3 * LEAF) for _ in range(6)]
    rng.shuffle(lengths)
    # every extent at this offset, then the same lengths with offsets that differ from extent to extent
    check(any_engine, arena, oracle, [(rand_bytes(rng, n), off) for n in lengths], CHUNK, LEAF, FANOUT)
    check(any_engine, arena, oracle, [(rand_bytes(rng, n), (off + 7 * i) % 16) for i, n in enumerate(lengths)],
          CHUNK, LEAF, FANOUT)


def test_one_leaf_of_many_tiny_extents(any_engine, arena, oracle):
    rng = random.Random(7)
    pieces = [(rand_bytes(rng, 5000), 4)]
    pieces += [(rand_bytes(rng, rng.randrange(1, 9)), rng.randrange(16)) for _ in range(150)]   # < 1 leaf in all
    pieces += [(rand_bytes(rng, 3000), 9)]
    check(any_engine, arena, oracle, pieces, CHUNK, LEAF, FANOUT)
    check(any_engine, arena, oracle, pieces, 256, 64, 2)             # 64-byte leaves: every block crosses extents


def test_repeated_and_overlapping_extents(any_engine, arena, oracle):
    rng = random.Random(8)
    extents, data, keep = lay_out(arena, [(rand_bytes(rng, 5000), 3), (rand_bytes(rng, 2 * LEAF + 5), 0), ("same", 0)])
    a, b = extents[0], extents[1]
    extents += [(a[0] + 100, 2000), (a[0] + 1, 63)]                 # overlaps of extent 0
    host = np.concatenate([data, data[100:2100], data[1:64]])
    got = digest_extents(any_engine, arena, extents, CHUNK, LEAF, FANOUT)
    want_chunks, _, want_root = oracle.tree_digest(host, CHUNK, LEAF, FANOUT)
    assert got == (want_chunks, want_root)


def test_warps_with_mixed_alignments(any_engine, arena, oracle):
    """Extents of 2.4 leaves at changing offsets: the 32 leaves of a warp sit in extents of different address classes,
    and many of their blocks straddle two extents."""
    rng = random.Random(9)
    pieces = [(rand_bytes(rng, 2 * LEAF + 400 + rng.randrange(64)), rng.randrange(16)) for _ in range(60)]
    check(any_engine, arena, oracle, pieces, CHUNK, LEAF, FANOUT)


@pytest.mark.parametrize("mod16", [0, 8])
def test_safetensors_shaped_layout(any_engine, arena, oracle, mod16):
    rng = random.Random(10 + mod16)
    sizes = [("a", "F16", (64, 50), 6400), ("b", "F16", (4096,), 8192), ("c", "F32", (1000,), 4000),
             ("d", "F16", (3, 1024), 6144), ("e", "I8", (17,), 17), ("f", "F16", (2048, 5), 20480)]
    header = header_in_order(sizes, mod16)
    assert len(header) % 16 == mod16
    pieces = [(np.frombuffer(header, np.uint8), 0)] + [(rand_bytes(rng, n), 0) for *_, n in sizes]
    check(any_engine, arena, oracle, pieces, CHUNK, LEAF, FANOUT)


@pytest.mark.parametrize("size,chunk,leaf,fanout", TREE_CASES)
def test_tree_cases_split_into_extents(any_engine, arena, oracle, size, chunk, leaf, fanout):
    rng = random.Random(size * 31 + fanout)
    blob = np.frombuffer(oracle.gen(7, size, SEED), np.uint8) if size else np.zeros(0, np.uint8)
    cuts = sorted(rng.sample(range(size + 1), min(size + 1, 40)))
    bounds = [0] + cuts + [size]
    pieces = [(blob[a:b], rng.randrange(16)) for a, b in zip(bounds, bounds[1:])]
    check(any_engine, arena, oracle, pieces, chunk, leaf, fanout)


def test_without_chunk_output(any_engine, arena, oracle):
    rng = random.Random(11)
    extents, data, keep = lay_out(arena, [(rand_bytes(rng, 70_000), 5), (rand_bytes(rng, 33_333), 8)])
    _, root = digest_extents(any_engine, arena, extents, CHUNK, LEAF, FANOUT, with_chunks=False)
    assert root == oracle.tree_digest(data, CHUNK, LEAF, FANOUT)[2]


# ---- argument rejection: on the host, before anything is enqueued --------------------------------------------------
def test_rejects_bad_arguments(any_engine, arena):
    lib, ctx = any_engine._lib, any_engine.handle
    rng = random.Random(12)
    extents, data, keep = lay_out(arena, [(rand_bytes(rng, 5000), 0)])
    ptr = extents[0][0]
    nch = 4
    o_chunks, o_root = Out(arena, nch * 32), Out(arena, 32)
    good_tp = N.TreeParams(CHUNK, LEAF, FANOUT, 0)

    def call(ext, n=None, tp=good_tp, chunks=None, root=None, dev=0, handle=ctx, use_none=False):
        n = len(ext) if n is None else n
        arr = None if use_none else (N.Span * max(len(ext), 1))(*[N.Span(p, ln) for p, ln in ext])
        return lib.mxd_dev_tree_digest_extents(handle, dev, arr, n, C.byref(tp) if tp is not None else None,
                                               o_chunks.ptr if chunks is None else chunks,
                                               o_root.ptr if root is None else root, None)

    good = [(ptr, 5000)]
    cases = {
        "NULL handle": dict(ext=good, handle=None),
        "device index past the engine's devices": dict(ext=good, dev=any_engine.device_count()),
        "negative device index": dict(ext=good, dev=-1),
        "n > 0 with a NULL extent array": dict(ext=[], n=2, use_none=True),
        "NULL extent with a nonzero length": dict(ext=[(ptr, 10), (0, 5)]),
        "total length overflows": dict(ext=[(ptr, 1 << 63), (ptr, 1 << 63)]),
        "total length overflows by one": dict(ext=[(ptr, (1 << 64) - 1), (ptr + 1, 1)]),
        "reserved != 0": dict(ext=good, tp=N.TreeParams(CHUNK, LEAF, FANOUT, 1)),
        "leaf not a multiple of 64": dict(ext=good, tp=N.TreeParams(100 * 16, 100, 4, 0)),
        "chunk not leaf * fanout^k": dict(ext=good, tp=N.TreeParams(CHUNK + 64, LEAF, FANOUT, 0)),
        "fanout 1": dict(ext=good, tp=N.TreeParams(LEAF, LEAF, 1, 0)),
        "NULL root": dict(ext=good, root=0),
        "root misaligned": dict(ext=good, root=o_root.ptr + 8),
        "chunk digests misaligned": dict(ext=good, chunks=o_chunks.ptr + 4),
    }
    launches = any_engine.stats()["kernel_launches"]
    for what, kw in cases.items():
        assert call(**kw) == N.MXD_ERR_INVALID, what
    arena.sync()
    assert o_chunks.take("chunks", slot=0) == bytes([UNSET]) * (nch * 32)
    assert o_root.take("root", slot=0) == bytes([UNSET]) * 32
    assert any_engine.stats()["kernel_launches"] == launches
    with pytest.raises(modelx_b200.MxdError) as ei:
        any_engine.dev_tree_digest_extents(0, [(0, 1)], (CHUNK, LEAF, FANOUT), o_chunks.ptr, o_root.ptr)
    assert ei.value.status == N.MXD_ERR_INVALID
    assert call(good) == N.MXD_OK                                     # the same outputs work with good arguments
    arena.sync()
    o_root.take("root")


# ---- modelx_b200.checkpoint: header construction and validation (CPU) ----------------------------------------------
def _cpu_dict():
    import torch
    return {"w": torch.zeros(4, 6, dtype=torch.float16), "b": torch.zeros(5, dtype=torch.float32),
            "i": torch.zeros(3, dtype=torch.int8), "e": torch.zeros(0, 3, dtype=torch.bfloat16)}


def test_safetensors_layout_header():
    from modelx_b200.checkpoint import parse_safetensors_header, safetensors_layout
    for meta in (None, {"format": "pt"}, {"k": "v" * 13}):
        header, names = safetensors_layout(_cpu_dict(), meta)
        assert len(header) % 8 == 0
        entries, payload = parse_safetensors_header(header)
        assert names == ["b", "e", "w", "i"]              # largest element size first, then by name
        assert payload == 5 * 4 + 0 + 24 * 2 + 3
        assert [entries[n]["data_offsets"][0] for n in names] == [0, 20, 20, 68]
        assert entries["w"] == {"dtype": "F16", "shape": [4, 6], "data_offsets": [20, 68]}
    with pytest.raises(ValueError, match="not contiguous"):
        safetensors_layout({"t": _cpu_dict()["w"].t()})


def _header(doc, pad=True):
    import json
    import struct
    text = json.dumps(doc).encode()
    if pad:
        text += b" " * (-len(text) % 8)
    return struct.pack("<Q", len(text)) + text


def test_header_validation_rejects():
    from modelx_b200.checkpoint import parse_safetensors_header
    ok = {"a": {"dtype": "F16", "shape": [2], "data_offsets": [0, 4]}, "b": {"dtype": "U8", "shape": [3], "data_offsets": [4, 7]}}
    assert parse_safetensors_header(_header(ok))[1] == 7
    bad = {
        "gap": {**ok, "b": {"dtype": "U8", "shape": [3], "data_offsets": [5, 8]}},
        "overlap": {**ok, "b": {"dtype": "U8", "shape": [3], "data_offsets": [3, 6]}},
        "does not start at 0": {"a": {"dtype": "F16", "shape": [2], "data_offsets": [4, 8]}},
        "size disagrees with shape": {"a": {"dtype": "F16", "shape": [3], "data_offsets": [0, 4]}},
        "unknown dtype": {"a": {"dtype": "F17", "shape": [2], "data_offsets": [0, 4]}},
        "offsets malformed": {"a": {"dtype": "F16", "shape": [2], "data_offsets": [0]}},
    }
    for what, doc in bad.items():
        with pytest.raises(ValueError, match="safetensors header"):
            parse_safetensors_header(_header(doc))
    h = _header(ok)
    for what, raw in {"truncated": h[:-3], "trailing bytes": h + b"  ", "shorter than 8": h[:5]}.items():
        with pytest.raises(ValueError, match="safetensors header"):
            parse_safetensors_header(raw)
    unpadded = b"{\"a\":{\"dtype\":\"U8\",\"shape\":[1],\"data_offsets\":[0,1]}}"
    assert len(unpadded) % 8
    with pytest.raises(ValueError, match="not padded"):
        parse_safetensors_header(len(unpadded).to_bytes(8, "little") + unpadded)


def test_tensor_mismatch_rejects(mock_lib):
    import torch
    from modelx_b200.checkpoint import safetensors_layout, tree_digest_safetensors
    eng = modelx_b200.Engine(devices=[0], lib_path=mock_lib)
    try:
        t = _cpu_dict()
        header, _ = safetensors_layout(t)
        cases = {
            "missing": ({k: v for k, v in t.items() if k != "b"}, "missing \\['b'\\]"),
            "extra": ({**t, "z": torch.zeros(1)}, "not in the header \\['z'\\]"),
            "dtype": ({**t, "b": torch.zeros(5, dtype=torch.int32)}, "dtype I32 but the header says F32"),
            "shape": ({**t, "w": torch.zeros(6, 4, dtype=torch.float16)}, "shape \\[6, 4\\] but the header says \\[4, 6\\]"),
            "non-contiguous": ({**t, "w": torch.zeros(6, 4, dtype=torch.float16).t()}, "not contiguous"),
            "not on a GPU": (t, "all tensors must be on one CUDA device"),
        }
        for what, (tensors, msg) in cases.items():
            with pytest.raises(ValueError, match=msg):
                tree_digest_safetensors(eng, header, tensors)
        with pytest.raises(ValueError, match="safetensors header"):
            tree_digest_safetensors(eng, header[:-1], t)
    finally:
        eng.close()


# ---- GPU only ------------------------------------------------------------------------------------------------------
def _torch():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    torch.cuda.set_device(0)
    return torch


@pytest.mark.gpu
def test_leaf_level_runs_the_extents_kernel(engine, oracle):
    torch = _torch()
    from torch.profiler import ProfilerActivity, profile
    arena = Arena(None)
    rng = random.Random(13)
    pieces = [(rand_bytes(rng, 300_000 + i), i % 16) for i in range(8)]
    extents, data, keep = lay_out(arena, pieces)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.ones(1, device="cuda").add_(1)
        got = digest_extents(engine, arena, extents, CHUNK, LEAF, FANOUT)
        torch.cuda.synchronize()
    names = [e.name for e in sorted(prof.events(), key=lambda e: e.time_range.start)
             if "k_tree_leaves_extents" in e.name or kernel_label(e.name)]
    assert names and "k_tree_leaves_extents" in names[0], names
    assert sum("k_tree_leaves_extents" in n for n in names) == 1, names
    assert got == tuple(oracle.tree_digest(data, CHUNK, LEAF, FANOUT)[::2])


def _fill_dict(torch, eng, shapes, seed, odd=None):
    """fp16 tensors filled by dev_gen_fill (plus an optional odd-length int8 tensor) -> {name: tensor}"""
    out = {}
    st = torch.cuda.current_stream().cuda_stream
    for i, (name, shape) in enumerate(shapes):
        t = torch.empty(shape, dtype=torch.float16, device="cuda")
        eng.dev_gen_fill(0, t.data_ptr(), 0, t.numel() * 2, seed + i, st)
        out[name] = t
    if odd:
        g = torch.Generator(device="cuda").manual_seed(seed)
        out["odd.int8"] = torch.randint(-128, 128, (odd,), dtype=torch.int8, device="cuda", generator=g)
    return out


def _specs(tensors, order):
    return [(n, "I8" if tensors[n].dtype.itemsize == 1 else "F16", tuple(tensors[n].shape),
             tensors[n].numel() * tensors[n].element_size()) for n in order]


def _gathered_digest(torch, eng, header, tensors, order, tp):
    """mxd_dev_tree_digest of header + tensors copied into one buffer: the existing contiguous path"""
    size = len(header) + sum(tensors[n].numel() * tensors[n].element_size() for n in order)
    buf = torch.empty(size, dtype=torch.uint8, device="cuda")
    buf[:len(header)].copy_(torch.frombuffer(bytearray(header), dtype=torch.uint8))
    pos = len(header)
    for n in order:
        nb = tensors[n].numel() * tensors[n].element_size()
        buf[pos:pos + nb].copy_(tensors[n].reshape(-1).view(torch.uint8))
        pos += nb
    nch = -(-size // tp[0])
    out = torch.empty(nch * 32 + 32, dtype=torch.uint8, device="cuda")
    eng.dev_tree_digest(0, buf.data_ptr(), size, tp, out.data_ptr(), out.data_ptr() + nch * 32,
                        torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    del buf
    raw = out.cpu().numpy().tobytes()
    return [raw[32 * i:32 * i + 32] for i in range(nch)], raw[nch * 32:], size


@pytest.mark.gpu
def test_llama_8b_shaped_checkpoint_equals_gathered_copy(engine):
    """About 16 GB in 291 tensors: header lengths = 0 and 8 mod 16, and an odd-length int8 tensor in front of the
    rest.  The extents path must equal mxd_dev_tree_digest of the same bytes gathered into one buffer."""
    torch = _torch()
    from modelx_b200.checkpoint import tree_digest_safetensors
    tp = (8 << 20, 16 << 10, 8)
    shapes = llama_shapes()
    tensors = _fill_dict(torch, engine, shapes, SEED, odd=4097)
    names = [n for n, _ in shapes]
    layouts = [(names, 0), (names, 8), (["odd.int8"] + names, 8)]
    for order, mod16 in layouts:
        header = header_in_order(_specs(tensors, order), mod16)
        sub = {n: tensors[n] for n in order}
        got = tree_digest_safetensors(engine, header, sub, *tp)
        want = _gathered_digest(torch, engine, header, tensors, order, tp)
        assert got[2] == want[2] > 16e9
        assert got[1] == want[1], (mod16, len(order))
        assert got[0] == want[0], (mod16, len(order))


@pytest.fixture(scope="module")
def small_dict():
    torch = _torch()
    import modelx_b200 as m
    with m.Engine(devices=[0]) as eng:
        tensors = _fill_dict(torch, eng, llama_shapes(**SMALL), SEED + 1000)
        torch.cuda.synchronize()
    return tensors


@pytest.mark.gpu
def test_file_of_the_same_bytes(engine, small_dict, tmp_path):
    torch = _torch()
    from modelx_b200.checkpoint import safetensors_layout, tree_digest_safetensors
    header, names = safetensors_layout(small_dict, {"format": "pt"})
    got = tree_digest_safetensors(engine, header, small_dict)
    path = str(tmp_path / "model.safetensors")
    with open(path, "wb") as f:
        f.write(header)
        for n in names:
            f.write(small_dict[n].reshape(-1).view(torch.uint8).cpu().numpy().tobytes())
    assert got == engine.tree_digest_file(path)
    assert got[2] > 0.9e9 and len(got[0]) == -(-got[2] // (8 << 20))
    st = pytest.importorskip("safetensors.torch")
    back = st.load_file(path)
    assert sorted(back) == sorted(small_dict)
    for n, t in small_dict.items():
        assert torch.equal(back[n].view(torch.uint8), t.cpu().view(torch.uint8)), n


@pytest.mark.gpu
def test_file_written_by_safetensors(engine, small_dict, tmp_path):
    torch = _torch()
    st = pytest.importorskip("safetensors.torch")
    from modelx_b200.checkpoint import tree_digest_safetensors
    path = str(tmp_path / "saved.safetensors")
    st.save_file({n: t.cpu() for n, t in small_dict.items()}, path, metadata={"format": "pt"})
    with open(path, "rb") as f:
        n = int.from_bytes(f.read(8), "little")
        header = n.to_bytes(8, "little") + f.read(n)
    loaded = {k: v.to("cuda") for k, v in st.load_file(path).items()}
    assert tree_digest_safetensors(engine, header, loaded) == engine.tree_digest_file(path)


@pytest.mark.gpu
def test_one_flipped_byte_changes_one_chunk(engine, small_dict):
    torch = _torch()
    from modelx_b200.checkpoint import parse_safetensors_header, safetensors_layout, tree_digest_safetensors
    header, names = safetensors_layout(small_dict)
    chunks, root, size = tree_digest_safetensors(engine, header, small_dict)
    entries, _ = parse_safetensors_header(header)
    name = names[len(names) // 2]
    t = small_dict[name].reshape(-1).view(torch.uint8)
    i = t.numel() // 3 + 5
    pos = len(header) + entries[name]["data_offsets"][0] + i
    old = t[i].item()
    t[i] = old ^ 0x40
    try:
        chunks2, root2, size2 = tree_digest_safetensors(engine, header, small_dict)
    finally:
        t[i] = old
    assert size2 == size and root2 != root
    assert [k for k in range(len(chunks)) if chunks[k] != chunks2[k]] == [pos // (8 << 20)]
    assert tree_digest_safetensors(engine, header, small_dict) == (chunks, root, size)
