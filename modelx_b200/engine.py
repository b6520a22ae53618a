"""Thin object wrapper over the C ABI: one ``Engine`` = one ``mxd_ctx``.

Everything here forwards to libmodelxdigest.so; no hashing happens in Python.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, List, Optional, Sequence, Tuple

from . import _native as N

DEFAULT_CHUNK = 8 << 20   # bytes covered by one chunk digest (the list a manifest carries)
DEFAULT_LEAF = 16 << 10   # bytes hashed by one GPU lane at the bottom of the tree
DEFAULT_FANOUT = 8        # digests per upper-level node; chunk = leaf * fanout**k


def _tp(chunk: int, leaf: int, fanout: int):
    return C.byref(N.TreeParams(chunk, leaf, fanout, 0))


def _buf(data):
    """(address, nbytes, keepalive) of a bytes-like / numpy array without copying when possible."""
    if isinstance(data, bytes):
        # pointer to the bytes object's own storage (no copy; valid while `data` is referenced by the caller)
        n = len(data)
        return (C.cast(C.c_char_p(data), C.c_void_p).value or 0), n, data
    if isinstance(data, bytearray):
        n = len(data)
        keep = (C.c_char * max(n, 1)).from_buffer(data)
        return C.addressof(keep), n, keep
    mv = memoryview(data)
    if not mv.contiguous:
        raise ValueError("buffer must be contiguous")
    n = mv.nbytes
    if hasattr(data, "ctypes"):  # numpy
        return data.ctypes.data, n, data
    keep = (C.c_char * max(n, 1)).from_buffer(mv) if not mv.readonly else C.create_string_buffer(mv.tobytes(), max(n, 1))
    return C.addressof(keep), n, keep


def digest_string(d: bytes) -> str:
    """go-digest string form: ``sha256:<hex>`` (what Descriptor.Digest carries, pkg/types/types.go:31)."""
    out = C.create_string_buffer(72)
    N.load().mxd_digest_string((C.c_uint8 * 32).from_buffer_copy(d), out)
    return out.value.decode()


def digest_parse(s: str) -> bytes:
    out = (C.c_uint8 * 32)()
    N.check(N.load().mxd_digest_parse(s.encode(), out), "mxd_digest_parse")
    return bytes(out)


def calc_parts(total: int, partscount: int) -> List[Tuple[int, int]]:
    """calcParts (pkg/client/extension_s3.go:99-112): [(offset, length)] for each part."""
    lib = N.load()
    if partscount > 0:
        parts = (N.Part * partscount)()
    else:
        parts = (N.Part * 1)()
    rc = lib.mxd_calc_parts(total, partscount, parts)
    if rc == N.MXD_ERR_DIV_ZERO:
        raise ZeroDivisionError("calcParts: integer divide by zero")   # the reference panics here
    N.check(rc, "mxd_calc_parts")
    return [(p.offset, p.length) for p in parts[:partscount]]


def batch_pays_off(n_blobs: int, total_bytes: int, max_blob_bytes: int = 0) -> bool:
    """Routing advice (mxd_batch_pays_off): is hashing these blobs together on the GPU expected to beat the
    reference's three SHA-NI goroutines?"""
    return bool(N.load().mxd_batch_pays_off(n_blobs, total_bytes, max_blob_bytes))


def server_part_count(size: int, force_multipart: bool = False) -> int:
    """Part count the modelxd S3 store chooses (pkg/registry/store_s3.go:198-203, 273-279)."""
    return int(N.load().mxd_server_part_count(size, 1 if force_multipart else 0))


def tree_shape(size: int, chunk: int = DEFAULT_CHUNK, leaf: int = DEFAULT_LEAF, fanout: int = DEFAULT_FANOUT) -> List[int]:
    """Node count per level, leaves first (level k, where chunk = leaf*fanout**k, is the chunk list)."""
    counts = (C.c_uint64 * 80)()
    klevel = C.c_int()
    lv = N.load().mxd_tree_shape(size, _tp(chunk, leaf, fanout), counts, 80, C.byref(klevel))
    if lv < 0:
        raise N.MxdError(lv, "mxd_tree_shape")
    return [int(counts[i]) for i in range(lv)]


class Engine:
    """One process-wide digest engine bound to one or more GPUs."""

    def __init__(self, devices: Optional[Sequence[int]] = None, ring_bytes: int = 0, lib_path: Optional[str] = None):
        self._lib = N.load(lib_path)
        self._ctx = C.c_void_p()
        self._parent = None
        devs = list(devices) if devices is not None else []
        self._devices = devs
        arr = (C.c_int * max(len(devs), 1))(*devs)
        self._check(self._lib.mxd_open(C.byref(self._ctx), arr if devs else None, len(devs), ring_bytes), "mxd_open")

    def _check(self, status: int, where: str):
        N.check(status, where, self._lib)

    def op(self) -> "Engine":
        """A new operation on this engine (mxd_op_begin): an Engine-shaped handle sharing the devices whose calls
        can be canceled on their own with ``.cancel()`` (one Go context, push.go:150-159).  Use as a context manager."""
        child = object.__new__(Engine)
        child._lib = self._lib
        child._ctx = C.c_void_p()
        child._parent = self
        child._devices = self._devices
        self._check(self._lib.mxd_op_begin(self._ctx, C.byref(child._ctx)), "mxd_op_begin")
        import weakref
        if not hasattr(self, "_children"):
            self._children = []
        self._children.append(weakref.ref(child))     # ended with the engine if the caller forgets (a handle must not outlive its context)
        return child

    # -- lifecycle ---------------------------------------------------------------------------
    def close(self):
        if self._ctx:
            if self._parent is not None:
                self._lib.mxd_op_end(self._ctx)
            else:
                for ref in getattr(self, "_children", []):
                    child = ref()
                    if child is not None:
                        child.close()
                self._lib.mxd_close(self._ctx)
            self._ctx = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def handle(self):
        return self._ctx

    def device_count(self) -> int:
        return self._lib.mxd_device_count(self._ctx)

    def device_index(self, ordinal: int) -> int:
        """The `dev` argument of the dev_* calls for CUDA device `ordinal`; ValueError if the engine does not drive it."""
        devs = self._devices or list(range(self.device_count()))
        if ordinal not in devs:
            raise ValueError(f"cuda:{ordinal} is not one of this engine's devices {devs}")
        return devs.index(ordinal)

    def stats(self) -> dict:
        st = N.Stats()
        self._check(self._lib.mxd_get_stats(self._ctx, C.byref(st)), "mxd_get_stats")
        return {"kernel_launches": st.kernel_launches, "bytes_hashed": st.bytes_hashed,
                "h2d_bytes": st.h2d_bytes, "d2h_bytes": st.d2h_bytes, "src_bytes_read": st.src_bytes_read,
                "open_files": st.open_files}

    def trace_enable(self, on: bool = True):
        self._check(self._lib.mxd_trace_enable(self._ctx, 1 if on else 0), "mxd_trace_enable")

    def trace_dump(self, path: str):
        self._check(self._lib.mxd_trace_dump(self._ctx, path.encode()), "mxd_trace_dump")

    def prof_enable(self, on: bool = True):
        self._check(self._lib.mxd_prof_enable(self._ctx, 1 if on else 0), "mxd_prof_enable")

    def prof_read(self) -> dict:
        ms, n, b = C.c_double(), C.c_uint64(), C.c_uint64()
        self._check(self._lib.mxd_prof_read(self._ctx, C.byref(ms), C.byref(n), C.byref(b)), "mxd_prof_read")
        return {"kernel_ms": ms.value, "launches": n.value, "bytes": b.value}

    def cancel(self):
        self._lib.mxd_cancel(self._ctx)

    def reset_cancel(self):
        self._lib.mxd_reset_cancel(self._ctx)

    def is_canceled(self) -> bool:
        return bool(self._lib.mxd_is_canceled(self._ctx))

    # -- whole-message digests (reference semantics) --------------------------------------------
    def sha256(self, data) -> bytes:
        addr, n, keep = _buf(data)
        out = (C.c_uint8 * 32)()
        self._check(self._lib.mxd_sha256(self._ctx, addr, n, out), "mxd_sha256")
        return bytes(out)

    def sha256_ptr(self, ptr: int, n: int) -> bytes:
        out = (C.c_uint8 * 32)()
        self._check(self._lib.mxd_sha256(self._ctx, ptr, n, out), "mxd_sha256")
        return bytes(out)

    def sha256_batch(self, items: Iterable) -> List[bytes]:
        bufs = [_buf(x) for x in items]
        n = len(bufs)
        spans = (N.Span * max(n, 1))()
        for i, (addr, ln, _) in enumerate(bufs):
            spans[i].ptr = addr
            spans[i].len = ln
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self._lib.mxd_sha256_batch(self._ctx, spans, n, out), "mxd_sha256_batch")
        raw = bytes(out)
        return [raw[32 * i:32 * i + 32] for i in range(n)]

    def sha256_batch_ptrs(self, spans_list: Sequence[Tuple[int, int]]) -> List[bytes]:
        n = len(spans_list)
        spans = (N.Span * max(n, 1))()
        for i, (addr, ln) in enumerate(spans_list):
            spans[i].ptr = addr
            spans[i].len = ln
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self._lib.mxd_sha256_batch(self._ctx, spans, n, out), "mxd_sha256_batch")
        raw = bytes(out)
        return [raw[32 * i:32 * i + 32] for i in range(n)]

    def sha256_file(self, path: str) -> Tuple[bytes, int]:
        out = (C.c_uint8 * 32)()
        size = C.c_uint64()
        self._check(self._lib.mxd_sha256_file(self._ctx, path.encode(), out, C.byref(size)), "mxd_sha256_file")
        return bytes(out), size.value

    def sha256_files(self, paths: Sequence[str]) -> Tuple[List[bytes], List[int]]:
        n = len(paths)
        arr = (C.c_char_p * max(n, 1))(*[p.encode() for p in paths])
        out = (C.c_uint8 * (32 * max(n, 1)))()
        sizes = (C.c_uint64 * max(n, 1))()
        self._check(self._lib.mxd_sha256_files(self._ctx, arr, n, out, sizes), "mxd_sha256_files")
        raw = bytes(out)
        return [raw[32 * i:32 * i + 32] for i in range(n)], [int(sizes[i]) for i in range(n)]

    def sha256_file_jobs(self, jobs: Sequence[dict]) -> List[dict]:
        """The general per-file form (mxd_sha256_file_jobs).  Each job: {"path": str, "ranges": [(off, len)...] or
        None, "sink": callable(offset, bytes) or None}.  Returns per job {"status", "size", "digests": [bytes]};
        never raises for a per-file failure."""
        n = len(jobs)
        arr = (N.FileJob * max(n, 1))()
        keep = []
        for i, jb in enumerate(jobs):
            rng = jb.get("ranges") or []
            parts = (N.Part * max(len(rng), 1))()
            for k, (off, ln) in enumerate(rng):
                parts[k].offset, parts[k].length = off, ln
            out = (C.c_uint8 * (32 * max(len(rng), 1)))()
            path = jb["path"].encode()
            cb = None
            if jb.get("sink"):
                sink = jb["sink"]

                def _cb(user, offset, data, nbytes, sink=sink):
                    try:
                        sink(offset, C.string_at(data, nbytes))
                        return 0
                    except Exception:
                        return 1
                cb = N.SINK_FN(_cb)
            arr[i].path = path
            arr[i].ranges = parts if rng else None
            arr[i].nranges = len(rng)
            arr[i].out = C.cast(out, C.POINTER(C.c_uint8))
            arr[i].sink = C.cast(cb, C.c_void_p) if cb else None
            keep.append((parts, out, path, cb))
        self._lib.mxd_sha256_file_jobs(self._ctx, arr, n)
        res = []
        for i in range(n):
            raw = bytes(keep[i][1])
            res.append({"status": arr[i].status, "size": arr[i].size,
                        "digests": [raw[32 * k:32 * k + 32] for k in range(len(raw) // 32)]})
        return res

    def sha256_file_ranges(self, path: str, ranges: Sequence[Tuple[int, int]], sink=None):
        """SHA-256 of each (offset, length) range of one file in ONE pass, optionally teeing every byte to
        ``sink(offset, data)``.  -> (digests, size)"""
        r = self.sha256_file_jobs([{"path": path, "ranges": list(ranges), "sink": sink}])[0]
        self._check(r["status"], "mxd_sha256_file_jobs")
        return r["digests"][:len(ranges)], r["size"]

    def sha256_file_parts(self, path: str, parts: Sequence[Tuple[int, int]]) -> List[bytes]:
        """SHA-256 of each (offset, length) range of a file, e.g. the ranges calc_parts() yields."""
        n = len(parts)
        arr = (N.Part * max(n, 1))()
        for i, (off, ln) in enumerate(parts):
            arr[i].offset, arr[i].length = off, ln
        out = (C.c_uint8 * (32 * max(n, 1)))()
        self._check(self._lib.mxd_sha256_file_parts(self._ctx, path.encode(), arr, n, out), "mxd_sha256_file_parts")
        raw = bytes(out)
        return [raw[32 * i:32 * i + 32] for i in range(n)]

    def verify_batch(self, items: Iterable, want: Sequence[bytes]) -> List[bool]:
        bufs = [_buf(x) for x in items]
        n = len(bufs)
        spans = (N.Span * max(n, 1))()
        for i, (addr, ln, _) in enumerate(bufs):
            spans[i].ptr = addr
            spans[i].len = ln
        w = (C.c_uint8 * (32 * max(n, 1))).from_buffer_copy(b"".join(want) + b"\0" * (32 * max(n, 1) - 32 * n))
        ok = (C.c_uint8 * max(n, 1))()
        self._check(self._lib.mxd_verify_batch(self._ctx, spans, w, n, ok), "mxd_verify_batch")
        return [bool(ok[i]) for i in range(n)]

    def verify_files(self, paths: Sequence[str], want: Sequence[bytes]) -> List[bool]:
        n = len(paths)
        arr = (C.c_char_p * max(n, 1))(*[p.encode() for p in paths])
        w = (C.c_uint8 * (32 * max(n, 1))).from_buffer_copy(b"".join(want) + b"\0" * (32 * max(n, 1) - 32 * n))
        ok = (C.c_uint8 * max(n, 1))()
        self._check(self._lib.mxd_verify_files(self._ctx, arr, w, n, ok), "mxd_verify_files")
        return [bool(ok[i]) for i in range(n)]

    # -- incremental hasher ------------------------------------------------------------------
    def hasher(self) -> "Hasher":
        return Hasher(self)

    # -- tree digests ------------------------------------------------------------------------
    def tree_digest(self, data, chunk: int = DEFAULT_CHUNK, leaf: int = DEFAULT_LEAF, fanout: int = DEFAULT_FANOUT):
        """-> (chunk_digests: list[bytes], root: bytes) for a bytes-like blob in host memory."""
        addr, n, keep = _buf(data)
        return self.tree_digest_ptr(addr, n, chunk, leaf, fanout)

    def tree_digest_ptr(self, ptr: int, n: int, chunk: int = DEFAULT_CHUNK, leaf: int = DEFAULT_LEAF,
                        fanout: int = DEFAULT_FANOUT):
        nch = max(1, -(-n // chunk))
        chunks = (C.c_uint8 * (32 * nch))()
        got = C.c_uint64()
        root = (C.c_uint8 * 32)()
        self._check(self._lib.mxd_tree_digest(self._ctx, ptr, n, _tp(chunk, leaf, fanout), chunks, C.byref(got), root),
                "mxd_tree_digest")
        raw = bytes(chunks)
        return [raw[32 * i:32 * i + 32] for i in range(got.value)], bytes(root)

    def tree_digest_file(self, path: str, chunk: int = DEFAULT_CHUNK, leaf: int = DEFAULT_LEAF,
                         fanout: int = DEFAULT_FANOUT):
        import os
        size = os.stat(path).st_size
        nch = max(1, -(-size // chunk))
        chunks = (C.c_uint8 * (32 * nch))()
        got = C.c_uint64()
        sz = C.c_uint64()
        root = (C.c_uint8 * 32)()
        self._check(self._lib.mxd_tree_digest_file(self._ctx, path.encode(), _tp(chunk, leaf, fanout), chunks, nch,
                                               C.byref(got), C.byref(sz), root), "mxd_tree_digest_file")
        raw = bytes(chunks)
        return [raw[32 * i:32 * i + 32] for i in range(got.value)], bytes(root), sz.value

    def tree_digest_file_tee(self, path: str, sink, chunk: int = DEFAULT_CHUNK, leaf: int = DEFAULT_LEAF,
                             fanout: int = DEFAULT_FANOUT):
        """Read-once digest: ``sink(offset, data: bytes)`` receives every piece that streams through the ring
        (possibly from several threads, any order).  -> (chunk_digests, root, size)"""
        import os
        size = os.stat(path).st_size
        nch = max(1, -(-size // chunk))
        chunks = (C.c_uint8 * (32 * nch))()
        got, sz = C.c_uint64(), C.c_uint64()
        root = (C.c_uint8 * 32)()

        def _cb(user, offset, data, nbytes):
            try:
                sink(offset, C.string_at(data, nbytes))
                return 0
            except Exception:
                return 1
        cb = N.SINK_FN(_cb)
        self._check(self._lib.mxd_tree_digest_file_tee(self._ctx, path.encode(), _tp(chunk, leaf, fanout), chunks, nch,
                                                   C.byref(got), C.byref(sz), root, C.cast(cb, C.c_void_p), None),
                "mxd_tree_digest_file_tee")
        raw = bytes(chunks)
        return [raw[32 * i:32 * i + 32] for i in range(got.value)], bytes(root), sz.value

    def tree_load_file(self, dev: int, path: str, extents: Sequence[Tuple[int, int]], chunk: int = DEFAULT_CHUNK,
                       leaf: int = DEFAULT_LEAF, fanout: int = DEFAULT_FANOUT):
        """Copy the file into the device spans [(ptr, nbytes), ...] on device index `dev`, whose lengths must add up to
        the file size, and tree-digest the bytes that landed there (mxd_tree_load_file).  Synchronous; nothing else
        may touch the spans during the call.  -> (chunk_digests, root, size), as ``tree_digest_file`` of the file."""
        import os
        try:
            size = os.stat(path).st_size
        except OSError:
            size = 0                  # the call reports the missing file
        n = len(extents)
        arr = (N.Span * max(n, 1))(*[N.Span(p, ln) for p, ln in extents])
        nch = max(1, -(-size // chunk))
        chunks = (C.c_uint8 * (32 * nch))()
        got, sz = C.c_uint64(), C.c_uint64()
        root = (C.c_uint8 * 32)()
        self._check(self._lib.mxd_tree_load_file(self._ctx, dev, path.encode(), arr if n else None, n, _tp(chunk, leaf, fanout),
                                                 chunks, nch, C.byref(got), C.byref(sz), root), "mxd_tree_load_file")
        raw = bytes(chunks)
        return [raw[32 * i:32 * i + 32] for i in range(got.value)], bytes(root), sz.value

    def tree_chunks_ptr(self, ptr: int, n: int, chunk: int = DEFAULT_CHUNK, leaf: int = DEFAULT_LEAF,
                        fanout: int = DEFAULT_FANOUT) -> bytes:
        nch = max(1, -(-n // chunk))
        chunks = (C.c_uint8 * (32 * nch))()
        self._check(self._lib.mxd_tree_chunks(self._ctx, ptr, n, _tp(chunk, leaf, fanout), chunks), "mxd_tree_chunks")
        return bytes(chunks)

    def tree_digest_files(self, paths: Sequence[str], chunk: int = DEFAULT_CHUNK, leaf: int = DEFAULT_LEAF,
                          fanout: int = DEFAULT_FANOUT):
        """Tree roots of many files in one pipelined pass -> (roots, sizes, statuses); per-file failures do not raise."""
        n = len(paths)
        arr = (C.c_char_p * max(n, 1))(*[p.encode() for p in paths])
        roots = (C.c_uint8 * (32 * max(n, 1)))()
        sizes = (C.c_uint64 * max(n, 1))()
        status = (C.c_int * max(n, 1))()
        rc = self._lib.mxd_tree_digest_files(self._ctx, arr, n, _tp(chunk, leaf, fanout), roots, sizes, status)
        if rc != 0 and all(status[i] == 0 for i in range(n)):
            self._check(rc, "mxd_tree_digest_files")
        raw = bytes(roots)
        return [raw[32 * i:32 * i + 32] for i in range(n)], [int(sizes[i]) for i in range(n)], [int(status[i]) for i in range(n)]

    def tree_chunks_file(self, path: str, offset: int, nbytes: int, chunk: int = DEFAULT_CHUNK, leaf: int = DEFAULT_LEAF,
                         fanout: int = DEFAULT_FANOUT) -> bytes:
        """Chunk digests of bytes [offset, offset+nbytes) of a file (offset on a chunk boundary): a rank's share."""
        nch = max(1, -(-nbytes // chunk))
        chunks = (C.c_uint8 * (32 * nch))()
        self._check(self._lib.mxd_tree_chunks_file(self._ctx, path.encode(), offset, nbytes, _tp(chunk, leaf, fanout), chunks),
                    "mxd_tree_chunks_file")
        return bytes(chunks)

    def tree_chunks(self, data, chunk: int = DEFAULT_CHUNK, leaf: int = DEFAULT_LEAF, fanout: int = DEFAULT_FANOUT) -> bytes:
        addr, n, keep = _buf(data)
        return self.tree_chunks_ptr(addr, n, chunk, leaf, fanout)

    def tree_finish(self, chunk_digests: bytes, size: int, chunk: int = DEFAULT_CHUNK, leaf: int = DEFAULT_LEAF,
                    fanout: int = DEFAULT_FANOUT) -> bytes:
        n = len(chunk_digests) // 32
        arr = (C.c_uint8 * len(chunk_digests)).from_buffer_copy(chunk_digests)
        root = (C.c_uint8 * 32)()
        self._check(self._lib.mxd_tree_finish(self._ctx, arr, n, size, _tp(chunk, leaf, fanout), root), "mxd_tree_finish")
        return bytes(root)

    # -- device-resident asynchronous forms (raw device pointers, cudaStream_t as int) -----------
    def dev_sha256_segments(self, dev: int, d_data: int, nbytes: int, seg: int, d_out: int, stream: int = 0):
        self._check(self._lib.mxd_dev_sha256_segments(self._ctx, dev, d_data, nbytes, seg, d_out, stream), "mxd_dev_sha256_segments")

    def dev_sha256_batch(self, dev: int, d_spans: int, n: int, d_out: int, stream: int = 0):
        self._check(self._lib.mxd_dev_sha256_batch(self._ctx, dev, d_spans, n, d_out, stream), "mxd_dev_sha256_batch")

    def dev_tree_chunks(self, dev: int, d_piece: int, nbytes: int, tp: Tuple[int, int, int], d_chunks: int, stream: int = 0):
        """tp = (chunk, leaf, fanout)"""
        self._check(self._lib.mxd_dev_tree_chunks(self._ctx, dev, d_piece, nbytes, _tp(*tp), d_chunks, stream), "mxd_dev_tree_chunks")

    def dev_tree_finish(self, dev: int, d_chunks: int, nchunks: int, size: int, tp: Tuple[int, int, int], d_root: int, stream: int = 0):
        self._check(self._lib.mxd_dev_tree_finish(self._ctx, dev, d_chunks, nchunks, size, _tp(*tp), d_root, stream), "mxd_dev_tree_finish")

    def dev_tree_digest(self, dev: int, d_data: int, size: int, tp: Tuple[int, int, int], d_chunks: int, d_root: int, stream: int = 0):
        self._check(self._lib.mxd_dev_tree_digest(self._ctx, dev, d_data, size, _tp(*tp), d_chunks, d_root, stream), "mxd_dev_tree_digest")

    def dev_tree_digest_extents(self, dev: int, extents: Sequence[Tuple[int, int]], tp: Tuple[int, int, int], d_chunks: int,
                                d_root: int, stream: int = 0):
        """Tree digest of the concatenation of device spans [(ptr, nbytes), ...] (mxd_dev_tree_digest_extents);
        d_chunks may be 0.  Asynchronous on `stream`."""
        n = len(extents)
        arr = (N.Span * max(n, 1))(*[N.Span(p, ln) for p, ln in extents])
        self._check(self._lib.mxd_dev_tree_digest_extents(self._ctx, dev, arr if n else None, n, _tp(*tp), d_chunks, d_root, stream),
                    "mxd_dev_tree_digest_extents")

    def dev_compare(self, dev: int, d_got: int, d_want: int, n: int, d_ok: int, stream: int = 0):
        self._check(self._lib.mxd_dev_compare(self._ctx, dev, d_got, d_want, n, d_ok, stream), "mxd_dev_compare")

    def dev_gen_fill(self, dev: int, d_dst: int, offset: int, n: int, seed: int, stream: int = 0):
        self._check(self._lib.mxd_dev_gen_fill(self._ctx, dev, d_dst, offset, n, seed, stream), "mxd_dev_gen_fill")

    # -- pinned memory -----------------------------------------------------------------------
    def host_alloc(self, nbytes: int) -> int:
        p = C.c_void_p()
        self._check(self._lib.mxd_host_alloc(self._ctx, C.byref(p), nbytes), "mxd_host_alloc")
        return p.value

    def host_free(self, ptr: int):
        self._lib.mxd_host_free(self._ctx, ptr)


class Hasher:
    """hash.Hash-shaped incremental SHA-256 (pkg/client/helper.go:46-49) running on the GPU."""

    def __init__(self, engine: Engine):
        self._e = engine
        self._h = C.c_void_p()
        engine._check(engine._lib.mxd_hasher_new(engine._ctx, C.byref(self._h)), "mxd_hasher_new")

    def write(self, data) -> int:
        addr, n, keep = _buf(data)
        self._e._check(self._e._lib.mxd_hasher_write(self._h, addr, n), "mxd_hasher_write")
        return n

    update = write

    def sum(self) -> bytes:
        out = (C.c_uint8 * 32)()
        self._e._check(self._e._lib.mxd_hasher_sum(self._h, out), "mxd_hasher_sum")
        return bytes(out)

    digest = sum

    def reset(self):
        self._e._check(self._e._lib.mxd_hasher_reset(self._h), "mxd_hasher_reset")

    def size(self) -> int:
        """hash.Hash.Size(): 32"""
        return int(self._e._lib.mxd_hasher_size(self._h))

    def block_size(self) -> int:
        return int(self._e._lib.mxd_hasher_block_size(self._h))

    def written(self) -> int:
        return int(self._e._lib.mxd_hasher_written(self._h))

    def close(self):
        if self._h:
            self._e._lib.mxd_hasher_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
