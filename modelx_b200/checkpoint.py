"""Tree digests of safetensors checkpoints held in GPU memory.

A ``.safetensors`` blob is an LE64 header length, a JSON header and then the tensors' bytes at the offsets the header
gives.  ``tree_digest_safetensors`` computes the ``modelx.tree.v1`` digest of that blob straight from the tensors in HBM
(``mxd_dev_tree_digest_extents``): no file is written and the tensors are not gathered into one buffer.  The root equals
``Engine.tree_digest_file`` of the file the same header and tensors form, so ``digest_string(root)`` is the
``modelx.tree.v1`` annotation of that file -- after a pull, to check a loaded model against its manifest; before a push,
to annotate a checkpoint that is still in GPU memory.

``load_safetensors`` is the pull-side counterpart: it reads a ``.safetensors`` file once, through the engine's pinned
ring, straight into one new CUDA tensor per entry (``mxd_tree_load_file``), and returns the tree digest of the bytes
that landed in those tensors; with ``expect`` it refuses weights that do not match the manifest.

Imports torch on first use; ``modelx_b200`` itself does not import this module.
"""
from __future__ import annotations

import json
import os
import struct
from typing import List, Mapping, Optional, Tuple, Union

from .engine import DEFAULT_CHUNK, DEFAULT_FANOUT, DEFAULT_LEAF, Engine, digest_parse

MAX_HEADER_BYTES = 100 << 20     # a safetensors JSON header larger than this is not taken from outside input


class DigestMismatch(ValueError):
    """The loaded bytes do not have the expected tree root.  Carries what was computed -- ``root``, ``chunk_digests``
    (one per chunk of the file, so the first differing chunk locates the damage) and ``size`` -- and ``expected``."""

    def __init__(self, path: str, expected: bytes, root: bytes, chunk_digests: List[bytes], size: int):
        from .engine import digest_string
        super().__init__(f"{path}: tree root {digest_string(root)}, expected {digest_string(expected)}")
        self.path, self.expected, self.root, self.chunk_digests, self.size = path, expected, root, chunk_digests, size


# safetensors dtype string -> (torch dtype attribute, bytes per element)
_DTYPES = {
    "BOOL": ("bool", 1), "U8": ("uint8", 1), "I8": ("int8", 1), "F8_E5M2": ("float8_e5m2", 1),
    "F8_E4M3": ("float8_e4m3fn", 1), "I16": ("int16", 2), "U16": ("uint16", 2), "F16": ("float16", 2),
    "BF16": ("bfloat16", 2), "I32": ("int32", 4), "U32": ("uint32", 4), "F32": ("float32", 4), "I64": ("int64", 8),
    "U64": ("uint64", 8), "F64": ("float64", 8),
}


def _dtype_name(t) -> str:
    import torch
    for name, (attr, _) in _DTYPES.items():
        if getattr(torch, attr, None) == t.dtype:
            return name
    raise ValueError(f"dtype {t.dtype} has no safetensors name")


def safetensors_layout(tensors: Mapping[str, "object"], metadata: Optional[Mapping[str, str]] = None) -> Tuple[bytes, List[str]]:
    """The safetensors header for `tensors` (name -> contiguous torch.Tensor) and the order their bytes follow it in.

    Tensors go largest element size first, then by name (the order safetensors.torch.save_file uses, which keeps every
    tensor aligned to its element size in the file), with contiguous ``data_offsets``.  The JSON is padded with spaces
    so that the whole header, length field included, is a multiple of 8 bytes.  -> (header bytes, names in data order)
    """
    if metadata is not None and (not isinstance(metadata, Mapping) or
                                 not all(isinstance(k, str) and isinstance(v, str) for k, v in metadata.items())):
        raise ValueError("metadata must map str to str")
    entries = []
    for name, t in tensors.items():
        if not isinstance(name, str) or name == "__metadata__":
            raise ValueError(f"invalid tensor name {name!r}")
        if not t.is_contiguous():
            raise ValueError(f"tensor {name!r} is not contiguous")
        dt = _dtype_name(t)
        entries.append((-_DTYPES[dt][1], name, dt, list(t.shape), t.numel() * _DTYPES[dt][1]))
    entries.sort()
    doc = {}
    if metadata:
        doc["__metadata__"] = dict(metadata)
    off = 0
    for _, name, dt, shape, nbytes in entries:
        doc[name] = {"dtype": dt, "shape": shape, "data_offsets": [off, off + nbytes]}
        off += nbytes
    text = json.dumps(doc, separators=(",", ":")).encode()
    text += b" " * (-len(text) % 8)
    return struct.pack("<Q", len(text)) + text, [e[1] for e in entries]


def parse_safetensors_header(header: bytes) -> Tuple[dict, int]:
    """Validate a complete safetensors header (length field + JSON) -> ({name: entry}, payload bytes).

    ValueError unless the header is exactly 8 + N bytes with N a multiple of 8, the JSON is an object of well-formed
    entries, and the entries' ``data_offsets`` tile [0, payload) with no gap or overlap."""
    header = bytes(header)
    if len(header) < 8:
        raise ValueError("safetensors header: shorter than its 8-byte length field")
    (n,) = struct.unpack("<Q", header[:8])
    if len(header) != 8 + n:
        raise ValueError(f"safetensors header: length field says {n} JSON bytes, got {len(header) - 8}")
    if n % 8:
        raise ValueError(f"safetensors header: JSON length {n} is not padded to a multiple of 8")
    try:
        doc = json.loads(header[8:].decode("utf-8"))
    except (UnicodeDecodeError, json.JSONDecodeError) as e:
        raise ValueError(f"safetensors header: not JSON ({e})") from None
    if not isinstance(doc, dict):
        raise ValueError("safetensors header: JSON is not an object")
    entries = {}
    for name, ent in doc.items():
        if name == "__metadata__":
            continue
        if not isinstance(ent, dict) or ent.get("dtype") not in _DTYPES or not isinstance(ent.get("shape"), list) or \
                not all(isinstance(d, int) and d >= 0 for d in ent["shape"]) or \
                not isinstance(ent.get("data_offsets"), list) or len(ent["data_offsets"]) != 2 or \
                not all(isinstance(o, int) and o >= 0 for o in ent["data_offsets"]):
            raise ValueError(f"safetensors header: malformed entry {name!r}")
        begin, end = ent["data_offsets"]
        numel = 1
        for d in ent["shape"]:
            numel *= d
        if end - begin != numel * _DTYPES[ent["dtype"]][1]:
            raise ValueError(f"safetensors header: {name!r} spans {end - begin} bytes, its dtype and shape need "
                             f"{numel * _DTYPES[ent['dtype']][1]}")
        entries[name] = ent
    pos = 0
    for name in sorted(entries, key=lambda k: tuple(entries[k]["data_offsets"])):
        begin, end = entries[name]["data_offsets"]
        if begin != pos:
            raise ValueError(f"safetensors header: {name!r} starts at {begin}, expected {pos} "
                             f"({'gap' if begin > pos else 'overlap'})")
        pos = end
    return entries, pos


def tree_digest_safetensors(engine: Engine, header: bytes, tensors: Mapping[str, "object"], chunk: int = DEFAULT_CHUNK,
                            leaf: int = DEFAULT_LEAF, fanout: int = DEFAULT_FANOUT, stream=None):
    """modelx.tree.v1 digest of the safetensors blob ``header || tensor bytes`` with the tensors in GPU memory.

    `header` is a complete safetensors header (from ``safetensors_layout`` or the first 8 + N bytes of a file);
    `tensors` maps each of its names to a contiguous CUDA tensor of that dtype and shape on one of the engine's
    devices.  Work is enqueued on `stream` (default: the current stream of the tensors' device) and waited for.
    -> (chunk_digests: list[bytes], root: bytes, size: int), like ``Engine.tree_digest_file`` of that file."""
    import torch
    entries, payload = parse_safetensors_header(header)
    missing = sorted(set(entries) - set(tensors))
    extra = sorted(set(tensors) - set(entries))
    if missing or extra:
        raise ValueError(f"tensors do not match the header: missing {missing[:8]}, not in the header {extra[:8]}")
    device = None
    for name, ent in entries.items():
        t = tensors[name]
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"{name!r} is not a torch.Tensor")
        if _dtype_name(t) != ent["dtype"]:
            raise ValueError(f"{name!r}: dtype {_dtype_name(t)} but the header says {ent['dtype']}")
        if list(t.shape) != ent["shape"]:
            raise ValueError(f"{name!r}: shape {list(t.shape)} but the header says {ent['shape']}")
        begin, end = ent["data_offsets"]
        if t.numel() * t.element_size() != end - begin:
            raise ValueError(f"{name!r}: {t.numel() * t.element_size()} bytes but the header says {end - begin}")
        if not t.is_contiguous():
            raise ValueError(f"{name!r} is not contiguous")
    for name in entries:
        t = tensors[name]
        if t.device.type != "cuda" or (device is not None and t.device != device):
            raise ValueError(f"{name!r} is on {t.device}; all tensors must be on one CUDA device")
        device = t.device
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device())
    dev = engine.device_index(device.index)
    nchunks = max(1, -(-(len(header) + payload) // chunk))
    with torch.cuda.device(device):
        st = stream if stream is not None else torch.cuda.current_stream(device)
        with torch.cuda.stream(st):
            d_header = torch.frombuffer(bytearray(header), dtype=torch.uint8).to(device, non_blocking=False)
            d_out = torch.empty(nchunks * 32 + 32, dtype=torch.uint8, device=device)   # chunk digests, then the root
        order = sorted(entries, key=lambda k: entries[k]["data_offsets"][0])
        extents = [(d_header.data_ptr(), len(header))] + \
            [(tensors[k].data_ptr(), tensors[k].numel() * tensors[k].element_size()) for k in order]
        engine.dev_tree_digest_extents(dev, extents, (chunk, leaf, fanout), d_out.data_ptr(), d_out.data_ptr() + nchunks * 32,
                                       st.cuda_stream)
        st.synchronize()
        raw = d_out.cpu().numpy().tobytes()
    return [raw[32 * i:32 * i + 32] for i in range(nchunks)], raw[nchunks * 32:], len(header) + payload


def _expected_root(expect: Union[bytes, str, None]) -> Optional[bytes]:
    if expect is None:
        return None
    if isinstance(expect, (bytes, bytearray)):
        if len(expect) != 32:
            raise ValueError(f"expect: a raw root is 32 bytes, got {len(expect)}")
        return bytes(expect)
    if isinstance(expect, str):
        try:
            return digest_parse(expect)
        except RuntimeError as e:
            raise ValueError(f"expect: {e}") from None
    raise ValueError(f"expect: want 32 bytes or 'sha256:<hex>', got {type(expect).__name__}")


def load_safetensors(engine: Engine, path: str, device=None, expect: Union[bytes, str, None] = None,
                     chunk: int = DEFAULT_CHUNK, leaf: int = DEFAULT_LEAF, fanout: int = DEFAULT_FANOUT):
    """Load a ``.safetensors`` file into new CUDA tensors on `device` (default: the current CUDA device), reading the
    file once through the engine's pinned ring, and tree-digest the bytes that landed in them.

    Every tensor is its own allocation, as ``safetensors.torch.load_file`` returns them.  `expect` (raw 32 bytes or
    ``"sha256:<hex>"``) is the tree root the file must have; on a mismatch ``DigestMismatch`` is raised and no tensor
    is returned.  -> (tensors: dict in header order, chunk_digests, root, size), where root and chunk digests equal
    ``Engine.tree_digest_file(path)``."""
    import torch
    want = _expected_root(expect)
    with open(path, "rb") as f:
        raw = f.read(8)
        if len(raw) < 8:
            raise ValueError(f"{path}: shorter than the 8-byte safetensors header length")
        (n,) = struct.unpack("<Q", raw)
        if n > MAX_HEADER_BYTES:
            raise ValueError(f"{path}: safetensors header of {n} bytes is over the {MAX_HEADER_BYTES}-byte limit")
        header = raw + f.read(n)
        file_size = os.fstat(f.fileno()).st_size
    entries, payload = parse_safetensors_header(header)
    if len(header) + payload != file_size:
        raise ValueError(f"{path}: header + tensors are {len(header) + payload} bytes, the file has {file_size}")
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if device.type != "cuda":
        raise ValueError(f"device {device} is not a CUDA device")
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    dev = engine.device_index(device.index)
    with torch.cuda.device(device):
        d_header = torch.empty(len(header), dtype=torch.uint8, device=device)
        tensors = {name: torch.empty(ent["shape"], dtype=getattr(torch, _DTYPES[ent["dtype"]][0]), device=device)
                   for name, ent in entries.items()}
        order = sorted(entries, key=lambda k: entries[k]["data_offsets"][0])
        extents = [(d_header.data_ptr(), len(header))] + \
            [(tensors[k].data_ptr(), tensors[k].numel() * tensors[k].element_size()) for k in order]
        # the caching allocator may have handed out memory that work still queued on this stream is using
        torch.cuda.current_stream(device).synchronize()
        chunks, root, size = engine.tree_load_file(dev, path, extents, chunk, leaf, fanout)
    del d_header
    if want is not None and root != want:
        tensors = None
        raise DigestMismatch(path, want, root, chunks, size)
    return tensors, chunks, root, size
