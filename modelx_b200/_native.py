"""ctypes binding of libmodelxdigest.so (the C ABI in include/modelx_digest.h).

The shared library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).  There is no
Python or CPU implementation behind this module: if the library is missing, importing the symbols
fails loudly, and if no CUDA device is present ``mxd_open`` returns MXD_ERR_NO_DEVICE.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# MODELX_B200_LIB lets a developer A/B an experimental build of the same library; default is the in-tree build.
LIB_PATH = os.environ.get("MODELX_B200_LIB") or os.path.join(_HERE, "libmodelxdigest.so")

MXD_OK = 0
MXD_ERR_INVALID = -1
MXD_ERR_NO_DEVICE = -2
MXD_ERR_CUDA = -3
MXD_ERR_IO = -4
MXD_ERR_NOMEM = -5
MXD_ERR_CANCELED = -6
MXD_ERR_DIV_ZERO = -7


class Span(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("len", C.c_uint64)]


class Part(C.Structure):
    _fields_ = [("offset", C.c_int64), ("length", C.c_int64)]


class TreeParams(C.Structure):
    _fields_ = [("chunk", C.c_uint64), ("leaf", C.c_uint64), ("fanout", C.c_uint32), ("reserved", C.c_uint32)]


SINK_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64)


class Stats(C.Structure):
    _fields_ = [("kernel_launches", C.c_uint64), ("bytes_hashed", C.c_uint64), ("h2d_bytes", C.c_uint64),
                ("d2h_bytes", C.c_uint64), ("src_bytes_read", C.c_uint64), ("open_files", C.c_uint64),
                ("reserved", C.c_uint64 * 2)]


class FileJob(C.Structure):
    _fields_ = [("path", C.c_char_p), ("ranges", C.POINTER(Part)), ("nranges", C.c_uint64), ("out", C.POINTER(C.c_uint8)),
                ("sink", C.c_void_p), ("sink_user", C.c_void_p), ("size", C.c_uint64), ("status", C.c_int)]


u8p = C.POINTER(C.c_uint8)
u64p = C.POINTER(C.c_uint64)
vp = C.c_void_p

# name -> (restype, argtypes); mirrors include/modelx_digest.h one to one
PROTOTYPES = {
    "mxd_open": (C.c_int, [C.POINTER(vp), C.POINTER(C.c_int), C.c_int, C.c_uint64]),
    "mxd_close": (None, [vp]),
    "mxd_device_count": (C.c_int, [vp]),
    "mxd_op_begin": (C.c_int, [vp, C.POINTER(vp)]),
    "mxd_op_end": (None, [vp]),
    "mxd_cancel": (None, [vp]),
    "mxd_reset_cancel": (None, [vp]),
    "mxd_is_canceled": (C.c_int, [vp]),
    "mxd_trace_enable": (C.c_int, [vp, C.c_int]),
    "mxd_trace_dump": (C.c_int, [vp, C.c_char_p]),
    "mxd_batch_pays_off": (C.c_int, [C.c_uint64, C.c_uint64, C.c_uint64]),
    "mxd_sha256_file_jobs": (C.c_int, [vp, C.POINTER(FileJob), C.c_uint64]),
    "mxd_sha256_file_ranges": (C.c_int, [vp, C.c_char_p, C.POINTER(Part), C.c_uint64, u8p, u64p, vp, vp]),
    "mxd_get_stats": (C.c_int, [vp, C.POINTER(Stats)]),
    "mxd_prof_enable": (C.c_int, [vp, C.c_int]),
    "mxd_prof_read": (C.c_int, [vp, C.POINTER(C.c_double), u64p, u64p]),
    "mxd_strerror": (C.c_char_p, [C.c_int]),
    "mxd_last_error": (C.c_char_p, []),
    "mxd_abi_version": (C.c_int, []),
    "mxd_sha256": (C.c_int, [vp, vp, C.c_uint64, u8p]),
    "mxd_sha256_batch": (C.c_int, [vp, C.POINTER(Span), C.c_uint64, u8p]),
    "mxd_sha256_file": (C.c_int, [vp, C.c_char_p, u8p, u64p]),
    "mxd_sha256_files": (C.c_int, [vp, C.POINTER(C.c_char_p), C.c_uint64, u8p, u64p]),
    "mxd_sha256_file_parts": (C.c_int, [vp, C.c_char_p, C.POINTER(Part), C.c_uint64, u8p]),
    "mxd_verify_batch": (C.c_int, [vp, C.POINTER(Span), u8p, C.c_uint64, u8p]),
    "mxd_verify_files": (C.c_int, [vp, C.POINTER(C.c_char_p), u8p, C.c_uint64, u8p]),
    "mxd_hasher_new": (C.c_int, [vp, C.POINTER(vp)]),
    "mxd_hasher_write": (C.c_int, [vp, vp, C.c_uint64]),
    "mxd_hasher_sum": (C.c_int, [vp, u8p]),
    "mxd_hasher_reset": (C.c_int, [vp]),
    "mxd_hasher_size": (C.c_uint64, [vp]),
    "mxd_hasher_block_size": (C.c_uint64, [vp]),
    "mxd_hasher_written": (C.c_uint64, [vp]),
    "mxd_hasher_free": (None, [vp]),
    "mxd_tree_shape": (C.c_int, [C.c_uint64, C.POINTER(TreeParams), u64p, C.c_int, C.POINTER(C.c_int)]),
    "mxd_tree_digest": (C.c_int, [vp, vp, C.c_uint64, C.POINTER(TreeParams), u8p, u64p, u8p]),
    "mxd_tree_digest_file": (C.c_int, [vp, C.c_char_p, C.POINTER(TreeParams), u8p, C.c_uint64, u64p, u64p, u8p]),
    "mxd_tree_digest_file_tee": (C.c_int, [vp, C.c_char_p, C.POINTER(TreeParams), u8p, C.c_uint64, u64p, u64p, u8p, vp, vp]),
    "mxd_tree_chunks": (C.c_int, [vp, vp, C.c_uint64, C.POINTER(TreeParams), u8p]),
    "mxd_tree_digest_files": (C.c_int, [vp, C.POINTER(C.c_char_p), C.c_uint64, C.POINTER(TreeParams), u8p, u64p, C.POINTER(C.c_int)]),
    "mxd_tree_chunks_file": (C.c_int, [vp, C.c_char_p, C.c_uint64, C.c_uint64, C.POINTER(TreeParams), u8p]),
    "mxd_tree_load_file": (C.c_int, [vp, C.c_int, C.c_char_p, C.POINTER(Span), C.c_uint64, C.POINTER(TreeParams), u8p,
                                     C.c_uint64, u64p, u64p, u8p]),
    "mxd_tree_finish": (C.c_int, [vp, u8p, C.c_uint64, C.c_uint64, C.POINTER(TreeParams), u8p]),
    "mxd_calc_parts": (C.c_int, [C.c_int64, C.c_int64, C.POINTER(Part)]),
    "mxd_server_part_count": (C.c_int64, [C.c_int64, C.c_int]),
    "mxd_digest_string": (None, [u8p, C.c_char_p]),
    "mxd_digest_parse": (C.c_int, [C.c_char_p, u8p]),
    "mxd_host_alloc": (C.c_int, [vp, C.POINTER(vp), C.c_uint64]),
    "mxd_host_free": (None, [vp, vp]),
    "mxd_host_register": (C.c_int, [vp, vp, C.c_uint64]),
    "mxd_host_unregister": (C.c_int, [vp, vp]),
    "mxd_dev_sha256_segments": (C.c_int, [vp, C.c_int, vp, C.c_uint64, C.c_uint64, vp, vp]),
    "mxd_dev_sha256_batch": (C.c_int, [vp, C.c_int, vp, C.c_uint64, vp, vp]),
    "mxd_dev_tree_chunks": (C.c_int, [vp, C.c_int, vp, C.c_uint64, C.POINTER(TreeParams), vp, vp]),
    "mxd_dev_tree_finish": (C.c_int, [vp, C.c_int, vp, C.c_uint64, C.c_uint64, C.POINTER(TreeParams), vp, vp]),
    "mxd_dev_tree_digest": (C.c_int, [vp, C.c_int, vp, C.c_uint64, C.POINTER(TreeParams), vp, vp, vp]),
    "mxd_dev_tree_digest_extents": (C.c_int, [vp, C.c_int, C.POINTER(Span), C.c_uint64, C.POINTER(TreeParams), vp, vp, vp]),
    "mxd_dev_compare": (C.c_int, [vp, C.c_int, vp, vp, C.c_uint64, vp, vp]),
    "mxd_dev_gen_fill": (C.c_int, [vp, C.c_int, vp, C.c_uint64, C.c_uint64, C.c_uint64, vp]),
}

cpp = C.POINTER(C.c_char_p)
# host-side mirror of pkg/client / pkg/registry (include/modelx_client.h)
PROTOTYPES.update({
    "mxc_last_error": (C.c_char_p, []),
    "mxc_free": (None, [C.c_void_p]),
    "mxc_parse_manifest": (C.c_int, [C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    "mxc_push_digest": (C.c_int, [vp, C.c_char_p, C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]),
    "mxc_pull_check": (C.c_int, [vp, C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    "mxc_fs_put_blob": (C.c_int, [vp, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int]),
    "mxc_fs_exists_blob": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p]),
    "mxc_fs_put_manifest": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p]),
    "mxc_fs_get_manifest": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    "mxc_blob_digest_path": (C.c_int, [C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    "mxc_push_local": (C.c_int, [vp, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_int, C.POINTER(C.c_void_p)]),
    "mxc_push_stream": (C.c_int, [vp, C.c_char_p, C.c_char_p, C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]),
    "mxc_tgz": (C.c_int, [vp, C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p), u64p]),
    "mxc_untgz": (C.c_int, [C.c_char_p, C.c_char_p]),
    "mxc_fs_get_index": (C.c_int, [C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    "mxc_push_local_tree": (C.c_int, [vp, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p)]),
    "mxc_pull_local": (C.c_int, [vp, C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, C.POINTER(C.c_void_p)]),
})

# mxc_uploader callbacks (include/modelx_client.h)
UP_BEGIN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint64, C.c_char_p, C.c_uint64, C.POINTER(Part), C.c_uint64)
UP_PART_WRITE = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_void_p, C.c_uint64)
UP_PART_RESTART = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint64, C.c_uint64)
UP_COMPLETE = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_uint64, C.c_char_p, C.POINTER(C.c_uint8), C.c_uint64, C.POINTER(C.c_char))
UP_ABORT = C.CFUNCTYPE(None, C.c_void_p, C.c_uint64)


class Uploader(C.Structure):
    _fields_ = [("user", C.c_void_p), ("max_concurrent", C.c_int), ("begin", UP_BEGIN), ("part_write", UP_PART_WRITE),
                ("part_restart", UP_PART_RESTART), ("complete", UP_COMPLETE), ("abort", UP_ABORT)]


MXC_ERR_DIGEST_INVALID = -20
MXC_ERR_UNSUPPORTED = -21
MXC_ERR_MANIFEST = -22
MXC_ERR_NOT_FOUND = -23

_libs = {}


def load(path: str = None) -> C.CDLL:
    """Load a build of the shared library (default: the in-tree CUDA build) and type every exported function.
    Tests of the host logic pass the path of the CPU test double built by tests/mock_build.py; nothing in the
    package does."""
    path = path or LIB_PATH
    lib = _libs.get(path)
    if lib is not None:
        return lib
    if not os.path.exists(path):
        raise ImportError(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). modelx_b200 has no pure-Python or CPU fallback.")
    lib = C.CDLL(path)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError here means header and library disagree
        fn.restype = res
        fn.argtypes = args
    _libs[path] = lib
    return lib


class MxdError(RuntimeError):
    def __init__(self, status: int, where: str, lib: C.CDLL = None):
        lib = lib or load()
        if where.startswith("mxc_"):
            detail = lib.mxc_last_error().decode(errors="replace")
        else:
            detail = lib.mxd_last_error().decode(errors="replace")
        super().__init__(f"{where}: {lib.mxd_strerror(status).decode()} ({status}) {detail}")
        self.status = status
        self.detail = detail


def check(status: int, where: str, lib: C.CDLL = None) -> None:
    if status != MXD_OK:
        raise MxdError(status, where, lib)
