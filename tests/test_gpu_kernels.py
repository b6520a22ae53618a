"""Every digest kernel across its launch contract, compared with hashlib (the battery is tests/kernel_routes.py), and
the device-resident entry points refusing pointers the kernels cannot use.

Each route runs in a fresh process because the knobs that select a kernel are read once, when the library loads."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import modelx_b200
from modelx_b200 import _native as N
from tests.kernel_routes import ROUTES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run_route(route, backend, timeout):
    out = subprocess.run([sys.executable, "-m", "tests.kernel_routes", "--route", route, "--backend", backend],
                         capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith("{")]
    assert out.returncode == 0 and lines, out.stdout + out.stderr
    res = json.loads(lines[-1])
    assert res["ok"] and res["route"] == route and res["cases"] > 0, out.stdout + out.stderr
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("route", list(ROUTES))
def test_kernel_route(route):
    res = _run_route(route, "cuda", timeout=1200)
    promised = ROUTES[route][1]
    kernels = set(res["kernels"])
    if promised is None:
        assert kernels, res
    else:
        assert promised <= kernels, res


def test_kernel_battery_on_mock(mock_lib):
    _run_route("default", "mock", timeout=600)


# ---- argument checks of the mxd_dev_* entry points (test double only: no misaligned pointer reaches a GPU) ------------
TP = (128, 64, 2)


def _calls(eng, a):
    """name -> (call with an unusable argument, the same call with a usable one).  `a` is a 256-byte aligned address with
    8 KiB behind it: data at a, outputs at a + 4096, spans at a + 6144."""
    out, spans = a + 4096, a + 6144
    return {
        "segments d_out+8": (lambda: eng.dev_sha256_segments(0, a, 100, 64, out + 8), lambda: eng.dev_sha256_segments(0, a, 100, 64, out)),
        "segments NULL data": (lambda: eng.dev_sha256_segments(0, 0, 32, 64, out), lambda: eng.dev_sha256_segments(0, 0, 0, 64, out)),
        "batch d_spans+4": (lambda: eng.dev_sha256_batch(0, spans + 4, 1, out), lambda: eng.dev_sha256_batch(0, spans, 1, out)),
        "batch d_out+8": (lambda: eng.dev_sha256_batch(0, spans, 1, out + 8), lambda: eng.dev_sha256_batch(0, spans, 1, out)),
        "tree_chunks d_chunk_digests+8": (lambda: eng.dev_tree_chunks(0, a, 200, TP, out + 8), lambda: eng.dev_tree_chunks(0, a, 200, TP, out)),
        "tree_chunks NULL piece": (lambda: eng.dev_tree_chunks(0, 0, 200, TP, out), lambda: eng.dev_tree_chunks(0, 0, 0, TP, out)),
        "tree_finish input+4": (lambda: eng.dev_tree_finish(0, a + 4, 2, 200, TP, out), lambda: eng.dev_tree_finish(0, a, 2, 200, TP, out)),
        "tree_finish d_root+8": (lambda: eng.dev_tree_finish(0, a, 2, 200, TP, out + 8), lambda: eng.dev_tree_finish(0, a, 2, 200, TP, out)),
        "tree_digest d_root+8": (lambda: eng.dev_tree_digest(0, a, 200, TP, out, out + 1032), lambda: eng.dev_tree_digest(0, a, 200, TP, out, out + 1024)),
        "tree_digest d_chunk_digests+8": (lambda: eng.dev_tree_digest(0, a, 200, TP, out + 8, out + 1024),
                                          lambda: eng.dev_tree_digest(0, a, 200, TP, out, out + 1024)),
        "tree_digest NULL data": (lambda: eng.dev_tree_digest(0, 0, 200, TP, out, out + 1024), lambda: eng.dev_tree_digest(0, 0, 0, TP, out, out + 1024)),
        "gen_fill dst+4": (lambda: eng.dev_gen_fill(0, out + 4, 0, 64, 1), lambda: eng.dev_gen_fill(0, out + 8, 0, 64, 1)),
        "gen_fill offset 4": (lambda: eng.dev_gen_fill(0, out, 4, 64, 1), lambda: eng.dev_gen_fill(0, out, 8, 64, 1)),
        "gen_fill n 12": (lambda: eng.dev_gen_fill(0, out, 0, 12, 1), lambda: eng.dev_gen_fill(0, out, 0, 16, 1)),
    }


@pytest.mark.parametrize("case", list(_calls(None, 0)))
def test_device_entry_points_reject_unusable_pointers(mock_lib, case):
    """A misaligned digest output, span array or chunk-digest input, a NULL data pointer with bytes to read, or a
    generator range off the 8-byte grid is MXD_ERR_INVALID, and nothing is launched or written."""
    mem = np.zeros(8192 + 256, dtype=np.uint8)
    a = mem.ctypes.data + (-mem.ctypes.data) % 256
    base = a - mem.ctypes.data
    with modelx_b200.Engine(devices=[0], lib_path=mock_lib) as eng:
        mem[base:base + 4096] = np.arange(4096) % 251
        mem[base + 6144:base + 6160].view(np.uint64)[:] = (a, 100)       # one span: 100 bytes at a
        mem[base + 4096:base + 6144] = 0x5A
        bad, good = _calls(eng, a)[case]
        before, snapshot = eng.stats()["kernel_launches"], mem.copy()
        with pytest.raises(modelx_b200.MxdError) as ei:
            bad()
        assert ei.value.status == N.MXD_ERR_INVALID
        assert eng.stats()["kernel_launches"] == before
        assert np.array_equal(mem, snapshot), "a refused call wrote memory"
        good()                                                            # the usable form of the same call is accepted
        assert not np.array_equal(mem, snapshot)
