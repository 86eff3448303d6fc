"""CPU: argument validation of the sparsifier's C-ABI entry points (gsb_sparsity_*, gsb_adc_prune_classify,
include/gsb200.h), with the conventions of test_cabi_validation.py: 0 for the empty cases, GSB_E_INVALID (-1) for null
or out-of-range arguments, GSB_E_WORKSPACE (-3) for a short or misaligned workspace.  No call reaches the device."""
import ctypes as C
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, E_INVALID, E_WORKSPACE = 0, -1, -3


@pytest.fixture(scope="module")
def lib(pkg):
    path = os.path.join(ROOT, "gaussian-splatting-cuda_b200", "lib", "libgsb200.so")
    if not os.path.exists(path):
        pkg.build()
    L = C.CDLL(path)
    L.gsb_sparsity_workspace.restype = C.c_size_t
    L.gsb_adc_workspace.restype = C.c_size_t
    return L


_buf = np.zeros(1 << 16, np.uint8)
_base = (_buf.ctypes.data + 255) & ~255
PTR = C.c_void_p(_base)            # 256-aligned: passes every alignment check
MIS = C.c_void_p(_base + 4)        # 4-byte aligned only
NULL = C.c_void_p(None)
u32, sz = C.c_uint32, C.c_size_t


def test_workspace_size_grows_with_N(lib):
    assert lib.gsb_sparsity_workspace(u32(0)) > 0
    assert lib.gsb_sparsity_workspace(u32(1000)) - lib.gsb_sparsity_workspace(u32(0)) >= 1000 * 4


def test_update_validation(lib):
    def update(N=8, o=PTR, z=PTR, u=PTR, k=4, ws=PTR, ws_bytes=None):
        nb = lib.gsb_sparsity_workspace(u32(N)) if ws_bytes is None else ws_bytes
        return lib.gsb_sparsity_update(u32(N), o, z, u, u32(k), C.c_int(0), ws, sz(nb), NULL)

    assert update(N=0, o=NULL, z=NULL, u=NULL, k=0) == OK              # nothing to do
    assert update(N=0, k=1) == E_INVALID                              # k > N
    assert update(k=9) == E_INVALID
    assert update(o=NULL) == E_INVALID
    assert update(z=NULL) == E_INVALID
    assert update(u=NULL) == E_INVALID
    assert update(ws=NULL) == E_WORKSPACE
    assert update(ws=MIS) == E_WORKSPACE                               # 256-byte alignment
    assert update(ws_bytes=lib.gsb_sparsity_workspace(u32(8)) - 1) == E_WORKSPACE


def test_loss_validation(lib):
    def loss(N=8, o=PTR, z=PTR, u=PTR, rho=PTR, v=PTR, out=PTR, ws=PTR, ws_bytes=None):
        nb = lib.gsb_sparsity_workspace(u32(N)) if ws_bytes is None else ws_bytes
        return lib.gsb_sparsity_loss(u32(N), o, z, u, rho, v, out, ws, sz(nb), NULL)

    assert loss(out=NULL) == E_INVALID
    assert loss(rho=NULL) == E_INVALID
    assert loss(o=NULL) == E_INVALID
    assert loss(z=NULL) == E_INVALID
    assert loss(u=NULL) == E_INVALID
    assert loss(v=NULL) == E_INVALID
    assert loss(ws=NULL) == E_WORKSPACE
    assert loss(ws=MIS) == E_WORKSPACE
    assert loss(ws_bytes=lib.gsb_sparsity_workspace(u32(8)) - 1) == E_WORKSPACE


def test_prune_classify_validation(lib):
    def prune(N=8, o=PTR, n_prune=4, counts=PTR, ws=PTR, ws_bytes=None):
        nb = lib.gsb_adc_workspace(u32(N)) if ws_bytes is None else ws_bytes
        return lib.gsb_adc_prune_classify(u32(N), o, u32(n_prune), counts, ws, sz(nb), NULL)

    assert prune(counts=NULL) == E_INVALID
    assert prune(n_prune=9) == E_INVALID                              # more rows than there are
    assert prune(o=NULL) == E_INVALID
    assert prune(N=1 << 30, ws_bytes=1 << 16) == E_INVALID             # gsb_adc_apply indexes 2N in int32
    assert prune(ws=NULL) == E_WORKSPACE
    assert prune(ws=MIS) == E_WORKSPACE
    assert prune(ws_bytes=lib.gsb_adc_workspace(u32(8)) - 1) == E_WORKSPACE
