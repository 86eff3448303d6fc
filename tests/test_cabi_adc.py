"""CPU: argument validation of the default strategy's C-ABI entry points (gsb_adc_*, include/gsb200.h), with the
conventions of test_cabi_validation.py: 0 for the empty cases, GSB_E_INVALID (-1) for null, misaligned or
out-of-range arguments, GSB_E_WORKSPACE (-3) for a short or misaligned workspace.  No call reaches the device."""
import ctypes as C
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, E_INVALID, E_WORKSPACE = 0, -1, -3


class GsbAdcParams(C.Structure):
    _fields_ = [("grad_threshold", C.c_float), ("grow_scale3d", C.c_float), ("prune_scale3d", C.c_float),
                ("scene_scale", C.c_float), ("prune_opacity", C.c_float), ("prune_too_big", C.c_int32),
                ("revised_opacity", C.c_int32)]


class GsbMcmcRows(C.Structure):
    _fields_ = [("means", C.c_void_p), ("sh0", C.c_void_p), ("shN", C.c_void_p), ("scaling_raw", C.c_void_p),
                ("rotation_raw", C.c_void_p), ("opacity_raw", C.c_void_p), ("shN_rows", C.c_uint32),
                ("exp_avg", C.c_void_p * 6), ("exp_avg_sq", C.c_void_p * 6)]


@pytest.fixture(scope="module")
def lib(pkg):
    path = os.path.join(ROOT, "gaussian-splatting-cuda_b200", "lib", "libgsb200.so")
    if not os.path.exists(path):
        pkg.build()
    L = C.CDLL(path)
    L.gsb_adc_workspace.restype = C.c_size_t
    return L


_buf = np.zeros(1 << 16, np.uint8)
_base = (_buf.ctypes.data + 255) & ~255
PTR = C.c_void_p(_base)            # 256-aligned: passes every alignment check
MIS = C.c_void_p(_base + 4)        # 4-byte aligned only
NULL = C.c_void_p(None)
u32, f32, sz = C.c_uint32, C.c_float, C.c_size_t
PARAMS = GsbAdcParams(2e-4, 0.01, 0.1, 1.0, 0.005, 0, 0)


def rows(rotation=PTR, shN_rows=0, shN=None):
    r = GsbMcmcRows()
    r.means = r.sh0 = r.scaling_raw = r.opacity_raw = PTR.value
    r.rotation_raw = rotation.value
    r.shN_rows, r.shN = shN_rows, shN
    return r


def classify(lib, N, info=PTR, rot=PTR, params=PARAMS, counts=PTR, ws=PTR, ws_bytes=None):
    nb = lib.gsb_adc_workspace(u32(N)) if ws_bytes is None else ws_bytes
    p = C.byref(params) if params is not None else NULL
    return lib.gsb_adc_classify(u32(N), info, PTR, rot, PTR, p, counts, ws, sz(nb), NULL)


def test_workspace_size_grows_with_N(lib):
    assert lib.gsb_adc_workspace(u32(0)) > 0
    assert lib.gsb_adc_workspace(u32(1000)) - lib.gsb_adc_workspace(u32(0)) >= 1000 * 25


def test_classify_validation(lib):
    assert classify(lib, 8, params=None) == E_INVALID
    assert classify(lib, 8, counts=NULL) == E_INVALID
    assert classify(lib, 8, rot=NULL) == E_INVALID
    assert classify(lib, 8, rot=MIS) == E_INVALID                      # rotation_raw is read as float4
    assert lib.gsb_adc_classify(u32(8), PTR, NULL, PTR, PTR, C.byref(PARAMS), PTR, PTR, sz(1 << 16), NULL) == E_INVALID
    assert classify(lib, (1 << 30), ws_bytes=1 << 16) == E_INVALID      # 2N does not fit int32
    assert classify(lib, 8, ws=NULL) == E_WORKSPACE
    assert classify(lib, 8, ws=MIS) == E_WORKSPACE                      # 256-byte alignment
    assert classify(lib, 8, ws_bytes=lib.gsb_adc_workspace(u32(8)) - 1) == E_WORKSPACE


def test_apply_validation(lib):
    src, dst = rows(), rows()
    nb = sz(lib.gsb_adc_workspace(u32(8)))
    p = C.byref(PARAMS)

    def apply(src_=src, dst_=dst, n_split=0, n_final=8, z=NULL, params=p, counts=PTR, ws=PTR, ws_bytes=nb, N=8):
        s = C.byref(src_) if src_ is not None else NULL
        d = C.byref(dst_) if dst_ is not None else NULL
        return lib.gsb_adc_apply(u32(N), s, d, u32(n_split), u32(n_final), z, params, counts, NULL, ws, ws_bytes, NULL)

    assert apply(src_=None) == E_INVALID
    assert apply(dst_=None) == E_INVALID
    assert apply(params=NULL) == E_INVALID
    assert apply(counts=NULL) == E_INVALID
    assert apply(n_final=17) == E_INVALID                               # more than 2N rows
    assert apply(n_split=9) == E_INVALID
    assert apply(n_split=2, z=NULL) == E_INVALID                        # z is needed when rows split
    assert apply(N=1 << 30, n_final=0) == E_INVALID                     # 2N does not fit int32
    assert apply(dst_=rows(rotation=MIS)) == E_INVALID
    assert apply(src_=rows(rotation=NULL)) == E_INVALID
    assert apply(src_=rows(shN_rows=15)) == E_INVALID                   # shN rows without shN
    assert apply(src_=rows(shN_rows=3, shN=PTR.value), dst_=rows(shN_rows=15, shN=PTR.value)) == E_INVALID
    assert apply(ws=MIS) == E_WORKSPACE
    assert apply(ws_bytes=sz(nb.value - 1)) == E_WORKSPACE
    assert apply(n_final=0) == OK                                       # everything pruned: nothing to write


def test_reset_opacity_validation(lib):
    assert lib.gsb_adc_reset_opacity(u32(0), NULL, f32(0.005), NULL, NULL, NULL) == OK
    assert lib.gsb_adc_reset_opacity(u32(8), NULL, f32(0.005), PTR, PTR, NULL) == E_INVALID
