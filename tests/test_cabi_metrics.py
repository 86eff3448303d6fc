"""CPU: argument validation of the evaluation metrics' C-ABI entry points (gsb_image_metrics*, include/gsb200.h), with
the conventions of test_cabi_validation.py: GSB_E_INVALID (-1) for null pointers, a zero size or unknown flags,
GSB_E_WORKSPACE (-3) for a short or misaligned workspace.  No call reaches the device."""
import ctypes as C
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OK, E_INVALID, E_WORKSPACE = 0, -1, -3
HWC = 1


@pytest.fixture(scope="module")
def lib(pkg):
    path = os.path.join(ROOT, "gaussian-splatting-cuda_b200", "lib", "libgsb200.so")
    if not os.path.exists(path):
        pkg.build()
    L = C.CDLL(path)
    L.gsb_image_metrics_workspace.restype = C.c_size_t
    return L


_buf = np.zeros(1 << 16, np.uint8)
_base = (_buf.ctypes.data + 255) & ~255
PTR = C.c_void_p(_base)            # 256-aligned: passes every alignment check
MIS = C.c_void_p(_base + 4)        # 4-byte aligned only
NULL = C.c_void_p(None)
u32, sz = C.c_uint32, C.c_size_t


def test_workspace_size_is_fixed_and_small(lib):
    n = lib.gsb_image_metrics_workspace()
    assert 0 < n <= 1 << 16  # a ticket and one pair of float64 partials per CTA, whatever the image size
    assert lib.gsb_image_metrics_workspace() == n


def test_metrics_validation(lib):
    def call(W=8, H=8, image=PTR, target=PTR, flags=0, out=PTR, ws=PTR, ws_bytes=None):
        nb = lib.gsb_image_metrics_workspace() if ws_bytes is None else ws_bytes
        return lib.gsb_image_metrics(u32(W), u32(H), image, target, u32(flags), out, ws, sz(nb), NULL)

    assert call(W=0) == E_INVALID
    assert call(H=0) == E_INVALID
    assert call(W=1 << 16, H=1 << 15) == E_INVALID                    # more than INT32_MAX values
    assert call(image=NULL) == E_INVALID
    assert call(target=NULL) == E_INVALID
    assert call(out=NULL) == E_INVALID
    assert call(flags=2) == E_INVALID                                  # unknown flag
    assert call(flags=HWC | 4) == E_INVALID
    assert call(ws=NULL) == E_WORKSPACE
    assert call(ws=MIS) == E_WORKSPACE                                 # 256-byte alignment
    assert call(ws_bytes=lib.gsb_image_metrics_workspace() - 1) == E_WORKSPACE
    assert call(flags=HWC, ws=NULL) == E_WORKSPACE                     # the layout flag itself is known
