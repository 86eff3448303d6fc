"""Backend over the REFERENCE's own fastgs rasterizer (oracle/_ref/libfastgs_ref.so, built by oracle/build_ref.py from
/root/reference/fastgs/rasterization, unmodified).  TEST INFRASTRUCTURE ONLY: the pin of oracle/fastgs_oracle.c and of
the H100 fastgs path, and the same-box GPU baseline of bench.py -- driven through the very same Python call sites as the
product backend (FastGsBackend of the package)."""
from __future__ import annotations

import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_SO = os.path.join(_HERE, "_ref", "libfastgs_ref.so")
_loaded = False


def available() -> bool:
    return os.path.exists(REF_SO)


def _ns():
    global _loaded
    if not _loaded:
        if not available():
            raise RuntimeError(f"{REF_SO} not built (python oracle/build_ref.py in the build container)")
        torch.ops.load_library(REF_SO)
        _loaded = True
    return torch.ops.fastgs_ref


def backend(fastgs_module):
    """A FastGsBackend (class from the product package's fastgs module) bound to the reference library."""
    return fastgs_module.FastGsBackend(_ns)
