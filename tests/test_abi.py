"""The C-ABI shared library loads without a GPU and exports every symbol include/dsk.h declares."""
import ctypes
import os
import re

import pytest

from deepspeaker_pytorch_b200 import _lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "dsk.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dsk_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_loads():
    lib = L.load()
    assert lib.dsk_version() >= 100


def test_every_declared_symbol_is_exported_and_bound():
    lib = L.load()
    syms = declared_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/dsk.h but not exported by libdsk.so"
        assert s in L.SIGNATURES, f"{s} has no ctypes signature in _lib.SIGNATURES"
    for s in L.SIGNATURES:
        assert s in syms, f"{s} bound in _lib.py but not declared in include/dsk.h"


def test_sass_is_hopper_native():
    """HGMMA (wgmma) and UTMALDG/UTMASTG (TMA) must be in the shipped SASS."""
    import shutil
    import subprocess

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", L.LIB_PATH], capture_output=True, text=True).stdout
    for mnem in ("HGMMA", "UTMALDG", "UTMASTG"):
        assert mnem in sass, f"{mnem} missing from libdsk.so SASS"
    assert "sm_90a" in subprocess.run([cuobjdump, "-lelf", L.LIB_PATH], capture_output=True, text=True).stdout


def test_error_convention_without_gpu():
    """No exceptions across the ABI: bad calls return a negative status and set dsk_last_error()."""
    import torch

    lib = L.load()
    h = ctypes.c_void_p()
    assert lib.dsk_create(None, 0, 0) < 0
    assert b"null" in lib.dsk_last_error()
    assert lib.dsk_create(ctypes.byref(h), 0, 7) < 0
    if not torch.cuda.is_available():
        rc = lib.dsk_create(ctypes.byref(h), 0, 0)      # no device: a CUDA error, reported not raised
        assert rc < 0 and len(lib.dsk_last_error()) > 0
        with pytest.raises(RuntimeError):
            L.check(rc, "dsk_create")
    assert lib.dsk_pairwise_distance(None, None, 0, 0, None, None) < 0
