"""CPU: the C-ABI library builds for sm_90a, loads, and exports every symbol include/hipie_b200.h declares.
No compute calls (no GPU here)."""
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from hipie_b200 import build, _lib
    build.build()
    return _lib.load()


def test_header_symbols_exported(lib):
    from hipie_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "hipie_b200.h")).read()
    declared = set(re.findall(r"\b(hipie_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    for name in sorted(declared):
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
        assert name in _lib.SYMBOLS, f"{name} has no ctypes signature in hipie_b200/_lib.py"
    assert set(_lib.SYMBOLS) <= declared | {"hipie_last_error"}


def test_abi_version_and_error_string(lib):
    assert lib.hipie_abi_version() == 1
    assert isinstance(lib.hipie_last_error(), bytes)
    assert lib.hipie_launch_count() == 0


def test_argument_validation_without_gpu(lib):
    import ctypes
    # null pointers must be rejected before any CUDA call
    rc = lib.hipie_msda_forward(None, None, None, None, None, None, 1, 1, 1, 1, 1, 1, 1, 0, 0, None)
    assert rc == -1 and b"null" in lib.hipie_last_error()
    rc = lib.hipie_gemm(None, None)
    assert rc == -1


def test_ops_refuse_cpu_tensors(lib):
    import torch
    from hipie_b200 import ops
    with pytest.raises(RuntimeError):
        ops.split(torch.zeros(8))


def test_sass_is_hopper_native(lib):
    import shutil
    import subprocess
    so = os.path.join(ROOT, "hipie_b200", "libhipie_b200.so")
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([cuobjdump, "-sass", so], capture_output=True, text=True).stdout
    assert "HGMMA" in sass, "16-bit wgmma missing from the GEMM / attention"
    assert "QGMMA" in sass, "e4m3 wgmma missing from the prec-6 GEMM"
    assert "UTMALDG" in sass, "TMA loads missing"
