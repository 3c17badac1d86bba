"""The C-ABI library loads on a CPU-only box and exports every function include/nfk.h declares."""
import ctypes
import os
import re

import pytest

from conftest import ROOT
from nflows_b200 import _native


def declared_functions():
    text = open(os.path.join(ROOT, "include", "nfk.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(nfk_[a-z0-9_]+)\s*\(", text)))


def test_header_and_binding_agree():
    assert declared_functions() == sorted(_native.EXPORTED_SYMBOLS)


def test_spline_bin_bound_matches_the_header():
    """The Python gates that send splines with more bins to the torch formulation use the header's NFK_MAX_BINS."""
    text = open(os.path.join(ROOT, "include", "nfk.h")).read()
    assert int(re.search(r"#define NFK_MAX_BINS (\d+)", text).group(1)) == _native.MAX_BINS


def test_library_exports_every_symbol():
    if not os.path.exists(_native.library_path()):
        import __graft_entry__
        __graft_entry__.build()
    lib = ctypes.CDLL(_native.library_path())
    for name in declared_functions():
        assert hasattr(lib, name), name
    loaded = _native.load()
    assert loaded.nfk_version() == 5
    assert loaded.nfk_launch_count() >= 0


def test_no_silent_fallback_on_missing_library(monkeypatch):
    monkeypatch.setattr(_native, "_lib", None)
    monkeypatch.setattr(_native, "_LIB_PATH", "/nonexistent/libnfk_sm90.so")
    with pytest.raises(_native.NativeUnavailable):
        _native.load()


def test_argument_validation_happens_before_any_cuda_call():
    """Bad shapes / NULL pointers are rejected with NFK_E_INVALID and a message by the entry points themselves, so this runs
    without a GPU (nothing is launched)."""
    lib = _native.load()
    lib.nfk_last_error.restype = ctypes.c_char_p
    assert lib.nfk_linear_f16x3_supported(784, 784, 784) == 1
    assert lib.nfk_linear_f16x3_supported(784, 784, 12) == 0           # K not a multiple of 8
    assert lib.nfk_linear_f16x3_supported(12, 784, 8) == 0             # row pitch not a multiple of 8 elements
    # no output requested
    rc = lib.nfk_linear_f16x3(16, 16, 8, 6, 16, 16, 8, 10, 0, 0, 0, 0, 0, 0, 0, 0, 6, 0, 0, 0, 0, 4, 8, 8, 0, 0)
    assert rc == -1 and b"no output" in lib.nfk_last_error()
    # y and the pair output are mutually exclusive in the fused kernel; both NULL is an error as well
    desc = _native.spline_desc(8, "linear", 3.0, 0, 1, 0, 1, 1e-3, 1e-3, 1e-3, False, 16.0)
    rc = lib.nfk_rq_coupling_final_f16x3(ctypes.byref(desc), 0, 16, 16, 64, 6, 16, 16, 64, 10, 16, 64, 16, 32, 0, 16, 4,
                                         0, 32, 0, 0, 0, 6, 0, 128, 0, 0)
    assert rc == -1 and b"either y" in lib.nfk_last_error()
    # unsupported bin count for the fused kernel
    assert lib.nfk_rq_coupling_final_supported(7, 1, 64, 64) == 0 and lib.nfk_rq_coupling_final_supported(8, 1, 64, 64) == 1
    assert lib.nfk_rq_coupling_final_padded_params(8, 1) == 24 and lib.nfk_rq_coupling_final_padded_params(8, 0) == 32
    # empty batches are a no-op success
    assert lib.nfk_split_f16(16, 8, 8, 0, 6, 16, 16, 8, 0, 0, 0) == 0
