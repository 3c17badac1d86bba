"""ctypes binding of libnfk_sm90.so (C ABI: include/nfk.h).

PyTorch is only the plumbing here: it owns device memory and the current CUDA stream; every kernel on
the hot path is one of ours, reached through this module.  There is NO fallback: if the shared library
is missing or the device is not sm_90, calls raise.
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_size_t, c_void_p

import torch

_LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libnfk_sm90.so")
_lib = None


class NativeUnavailable(RuntimeError):
    pass


class NfkSplineDesc(Structure):
    _fields_ = [
        ("num_bins", c_int32), ("linear_tails", c_int32),
        ("left", c_double), ("right", c_double), ("bottom", c_double), ("top", c_double),
        ("min_bin_width", c_double), ("min_bin_height", c_double), ("min_derivative", c_double),
        ("softplus_beta", c_double), ("wh_divisor", c_double),
    ]


_P = c_void_p  # device pointers travel as integers


class NfkCouplingStep(Structure):
    """include/nfk.h: NfkCouplingStep (field for field)."""
    _fields_ = [
        ("spline", POINTER(NfkSplineDesc)), ("inverse", c_int32),
        ("a_hi", _P), ("a_lo", _P), ("lda", c_int64), ("a_exp", c_int32), ("in_features", c_int32),
        ("w0_hi", _P), ("w0_lo", _P), ("ldw0", c_int64), ("w0_exp", c_int32),
        ("wt_hi", _P), ("wt_lo", _P), ("ldwt", c_int64), ("wt_exps", POINTER(c_int32)),
        ("bias_trunk", _P), ("layer_flags", POINTER(c_int32)), ("num_square_layers", c_int32), ("act_exp", c_int32),
        ("wp_hi", _P), ("wp_lo", _P), ("ldwp", c_int64), ("wp_exp", c_int32), ("bias_packed", _P), ("hidden_features", c_int32),
        ("x", _P), ("ldx", c_int64), ("t_cols", _P), ("t_col0", c_int32), ("d_t", c_int32),
        ("y", _P), ("ldy", c_int64), ("y_hi", _P), ("y_lo", _P), ("lds", c_int64), ("y_exp", c_int32),
        ("h_hi", _P), ("h_lo", _P), ("ldh", c_int64),
        ("lad_accum", _P), ("n_rows", c_int64),
        ("workspace", _P), ("workspace_bytes", c_size_t),
        ("flags", _P),
    ]


STEP_MAX_LAYERS = 9


class NfkRowTerm(Structure):
    _fields_ = [("add", _P), ("ld", c_int64)]


class NfkStepRowTerms(Structure):
    """include/nfk.h: NfkStepRowTerms -- per-row additive terms of the coupling-step kernel's trunk layers."""
    _fields_ = [("layer", NfkRowTerm * STEP_MAX_LAYERS)]


# include/nfk.h: NFK_ACT_* -- the activation codes of the dense layers and of the coupling-step layer flags
ACT_NONE, ACT_RELU, ACT_TANH, ACT_ELU, ACT_LEAKY_RELU, ACT_GELU, ACT_SILU = range(7)
ACT_COUNT = 7
STEP_ACT_SHIFT = 8          # layer-flag bits [8, 12): the activation of bits 1 and 8 (0 reads as relu)

MOG_MAX_COMPONENTS = 21     # include/nfk.h: NFK_MOG_MAX_COMPONENTS
MOG_LOG_PROB, MOG_SAMPLE = 0, 1


class NfkMogArgs(Structure):
    """include/nfk.h: NfkMogArgs -- the mixture epilogue's arguments of nfk_mog_made_step_f16x3."""
    _fields_ = [("num_components", c_int32), ("mode", c_int32), ("epsilon", c_float), ("u", _P), ("e", _P), ("ld_noise", c_int64)]


_SIGNATURES = {
    "nfk_version": (c_int, []),
    "nfk_last_error": (c_char_p, []),
    "nfk_launch_count": (c_int64, []),
    "nfk_check_device": (c_int, []),
    "nfk_rqs_elementwise": (c_int, [POINTER(NfkSplineDesc), c_int, _P, _P, _P, _P, c_int64, c_int64, c_int64, c_int64,
                                    _P, _P, c_int64, _P, _P]),
    "nfk_rqs_rows": (c_int, [POINTER(NfkSplineDesc), c_int, _P, c_int64, _P, _P, c_int32, _P, c_int32, _P, c_int64, _P,
                             c_int64, _P, _P]),
    "nfk_linear": (c_int, [_P, c_int64, _P, c_int64, _P, _P, c_int64, _P, c_int64, c_int64, c_int32, c_int32, c_int, c_int,
                           _P]),
    "nfk_linear_f16x3_supported": (c_int, [c_int64, c_int64, c_int32]),
    "nfk_linear_f16x3": (c_int, [_P, _P, c_int64, c_int32, _P, _P, c_int64, c_int32, _P, _P, c_int64, _P, c_int64, _P, _P, c_int64,
                                 c_int32, c_int32, c_int32, c_int, c_int, c_int64, c_int32, c_int32, _P, _P]),
    "nfk_absmax": (c_int, [_P, c_int64, c_int64, c_int32, _P, _P]),
    "nfk_split_f16": (c_int, [_P, c_int64, c_int32, c_int, c_int32, _P, _P, c_int64, c_int64, _P, _P]),
    "nfk_nchw_to_rows": (c_int, [_P, _P, c_int64, c_int32, c_int32, c_int, _P]),
    "nfk_squeeze_rows": (c_int, [_P, _P, c_int64, c_int32, c_int32, c_int32, c_int, _P]),
    "nfk_im2col3x3_f16": (c_int, [_P, _P, c_int64, _P, _P, c_int64, c_int64, c_int32, c_int32, c_int32, _P]),
    "nfk_segment_sum": (c_int, [_P, _P, c_int64, c_int32, _P]),
    "nfk_affine_coupling_final_f16x3": (c_int, [_P, _P, c_int64, c_int32, _P, _P, c_int64, c_int32, _P, c_int32, _P, c_int64, _P, c_int32,
                                                c_int32, c_int32, c_int32, c_int, _P, c_int64, _P, c_int64, _P, _P]),
    "nfk_glu_skip_rows": (c_int, [_P, c_int64, _P, c_int64, _P, c_int64, _P, c_int64, _P, _P, c_int64, c_int32, c_int, c_int64, c_int32,
                                  _P, _P]),
    "nfk_rq_coupling_final_supported": (c_int, [c_int32, c_int32, c_int32, c_int64]),
    "nfk_rq_coupling_final_padded_params": (c_int32, [c_int32, c_int32]),
    "nfk_rq_coupling_final_f16x3": (c_int, [POINTER(NfkSplineDesc), c_int, _P, _P, c_int64, c_int32, _P, _P, c_int64, c_int32, _P,
                                            c_int32, _P, c_int64, _P, c_int32, c_int32, _P, c_int64, _P, _P, c_int64, c_int32, _P,
                                            c_int64, _P, _P]),
    "nfk_rq_coupling_step_supported": (c_int, [c_int32, c_int32, c_int32, c_int32, c_int32]),
    "nfk_rq_coupling_step_workspace_bytes": (c_size_t, [c_int32]),
    "nfk_rq_coupling_step_f16x3": (c_int, [POINTER(NfkCouplingStep), _P]),
    "nfk_rq_coupling_step_terms_f16x3": (c_int, [POINTER(NfkCouplingStep), POINTER(NfkStepRowTerms), _P]),
    "nfk_affine_ar_step_f16x3": (c_int, [POINTER(NfkCouplingStep), POINTER(NfkStepRowTerms), _P]),
    "nfk_mog_made_padded_rows": (c_int32, [c_int32]),
    "nfk_mog_made_step_f16x3": (c_int, [POINTER(NfkCouplingStep), POINTER(NfkStepRowTerms), POINTER(NfkMogArgs), _P]),
    "nfk_gather_cols": (c_int, [_P, c_int64, _P, c_int32, _P, c_int64, c_int64, _P]),
    "nfk_actnorm": (c_int, [_P, c_int64, _P, _P, _P, c_int64, _P, c_float, c_int64, c_int32, c_int, _P]),
    "nfk_add_const": (c_int, [_P, c_float, c_int64, _P]),
    "nfk_fill": (c_int, [_P, c_float, c_int64, _P]),
    "nfk_affine_coupling_rows": (c_int, [_P, c_int64, _P, c_int32, c_int32, c_int, _P, c_int32, _P, c_int32, _P, c_int64,
                                         _P, c_int64, _P]),
    "nfk_std_normal_log_prob": (c_int, [_P, c_int64, c_int32, c_float, _P, _P, c_int64, _P]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def library_path():
    return _LIB_PATH


def load():
    """Load the shared library (once).  Raises NativeUnavailable when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise NativeUnavailable(
            "libnfk_sm90.so not found at {}; run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). nflows_b200 has no CPU/PyTorch fallback for CUDA tensors.".format(_LIB_PATH))
    lib = ctypes.CDLL(_LIB_PATH)
    for name, (restype, argtypes) in _SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError here means header and library disagree
        fn.restype = restype
        fn.argtypes = argtypes
    if lib.nfk_version() != 5:
        raise NativeUnavailable("libnfk_sm90.so ABI version {} != 5".format(lib.nfk_version()))
    _lib = lib
    return lib


_devices_checked = set()


def lib():
    """The library, after checking once per device that the CURRENT CUDA device can run it."""
    l = load()
    if not torch.cuda.is_available():
        raise NativeUnavailable("nflows_b200 native kernels need a CUDA device (H100, sm_90a)")
    dev = torch.cuda.current_device()
    if dev not in _devices_checked:
        check(l.nfk_check_device(), l)
        _devices_checked.add(dev)
    return l


def check(rc, l=None):
    if rc != 0:
        l = l or load()
        raise RuntimeError("libnfk_sm90: {} (code {})".format(l.nfk_last_error().decode(), rc))


def launch_count():
    return int(load().nfk_launch_count())


def stream():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return 0 if t is None else t.data_ptr()


def check_bin_sizes(num_bins, min_bin_width, min_bin_height):
    """The reference's checks of the minimal bin sizes (rational_quadratic.py:49-52)."""
    if min_bin_width * num_bins > 1.0:
        raise ValueError("Minimal bin width too large for the number of bins")
    if min_bin_height * num_bins > 1.0:
        raise ValueError("Minimal bin height too large for the number of bins")


def spline_desc(num_bins, tails, tail_bound, left, right, bottom, top, min_bin_width, min_bin_height, min_derivative,
                enable_identity_init=False, wh_divisor=1.0):
    """Validated NfkSplineDesc of a rational-quadratic spline (raises the reference's ValueError before anything is launched)."""
    import math
    check_bin_sizes(num_bins, min_bin_width, min_bin_height)
    if tails is None:
        lt, l, r, b, t = 0, left, right, bottom, top
    elif tails == "linear":
        lt, l, r, b, t = 1, -tail_bound, tail_bound, -tail_bound, tail_bound
    else:
        raise RuntimeError("{} tails are not implemented.".format(tails))
    beta = math.log(2) / (1 - min_derivative) if enable_identity_init else 1.0
    return NfkSplineDesc(int(num_bins), lt, float(l), float(r), float(b), float(t), float(min_bin_width),
                         float(min_bin_height), float(min_derivative), float(beta), float(wh_divisor))
