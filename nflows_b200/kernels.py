"""Tensor-level wrappers over the C ABI (include/nfk.h).  Each function enqueues exactly the kernels the
C entry point launches on the current CUDA stream; tensors are only used for their storage."""
import ctypes

import torch

from . import _native as N


#: bench.py sets this to a list to collect (tag, rows, start_event, end_event) around tagged launches
TIMELINE = None


class timed:
    """Brackets a launch with CUDA events on the current stream when bench.py asked for a timeline."""

    def __init__(self, tag, rows):
        self.tag, self.rows = tag, rows

    def __enter__(self):
        if TIMELINE is not None:
            self.e0 = torch.cuda.Event(enable_timing=True)
            self.e0.record()

    def __exit__(self, *exc):
        if TIMELINE is not None:
            e1 = torch.cuda.Event(enable_timing=True)
            e1.record()
            TIMELINE.append((self.tag, self.rows, self.e0, e1))


def _rows2d(t, name):
    if not (t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.stride(1) == 1):
        raise ValueError("{} must be a 2-D float32 CUDA tensor with unit column stride".format(name))
    return t


def _operand(t, name, shape, device, dtype=torch.float32):
    """t, checked to be a `dtype` tensor of exactly `shape` on `device` with unit column stride (a row pitch is all the kernels
    take), before anything is launched."""
    if not (torch.is_tensor(t) and t.dtype == dtype and t.device == device and tuple(t.shape) == tuple(shape)
            and (t.dim() == 1 or t.stride(1) == 1)):
        raise ValueError("{} must be a {} tensor of shape {} on {} with unit column stride, got {} {} {}".format(
            name, dtype, tuple(shape), device, tuple(t.shape) if torch.is_tensor(t) else type(t).__name__,
            getattr(t, "dtype", ""), getattr(t, "device", "")))
    return t


def _bias(bias, o, device):
    return None if bias is None else _operand(bias, "bias", (o,), device).contiguous()


def native_ok(t, context=None):
    """True when `t` is something the native path takes: CUDA, fp32, no autograd graph to build -- neither through `t` nor
    through a context tensor (the kernels take raw pointers: a graph to the context / embedding net would be dropped)."""
    if not (t.is_cuda and t.dtype == torch.float32):
        return False
    if torch.is_grad_enabled() and (t.requires_grad or (torch.is_tensor(context) and context.requires_grad)):
        return False
    return True


def on_device_of(t):
    """Context manager: make t's device current, so the launches below go to its current stream and every per-device
    resource (function attributes, SM count, workspaces) is the right one.  Every native entry point runs under it."""
    return torch.cuda.device(t.device)


_warned_eager = [False]


def warn_eager_cuda(t, module=None):
    """One warning when a CUDA fp32 call takes the differentiable PyTorch path only because autograd is on.  Quiet with
    config.native_training on: the user asked for training on this path (its splines run on the kernels)."""
    from . import config
    if config.native_training or _warned_eager[0] or not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32 and torch.is_grad_enabled()):
        return
    _warned_eager[0] = True
    import warnings
    warnings.warn("nflows_b200: this CUDA call runs the differentiable PyTorch formulation, not the native kernels, because "
                  "autograd is enabled and the inputs or parameters require grad; wrap inference in torch.no_grad() (or freeze "
                  "the parameters) to run the sm_90a kernels.", RuntimeWarning, stacklevel=3)


_DEFERRED = [None]


class deferred_flags:
    """`with deferred_flags(device) as d:` -- native calls inside the block share ONE device flag word and do not read it back
    (no host synchronisation per call: a caller that streams many chunks through a flow keeps the GPU fed); the caller reads
    `d.value()` once at the end and acts on it (raise_for_flag_value, or repeat with a smaller activation exponent)."""

    def __init__(self, device):
        self.flags = torch.zeros(1, dtype=torch.int32, device=device)

    def __enter__(self):
        self.prev, _DEFERRED[0] = _DEFERRED[0], self
        return self

    def __exit__(self, *exc):
        _DEFERRED[0] = self.prev

    def value(self):
        return int(self.flags.item())


def new_flags(device):
    d = _DEFERRED[0]
    if d is not None and d.flags.device == torch.device(device):
        return d.flags
    return torch.zeros(1, dtype=torch.int32, device=device)


def index_tensor(idx, device):
    return idx.to(device=device, dtype=torch.int32).contiguous()


def fill_(t, value):
    N.check(N.lib().nfk_fill(t.data_ptr(), float(value), t.numel(), N.stream()))
    return t


def add_const_(lad, c):
    N.check(N.lib().nfk_add_const(lad.data_ptr(), float(c), lad.numel(), N.stream()))
    return lad


def zeros_lad(x):
    return fill_(torch.empty(x.shape[0], dtype=torch.float32, device=x.device), 0.0)


def linear(x, weight, bias=None, residual=None, relu_in=False, relu_out=False, out=None):
    """out = post(pre(x) @ weight.T + bias) + residual; weight is [out_features, in_features] (nn.Linear layout)."""
    _rows2d(x, "x")
    _rows2d(weight, "weight")
    n, k = x.shape
    o = weight.shape[0]
    if weight.shape[1] != k:
        raise ValueError("weight is {}x{}, x has {} features".format(o, weight.shape[1], k))
    if out is None:
        out = torch.empty(n, o, dtype=torch.float32, device=x.device)
    _operand(out, "out", (n, o), x.device)
    bias = _bias(bias, o, x.device)
    if residual is not None:
        _operand(residual, "residual", (n, o), x.device)
    N.check(N.lib().nfk_linear(x.data_ptr(), x.stride(0), weight.data_ptr(), weight.stride(0), N.ptr(bias),
                               N.ptr(residual), residual.stride(0) if residual is not None else 0, out.data_ptr(),
                               out.stride(0), n, k, o, int(relu_in), int(relu_out), N.stream()))
    return out


def gather_cols(x, cols_i32, out=None):
    _rows2d(x, "x")
    n = x.shape[0]
    c = cols_i32.numel()
    if out is None:
        out = torch.empty(n, c, dtype=torch.float32, device=x.device)
    N.check(N.lib().nfk_gather_cols(x.data_ptr(), x.stride(0), cols_i32.data_ptr(), c, out.data_ptr(), out.stride(0), n,
                                    N.stream()))
    return out


def actnorm(x, scale, shift, lad_accum, lad_const, inverse):
    _rows2d(x, "x")
    y = torch.empty_like(x, memory_format=torch.contiguous_format)
    N.check(N.lib().nfk_actnorm(x.data_ptr(), x.stride(0), scale.data_ptr(), shift.data_ptr(), y.data_ptr(), y.stride(0),
                                N.ptr(lad_accum), float(lad_const), x.shape[0], x.shape[1], int(inverse), N.stream()))
    return y


def rqs_rows(desc, inverse, x, params, t_cols, id_cols, lad_accum, flags, out=None):
    """t_cols None: every column of x is transformed (d_t = x.shape[1], consecutive columns, no index list)."""
    _rows2d(x, "x")
    _rows2d(params, "params")
    if not params.is_contiguous():
        raise ValueError("params must be contiguous")
    y = torch.empty_like(x, memory_format=torch.contiguous_format) if out is None else out
    d_t = x.shape[1] if t_cols is None else t_cols.numel()
    N.check(N.lib().nfk_rqs_rows(ctypes.byref(desc), int(inverse), x.data_ptr(), x.stride(0), params.data_ptr(),
                                 N.ptr(t_cols), d_t, N.ptr(id_cols), 0 if id_cols is None else id_cols.numel(),
                                 y.data_ptr(), y.stride(0),
                                 N.ptr(lad_accum), x.shape[0], N.ptr(flags), N.stream()))
    return y


def rqs_rows_backward(desc, inverse, x, params, grad_y, grad_lad, want_grad_x=True):
    """Backward of rqs_rows over every column of x (include/nfk.h: nfk_rqs_rows_backward): returns (grad_x or None, grad_params)
    for the cotangents grad_y ([n, d_t], unit column stride, or None) and grad_lad ([n] of the summed log|det|, or None)."""
    _rows2d(x, "x")
    _rows2d(params, "params")
    if not params.is_contiguous():
        raise ValueError("params must be contiguous")
    n, d_t = x.shape
    if grad_y is not None:
        _rows2d(grad_y, "grad_y")
        if tuple(grad_y.shape) != (n, d_t):
            raise ValueError("grad_y is {}, x is {}".format(tuple(grad_y.shape), tuple(x.shape)))
    if grad_lad is not None:
        if not (grad_lad.is_cuda and grad_lad.dtype == torch.float32 and grad_lad.numel() == n):
            raise ValueError("grad_lad must be a float32 CUDA tensor of {} entries".format(n))
        grad_lad = grad_lad.contiguous()
    grad_params = torch.empty_like(params)
    grad_x = torch.empty(n, d_t, dtype=torch.float32, device=x.device) if want_grad_x else None
    with timed("rqs_rows_backward", n):
        N.check(N.lib().nfk_rqs_rows_backward(ctypes.byref(desc), int(inverse), x.data_ptr(), x.stride(0), params.data_ptr(),
                                              N.ptr(grad_y), grad_y.stride(0) if grad_y is not None else 0, N.ptr(grad_lad),
                                              N.ptr(grad_x), grad_x.stride(0) if grad_x is not None else 0,
                                              grad_params.data_ptr(), d_t, n, N.stream()))
    return grad_x, grad_params


def _planes_shapes(x, params, m):
    """(n, c_t, pixels) of a 4-D contiguous fp32 CUDA x [n, c_t, h, w] and params [n, c_t * m, h, w], checked."""
    for t, name in ((x, "x"), (params, "params")):
        if not (t.is_cuda and t.dtype == torch.float32 and t.dim() == 4 and t.is_contiguous()):
            raise ValueError("{} must be a contiguous 4-D float32 CUDA tensor".format(name))
    n, c_t, h, w = x.shape
    if tuple(params.shape) != (n, c_t * m, h, w) or params.device != x.device:
        raise ValueError("params is {}, expected {} on {}".format(tuple(params.shape), (n, c_t * m, h, w), x.device))
    return n, c_t, h * w


def rqs_planes(desc, inverse, x, params, lad_accum, flags):
    """Spline of an image coupling on the plane layout (include/nfk.h: nfk_rqs_planes): x [n, c_t, h, w], params [n, c_t * M, h, w]
    (the conditioner's output as it is), both contiguous; returns y like x and adds each sample's log|det| to lad_accum [n]."""
    n, c_t, pixels = _planes_shapes(x, params, N.spline_param_count(desc.num_bins, desc.linear_tails))
    y = torch.empty_like(x)
    with timed("rqs_planes", n):
        N.check(N.lib().nfk_rqs_planes(ctypes.byref(desc), int(inverse), x.data_ptr(), c_t * pixels, params.data_ptr(),
                                       params[0].numel() if n else 0, c_t, pixels, y.data_ptr(), c_t * pixels, N.ptr(lad_accum), n,
                                       N.ptr(flags), N.stream()))
    return y


def rqs_planes_backward(desc, inverse, x, params, grad_y, grad_lad, want_grad_x=True):
    """Backward of rqs_planes (include/nfk.h: nfk_rqs_planes_backward): returns (grad_x or None, grad_params) for the cotangents
    grad_y (like x, or None) and grad_lad ([n] of the per-sample log|det|, or None)."""
    n, c_t, pixels = _planes_shapes(x, params, N.spline_param_count(desc.num_bins, desc.linear_tails))
    if grad_y is not None:
        if tuple(grad_y.shape) != tuple(x.shape) or grad_y.dtype != torch.float32 or grad_y.device != x.device:
            raise ValueError("grad_y is {}, x is {}".format(tuple(grad_y.shape), tuple(x.shape)))
        grad_y = grad_y.contiguous()
    if grad_lad is not None:
        if not (grad_lad.is_cuda and grad_lad.dtype == torch.float32 and grad_lad.numel() == n):
            raise ValueError("grad_lad must be a float32 CUDA tensor of {} entries".format(n))
        grad_lad = grad_lad.contiguous()
    grad_params = torch.empty_like(params)
    grad_x = torch.empty_like(x) if want_grad_x else None
    ld, ldp = c_t * pixels, params[0].numel() if n else 0
    with timed("rqs_planes_backward", n):
        N.check(N.lib().nfk_rqs_planes_backward(ctypes.byref(desc), int(inverse), x.data_ptr(), ld, params.data_ptr(), ldp,
                                                N.ptr(grad_y), ld, N.ptr(grad_lad), N.ptr(grad_x), ld, grad_params.data_ptr(), ldp,
                                                c_t, pixels, n, N.stream()))
    return grad_x, grad_params


def rqs_shared_backward(desc, inverse, x, uw, uh, ud, grad_y, grad_lad, want_grad_x=True):
    """Backward of the batch-shared spline of PiecewiseRationalQuadraticCDF (include/nfk.h: nfk_rqs_shared_backward): x [n, F]
    contiguous, uw / uh [F, K], ud [F, K -+ 1]; cotangents grad_y [n, F] or None, grad_lad [n] or None.  Returns
    (grad_x or None, grad_uw, grad_uh, grad_ud), the parameter gradients summed over the rows."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.is_contiguous()):
        raise ValueError("x must be a contiguous 2-D float32 CUDA tensor")
    n, f = x.shape
    k = desc.num_bins
    nd = N.spline_param_count(k, desc.linear_tails) - 2 * k
    uw = _operand(uw, "uw", (f, k), x.device).contiguous()
    uh = _operand(uh, "uh", (f, k), x.device).contiguous()
    ud = _operand(ud, "ud", (f, nd), x.device).contiguous()
    if grad_y is not None:
        grad_y = _operand(grad_y, "grad_y", (n, f), x.device).contiguous()
    if grad_lad is not None:
        grad_lad = _operand(grad_lad.reshape(-1), "grad_lad", (n,), x.device).contiguous()
    lib = N.lib()
    ws = torch.empty(int(lib.nfk_rqs_shared_backward_workspace(n, f, k, int(desc.linear_tails))) // 4, dtype=torch.float32,
                     device=x.device)
    grad_x = torch.empty_like(x) if want_grad_x else None
    guw, guh, gud = torch.empty_like(uw), torch.empty_like(uh), torch.empty_like(ud)
    with timed("rqs_shared_backward", n):
        N.check(lib.nfk_rqs_shared_backward(ctypes.byref(desc), int(inverse), x.data_ptr(), uw.data_ptr(), uh.data_ptr(),
                                            N.ptr(ud) if nd else 0, N.ptr(grad_y), N.ptr(grad_lad), N.ptr(grad_x), guw.data_ptr(),
                                            guh.data_ptr(), N.ptr(gud) if nd else 0, f, n, N.ptr(ws) if ws.numel() else 0,
                                            ws.numel() * 4, N.stream()))
    return grad_x, guw, guh, gud


def rqs_elementwise(desc, inverse, x, uw, uh, ud, param_period=0, flags=None):
    """x: any shape (contiguous); uw/uh/ud: [..., K], [..., K], [..., K-1|K+1] contiguous on the last dim."""
    x = x.contiguous()
    uw, uh, ud = uw.contiguous(), uh.contiguous(), ud.contiguous()
    y = torch.empty_like(x)
    lad = torch.empty_like(x)
    N.check(N.lib().nfk_rqs_elementwise(ctypes.byref(desc), int(inverse), x.data_ptr(), uw.data_ptr(), uh.data_ptr(),
                                        ud.data_ptr(), uw.shape[-1], uh.shape[-1], ud.shape[-1], int(param_period),
                                        y.data_ptr(), lad.data_ptr(), x.numel(), N.ptr(flags), N.stream()))
    return y, lad


def affine_coupling_rows(x, params, mult, scale_activation, inverse, t_cols, id_cols, lad_accum, out=None):
    _rows2d(x, "x")
    if not params.is_contiguous():
        raise ValueError("params must be contiguous")
    y = torch.empty_like(x, memory_format=torch.contiguous_format) if out is None else out
    N.check(N.lib().nfk_affine_coupling_rows(x.data_ptr(), x.stride(0), params.data_ptr(), int(mult), int(scale_activation),
                                             int(inverse), N.ptr(t_cols), t_cols.numel(), N.ptr(id_cols), id_cols.numel(),
                                             y.data_ptr(), y.stride(0), N.ptr(lad_accum), x.shape[0], N.stream()))
    return y


def std_normal_log_prob(z, log_z, lad=None):
    _rows2d(z, "z")
    out = torch.empty(z.shape[0], dtype=torch.float32, device=z.device)
    N.check(N.lib().nfk_std_normal_log_prob(z.data_ptr(), z.stride(0), z.shape[1], float(log_z), N.ptr(lad), out.data_ptr(),
                                            z.shape[0], N.stream()))
    return out


class Float16RangeError(RuntimeError):
    """A value left the representable range of the fp16 split pairs (NFK_FLAG_F16_RANGE)."""


def raise_for_flags(flags):
    """Mirror the reference's exceptions (rational_quadratic.py:81-82, :142).  One device->host read."""
    raise_for_flag_value(int(flags.item()))


def raise_for_flag_value(v):
    from .transforms.base import InputOutsideDomain
    if v & 1:
        raise InputOutsideDomain()
    if v & 2:
        raise AssertionError("rational-quadratic spline inverse: negative discriminant")
    if v & 4:
        raise Float16RangeError("an activation exceeded the fp16 split range of the tensor-core dense layers "
                                "(|value| * 2^config.activation_exp > 65000) and config.auto_activation_exp is off or exhausted: "
                                "lower nflows_b200.config.activation_exp or set NFLOWS_B200_GEMM=simt")


_warned_rescale = [False]


def run_with_activation_rescale(fn):
    """fn() -> (outputs, lad, flags): runs it, reads the flag word (config.check_domain) and, when a value left the fp16 split
    range, runs it again with a smaller power-of-two scale for the activation pairs (config.auto_activation_exp) -- an input
    magnitude the reference accepts must not raise here.  Other flags raise the reference's exceptions."""
    from . import config
    saved = config.activation_exp
    try:
        while True:
            out, lad, flags = fn()
            if not config.check_domain or (_DEFERRED[0] is not None and flags is _DEFERRED[0].flags):
                return out, lad
            v = int(flags.item())
            if (v & 4) and config.auto_activation_exp and config.activation_exp > -24:
                config.activation_exp = max(-24, config.activation_exp - 5)      # results of this attempt are discarded
                if not _warned_rescale[0]:
                    _warned_rescale[0] = True
                    import warnings
                    warnings.warn("nflows_b200: an activation left the fp16 split range at activation_exp=%d; the call is "
                                  "repeated with smaller exponents (set config.activation_exp lower to avoid the repeat)" % saved,
                                  RuntimeWarning, stacklevel=4)
                continue
            raise_for_flag_value(v)
            return out, lad
    finally:
        config.activation_exp = saved


# ---- split-fp16 tensor-core dense layers ------------------------------------------------------------------------------
class Pair16:
    """fp16 split pair of an fp32 matrix: value * 2^exp = hi + lo (include/nfk.h, nfk_linear_f16x3)."""
    __slots__ = ("hi", "lo", "exp")

    def __init__(self, hi, lo, exp):
        self.hi, self.lo, self.exp = hi, lo, int(exp)

    @classmethod
    def empty(cls, rows, cols, exp, device):
        return cls(torch.empty(rows, cols, dtype=torch.float16, device=device),
                   torch.empty(rows, cols, dtype=torch.float16, device=device), exp)

    @classmethod
    def zeros(cls, rows, cols, exp, device):
        p = cls.empty(rows, cols, exp, device)
        for t in (p.hi, p.lo):
            if t.numel() and t.numel() % 2 == 0:
                fill_(t.view(-1).view(torch.float32), 0.0)      # two fp16 zeros per fp32 zero
            else:
                t.zero_()
        return p

    @property
    def shape(self):
        return self.hi.shape

    def rows(self, r0, r1):
        return Pair16(self.hi[r0:r1], self.lo[r0:r1], self.exp)

    def cols(self, c0, c1):
        return Pair16(self.hi[:, c0:c1], self.lo[:, c0:c1], self.exp)

    def float(self):
        """The represented fp32 values (tests)."""
        return (self.hi.double() + self.lo.double()).mul_(2.0 ** -self.exp).float()


def weight_exp(w):
    """Power-of-two exponent that lifts max |w| to 2^14: the whole matrix, including the lo parts, stays clear of fp16's
    subnormals and of its overflow."""
    import math
    w = _rows2d(w.detach(), "w")
    out = fill_(torch.empty(1, dtype=torch.float32, device=w.device), 0.0)
    N.check(N.lib().nfk_absmax(w.data_ptr(), w.stride(0), w.shape[0], w.shape[1], out.data_ptr(), N.stream()))
    amax = float(out.item())
    if not (amax > 0.0) or not math.isfinite(amax):
        return 0
    return max(-40, min(40, 14 - math.ceil(math.log2(amax))))


def split_f16(x, exp, relu=False, out=None, flags=None):
    """Pair16 of pre(x) (x: 2-D fp32, unit column stride; may be a strided column block)."""
    _rows2d(x, "x")
    n, c = x.shape
    pair = out if out is not None else Pair16.empty(n, c, exp, x.device)
    if pair.exp != exp:
        raise ValueError("destination pair has exponent {}, asked for {}".format(pair.exp, exp))
    with timed("split_%d" % c, n):
        N.check(N.lib().nfk_split_f16(x.data_ptr(), x.stride(0), c, int(relu), int(exp), pair.hi.data_ptr(), pair.lo.data_ptr(),
                                      pair.hi.stride(0), n, N.ptr(flags), N.stream()))
    return pair


def glu_skip(t, gate, skip=None, want_y=True, want_split=False, split_relu=False, split_exp=None, pair_out=None, flags=None):
    """skip + t * sigmoid(gate) (the context gate of a residual block, nn/nets/resnet.py:50-53) in one pass.
    Returns (y fp32 or None, Pair16 of pre(y) or None)."""
    _rows2d(t, "t"); _rows2d(gate, "gate")
    n, c = t.shape
    y = torch.empty(n, c, dtype=torch.float32, device=t.device) if want_y else None
    pair = None
    if want_split:
        from . import config
        exp = config.activation_exp if split_exp is None else split_exp
        pair = pair_out if pair_out is not None else Pair16.empty(n, c, exp, t.device)
    with timed("glu_skip_%d" % c, n):
        N.check(N.lib().nfk_glu_skip_rows(
            t.data_ptr(), t.stride(0), gate.data_ptr(), gate.stride(0), N.ptr(skip), skip.stride(0) if skip is not None else 0,
            N.ptr(y), y.stride(0) if y is not None else 0, pair.hi.data_ptr() if pair else 0, pair.lo.data_ptr() if pair else 0,
            pair.hi.stride(0) if pair else 0, pair.exp if pair else 0, int(split_relu), n, c, N.ptr(flags), N.stream()))
    return y, pair


def _t_cols(t_cols):
    """(pointer, first column, count) of the transformed columns: an int32 index tensor (first column -1), or (first, count)
    when they are consecutive (null pointer)."""
    if isinstance(t_cols, tuple):
        return 0, int(t_cols[0]), int(t_cols[1])
    return t_cols.data_ptr(), -1, t_cols.numel()


def affine_coupling_final(a, w, bias, x, t_cols, mult, scale_activation, inverse, y, lad_accum, flags=None):
    """Last conditioner layer + affine / additive coupling in one wgmma kernel (include/nfk.h:
    nfk_affine_coupling_final_f16x3).  a: Pair16 of the trunk output; w, bias: dense.pack_final_affine (interleaved rows);
    t_cols: int32 index tensor of the transformed columns or (first_column, count); writes the transformed columns of y."""
    cols_ptr, col0, d_t = _t_cols(t_cols)
    with timed("affine_coupling_final", x.shape[0]):
        N.check(N.lib().nfk_affine_coupling_final_f16x3(
            a.hi.data_ptr(), a.lo.data_ptr(), a.hi.stride(0), a.exp, w.hi.data_ptr(), w.lo.data_ptr(), w.hi.stride(0), w.exp,
            bias.data_ptr(), a.shape[1], x.data_ptr(), x.stride(0), cols_ptr, col0, d_t, int(mult), int(scale_activation), int(inverse),
            y.data_ptr(), y.stride(0), N.ptr(lad_accum), x.shape[0], N.ptr(flags), N.stream()))
    return y


# ---- image path: pixel rows (include/nfk.h, "image path") ----------------------------------------------------------------
def nchw_to_rows(x):
    """[B, C, H, W] fp32 -> pixel rows [B*H*W, C]."""
    b, c, h, w = x.shape
    x = x.contiguous()
    rows = torch.empty(b * h * w, c, dtype=torch.float32, device=x.device)
    with timed("nchw_to_rows", b * h * w):
        N.check(N.lib().nfk_nchw_to_rows(x.data_ptr(), rows.data_ptr(), b, c, h * w, 0, N.stream()))
    return rows


def rows_to_nchw(rows, b, c, h, w):
    out = torch.empty(b, c, h, w, dtype=torch.float32, device=rows.device)
    rows = rows.contiguous()
    with timed("rows_to_nchw", b * h * w):
        N.check(N.lib().nfk_nchw_to_rows(rows.data_ptr(), out.data_ptr(), b, c, h * w, 1, N.stream()))
    return out


def squeeze_rows(rows, b, c, h, w, inverse=False):
    """SqueezeTransform(2) on pixel rows of a [b, c, h, w] image; returns (rows, (c, h, w)) of the result."""
    rows = rows.contiguous()
    if not inverse:
        if h % 2 or w % 2:
            raise ValueError("Input image size not compatible with the factor.")
        out = torch.empty(b * (h // 2) * (w // 2), 4 * c, dtype=torch.float32, device=rows.device)
        N.check(N.lib().nfk_squeeze_rows(rows.data_ptr(), out.data_ptr(), b, h // 2, w // 2, c, 0, N.stream()))
        return out, (4 * c, h // 2, w // 2)
    if c < 4 or c % 4:
        raise ValueError("Invalid number of channel dimensions.")
    out = torch.empty(b * h * w * 4, c // 4, dtype=torch.float32, device=rows.device)
    N.check(N.lib().nfk_squeeze_rows(rows.data_ptr(), out.data_ptr(), b, h, w, c // 4, 1, N.stream()))
    return out, (c // 4, 2 * h, 2 * w)


def im2col3x3(pair, n_images, h, w):
    """Pair16 [n_images*h*w, C] -> Pair16 [n_images*h*w, 9*C]: the operand of a 3x3 / padding-1 convolution as a dense layer."""
    n, c = pair.shape
    if n != n_images * h * w:
        raise ValueError("{} rows are not {} images of {}x{} pixels".format(n, n_images, h, w))
    out = Pair16.empty(n, 9 * c, pair.exp, pair.hi.device)
    with timed("im2col3x3_%d" % c, n):
        N.check(N.lib().nfk_im2col3x3_f16(pair.hi.data_ptr(), pair.lo.data_ptr(), pair.hi.stride(0), out.hi.data_ptr(), out.lo.data_ptr(),
                                          out.hi.stride(0), n_images, h, w, c, N.stream()))
    return out


def segment_sum_(values, out_accum, segment_len):
    """out_accum[s] += sum(values[s*segment_len : (s+1)*segment_len])."""
    N.check(N.lib().nfk_segment_sum(values.data_ptr(), out_accum.data_ptr(), out_accum.numel(), int(segment_len), N.stream()))
    return out_accum


def f16x3_supported(lda, ldw, in_features):
    return bool(N.load().nfk_linear_f16x3_supported(int(lda), int(ldw), int(in_features)))


def linear_f16x3(a, w, bias=None, residual=None, relu_out=False, want_y=True, want_split=False, split_relu=False,
                 split_exp=None, split_cols=0, y_out=None, pair_out=None, flags=None, y_first_col=0):
    """wgmma dense layer on Pair16 operands.  Returns (y or None, Pair16 or None); y_out / pair_out are caller-provided
    destinations (row slices of larger buffers).  The pair output covers the first split_cols columns (0 = all); y_first_col > 0:
    the fp32 result is only needed from that column on (the columns before it may stay unwritten)."""
    n, k = a.shape
    o = w.shape[0]
    dev = a.hi.device
    y = (y_out if y_out is not None else torch.empty(n, o, dtype=torch.float32, device=dev)) if want_y else None
    if y_out is not None and want_y:
        _operand(y_out, "y_out", (n, o), dev)
    pair = None
    if want_split:
        from . import config
        exp = config.activation_exp if split_exp is None else split_exp
        pair = pair_out if pair_out is not None else Pair16.empty(n, o, exp, dev)
        if pair_out is not None:
            _operand(pair.hi, "pair_out.hi", (n, o), dev, torch.float16)
            _operand(pair.lo, "pair_out.lo", (n, o), dev, torch.float16)
            if pair.hi.stride(0) != pair.lo.stride(0):
                raise ValueError("pair_out.hi and pair_out.lo must share one row pitch")
    bias = _bias(bias, o, dev)
    if residual is not None:
        _operand(residual, "residual", (n, o), dev)
    with timed("linear_%dx%d" % (k, o), n):
        N.check(N.lib().nfk_linear_f16x3(
            a.hi.data_ptr(), a.lo.data_ptr(), a.hi.stride(0), a.exp, w.hi.data_ptr(), w.lo.data_ptr(), w.hi.stride(0), w.exp,
            N.ptr(bias), N.ptr(residual), residual.stride(0) if residual is not None else 0, N.ptr(y),
            y.stride(0) if y is not None else 0, pair.hi.data_ptr() if pair else 0, pair.lo.data_ptr() if pair else 0,
            pair.hi.stride(0) if pair else 0, pair.exp if pair else 0, int(split_cols), int(y_first_col), int(relu_out),
            int(split_relu), n, k, o, N.ptr(flags), N.stream()))
    return y, pair


def absmax_start(x):
    """Enqueues max |x| over a 2-D fp32 matrix (unit column stride) and its copy to pinned host memory; returns a function that
    waits for that copy (not for the rest of the stream) and gives the value.  Work enqueued between the two keeps the GPU busy
    while the host waits."""
    _rows2d(x, "x")
    out = fill_(torch.empty(1, dtype=torch.float32, device=x.device), 0.0)
    with timed("absmax", x.shape[0]):
        N.check(N.lib().nfk_absmax(x.data_ptr(), x.stride(0), x.shape[0], x.shape[1], out.data_ptr(), N.stream()))
    host = torch.empty(1, dtype=torch.float32, pin_memory=True)
    host.copy_(out, non_blocking=True)
    done = torch.cuda.Event()
    done.record()

    def read():
        done.synchronize()
        return float(host[0])
    return read


def absmax(x):
    """max |x| over a 2-D fp32 matrix (unit column stride), read back to the host."""
    return absmax_start(x)()


def gradient_exp(amax):
    """Exponent of a gradient pair whose largest element has magnitude amax: amax * 2^exp lands in [2^13, 2^14), as for weights
    (kernels.weight_exp).  Every element v is then carried within 2^-22 |v| + 2^-38 amax (the second term: half the fp16 subnormal
    spacing of lo), so gradients of any overall scale down to amax = 2^-46 (the exponent's range is +-60) keep their accuracy;
    elements below 2^-39 amax are flushed to zero.  0 for an all-zero (or non-finite) tensor."""
    import math
    if not (amax > 0.0) or not math.isfinite(amax):
        return 0
    return max(-60, min(60, 14 - math.ceil(math.log2(amax))))


def linear_wgrad(g, a, want_bias=True):
    """(dW [out, in], db [out] or None) of a split-fp16 dense layer (include/nfk.h: nfk_linear_f16x3_wgrad): dW = G^T A, db = the
    column sums of G.  g: Pair16 of the pre-activation gradient [n, >= out] (columns past `out` ignored), a: Pair16 of the layer
    input [n, in]; out = g's column count unless g is padded (pass the Pair16 cols view)."""
    n, o = g.shape
    k = a.shape[1]
    dev = a.hi.device
    if a.shape[0] != n or g.hi.device != dev:
        raise ValueError("gradient pair {} and input pair {} must have the same rows on one device".format(tuple(g.shape), tuple(a.shape)))
    for t, name in ((g.hi, "g.hi"), (g.lo, "g.lo"), (a.hi, "a.hi"), (a.lo, "a.lo")):
        if not (t.dtype == torch.float16 and t.dim() == 2 and (t.shape[0] == 0 or t.stride(1) == 1)):
            raise ValueError("{} must be a 2-D float16 tensor with unit column stride".format(name))
    if g.hi.stride(0) != g.lo.stride(0) or a.hi.stride(0) != a.lo.stride(0):
        raise ValueError("the halves of a pair must share one row pitch")
    lib = N.lib()
    ws = torch.empty((int(lib.nfk_linear_f16x3_wgrad_workspace(n, o, k, int(want_bias))) + 3) // 4, dtype=torch.float32, device=dev)
    dw = torch.empty(o, k, dtype=torch.float32, device=dev)
    db = torch.empty(o, dtype=torch.float32, device=dev) if want_bias else None
    with timed("linear_wgrad_%dx%d" % (k, o), n):
        N.check(lib.nfk_linear_f16x3_wgrad(g.hi.data_ptr(), g.lo.data_ptr(), g.hi.stride(0), g.exp, a.hi.data_ptr(), a.lo.data_ptr(),
                                           a.hi.stride(0), a.exp, dw.data_ptr(), dw.stride(0), N.ptr(db), n, o, k,
                                           N.ptr(ws) if ws.numel() else 0, ws.numel() * 4, N.stream()))
    return dw, db


def mask_split(da, exp, mask=None, skip=None, cols_pad=None, want_y=False, flags=None):
    """(Pair16 [n, cols_pad] of v * 2^exp, fp32 v [n, c] or None) for v = da * [mask != 0] + skip (include/nfk.h:
    nfk_mask_split_f16): the gradient of the layer in front of a relu (mask: the Pair16 the forward saved) and / or a skip
    connection, split for the tensor cores; the pair's columns past c are zero."""
    _rows2d(da, "da")
    n, c = da.shape
    cols_pad = c if cols_pad is None else int(cols_pad)
    if mask is not None:
        if tuple(mask.shape[:1]) != (n,) or mask.shape[1] < c or mask.hi.stride(0) != mask.lo.stride(0):
            raise ValueError("mask pair {} does not cover da {}".format(tuple(mask.shape), (n, c)))
    if skip is not None:
        _operand(skip, "skip", (n, c), da.device)
    pair = Pair16.empty(n, cols_pad, exp, da.device)
    y = torch.empty(n, c, dtype=torch.float32, device=da.device) if want_y else None
    with timed("mask_split_%d" % c, n):
        N.check(N.lib().nfk_mask_split_f16(da.data_ptr(), da.stride(0), mask.hi.data_ptr() if mask is not None else 0,
                                           mask.lo.data_ptr() if mask is not None else 0, mask.hi.stride(0) if mask is not None else 0,
                                           N.ptr(skip), skip.stride(0) if skip is not None else 0, c, cols_pad, int(exp),
                                           pair.hi.data_ptr(), pair.lo.data_ptr(), pair.hi.stride(0), N.ptr(y),
                                           y.stride(0) if y is not None else 0, n, N.ptr(flags), N.stream()))
    return pair, y


def rq_coupling_final_supported(num_bins, tails, hidden, lda):
    return bool(N.load().nfk_rq_coupling_final_supported(int(num_bins), 1 if tails == "linear" else 0, int(hidden), int(lda)))


def rq_coupling_final_padded_params(num_bins, tails):
    return int(N.load().nfk_rq_coupling_final_padded_params(int(num_bins), 1 if tails == "linear" else 0))


def rq_coupling_final(desc, inverse, a, wp, bias_packed, x, t_cols, y, lad_accum, flags, y_pair=None):
    """Fused final conditioner layer + RQ spline + scatter + log|det| (one wgmma kernel).  a, wp: Pair16; y may be x.
    t_cols: int32 column index tensor of the transformed features, or (first_column, count) when they are consecutive.
    y_pair (with y=None): write the fp16 split pair of the outputs into this Pair16 (same shape as x) instead of fp32."""
    cols_ptr, col0, d_t = _t_cols(t_cols)
    N.check(N.lib().nfk_rq_coupling_final_f16x3(
        ctypes.byref(desc), int(inverse), a.hi.data_ptr(), a.lo.data_ptr(), a.hi.stride(0), a.exp, wp.hi.data_ptr(),
        wp.lo.data_ptr(), wp.hi.stride(0), wp.exp, bias_packed.data_ptr(), a.shape[1], x.data_ptr(), x.stride(0),
        cols_ptr, col0, d_t, N.ptr(y), y.stride(0) if y is not None else 0, y_pair.hi.data_ptr() if y_pair is not None else 0,
        y_pair.lo.data_ptr() if y_pair is not None else 0, y_pair.hi.stride(0) if y_pair is not None else 0,
        y_pair.exp if y_pair is not None else 0, N.ptr(lad_accum), x.shape[0], N.ptr(flags), N.stream()))
    return y


# ---- the whole RQ-coupling step in one kernel --------------------------------------------------------------------------
def rq_coupling_step_supported(num_bins, tails, hidden, in_features, num_square_layers):
    return bool(N.load().nfk_rq_coupling_step_supported(int(num_bins), 1 if tails == "linear" else 0, int(hidden), int(in_features),
                                                        int(num_square_layers)))


_STEP_WORKSPACE = {}


def step_workspace(device, hidden):
    """Scratch of the coupling-step kernel (skip tensors, one 128 x hidden tile per CTA), one buffer per (device, stream)."""
    key = (str(device), torch.cuda.current_stream(device).cuda_stream, int(hidden))
    ws = _STEP_WORKSPACE.get(key)
    if ws is None:
        nbytes = int(N.lib().nfk_rq_coupling_step_workspace_bytes(int(hidden)))
        ws = torch.empty(nbytes // 4, dtype=torch.float32, device=device)
        _STEP_WORKSPACE[key] = ws
    return ws


def _trunk_descriptor(plan, a, flags):
    """NfkCouplingStep with the trunk of `plan` (dense.StepPlan) on the conditioner input pair `a` filled in."""
    n, k0 = a.shape
    h = plan.hidden
    ws = step_workspace(a.hi.device, h)
    d = N.NfkCouplingStep()
    d.a_hi, d.a_lo, d.lda, d.a_exp, d.in_features = a.hi.data_ptr(), a.lo.data_ptr(), a.hi.stride(0), a.exp, k0
    d.w0_hi, d.w0_lo, d.ldw0, d.w0_exp = plan.w0.hi.data_ptr(), plan.w0.lo.data_ptr(), plan.w0.hi.stride(0), plan.w0.exp
    nsq = len(plan.layer_flags) - 1
    if nsq:
        d.wt_hi, d.wt_lo, d.ldwt = plan.wt_hi.data_ptr(), plan.wt_lo.data_ptr(), plan.wt_hi.stride(0)
        d.wt_exps = plan.wt_exps_c
    d.bias_trunk = plan.bias.data_ptr()
    d.layer_flags = plan.layer_flags_c
    d.num_square_layers = nsq
    d.act_exp = plan.act_exp
    d.hidden_features = h
    d.n_rows = n
    d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel() * 4
    d.flags = N.ptr(flags)
    return d


def _row_terms(terms, plan, a):
    """NfkStepRowTerms of per-trunk-layer fp32 terms (None entries: no term on that layer), checked against the launch."""
    n, h = a.shape[0], plan.hidden
    if len(terms) > len(plan.layer_flags):
        raise ValueError("{} row terms for a trunk of {} layers".format(len(terms), len(plan.layer_flags)))
    rt = N.NfkStepRowTerms()
    for l, t in enumerate(terms):
        if t is None:
            continue
        if not (t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.stride(1) == 1 and t.shape[0] >= n
                and t.shape[1] >= h and t.device == a.hi.device):
            raise ValueError("row term of layer {}: need a 2-D float32 CUDA tensor of at least {} x {} with unit column stride on {}, "
                             "got {} {} {}".format(l, n, h, a.hi.device, tuple(t.shape), t.dtype, t.device))
        rt.layer[l].add, rt.layer[l].ld = t.data_ptr(), t.stride(0)
    return rt


def rq_coupling_step(plan, a, desc=None, inverse=False, wp=None, bias_packed=None, x=None, t_cols=None, y=None, lad_accum=None,
                     flags=None, y_pair=None, h_pair=None, terms=None):
    """ONE launch for conditioner + spline of an RQ coupling (include/nfk.h: nfk_rq_coupling_step_f16x3).
    plan: dense.StepPlan (packed trunk weights, layer flags); a: Pair16 of the conditioner input.
    Either (desc, wp, bias_packed, x, t_cols, y | y_pair, lad_accum) for the full step, or h_pair (Pair16 [n, hidden]) to stop after
    the trunk and get its output pair.
    terms: per trunk layer an fp32 [>= n, >= hidden] tensor (unit column stride) added to that layer's pre-activation, or None
    (include/nfk.h: nfk_rq_coupling_step_terms_f16x3); full step only."""
    n = a.shape[0]
    h = plan.hidden
    nsq = len(plan.layer_flags) - 1
    d = _trunk_descriptor(plan, a, flags)
    d.spline = ctypes.pointer(desc) if desc is not None else None
    d.inverse = int(inverse)
    if h_pair is not None:
        if h_pair.exp != plan.act_exp:
            raise ValueError("trunk output pair must carry the plan's activation exponent")
        d.h_hi, d.h_lo, d.ldh = h_pair.hi.data_ptr(), h_pair.lo.data_ptr(), h_pair.hi.stride(0)
        tag = "trunk_step_%dx%d" % (h, nsq + 1)
    else:
        d.t_cols, d.t_col0, d.d_t = _t_cols(t_cols)
        d.wp_hi, d.wp_lo, d.ldwp, d.wp_exp = wp.hi.data_ptr(), wp.lo.data_ptr(), wp.hi.stride(0), wp.exp
        d.bias_packed = bias_packed.data_ptr()
        d.x, d.ldx = x.data_ptr(), x.stride(0)
        if y is not None:
            d.y, d.ldy = y.data_ptr(), y.stride(0)
        if y_pair is not None:
            d.y_hi, d.y_lo, d.lds, d.y_exp = y_pair.hi.data_ptr(), y_pair.lo.data_ptr(), y_pair.hi.stride(0), y_pair.exp
        d.lad_accum = N.ptr(lad_accum)
        tag = "rq_coupling_step"
    if terms is None:
        with timed(tag, n):
            N.check(N.lib().nfk_rq_coupling_step_f16x3(ctypes.byref(d), N.stream()))
        return y if y is not None else (y_pair if y_pair is not None else h_pair)
    rt = _row_terms(terms, plan, a)
    with timed(tag, n):
        N.check(N.lib().nfk_rq_coupling_step_terms_f16x3(ctypes.byref(d), ctypes.byref(rt), N.stream()))
    return y if y is not None else (y_pair if y_pair is not None else h_pair)


# ---- the masked affine autoregressive step in one kernel ---------------------------------------------------------------
def affine_ar_step(plan, a, wf, bias, x, cols, y, lad_accum, flags, inverse, terms=None):
    """ONE launch for MADE + the affine map of MaskedAffineAutoregressiveTransform (include/nfk.h: nfk_affine_ar_step_f16x3).
    plan: dense.StepPlan of the trunk; a: Pair16 of the conditioner input; wf: Pair16 of the final layer [2 d_t, hidden] in MADE's
    row order, bias [2 d_t]; features cols = (first column, count) of x are written to the same columns of y (fp32);
    lad_accum += +-sum log scale.  terms: per-row trunk terms as for rq_coupling_step, or None."""
    n = a.shape[0]
    d = _trunk_descriptor(plan, a, flags)
    d.inverse = int(inverse)
    d.t_col0, d.d_t = int(cols[0]), int(cols[1])
    d.wp_hi, d.wp_lo, d.ldwp, d.wp_exp = wf.hi.data_ptr(), wf.lo.data_ptr(), wf.hi.stride(0), wf.exp
    d.bias_packed = bias.data_ptr()
    d.x, d.ldx = x.data_ptr(), x.stride(0)
    d.y, d.ldy = y.data_ptr(), y.stride(0)
    d.lad_accum = N.ptr(lad_accum)
    rt = None if terms is None else _row_terms(terms, plan, a)
    with timed("affine_ar_step", n):
        N.check(N.lib().nfk_affine_ar_step_f16x3(ctypes.byref(d), None if rt is None else ctypes.byref(rt), N.stream()))
    return y


# ---- the mixture-of-Gaussians MADE step in one kernel ------------------------------------------------------------------
def mog_made_padded_rows(num_components):
    """Packed rows per feature of the mixture step's final layer, 0 when num_components has no instance."""
    return int(N.load().nfk_mog_made_padded_rows(int(num_components)))


def mog_made_step(plan, a, wf, bias, num_components, epsilon, cols, x=None, lad_accum=None, y=None, noise=None, flags=None,
                  terms=None):
    """ONE launch for MADE + the mixture epilogue of MixtureOfGaussiansMADE (include/nfk.h: nfk_mog_made_step_f16x3).
    plan: dense.StepPlan of the trunk; a: Pair16 of the conditioner input; wf, bias: dense.mog_operands (packed to
    mog_made_padded_rows rows per feature); cols = (first column, count) of the features.
    log_prob (noise None): lad_accum += the features' mixture log-density at x.  sample: noise = (u, e), fp32 [n, >= count]
    with unit column stride, feature j of cols in column j; y[:, cols] = the draws.  terms: per-row trunk terms or None."""
    n = a.shape[0]
    d = _trunk_descriptor(plan, a, flags)
    d.t_col0, d.d_t = int(cols[0]), int(cols[1])
    d.wp_hi, d.wp_lo, d.ldwp, d.wp_exp = wf.hi.data_ptr(), wf.lo.data_ptr(), wf.hi.stride(0), wf.exp
    d.bias_packed = bias.data_ptr()
    g = N.NfkMogArgs(int(num_components), N.MOG_LOG_PROB if noise is None else N.MOG_SAMPLE, float(epsilon))
    if noise is None:
        d.x, d.ldx = x.data_ptr(), x.stride(0)
        d.lad_accum = N.ptr(lad_accum)
    else:
        u, e = noise
        if u.stride() != e.stride() or u.stride(1) != 1:
            raise ValueError("u and e must share one row pitch and have unit column stride")
        d.y, d.ldy = y.data_ptr(), y.stride(0)
        g.u, g.e, g.ld_noise = u.data_ptr(), e.data_ptr(), u.stride(0)
    rt = None if terms is None else _row_terms(terms, plan, a)
    with timed("mog_made_step", n):
        N.check(N.lib().nfk_mog_made_step_f16x3(ctypes.byref(d), None if rt is None else ctypes.byref(rt), ctypes.byref(g),
                                                N.stream()))
    return y if noise is not None else lad_accum
