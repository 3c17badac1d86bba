"""Training path of the rational-quadratic spline on the kernels (config.native_training).

Under autograd the spline of an RQ coupling or of a masked autoregressive RQ transform is the one place where the torch
formulation is expensive: hundreds of small ops whose intermediates (knots, bin sizes, gathered parameters) autograd keeps for
the backward.  `RQSplineRows` runs the forward on `nfk_rqs_rows` and the backward on `nfk_rqs_rows_backward`, which rebuilds the
knots from the saved input and parameters instead -- only those two tensors are kept.  The conditioner that produces the
parameters stays torch (its GEMMs are cuBLAS under autograd either way).

`RQSplinePlanes` does the same for image couplings on the conditioner's [B, C_t * M, H, W] output as it is (`nfk_rqs_planes` /
`nfk_rqs_planes_backward`), and `RQSplineShared` for PiecewiseRationalQuadraticCDF, whose parameters every row shares: its forward
is the inference kernel `nfk_rqs_elementwise`, its backward `nfk_rqs_shared_backward` sums the parameter gradients over the batch
in a fixed order."""
import torch
from torch.autograd.function import once_differentiable

from ... import _native as N
from ... import config
from ... import kernels as K


class RQSplineRows(torch.autograd.Function):
    """(outputs [B, d_t], summed log|det| [B]) of the spline of desc on every column of `inputs` [B, d_t] with parameters
    [B, d_t * M] (column j * M + k = parameter k of feature j, widths and heights before the softmax divisor of desc)."""

    @staticmethod
    def forward(ctx, inputs, params, desc, inverse):
        ctx.set_materialize_grads(False)
        with K.on_device_of(inputs):
            flags = K.new_flags(inputs.device)
            lad = K.zeros_lad(inputs)
            with K.timed("rqs_rows", inputs.shape[0]):
                outputs = K.rqs_rows(desc, inverse, inputs, params, None, None, lad, flags)
            if config.check_domain:
                K.raise_for_flags(flags)
        ctx.save_for_backward(inputs, params)
        ctx.desc, ctx.inverse = desc, inverse
        return outputs, lad

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_outputs, grad_lad):
        inputs, params = ctx.saved_tensors
        want_x, want_params = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if grad_outputs is None and grad_lad is None:
            return None, None, None, None
        if grad_outputs is not None and grad_outputs.stride(-1) != 1:
            grad_outputs = grad_outputs.contiguous()
        with K.on_device_of(inputs):
            grad_x, grad_params = K.rqs_rows_backward(ctx.desc, ctx.inverse, inputs, params, grad_outputs, grad_lad,
                                                      want_grad_x=want_x)
        return grad_x, (grad_params if want_params else None), None, None


class RQSplinePlanes(torch.autograd.Function):
    """(outputs [B, C_t, H, W], summed log|det| [B]) of the spline of desc on every element of `inputs` with parameters
    [B, C_t * M, H, W] (channel j * M + k = parameter k of channel j, widths and heights before the softmax divisor of desc)."""

    @staticmethod
    def forward(ctx, inputs, params, desc, inverse):
        ctx.set_materialize_grads(False)
        with K.on_device_of(inputs):
            flags = K.new_flags(inputs.device)
            lad = K.zeros_lad(inputs)
            outputs = K.rqs_planes(desc, inverse, inputs, params, lad, flags)
            if config.check_domain:
                K.raise_for_flags(flags)
        ctx.save_for_backward(inputs, params)
        ctx.desc, ctx.inverse = desc, inverse
        return outputs, lad

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_outputs, grad_lad):
        inputs, params = ctx.saved_tensors
        want_x, want_params = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if grad_outputs is None and grad_lad is None:
            return None, None, None, None
        with K.on_device_of(inputs):
            grad_x, grad_params = K.rqs_planes_backward(ctx.desc, ctx.inverse, inputs, params, grad_outputs, grad_lad,
                                                        want_grad_x=want_x)
        return grad_x, (grad_params if want_params else None), None, None


class RQSplineShared(torch.autograd.Function):
    """(outputs [B, F], summed log|det| [B]) of the spline of desc on `inputs` [B, F] with the parameters uw, uh [F, K] and
    ud [F, K - 1 | K + 1] that every row shares (PiecewiseRationalQuadraticCDF)."""

    @staticmethod
    def forward(ctx, inputs, uw, uh, ud, desc, inverse):
        ctx.set_materialize_grads(False)
        with K.on_device_of(inputs):
            flags = K.new_flags(inputs.device)
            with K.timed("rqs_elementwise", inputs.shape[0]):
                outputs, lad_el = K.rqs_elementwise(desc, inverse, inputs, uw, uh, ud, param_period=inputs.shape[1], flags=flags)
            lad = K.zeros_lad(inputs)
            if inputs.numel():
                K.segment_sum_(lad_el, lad, inputs.shape[1])
            if config.check_domain:
                K.raise_for_flags(flags)
        ctx.save_for_backward(inputs, uw, uh, ud)
        ctx.desc, ctx.inverse = desc, inverse
        return outputs, lad

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_outputs, grad_lad):
        inputs, uw, uh, ud = ctx.saved_tensors
        want = ctx.needs_input_grad
        if grad_outputs is None and grad_lad is None:
            return None, None, None, None, None, None
        with K.on_device_of(inputs):
            grad_x, guw, guh, gud = K.rqs_shared_backward(ctx.desc, ctx.inverse, inputs, uw, uh, ud, grad_outputs, grad_lad,
                                                          want_grad_x=want[0])
        return (grad_x, guw if want[1] else None, guh if want[2] else None, gud if want[3] else None, None, None)


def _device_ok(t):
    return t.is_cuda and t.dtype == torch.float32 and t.dim() == 2


def _cuda_fp32(t):
    return t.is_cuda and t.dtype == torch.float32


def routed(inputs, params, num_bins, tails):
    """True when a spline call should run on RQSplineRows: config.native_training on, a gradient to compute, CUDA fp32 2-D
    tensors on one device with params [B, d_t * M], a bin count the kernels are instantiated for and linear or no tails."""
    if not (config.native_training and torch.is_grad_enabled() and (inputs.requires_grad or params.requires_grad)):
        return False
    if tails not in (None, "linear") or not 1 <= num_bins <= N.MAX_BINS:
        return False
    if not (_device_ok(inputs) and _device_ok(params)):
        return False
    m = N.spline_param_count(num_bins, tails == "linear")
    return (inputs.device == params.device and inputs.shape[1] >= 1 and params.shape[0] == inputs.shape[0]
            and params.shape[1] == inputs.shape[1] * m)


def _wants_grad(*tensors):
    return config.native_training and torch.is_grad_enabled() and any(t.requires_grad for t in tensors)


def routed_planes(inputs, params, num_bins, tails):
    """True when the spline of an image coupling should run on RQSplinePlanes: config.native_training on, a gradient to compute,
    CUDA fp32 4-D tensors on one device with inputs [B, C_t, H, W] and params [B, C_t * M, H, W], a bin count the kernels are
    instantiated for and linear or no tails."""
    if not _wants_grad(inputs, params):
        return False
    if tails not in (None, "linear") or not 1 <= num_bins <= N.MAX_BINS:
        return False
    if not (_cuda_fp32(inputs) and _cuda_fp32(params) and inputs.dim() == 4 and params.dim() == 4):
        return False
    m = N.spline_param_count(num_bins, tails == "linear")
    b, c, h, w = inputs.shape
    return inputs.device == params.device and c >= 1 and tuple(params.shape) == (b, c * m, h, w)


def routed_shared(inputs, widths, heights, derivatives, tails):
    """True when a PiecewiseRationalQuadraticCDF call should run on RQSplineShared: config.native_training on, a gradient to
    compute, CUDA fp32 tensors on one device, inputs [B, *shape] with parameters [*shape, K], K <= NFK_MAX_BINS and linear or no
    tails."""
    if not _wants_grad(inputs, widths, heights, derivatives):
        return False
    if tails not in (None, "linear") or not 1 <= widths.shape[-1] <= N.MAX_BINS:
        return False
    if not all(_cuda_fp32(t) and t.device == inputs.device for t in (inputs, widths, heights, derivatives)):
        return False
    return inputs.dim() >= 2 and tuple(inputs.shape[1:]) == tuple(widths.shape[:-1])


def rq_spline_planes(inputs, params, inverse, num_bins, tails, tail_bound, min_bin_width, min_bin_height, min_derivative,
                     divisor):
    """Spline of an image coupling on the kernels with autograd: (outputs [B, C_t, H, W], log|det| summed per sample [B])."""
    desc = N.spline_desc(num_bins, tails, tail_bound, 0.0, 1.0, 0.0, 1.0, min_bin_width, min_bin_height, min_derivative, False,
                         1.0 if divisor is None else divisor)
    return RQSplinePlanes.apply(inputs.contiguous(), params.contiguous(), desc, bool(inverse))


def rq_spline_shared(inputs, widths, heights, derivatives, inverse, tails, tail_bound, min_bin_width, min_bin_height,
                     min_derivative):
    """PiecewiseRationalQuadraticCDF on the kernels with autograd: (outputs like inputs, log|det| summed per row [B]).  The
    bounds are [-tail_bound, tail_bound] for linear tails, [0, 1] without tails."""
    k = widths.shape[-1]
    desc = N.spline_desc(k, tails, tail_bound, 0.0, 1.0, 0.0, 1.0, min_bin_width, min_bin_height, min_derivative)
    b = inputs.shape[0]
    f = widths[..., 0].numel()
    flat = lambda p: p.reshape(f, p.shape[-1])
    outputs, lad = RQSplineShared.apply(inputs.reshape(b, f).contiguous(), flat(widths), flat(heights), flat(derivatives), desc,
                                        bool(inverse))
    return outputs.reshape(inputs.shape), lad


def rq_spline_rows(inputs, params, inverse, num_bins, tails, tail_bound, min_bin_width, min_bin_height, min_derivative,
                   divisor):
    """Spline of a coupling / autoregressive layer on the kernels with autograd: (outputs [B, d_t], log|det| summed per row [B]).
    The bounds are [-tail_bound, tail_bound] for linear tails, [0, 1] without tails, as the layers use them."""
    desc = N.spline_desc(num_bins, tails, tail_bound, 0.0, 1.0, 0.0, 1.0, min_bin_width, min_bin_height, min_derivative, False,
                         1.0 if divisor is None else divisor)
    x = inputs if inputs.stride(-1) == 1 else inputs.contiguous()
    return RQSplineRows.apply(x, params.contiguous(), desc, bool(inverse))
