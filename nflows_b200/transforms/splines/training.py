"""Training path of the rational-quadratic spline on the kernels (config.native_training).

Under autograd the spline of an RQ coupling or of a masked autoregressive RQ transform is the one place where the torch
formulation is expensive: hundreds of small ops whose intermediates (knots, bin sizes, gathered parameters) autograd keeps for
the backward.  `RQSplineRows` runs the forward on `nfk_rqs_rows` and the backward on `nfk_rqs_rows_backward`, which rebuilds the
knots from the saved input and parameters instead -- only those two tensors are kept.  The conditioner that produces the
parameters stays torch (its GEMMs are cuBLAS under autograd either way)."""
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


def _device_ok(t):
    return t.is_cuda and t.dtype == torch.float32 and t.dim() == 2


def routed(inputs, params, num_bins, tails):
    """True when a spline call should run on RQSplineRows: config.native_training on, a gradient to compute, CUDA fp32 2-D
    tensors on one device with params [B, d_t * M], a bin count the kernels are instantiated for and linear or no tails."""
    if not (config.native_training and torch.is_grad_enabled() and (inputs.requires_grad or params.requires_grad)):
        return False
    if tails not in (None, "linear") or not 1 <= num_bins <= N.MAX_BINS:
        return False
    if not (_device_ok(inputs) and _device_ok(params)):
        return False
    m = 3 * num_bins - 1 if tails == "linear" else 3 * num_bins + 1
    return (inputs.device == params.device and inputs.shape[1] >= 1 and params.shape[0] == inputs.shape[0]
            and params.shape[1] == inputs.shape[1] * m)


def rq_spline_rows(inputs, params, inverse, num_bins, tails, tail_bound, min_bin_width, min_bin_height, min_derivative,
                   divisor):
    """Spline of a coupling / autoregressive layer on the kernels with autograd: (outputs [B, d_t], log|det| summed per row [B]).
    The bounds are [-tail_bound, tail_bound] for linear tails, [0, 1] without tails, as the layers use them."""
    desc = N.spline_desc(num_bins, tails, tail_bound, 0.0, 1.0, 0.0, 1.0, min_bin_width, min_bin_height, min_derivative, False,
                         1.0 if divisor is None else divisor)
    x = inputs if inputs.stride(-1) == 1 else inputs.contiguous()
    return RQSplineRows.apply(x, params.contiguous(), desc, bool(inverse))
