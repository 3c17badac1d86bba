"""Unconditional elementwise spline transform (reference nflows/transforms/nonlinearities.py:386-467); the other
elementwise nonlinearities of that file are out of the hot-path scope (SURVEY.md section 2, row 11)."""
import numpy as np
import torch
from torch import nn

from .. import _native as N
from .. import config
from .. import kernels as K
from . import splines
from .base import Transform, params_frozen


class PiecewiseRationalQuadraticCDF(Transform):
    """Rational-quadratic spline with its own (batch-independent) parameters per input element of shape `shape`.
    This is what `apply_unconditional_transform=True` puts on the identity half of a spline coupling."""

    def __init__(self, shape, num_bins=10, tails=None, tail_bound=1.0, identity_init=False,
                 min_bin_width=splines.rational_quadratic.DEFAULT_MIN_BIN_WIDTH,
                 min_bin_height=splines.rational_quadratic.DEFAULT_MIN_BIN_HEIGHT,
                 min_derivative=splines.rational_quadratic.DEFAULT_MIN_DERIVATIVE):
        super().__init__()
        self.min_bin_width = min_bin_width
        self.min_bin_height = min_bin_height
        self.min_derivative = min_derivative
        self.tail_bound = tail_bound
        self.tails = tails
        if isinstance(shape, int):
            shape = (shape,)
        num_derivatives = (num_bins - 1) if tails == "linear" else (num_bins + 1)
        if identity_init:
            self.unnormalized_widths = nn.Parameter(torch.zeros(*shape, num_bins))
            self.unnormalized_heights = nn.Parameter(torch.zeros(*shape, num_bins))
            edge = np.log(np.exp(1 - min_derivative) - 1)
            self.unnormalized_derivatives = nn.Parameter(edge * torch.ones(*shape, num_derivatives))
        else:
            self.unnormalized_widths = nn.Parameter(torch.rand(*shape, num_bins))
            self.unnormalized_heights = nn.Parameter(torch.rand(*shape, num_bins))
            self.unnormalized_derivatives = nn.Parameter(torch.rand(*shape, num_derivatives))

    def _native_ready(self, inputs, context):
        return (K.native_ok(inputs, context) and params_frozen(self) and self.tails in (None, "linear")
                and inputs.shape[1:] == self.unnormalized_widths.shape[:-1] and self.unnormalized_widths.shape[-1] <= N.MAX_BINS)

    def _native_apply(self, inputs, lad, flags, inverse, context=None):
        k = self.unnormalized_widths.shape[-1]
        desc = N.spline_desc(k, self.tails, self.tail_bound, 0.0, 1.0, 0.0, 1.0, self.min_bin_width, self.min_bin_height,
                             self.min_derivative)
        period = int(np.prod(inputs.shape[1:]))
        flat = lambda p: p.detach().reshape(period, p.shape[-1])
        y, l = K.rqs_elementwise(desc, inverse, inputs, flat(self.unnormalized_widths), flat(self.unnormalized_heights),
                                 flat(self.unnormalized_derivatives), param_period=period, flags=flags)
        lad += l.reshape(inputs.shape[0], -1).sum(dim=1)
        return y

    def _run(self, inputs, context, inverse):
        # same dispatch as Transform._run, but inputs may have any number of event dimensions
        if torch.is_tensor(inputs) and self._native_ready(inputs, context):
            with K.on_device_of(inputs):
                x = inputs.contiguous()
                lad = K.zeros_lad(x)
                flags = K.new_flags(x.device)
                out = self._native_apply(x, lad, flags, inverse, context)
                if config.check_domain:
                    K.raise_for_flags(flags)
            return out, lad
        return self._eager(inputs, context, inverse)

    def _eager(self, inputs, context, inverse):
        batch = inputs.shape[0]
        share = lambda p: p[None, ...].expand(batch, *p.shape)
        kwargs = dict(inputs=inputs, unnormalized_widths=share(self.unnormalized_widths),
                      unnormalized_heights=share(self.unnormalized_heights),
                      unnormalized_derivatives=share(self.unnormalized_derivatives), inverse=inverse,
                      min_bin_width=self.min_bin_width, min_bin_height=self.min_bin_height,
                      min_derivative=self.min_derivative)
        if self.tails is None:
            outputs, logabsdet = splines.rational_quadratic_spline(**kwargs)
        else:
            outputs, logabsdet = splines.unconstrained_rational_quadratic_spline(tails=self.tails, tail_bound=self.tail_bound,
                                                                               **kwargs)
        return outputs, logabsdet.reshape(batch, -1).sum(dim=1)
