"""Masked autoregressive transforms (reference nflows/transforms/autoregressive.py:24-62, 64-128, 404-495).

Forward is one MADE pass + an elementwise map: ONE launch of the coupling-step kernel (masked conditioner + spline or affine map).  The
inverse is inherently sequential: feature i of the output needs the conditioner evaluated on outputs 1..i-1, so -- like the
reference (:43-52) -- it runs D passes; here pass i is one launch of the same kernel on the degree-sorted SUB-network feature
i can see (hidden units of degree <= i are a prefix once sorted) with the final layer of feature i alone."""
import numpy as np
import torch
from torch.nn import functional as F

from .. import dense as D
from .. import kernels as K
from . import made as made_module
from . import splines
from .base import Transform, params_frozen


class AutoregressiveTransform(Transform):
    """outputs_i = f(inputs_i; params_i(inputs_<i)).  Subclasses define the elementwise map and its parameter count."""

    def __init__(self, autoregressive_net):
        super().__init__()
        self.autoregressive_net = autoregressive_net

    def _eager(self, inputs, context, inverse):
        if not inverse:
            return self._elementwise_forward(inputs, self.autoregressive_net(inputs, context))
        outputs = torch.zeros_like(inputs)
        logabsdet = None
        for _ in range(int(np.prod(inputs.shape[1:]))):
            outputs, logabsdet = self._elementwise_inverse(inputs, self.autoregressive_net(outputs, context))
        return outputs, logabsdet

    def _output_dim_multiplier(self):
        raise NotImplementedError()

    def _elementwise_forward(self, inputs, autoregressive_params):
        raise NotImplementedError()

    def _elementwise_inverse(self, inputs, autoregressive_params):
        raise NotImplementedError()


class MaskedAffineAutoregressiveTransform(AutoregressiveTransform):
    """MAF layer: y_i = scale_i * x_i + shift_i, scale_i = softplus(u_i) + 1e-3 with (u_i, shift_i) = MADE(x)[i, :] (reference
    :64-128).  On the native path the forward is one launch of the coupling-step kernel with its affine epilogue
    (nfk_affine_ar_step_f16x3), the inverse one launch per feature on the degree-sorted sub-networks."""

    def __init__(self, features, hidden_features, context_features=None, num_blocks=2, use_residual_blocks=True,
                 random_mask=False, activation=F.relu, dropout_probability=0.0, use_batch_norm=False):
        self.features = features
        net = made_module.MADE(features=features, hidden_features=hidden_features, context_features=context_features,
                               num_blocks=num_blocks, output_multiplier=self._output_dim_multiplier(),
                               use_residual_blocks=use_residual_blocks, random_mask=random_mask, activation=activation,
                               dropout_probability=dropout_probability, use_batch_norm=use_batch_norm)
        self._epsilon = 1e-3
        super().__init__(net)

    def _output_dim_multiplier(self):
        return 2

    def _scale_shift(self, params):
        params = params.view(-1, self.features, self._output_dim_multiplier())
        return F.softplus(params[..., 0]) + self._epsilon, params[..., 1]

    def _elementwise_forward(self, inputs, autoregressive_params):
        scale, shift = self._scale_shift(autoregressive_params)
        return scale * inputs + shift, torch.sum(torch.log(scale), dim=1)

    def _elementwise_inverse(self, inputs, autoregressive_params):
        scale, shift = self._scale_shift(autoregressive_params)
        return (inputs - shift) / scale, -torch.sum(torch.log(scale), dim=1)

    # ---- native ----------------------------------------------------------------------------------------------------
    def _native_ready(self, inputs, context):
        """The step route on MADE's padded chain.  A hidden width that is not a multiple of 32 (sbi's 50) is padded only with
        config.native_activations on; otherwise it keeps the torch path."""
        from .. import config
        net = self.autoregressive_net
        if not (K.native_ok(inputs, context) and inputs.dim() == 2 and params_frozen(self)
                and net.native_context_ok(inputs, context)
                and (net.initial_layer.out_features % 32 == 0 or config.native_activations)):
            return False
        chain = net.padded_chain(context)
        return chain is not None and net.degrees_kept() and D.made_step_ready(chain, net.in_pad())

    def _native_apply(self, inputs, lad, flags, inverse, context=None):
        """Forward: one launch per row block (the whole batch without a context).  Inverse: per row block, the D passes of
        made.MADE.sequential_passes on the degree-sorted sub-networks.  A context is projected once per row block of
        config.coupling_block_rows (made.ContextProjection) and every launch of the block reads the projections as per-row trunk
        terms."""
        if inputs.shape[1] != self.features:
            raise ValueError("Expected features = {}, got {}.".format(self.features, inputs.shape[1]))
        net = self.autoregressive_net
        chain = net.padded_chain(context)
        n, d = inputs.shape
        outputs = torch.empty_like(inputs, memory_format=torch.contiguous_format)
        sub = net.sorted_subnets(chain, D.ar_affine_operands) if inverse else None
        proj = net.context_projection(sort=inverse, width=net.hidden_pad()) if context is not None else None
        ctx = None if context is None else (context if context.stride(1) == 1 else context.contiguous())
        for r0, r1 in net.row_blocks(n, context):
            xs, ys, ls = inputs[r0:r1], outputs[r0:r1], lad[r0:r1]
            terms = None if proj is None else proj.terms(ctx[r0:r1], flags)
            if inverse:
                net.sequential_passes(sub, ys, flags, lambda plan, pair, wf, bias, i: K.affine_ar_step(
                    plan, pair, wf, bias, xs, (i, 1), ys, ls, flags, True, terms=terms))
            else:
                wf, bias, _ = D.ar_affine_operands(chain[-1][0], chain[-1][1])
                K.affine_ar_step(D.step_plan(chain), net.input_pair(xs, flags), wf, bias, xs, (0, d), ys, ls, flags, False,
                                 terms=terms)
        return outputs


class MaskedPiecewiseRationalQuadraticAutoregressiveTransform(AutoregressiveTransform):
    """Autoregressive neural spline layer: feature i goes through an RQ spline whose 3K-1 / 3K+1 parameters are rows
    i*M .. i*M+M-1 of the MADE output (feature-major, like the coupling layout)."""

    def __init__(self, features, hidden_features, context_features=None, num_bins=10, tails=None, tail_bound=1.0,
                 num_blocks=2, use_residual_blocks=True, random_mask=False, activation=F.relu, dropout_probability=0.0,
                 use_batch_norm=False, min_bin_width=splines.rational_quadratic.DEFAULT_MIN_BIN_WIDTH,
                 min_bin_height=splines.rational_quadratic.DEFAULT_MIN_BIN_HEIGHT,
                 min_derivative=splines.rational_quadratic.DEFAULT_MIN_DERIVATIVE):
        self.num_bins = num_bins
        self.min_bin_width = min_bin_width
        self.min_bin_height = min_bin_height
        self.min_derivative = min_derivative
        self.tails = tails
        self.tail_bound = tail_bound
        self.features = features
        net = made_module.MADE(features=features, hidden_features=hidden_features, context_features=context_features,
                               num_blocks=num_blocks, output_multiplier=self._output_dim_multiplier(),
                               use_residual_blocks=use_residual_blocks, random_mask=random_mask, activation=activation,
                               dropout_probability=dropout_probability, use_batch_norm=use_batch_norm)
        super().__init__(net)

    def _output_dim_multiplier(self):
        if self.tails == "linear":
            return self.num_bins * 3 - 1
        if self.tails is None:
            return self.num_bins * 3 + 1
        raise ValueError

    def _softmax_divisor(self):
        net = self.autoregressive_net
        return float(np.sqrt(net.hidden_features)) if hasattr(net, "hidden_features") else None

    def _elementwise(self, inputs, autoregressive_params, inverse=False):
        b, d = inputs.shape[0], inputs.shape[1]
        params = autoregressive_params.view(b, d, self._output_dim_multiplier())
        k = self.num_bins
        widths, heights, derivatives = params[..., :k], params[..., k:2 * k], params[..., 2 * k:]
        divisor = self._softmax_divisor()
        if divisor is not None:
            widths, heights = widths / divisor, heights / divisor
        common = dict(inputs=inputs, unnormalized_widths=widths, unnormalized_heights=heights,
                      unnormalized_derivatives=derivatives, inverse=inverse, min_bin_width=self.min_bin_width,
                      min_bin_height=self.min_bin_height, min_derivative=self.min_derivative)
        if self.tails is None:
            outputs, logabsdet = splines.rational_quadratic_spline(**common)
        elif self.tails == "linear":
            outputs, logabsdet = splines.unconstrained_rational_quadratic_spline(tails=self.tails, tail_bound=self.tail_bound,
                                                                               **common)
        else:
            raise ValueError
        return outputs, torch.sum(logabsdet.reshape(b, -1), dim=1)

    def _elementwise_forward(self, inputs, autoregressive_params):
        return self._elementwise(inputs, autoregressive_params)

    def _elementwise_inverse(self, inputs, autoregressive_params):
        return self._elementwise(inputs, autoregressive_params, inverse=True)

    # ---- native ----------------------------------------------------------------------------------------------------
    def _native_ready(self, inputs, context):
        net = self.autoregressive_net
        if not (K.native_ok(inputs, context) and inputs.dim() == 2 and params_frozen(self) and self.num_bins <= 64
                and net.native_context_ok(inputs, context)):
            return False
        chain = net.dense_chain(context)
        return chain is not None and (context is None or self._native_head(chain).route == "step")

    def _native_head(self, chain):
        return D.spline_head(chain, self, self._softmax_divisor(), self.features, self.features)

    def _pack_final(self, weight, bias):
        return D.spline_operands(weight, bias, self.num_bins, self.tails, self.features)

    def _native_apply(self, inputs, lad, flags, inverse, context=None):
        """Per row block (the whole batch without a context), the forward is one head.run and the inverse the D passes of
        made.MADE.sequential_passes on the degree-sorted sub-networks (step route), else D full passes.  A context (step route
        only) is projected once per row block of config.coupling_block_rows -- (1 + num_blocks) * rows * hidden * 4 bytes of
        terms -- and every launch of the block reads the projections: in the sorted hidden order for the sub-networks, pass i
        reading their first h_i columns, else at full width.  The chain is MADE's unpadded one: the step route needs features a
        multiple of 8 and a hidden width a multiple of 32 as they stand."""
        if inputs.shape[1] != self.features:
            raise ValueError("Expected features = {}, got {}.".format(self.features, inputs.shape[1]))
        net = self.autoregressive_net
        chain = net.dense_chain(context)
        head = self._native_head(chain)
        n, d = inputs.shape
        sub = net.sorted_subnets(chain, self._pack_final) if inverse and head.route == "step" and net.degrees_kept() else None
        proj = None if context is None else net.context_projection(sort=sub is not None)
        ctx = None if context is None else (context if context.stride(1) == 1 else context.contiguous())
        outputs = torch.empty_like(inputs, memory_format=torch.contiguous_format)
        for r0, r1 in net.row_blocks(n, context):
            xs, ys, ls = inputs[r0:r1], outputs[r0:r1], lad[r0:r1]
            terms = None if proj is None else proj.terms(ctx[r0:r1], flags)
            if not inverse:
                head.run(chain, (xs, None), xs, (0, d), ys, ls, flags, False, terms=terms)
            elif sub is not None:
                net.sequential_passes(sub, ys, flags, lambda plan, pair, wf, bias, i: head.step(
                    plan, pair, wf, bias, xs, (i, 1), ys, ls, flags, True, terms=terms))
            else:
                # D passes, each conditioned on the outputs of the one before: after pass i, features 0..i are exact
                cur = K.fill_(torch.empty_like(xs, memory_format=torch.contiguous_format), 0.0)
                for i in range(d):
                    nxt = ys if i == d - 1 else torch.empty_like(xs, memory_format=torch.contiguous_format)
                    head.run(chain, (cur, None), xs, (0, d), nxt, ls if i == d - 1 else None, flags, True, terms=terms)
                    cur = nxt
        return outputs
