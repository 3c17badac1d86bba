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

    # ---- native: what the spline and the affine transform share ---------------------------------------------------------
    def _native_context_ok(self, inputs, context):
        """A context runs natively on the step route only: its projections enter the step kernel's trunk layers as row terms.
        A context of another batch size or width stays on the torch path, which broadcasts or raises as the reference does."""
        return (torch.is_tensor(context) and K.native_ok(context) and context.dim() == 2 and context.device == inputs.device
                and context.shape[0] == inputs.shape[0])

    def _pack_final(self, weight, bias):
        """(Pair16, bias, rows per feature) of the final layer as the step kernel's epilogue reads it."""
        raise NotImplementedError()

    def _sorted_subnets(self, chain):
        """Degree-sorted copies of the MADE weights for the inverse (sorted_subnets).  Hidden units the chain pads take degree D,
        so they sort last and no feature's prefix needs them."""
        net = self.autoregressive_net
        hp = chain[0][0].shape[0]
        pad = lambda dg: torch.cat([dg, dg.new_full((hp - dg.numel(),), self.features)]) if hp != dg.numel() else dg
        return sorted_subnets(self, chain, [pad(net.initial_layer.degrees)] + [pad(block.degrees) for block in net.blocks],
                              self.features, self._pack_final)


def sorted_subnets(owner, chain, degrees, features, pack_final):
    """Degree-sorted copies of a MADE chain's weights for the D sequential passes (the autoregressive inverse, the sampler of
    MixtureOfGaussiansMADE).  Feature i (degree i + 1) only sees hidden units of degree <= i; with the hidden units sorted by
    degree (one permutation for every hidden layer: the residual blocks keep degrees per index) those are a PREFIX, so pass i
    runs the sub-network of the first H_i units (rounded up to 32) and the final layer of feature i alone -- the total work of
    the D passes is ~1/8 of D full passes.  degrees: the hidden degrees of the initial layer, then of every block (None unless
    they all agree); pack_final(weight, bias) -> (Pair16, bias, rows per feature).  Cached on `owner` per parameter version."""
    def build():
        deg = degrees[0].to(chain[0][0].device)
        for block_degrees in degrees[1:]:
            if not torch.equal(block_degrees.to(deg.device), deg):
                return None
        perm = torch.argsort(deg, stable=True)
        sorted_deg = deg[perm].cpu()
        hidden = deg.numel()
        body = []
        for li, (w, b, relu_in, relu_out, res) in enumerate(chain[:-1]):
            w = w.detach()
            w = w[perm] if li == 0 else w[perm][:, perm]
            body.append((w.contiguous(), b.detach()[perm].contiguous(), relu_in, relu_out, res))
        wf = chain[-1][0].detach()[:, perm].contiguous()
        wp_pair, bias_packed, mp = pack_final(wf, chain[-1][1].detach())
        flags_l = D.plan_step_kernel(body + [chain[-1]])
        plans, widths = {}, []
        for i in range(features):
            count = int((sorted_deg <= i).sum())
            h = min(hidden, max(32, (count + 31) // 32 * 32))
            widths.append(h)
            if h not in plans:
                sub = [((w[:h] if li == 0 else w[:h, :h]).contiguous(), b[:h].contiguous(), ri, ro, rs)
                       for li, (w, b, ri, ro, rs) in enumerate(body)]
                plans[h] = D.StepPlan(sub).set_flags(flags_l)
        return plans, widths, wp_pair, bias_packed, mp
    return D.derived(owner, "_subnets", [t for layer in chain for t in layer[:2]], build, extra=(D.act_exp(),))


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
    def _in_pad(self):
        return (self.features + 7) // 8 * 8

    def _hidden_pad(self):
        return (self.autoregressive_net.initial_layer.out_features + 31) // 32 * 32

    def _native_chain(self, context):
        """MADE's dense chain with the initial layer's columns zero padded to a multiple of 8 (TMA rows are multiples of 16 bytes;
        the input pair is padded the same way) and the hidden units to a multiple of 32 (rows of the trunk weights and biases,
        columns of the square and final weights: sbi's H = 50 runs as 64), cached per parameter version.  Exact: every
        activation the kernels run maps 0 to 0, so a zero hidden unit stays zero."""
        from .. import config
        chain = self.autoregressive_net.dense_chain(context)
        d, dp, hp = self.features, self._in_pad(), self._hidden_pad()
        if chain is None or (dp == d and hp == chain[0][0].shape[0]):
            return chain
        if hp != chain[0][0].shape[0] and not config.native_activations:
            return None
        if hp == chain[0][0].shape[0]:                   # the initial layer's columns only
            w = chain[0][0]

            def padded_w0():
                out = w.new_zeros(w.shape[0], dp)
                out[:, :d] = w
                return out
            return [(D.derived(self, "_w0_padded", [w], padded_w0),) + tuple(chain[0][1:])] + list(chain[1:])

        def padded():
            out = []
            for li, (w, b, act_in, act_out, res) in enumerate(chain):
                last = li == len(chain) - 1
                wp = w.new_zeros(w.shape[0] if last else hp, dp if li == 0 else hp)
                wp[:w.shape[0], :w.shape[1]] = w.detach()
                bp = b.detach().new_zeros(w.shape[0] if last else hp)
                bp[:b.numel()] = b.detach()
                out.append((wp, bp, act_in, act_out, res))
            return out
        return D.derived(self, "_padded_chain", [t for layer in chain for t in layer[:2]], padded)

    def _degrees_kept(self):
        """The residual blocks keep the initial layer's hidden degrees (so the inverse's sub-networks are prefixes)."""
        net = self.autoregressive_net
        degrees = [net.initial_layer.degrees] + [block.degrees for block in net.blocks]
        return D.derived(self, "_degrees_match", degrees, lambda: all(torch.equal(d.cpu(), degrees[0].cpu()) for d in degrees[1:]))

    def _native_ready(self, inputs, context):
        if not (K.native_ok(inputs, context) and inputs.dim() == 2 and params_frozen(self)):
            return False
        net = self.autoregressive_net
        if context is not None and not (self._native_context_ok(inputs, context) and net._has_context_layers()
                                        and context.shape[1] == net.context_layer.in_features):
            return False
        chain = self._native_chain(context)
        return chain is not None and self._degrees_kept() and D.AffineARHead(chain, self._in_pad()).route == "step"

    def _pack_final(self, weight, bias):
        return D.ar_affine_operands(weight, bias)

    def _input_pair(self, x, flags):
        """Pair16 of x, zero padded to _in_pad() columns."""
        n, d = x.shape
        if self._in_pad() == d:
            return K.split_f16(x, D.act_exp(), flags=flags)
        pair = K.Pair16.zeros(n, self._in_pad(), D.act_exp(), x.device)
        K.split_f16(x, D.act_exp(), out=pair.cols(0, d), flags=flags)
        return pair

    def _native_apply(self, inputs, lad, flags, inverse, context=None):
        """Forward: one launch per row block (the whole batch without a context).  Inverse: per row block, D launches on the
        degree-sorted sub-networks, pass i writing feature i and splitting it into the input pair of pass i + 1.  A context is
        projected once per row block of config.coupling_block_rows (made.ContextProjection) and every launch of the block reads
        the projections as per-row trunk terms."""
        from .. import config
        if inputs.shape[1] != self.features:
            raise ValueError("Expected features = {}, got {}.".format(self.features, inputs.shape[1]))
        net = self.autoregressive_net
        chain = self._native_chain(context)
        head = D.AffineARHead(chain, self._in_pad())
        n, d = inputs.shape
        outputs = torch.empty_like(inputs, memory_format=torch.contiguous_format)
        sub = self._sorted_subnets(chain) if inverse else None
        proj = net.context_projection(sort=inverse, width=self._hidden_pad()) if context is not None else None
        ctx = None if context is None else (context if context.stride(1) == 1 else context.contiguous())
        block = n if context is None else max(128, int(config.coupling_block_rows))
        for r0 in range(0, n, max(1, block)):
            r1 = min(n, r0 + block)
            xs, ys, ls = inputs[r0:r1], outputs[r0:r1], lad[r0:r1]
            terms = None if proj is None else proj.terms(ctx[r0:r1], flags)
            if not inverse:
                wf, bias, _ = D.ar_affine_operands(chain[-1][0], chain[-1][1])
                head.step(D.step_plan(chain), self._input_pair(xs, flags), wf, bias, xs, (0, d), ys, ls, flags, False, terms=terms)
                continue
            plans, widths, wf, bias, mp = sub
            pair = K.Pair16.zeros(r1 - r0, self._in_pad(), D.act_exp(), inputs.device)
            for i in range(d):
                h = widths[i]
                wf_i = K.Pair16(wf.hi[i * mp:(i + 1) * mp, :h], wf.lo[i * mp:(i + 1) * mp, :h], wf.exp)
                head.step(plans[h], pair, wf_i, bias[i * mp:(i + 1) * mp], xs, (i, 1), ys, ls, flags, True, terms=terms)
                if i + 1 < d:
                    K.split_f16(ys[:, i:i + 1], pair.exp, out=pair.cols(i, i + 1), flags=flags)
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
        if not (K.native_ok(inputs, context) and inputs.dim() == 2 and params_frozen(self) and self.num_bins <= 64):
            return False
        net = self.autoregressive_net
        if context is None:
            return net.dense_chain(None) is not None
        if not self._native_context_ok(inputs, context):
            return False
        chain = net.dense_chain(context)
        return (chain is not None and context.shape[1] == net.context_layer.in_features
                and self._native_head(chain).route == "step")

    def _native_head(self, chain):
        return D.spline_head(chain, self, self._softmax_divisor(), self.features, self.features)

    def _pack_final(self, weight, bias):
        return D.spline_operands(weight, bias, self.num_bins, self.tails, self.features)

    def _native_inverse_step(self, head, chain, inputs, lad, flags, terms=None, outputs=None):
        """The D per-feature launches on the degree-sorted sub-networks (None when the blocks do not keep the degrees).  terms:
        the row terms of the trunk layers with their columns in the sorted order (context); outputs: where to write."""
        sub = self._sorted_subnets(chain)
        if sub is None:
            return None
        plans, widths, wp_pair, bias_packed, mp = sub
        n, d = inputs.shape
        if outputs is None:
            outputs = torch.zeros_like(inputs, memory_format=torch.contiguous_format)
        pair = K.Pair16(torch.zeros(n, d, dtype=torch.float16, device=inputs.device),
                        torch.zeros(n, d, dtype=torch.float16, device=inputs.device), D.act_exp())
        for i in range(d):
            h = widths[i]
            wp_i = K.Pair16(wp_pair.hi[i * mp:(i + 1) * mp, :h], wp_pair.lo[i * mp:(i + 1) * mp, :h], wp_pair.exp)
            head.step(plans[h], pair, wp_i, bias_packed[i * mp:(i + 1) * mp], inputs, (i, 1), outputs, lad, flags, True,
                      terms=terms)
            if i + 1 < d:
                K.split_f16(outputs[:, i:i + 1], pair.exp, out=pair.cols(i, i + 1), flags=flags)
        return outputs

    def _native_apply(self, inputs, lad, flags, inverse, context=None):
        if inputs.shape[1] != self.features:
            raise ValueError("Expected features = {}, got {}.".format(self.features, inputs.shape[1]))
        if context is not None:
            return self._native_conditional(inputs, context, lad, flags, inverse)
        chain = self.autoregressive_net.dense_chain(None)
        head = self._native_head(chain)
        d = self.features
        if not inverse:
            outputs = torch.empty_like(inputs, memory_format=torch.contiguous_format)
            head.run(chain, (inputs, None), inputs, (0, d), outputs, lad, flags, False)
            return outputs
        if head.route == "step":
            outputs = self._native_inverse_step(head, chain, inputs, lad, flags)
            if outputs is not None:
                return outputs
        # D passes, each conditioned on the outputs of the one before: after pass i, features 0..i are exact
        outputs = K.fill_(torch.empty_like(inputs, memory_format=torch.contiguous_format), 0.0)
        for i in range(d):
            nxt = torch.empty_like(inputs, memory_format=torch.contiguous_format)
            head.run(chain, (outputs, None), inputs, (0, d), nxt, lad if i == d - 1 else None, flags, True)
            outputs = nxt
        return outputs

    def _native_conditional(self, inputs, context, lad, flags, inverse):
        """The context-conditioned transform on the step route.  The context projections (made.ContextProjection) are computed
        once per row block of config.coupling_block_rows -- (1 + num_blocks) * rows * hidden * 4 bytes of terms -- and every
        launch of the block reads them: the forward launch, or all D passes of the inverse (sorted sub-networks: the terms in
        the sorted hidden order, pass i reading their first h_i columns; else D full passes reading them at full width)."""
        from .. import config
        net = self.autoregressive_net
        chain = net.dense_chain(context)
        head = self._native_head(chain)
        n, d = inputs.shape
        sub = self._sorted_subnets(chain) if inverse else None
        proj = net.context_projection(sort=sub is not None)
        ctx = context if context.stride(1) == 1 else context.contiguous()
        outputs = torch.empty_like(inputs, memory_format=torch.contiguous_format)
        block = max(128, int(config.coupling_block_rows))
        for r0 in range(0, n, block):
            r1 = min(n, r0 + block)
            xs, ys, ls = inputs[r0:r1], outputs[r0:r1], lad[r0:r1]
            terms = proj.terms(ctx[r0:r1], flags)
            if not inverse:
                head.run(chain, (xs, None), xs, (0, d), ys, ls, flags, False, terms=terms)
            elif sub is not None:
                self._native_inverse_step(head, chain, xs, ls, flags, terms=terms, outputs=ys)
            else:
                cur = K.fill_(torch.empty_like(xs, memory_format=torch.contiguous_format), 0.0)
                for i in range(d):
                    nxt = ys if i == d - 1 else torch.empty_like(xs, memory_format=torch.contiguous_format)
                    head.run(chain, (cur, None), xs, (0, d), nxt, ls if i == d - 1 else None, flags, True, terms=terms)
                    cur = nxt
        return outputs
