"""Coupling transforms (reference nflows/transforms/coupling.py:20-142, 212-296, 502-582).

A coupling layer leaves the `identity` features unchanged, feeds them to a conditioner network and uses its
output as the parameters of an elementwise invertible map of the `transform` features.

Native execution (CUDA fp32, 2-D inputs, no autograd):
  gather identity columns -> conditioner as a chain of `nfk_linear` launches (or the user's torch module if it
  is not a recognised relu ResidualNet/MLP) -> ONE epilogue kernel (`nfk_rqs_rows` / `nfk_affine_coupling_rows`)
  that evaluates the elementwise map, scatters both halves into the output and adds the per-row log|det| into
  the running buffer.  The conditioner output is produced in row chunks small enough to stay resident in the
  L2 (50 MB on an H100), so the [B, d_t * M] parameter tensor the reference materialises never makes a full HBM round trip.
"""
import warnings

import numpy as np
import torch
from torch.nn.functional import softplus

from .. import _native as N
from .. import config
from .. import dense as D
from .. import kernels as K
from . import splines
from .base import Transform, params_frozen


class CouplingTransform(Transform):
    """Base class.  `mask[i] > 0` marks feature i as transformed, `<= 0` as identity (conditioner input)."""

    def __init__(self, mask, transform_net_create_fn, unconditional_transform=None):
        mask = torch.as_tensor(mask)
        if mask.dim() != 1:
            raise ValueError("Mask must be a 1-dim tensor.")
        if mask.numel() <= 0:
            raise ValueError("Mask can't be empty.")
        super().__init__()
        self.features = len(mask)
        index = torch.arange(self.features)
        self.register_buffer("identity_features", index.masked_select(mask <= 0))
        self.register_buffer("transform_features", index.masked_select(mask > 0))
        assert self.num_identity_features + self.num_transform_features == self.features
        self.transform_net = transform_net_create_fn(
            self.num_identity_features, self.num_transform_features * self._transform_dim_multiplier())
        if unconditional_transform is None:
            self.unconditional_transform = None
        else:
            self.unconditional_transform = unconditional_transform(features=self.num_identity_features)

    @property
    def num_identity_features(self):
        return len(self.identity_features)

    @property
    def num_transform_features(self):
        return len(self.transform_features)

    def _check_inputs(self, inputs):
        if inputs.dim() not in (2, 4):
            raise ValueError("Inputs must be a 2D or a 4D tensor.")
        if inputs.shape[1] != self.features:
            raise ValueError("Expected features = {}, got {}.".format(self.features, inputs.shape[1]))

    # ---- torch path (device-agnostic, differentiable) -----------------------------------------------------
    def _eager(self, inputs, context, inverse):
        self._check_inputs(inputs)
        identity = inputs[:, self.identity_features, ...]
        moved = inputs[:, self.transform_features, ...]
        if inverse:
            logabsdet = 0.0
            if self.unconditional_transform is not None:
                identity, logabsdet = self.unconditional_transform.inverse(identity, context)
            params = self._conditioner(identity, context)
            moved, lad = self._coupling_transform_inverse(inputs=moved, transform_params=params)
            logabsdet = logabsdet + lad
        else:
            params = self._conditioner(identity, context)
            moved, logabsdet = self._coupling_transform_forward(inputs=moved, transform_params=params)
            if self.unconditional_transform is not None:
                identity, lad = self.unconditional_transform(identity, context)
                logabsdet = logabsdet + lad
        outputs = torch.empty_like(inputs)
        outputs[:, self.identity_features, ...] = identity
        outputs[:, self.transform_features, ...] = moved
        return outputs, logabsdet

    def _conditioner(self, identity, context):
        """transform_net(identity, context); under autograd with config.native_training on, a dense ResidualNet / MLP runs its
        forward and backward on the tensor-core dense layers (splines.training.routed_conditioner)."""
        net = self.transform_net
        if splines.training.routed_conditioner(net, identity, context):
            return D.train_chain(net.dense_chain(None), identity)
        return net(identity, context)

    # ---- native path --------------------------------------------------------------------------------------
    def _native_ready(self, inputs, context):
        return K.native_ok(inputs, context) and inputs.dim() == 2 and params_frozen(self) and self._native_epilogue_supported()

    def _native_epilogue_supported(self):
        return False

    def _cols(self, device):
        idf, tf = self.identity_features, self.transform_features
        return D.derived(self, "_col_index", [idf, tf], lambda: (K.index_tensor(idf, device), K.index_tensor(tf, device)),
                         extra=(device,))

    def _native_layout(self, inputs, context):
        """Column order this coupling wants its input in -- identity features first, transformed features last -- when it
        runs on the fused tensor-core path (CompositeTransform._native_apply arranges it), else None."""
        if self.unconditional_transform is not None or not self._native_ready(inputs, context):
            return None
        net = self.transform_net
        chain = net.dense_chain(context) if hasattr(net, "dense_chain") else None
        if chain is None or self._native_head(chain).route == "rows":
            return None
        if (self.num_identity_features % 8) or (self.features % 8):
            return None                                   # the strided fp16 identity view must be TMA-addressable
        from .fused_affine import Layout
        idf, tf = self.identity_features, self.transform_features
        return D.derived(self, "_layout", [idf, tf], lambda: Layout(torch.cat([idf, tf]).cpu().numpy()))

    def _native_packed(self, x, lad, flags, inverse, context, owned, carry=None):
        """Fused path on a tensor already in the [identity | transformed] column order: the conditioner reads the fp16 pair of
        the identity block (written by the affine run in front, else split here), the fused kernel overwrites the transformed
        block in place -- or, when only a folded affine run reads the result, writes just its fp16 pair -- and the pair of the
        whole row is handed to the affine run behind; nothing is copied."""
        if not owned:
            x = x.clone()
        d_id = self.num_identity_features
        chain = self.transform_net.dense_chain(context)
        pair = carry["pair"] if carry is not None else None
        # the next leaf is a folded affine run: it multiplies the fp16 pair of this output, never the fp32 values, so the
        # fused kernel writes only the pair of the transformed block (x's transformed block is then stale and unread)
        pair_only = bool(carry is not None and carry.get("pair_only") and d_id % 8 == 0 and self._fused_pair_output)
        if pair is None:
            pair = K.Pair16.empty(x.shape[0], self.features, D.act_exp(), x.device)
            K.split_f16(x[:, :d_id], pair.exp, out=pair.cols(0, d_id), flags=flags)
        self._native_fused(chain, x, pair.cols(0, d_id), (d_id, self.features - d_id), lad, flags, inverse,
                           y_pair=pair if pair_only else None)
        if carry is not None:
            if pair_only:
                carry["pair"] = pair
            elif carry.get("pair_only"):          # an affine run follows but this coupling cannot write the pair alone
                K.split_f16(x[:, d_id:], pair.exp, out=pair.cols(d_id, self.features), flags=flags)
                carry["pair"] = pair
            else:                                 # nobody multiplies this output on the tensor cores
                carry["pair"] = None
        return x

    def _native_fused(self, chain, x, a, t_cols, lad, flags, inverse, y_pair=None):
        """The fused routes over row blocks of x (config.coupling_block_rows), transformed columns overwritten in place or their
        fp16 pair written to y_pair.  a: Pair16 of the conditioner input (packed path), or the identity column indices of x."""
        head = self._native_head(chain)
        block = D.whole_images(max(128, int(config.coupling_block_rows)))
        for r0 in range(0, x.shape[0], block):
            r1 = min(x.shape[0], r0 + block)
            xs = x[r0:r1]
            head.run(D.chain_rows(chain, r0, r1), a.rows(r0, r1) if isinstance(a, K.Pair16) else (xs, a), xs, t_cols,
                     None if y_pair is not None else xs, lad[r0:r1], flags, inverse,
                     y_pair=None if y_pair is None else y_pair.rows(r0, r1))

    def _native_apply(self, inputs, lad, flags, inverse, context=None, layout=None, owned=False, carry=None):
        self._check_inputs(inputs)
        if layout is not None:
            return self._native_packed(inputs, lad, flags, inverse, context, owned, carry)
        if self.unconditional_transform is None:
            return self._native_coupling(inputs, lad, flags, inverse, context)
        # identity half additionally goes through its own elementwise transform (coupling.py:90-94 forward: after the
        # conditioner has seen the untouched identity half; :114-118 inverse: before the conditioner)
        idf = self.identity_features
        if inverse:
            identity, lad_id = self.unconditional_transform.inverse(inputs[:, idf], context)
            staged = inputs.clone()
            staged[:, idf] = identity
            outputs = self._native_coupling(staged, lad, flags, True, context)
        else:
            outputs = self._native_coupling(inputs, lad, flags, False, context)
            identity, lad_id = self.unconditional_transform(inputs[:, idf], context)
            outputs[:, idf] = identity
        lad += lad_id
        return outputs

    def _native_coupling(self, inputs, lad, flags, inverse, context=None):
        id_cols, t_cols = self._cols(inputs.device)
        n = inputs.shape[0]
        outputs = torch.empty_like(inputs, memory_format=torch.contiguous_format)
        net = self.transform_net
        chain = net.dense_chain(context) if hasattr(net, "dense_chain") else None
        n_params = self.num_transform_features * self._transform_dim_multiplier()
        trunk_rows = D.whole_images(1 << 15)
        if chain is None and net.training and any(isinstance(m, torch.nn.modules.batchnorm._BatchNorm) for m in net.modules()):
            trunk_rows = max(1, n)      # a batch-dependent conditioner must see the whole batch (statistics, running averages)
        head = self._native_head(chain)
        if head.route != "rows":
            # stand-alone call (no composite arranging the column order): gather into [identity | transformed], run the
            # packed path in place, scatter back
            layout = self._native_layout(inputs, context)
            if layout is not None:
                packed = self._native_packed(K.gather_cols(inputs, layout.cols(inputs.device)), lad, flags, inverse, context,
                                             True)
                return K.gather_cols(packed, layout.cols(inputs.device, inverse=True), out=outputs)
            # feature counts not multiples of 8 (no TMA-addressable fp16 identity view): gathered trunk input, full copy of the
            # input as the output, transformed columns overwritten in place
            all_cols = D.derived(self, "_all_cols", [], lambda: torch.arange(self.features, dtype=torch.int32, device=inputs.device),
                                 extra=(inputs.device,))
            K.gather_cols(inputs, all_cols, out=outputs)
            self._native_fused(chain, outputs, id_cols, t_cols, lad, flags, inverse)
            return outputs
        for r0 in range(0, n, trunk_rows):
            r1 = min(n, r0 + trunk_rows)
            xs = inputs[r0:r1]
            if chain is None:
                identity = K.gather_cols(xs, id_cols)
                if context is not None:
                    context_rows = context[r0:r1]
                else:
                    context_rows = None
                params = net(identity, context_rows)
                if params.dim() != 2 or params.shape[1] != n_params:
                    raise ValueError("conditioner returned shape {}, expected [B, {}]".format(tuple(params.shape), n_params))
                self._native_epilogue(xs, params.float().contiguous(), t_cols, id_cols, outputs[r0:r1], lad[r0:r1], flags,
                                      inverse)
                continue
            head.run(D.chain_rows(chain, r0, r1), (xs, id_cols), xs, t_cols, outputs[r0:r1], lad[r0:r1], flags, inverse)
        return outputs

    def _native_epilogue(self, x, params, t_cols, id_cols, out, lad, flags, inverse):
        raise NotImplementedError()

    def _native_head(self, chain):
        """What runs the elementwise map from the conditioner (chain None: a module that is not a dense chain): `.route` is
        "rows" (last layer into HBM, then the epilogue kernel) or a fused route; `.run(...)` runs one row block of it."""
        raise NotImplementedError()

    _fused_pair_output = True      # the fused final kernel can write the fp16 pair of its outputs instead of fp32

    # ---- subclass API (same names as the reference) -------------------------------------------------------
    def _transform_dim_multiplier(self):
        raise NotImplementedError()

    def _coupling_transform_forward(self, inputs, transform_params):
        raise NotImplementedError()

    def _coupling_transform_inverse(self, inputs, transform_params):
        raise NotImplementedError()


class AffineCouplingTransform(CouplingTransform):
    """RealNVP affine coupling: y = x * scale(params) + shift(params) on the transformed features.
    Conditioner output layout is BLOCKED: first d_t columns = shift, last d_t = unconstrained scale."""

    DEFAULT_SCALE_ACTIVATION = lambda x: torch.sigmoid(x + 2) + 1e-3
    GENERAL_SCALE_ACTIVATION = lambda x: (softplus(x) + 1e-3).clamp(0, 3)

    def __init__(self, mask, transform_net_create_fn, unconditional_transform=None,
                 scale_activation=DEFAULT_SCALE_ACTIVATION):
        self.scale_activation = scale_activation
        super().__init__(mask, transform_net_create_fn, unconditional_transform)

    def _transform_dim_multiplier(self):
        return 2

    def _scale_and_shift(self, transform_params):
        raw_scale = transform_params[:, self.num_transform_features:, ...]
        shift = transform_params[:, :self.num_transform_features, ...]
        return self.scale_activation(raw_scale), shift

    def _coupling_transform_forward(self, inputs, transform_params):
        scale, shift = self._scale_and_shift(transform_params)
        log_scale = torch.log(scale)
        return inputs * scale + shift, torch.sum(log_scale.reshape(log_scale.shape[0], -1), dim=1)

    def _coupling_transform_inverse(self, inputs, transform_params):
        scale, shift = self._scale_and_shift(transform_params)
        log_scale = torch.log(scale)
        return (inputs - shift) / scale, -torch.sum(log_scale.reshape(log_scale.shape[0], -1), dim=1)

    def _activation_code(self):
        cls = AffineCouplingTransform
        if self.scale_activation is cls.__dict__["DEFAULT_SCALE_ACTIVATION"]:
            return 0
        if self.scale_activation is cls.__dict__["GENERAL_SCALE_ACTIVATION"]:
            return 1
        return None

    def _native_epilogue_supported(self):
        return self._activation_code() is not None

    def _native_epilogue(self, x, params, t_cols, id_cols, out, lad, flags, inverse):
        K.affine_coupling_rows(x, params, self._transform_dim_multiplier(), self._activation_code() or 0, inverse, t_cols,
                               id_cols, lad, out=out)

    # the last conditioner layer fused with the coupling (nfk_affine_coupling_final_f16x3): the [B, 2*d_t] parameter tensor of
    # coupling.py:229-232 is never written
    _fused_pair_output = False

    def _native_head(self, chain):
        return _AffineHead(self, chain)

    def _fused_final_ready(self, chain):
        hidden = chain[-1][0].shape[1]
        return D.fused_last_layer_ok(chain) and self._activation_code() is not None and K.f16x3_supported(hidden, hidden, hidden)

    def _fused_final(self, chain, state, x, t_cols, out, lad, flags, inverse, y_pair=None):
        weight, bias = chain[-1][0], chain[-1][1]
        mult = self._transform_dim_multiplier()
        w_pair, bias_i = D.pack_final_affine(weight, bias, self.num_transform_features, mult)
        K.affine_coupling_final(state.pair, w_pair, bias_i, x, t_cols, mult, self._activation_code() or 0, inverse, out, lad, flags)


class _AffineHead:
    """Affine / additive counterpart of dense.SplineHead: route "final" runs the trunk and the last layer fused with the coupling
    (nfk_affine_coupling_final_f16x3), route "rows" the trunk, the last layer into HBM and nfk_affine_coupling_rows."""

    def __init__(self, coupling, chain):
        self.coupling = coupling
        self.use_tc = chain is not None and D.chain_uses_tc(chain, coupling.num_identity_features)
        self.route = "final" if self.use_tc and coupling._fused_final_ready(chain) else "rows"

    def run(self, chain, a, x, t_cols, y, lad, flags, inverse, y_pair=None):
        c = self.coupling
        (src, id_cols), pair = ((x, None), a) if isinstance(a, K.Pair16) else (a, None)
        state = D.run_trunk(chain, src, id_cols, self.use_tc, x_pair=pair, flags=flags)
        if self.route == "final":
            with K.timed("rq_coupling_final", x.shape[0]):
                c._fused_final(chain, state, x, t_cols, y, lad, flags, inverse)
            return
        D.run_last_chunks(chain, state, self.use_tc, x.shape[0], c.num_transform_features * c._transform_dim_multiplier(), flags,
                          lambda params, q0, q1: c._native_epilogue(x[q0:q1], params, t_cols, id_cols, y[q0:q1], lad[q0:q1],
                                                                    flags, inverse))


class AdditiveCouplingTransform(AffineCouplingTransform):
    """NICE additive coupling: y = x + shift(params); log|det| = 0."""

    def _transform_dim_multiplier(self):
        return 1

    def _scale_and_shift(self, transform_params):
        return torch.ones_like(transform_params), transform_params

    def _native_epilogue_supported(self):
        return True


class PiecewiseCouplingTransform(CouplingTransform):
    def _coupling_transform_forward(self, inputs, transform_params):
        return self._coupling_transform(inputs, transform_params, inverse=False)

    def _coupling_transform_inverse(self, inputs, transform_params):
        return self._coupling_transform(inputs, transform_params, inverse=True)

    def _coupling_transform(self, inputs, transform_params, inverse=False):
        routed = self._native_training_spline(inputs, transform_params, inverse)
        if routed is not None:
            return routed
        if inputs.dim() == 4:
            b, c, h, w = inputs.shape
            # conditioner channels are ordered (feature, param): B x (C*M) x H x W -> B x C x H x W x M
            transform_params = transform_params.reshape(b, c, -1, h, w).permute(0, 1, 3, 4, 2)
        elif inputs.dim() == 2:
            b, d = inputs.shape
            transform_params = transform_params.reshape(b, d, -1)
        outputs, logabsdet = self._piecewise_cdf(inputs, transform_params, inverse)
        return outputs, torch.sum(logabsdet.reshape(logabsdet.shape[0], -1), dim=1)

    def _piecewise_cdf(self, inputs, transform_params, inverse=False):
        raise NotImplementedError()

    def _native_training_spline(self, inputs, transform_params, inverse):
        """(outputs, log|det|) of the spline on the kernels under autograd (config.native_training), or None."""
        return None


class PiecewiseRationalQuadraticCouplingTransform(PiecewiseCouplingTransform):
    """Neural-spline-flow coupling: each transformed feature goes through a monotonic rational-quadratic spline
    with `num_bins` bins whose 3K-1 (linear tails) or 3K+1 parameters come from the conditioner, laid out
    INTERLEAVED: conditioner column j*M + k is parameter k of transformed feature j."""

    def __init__(self, mask, transform_net_create_fn, num_bins=10, tails=None, tail_bound=1.0,
                 apply_unconditional_transform=False, img_shape=None,
                 min_bin_width=splines.rational_quadratic.DEFAULT_MIN_BIN_WIDTH,
                 min_bin_height=splines.rational_quadratic.DEFAULT_MIN_BIN_HEIGHT,
                 min_derivative=splines.rational_quadratic.DEFAULT_MIN_DERIVATIVE):
        self.num_bins = num_bins
        self.min_bin_width = min_bin_width
        self.min_bin_height = min_bin_height
        self.min_derivative = min_derivative
        self.tails = tails
        self.tail_bound = tail_bound
        if apply_unconditional_transform:
            from .nonlinearities import PiecewiseRationalQuadraticCDF
            unconditional_transform = lambda features: PiecewiseRationalQuadraticCDF(
                shape=[features] + (img_shape if img_shape else []), num_bins=num_bins, tails=tails,
                tail_bound=tail_bound, min_bin_width=min_bin_width, min_bin_height=min_bin_height,
                min_derivative=min_derivative)
        else:
            unconditional_transform = None
        super().__init__(mask, transform_net_create_fn, unconditional_transform=unconditional_transform)

    def _transform_dim_multiplier(self):
        return self.num_bins * 3 - 1 if self.tails == "linear" else self.num_bins * 3 + 1

    def _softmax_divisor(self, warn=True):
        net = self.transform_net
        if hasattr(net, "hidden_features"):
            return float(np.sqrt(net.hidden_features))
        if hasattr(net, "hidden_channels"):
            return float(np.sqrt(net.hidden_channels))
        if warn:
            warnings.warn("Inputs to the softmax are not scaled down: initialization might be bad.")
        return None

    def _piecewise_cdf(self, inputs, transform_params, inverse=False):
        k = self.num_bins
        widths = transform_params[..., :k]
        heights = transform_params[..., k:2 * k]
        derivatives = transform_params[..., 2 * k:]
        divisor = self._softmax_divisor()
        if divisor is not None:
            widths = widths / divisor
            heights = heights / divisor
        common = dict(inputs=inputs, unnormalized_widths=widths, unnormalized_heights=heights,
                      unnormalized_derivatives=derivatives, inverse=inverse, min_bin_width=self.min_bin_width,
                      min_bin_height=self.min_bin_height, min_derivative=self.min_derivative)
        if self.tails is None:
            return splines.rational_quadratic_spline(**common)
        return splines.unconstrained_rational_quadratic_spline(tails=self.tails, tail_bound=self.tail_bound, **common)

    def _native_training_spline(self, inputs, transform_params, inverse):
        args = (inputs, transform_params, inverse, self.num_bins, self.tails, self.tail_bound, self.min_bin_width,
                self.min_bin_height, self.min_derivative)
        if splines.training.routed(inputs, transform_params, self.num_bins, self.tails):
            return splines.training.rq_spline_rows(*args, self._softmax_divisor())
        if splines.training.routed_planes(inputs, transform_params, self.num_bins, self.tails):
            # image couplings: the conditioner's [B, C_t * M, H, W] output is read in place (no reshape / permute copy)
            return splines.training.rq_spline_planes(*args, self._softmax_divisor())
        return None

    def _native_epilogue_supported(self):
        if self.tails not in (None, "linear"):
            raise RuntimeError("{} tails are not implemented.".format(self.tails))
        return self.num_bins <= N.MAX_BINS

    def _native_head(self, chain):
        return D.spline_head(chain, self, self._softmax_divisor(), self.num_transform_features, self.num_identity_features)

    def _native_epilogue(self, x, params, t_cols, id_cols, out, lad, flags, inverse):
        K.rqs_rows(self._native_head(None).desc, inverse, x, params, t_cols, id_cols, lad, flags, out=out)
