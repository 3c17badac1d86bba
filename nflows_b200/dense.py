"""Execution of dense-layer chains (conditioner networks, folded affine maps) on the native GEMM kernels.

Two kernels implement the same contract (fp32-equivalent products, fp32 accumulation):
  * "tc"   -- `nfk_linear_f16x3`: wgmma tensor cores, operands carried as fp16 (hi, lo) split pairs (kernels.Pair16);
              the default.
  * "simt" -- `nfk_linear`: FP32 FFMA pipe; used for shapes the TMA path cannot address (in_features not a multiple
              of 8) and selectable with NFLOWS_B200_GEMM=simt for A/B comparisons.
Both are CUDA kernels of this library; there is no PyTorch/cuBLAS path here."""
import os

import torch
from torch.autograd.function import once_differentiable
from torch.utils.weak import WeakIdKeyDictionary

from . import _native as N
from . import kernels as K


def backend():
    return os.environ.get("NFLOWS_B200_GEMM", "tc")


def cache_epoch():
    from . import config
    return config.cache_epoch


def act_exp():
    from . import config
    return int(config.activation_exp)


def activation_code(fn):
    """The activation code (include/nfk.h: NFK_ACT_*) under which the native kernels compute the conditioner activation `fn`,
    or None when they do not: F.relu / torch.relu / nn.ReLU (1), torch.tanh / F.tanh / nn.Tanh (2), F.elu / nn.ELU with alpha 1
    (3), F.leaky_relu / nn.LeakyReLU with slope 0.01 (4), F.gelu / nn.GELU with approximate='none' (5), F.silu / nn.SiLU (6).
    The functions are recognised with their default parameters only; anything else (sigmoid, lambdas, custom modules, other
    parameters) keeps the torch formulation.  This is the only place that maps a callable to a code."""
    from torch import nn
    from torch.nn import functional as F
    for fns, code in (((F.relu, torch.relu), N.ACT_RELU), ((torch.tanh, F.tanh), N.ACT_TANH), ((F.elu,), N.ACT_ELU),
                      ((F.leaky_relu,), N.ACT_LEAKY_RELU), ((F.gelu,), N.ACT_GELU), ((F.silu,), N.ACT_SILU)):
        if any(fn is f for f in fns):
            return code
    t = type(fn)
    if t is nn.ReLU:
        return N.ACT_RELU
    if t is nn.Tanh:
        return N.ACT_TANH
    if t is nn.ELU and fn.alpha == 1.0:
        return N.ACT_ELU
    if t is nn.LeakyReLU and fn.negative_slope == 0.01:
        return N.ACT_LEAKY_RELU
    if t is nn.GELU and fn.approximate == "none":
        return N.ACT_GELU
    if t is nn.SiLU:
        return N.ACT_SILU
    return None


def native_activation(fn):
    """activation_code(fn) where the native path runs it: relu always, the other codes with config.native_activations on;
    else None (the net keeps its torch formulation)."""
    from . import config
    code = activation_code(fn)
    return code if code == N.ACT_RELU or config.native_activations else None


_TENSOR_ENTRIES = WeakIdKeyDictionary()      # tensor -> {name: entry}; Tensor.__eq__ is elementwise, so keys compare by id


def derived(owner, name, sources, build, extra=()):
    """build(), cached as entry `name` of `owner` until its signature changes: (data_ptr, _version, device, shape) of every
    tensor in `sources`, config.cache_epoch and `extra` (plain values, no tensors).  A changed signature rebuilds the entry in
    place, so an owner has one entry per name, and the entry is freed with its owner: in the owner's __dict__ (a module or any
    other object), or beside it (a tensor).  The entry keeps the sources other than the owner alive, so no new tensor can take
    over their (data_ptr, _version) while it compares against them; the built value must not reference the owner, and `name`
    must not be an attribute of the owner's class (an entry in the __dict__ would hide it).
    The operands of the native path -- split pairs, packed final layers, step plans, masked, padded, sorted or folded weights --
    are all derived from parameters this way, once per parameter version."""
    sig = tuple((t.data_ptr(), t._version, t.device, t.shape) for t in sources) + (cache_epoch(),) + tuple(extra)
    entries = _TENSOR_ENTRIES.setdefault(owner, {}) if torch.is_tensor(owner) else owner.__dict__
    hit = entries.get(name)
    if hit is None or hit[0] != sig:
        hit = entries[name] = (sig, build(), [t for t in sources if t is not owner])
    return hit[1]


def split_weight(weight):
    """Pair16 of a weight matrix (scaled so that max |w| sits at 2^14), cached on the weight until it is modified."""
    def build():
        w = weight.detach().contiguous()
        return K.split_f16(w, K.weight_exp(w))
    return derived(weight, "_split", [weight], build)


def chain_uses_tc(chain, first_in_features):
    if backend() != "tc":
        return False
    k = first_in_features
    conv = getattr(chain, "conv3x3", ())
    if isinstance(chain, ConvChain):
        if k != chain.in_features or current_geometry() is None:
            return False
        k = chain.in_pad
    for i, (weight, _, _, _, _) in enumerate(chain):
        kk = 9 * k if i in conv else k
        if weight.shape[1] != kk or not K.f16x3_supported(kk, weight.stride(0), kk):
            return False
        k = weight.shape[0]
    return True


class StepPlan:
    """Operands of nfk_rq_coupling_step_f16x3 for every layer of a conditioner but the last: Pair16 of the initial layer's weight,
    stacked pairs + exponents of the square layers, stacked biases, layer flags."""

    def __init__(self, body):
        import ctypes
        h = body[0][0].shape[0]
        dev = body[0][0].device
        self.hidden = h
        self.act_exp = act_exp()
        w0 = body[0][0].detach().contiguous()
        self.w0 = K.split_f16(w0, K.weight_exp(w0))
        tail = body[1:]
        self.wt_hi = self.wt_lo = None
        exps = []
        if tail:
            self.wt_hi = torch.empty(len(tail) * h, h, dtype=torch.float16, device=dev)
            self.wt_lo = torch.empty_like(self.wt_hi)
            for l, layer in enumerate(tail):
                w = layer[0].detach().contiguous()
                e = K.weight_exp(w)
                K.split_f16(w, e, out=K.Pair16(self.wt_hi[l * h:(l + 1) * h], self.wt_lo[l * h:(l + 1) * h], e))
                exps.append(e)
        self.wt_exps_c = (ctypes.c_int32 * max(1, len(exps)))(*exps)
        self.bias = torch.cat([layer[1].detach().reshape(-1).float() for layer in body]).contiguous()
        self.layer_flags = None
        self.layer_flags_c = None

    def set_flags(self, flags):
        import ctypes
        self.layer_flags = list(flags)
        self.layer_flags_c = (ctypes.c_int32 * len(flags))(*[int(f) for f in flags])
        return self


def plan_step_kernel(chain):
    """Layer flags of nfk_rq_coupling_step_f16x3 for chain[:-1] (initial layer + square hidden layers), or None when the chain
    does not have that shape: one hidden width (a multiple of 32, <= 256), biases everywhere, skip adds that take the output
    of the layer two before (ResidualNet blocks), no activation on the first layer's input or between a skip add and its
    accumulate, and one activation per layer for its output and its consumer's input.  The chain's activation slots hold
    codes (include/nfk.h: NFK_ACT_*; True is relu); a code other than relu goes into flag bits [8, 12)."""
    body = chain[:-1]
    if not body or chain[0][2]:
        return None
    h = body[0][0].shape[0]
    flags = []
    saved = None                                     # index of the layer whose fp32 output is the saved skip tensor
    for i, (weight, bias, relu_in, relu_out, residual) in enumerate(body):
        if bias is None or weight.shape[0] != h or (i > 0 and weight.shape[1] != h):
            return None
        f = 1 if relu_out else 0
        if residual == "skip":
            if relu_out or saved is None or saved != i - 2:
                return None
            f |= 2
        elif residual is not None:
            return None
        if i + 2 < len(chain) and chain[i + 2][4] == "skip":
            f |= 4
            saved = i
        if chain[i + 1][2]:
            f |= 8
        acts = {int(a) for a in (relu_out, chain[i + 1][2]) if a}
        if len(acts) > 1 or not acts <= set(range(1, N.ACT_COUNT)):
            return None
        if acts and acts != {N.ACT_RELU}:
            f |= acts.pop() << N.STEP_ACT_SHIFT
        flags.append(f)
    return flags


def step_kernel_ready(chain, in_features, num_bins=8, tails="linear"):
    """True when nfk_rq_coupling_step_f16x3 runs chain[:-1] as its trunk on an input pair of in_features columns (the shape
    plan_step_kernel accepts, config.coupling_step_kernel on).  The trunk-only launch is the kernel's (8, linear) instance."""
    from . import config
    return bool(config.coupling_step_kernel and plan_step_kernel(chain) is not None
                and K.rq_coupling_step_supported(num_bins, tails, chain[0][0].shape[0], in_features, len(chain) - 2))


def fused_last_layer_ok(chain):
    """The last layer has the form the fused final-layer kernels take: bias, no output relu, no residual (config.fuse_coupling)."""
    from . import config
    _, bias, _, relu_out, residual = chain[-1]
    return bool(config.fuse_coupling and bias is not None and not relu_out and residual is None)


class SplineHead:
    """A rational-quadratic spline fed by the last layer of a conditioner chain: its validated descriptor and the kernel route
    that runs it,
      "step"  -- nfk_rq_coupling_step_f16x3: conditioner and spline in one launch;
      "final" -- the trunk, then nfk_rq_coupling_final_f16x3 (last layer fused with the spline);
      "rows"  -- the trunk, the last layer into HBM in L2-sized chunks, then nfk_rqs_rows (also the route of a conditioner
                 that is not a dense chain: chain None).
    `spline` carries the settings (num_bins, tails, tail_bound, min_bin_width, min_bin_height, min_derivative); widths and
    heights are divided by `divisor` (None: 1) before the softmax; d_t features are transformed; the conditioner input has
    in_features columns."""

    def __init__(self, chain, spline, divisor, d_t, in_features):
        self.desc = N.spline_desc(spline.num_bins, spline.tails, spline.tail_bound, 0.0, 1.0, 0.0, 1.0, spline.min_bin_width,
                                  spline.min_bin_height, spline.min_derivative, False, 1.0 if divisor is None else divisor)
        self.num_bins, self.tails, self.d_t = spline.num_bins, spline.tails, d_t
        self.use_tc = chain is not None and chain_uses_tc(chain, in_features)
        self.route = "rows"
        if self.use_tc and fused_last_layer_ok(chain):
            hidden = chain[-1][0].shape[1]
            if K.rq_coupling_final_supported(self.num_bins, self.tails, hidden, hidden):
                self.route = "step" if step_kernel_ready(chain, in_features, self.num_bins, self.tails) else "final"

    def run(self, chain, a, x, t_cols, y, lad, flags, inverse, y_pair=None, terms=None):
        """One row block: y[:, t_cols] = spline(x[:, t_cols]; conditioner(a)), lad += log|det| (lad may be None).
        a: Pair16 of the conditioner input, or (fp32 rows, identity column indices or None).  t_cols: int32 index tensor or
        (first, count).  y_pair (with y None): write the fp16 pair of the outputs instead (step / final routes).  A gathered
        input (identity columns given) takes the trunk and the fused final layer, never the step kernel.
        terms: per-row additive terms of the trunk layers (see step); the step route only."""
        if isinstance(a, K.Pair16):
            src, id_cols, pair = x, None, a
        else:
            (src, id_cols), pair = a, None
        if terms is not None and (self.route != "step" or id_cols is not None):
            raise ValueError("per-row trunk terms need the step route on an ungathered input")
        if self.route == "step" and id_cols is None:
            wp, bias, _ = spline_operands(chain[-1][0], chain[-1][1], self.num_bins, self.tails, self.d_t)
            if pair is None:
                pair = K.split_f16(src, act_exp(), flags=flags)
            self.step(step_plan(chain), pair, wp, bias, x, t_cols, y, lad, flags, inverse, y_pair, terms=terms)
            return
        state = run_trunk(chain, src, id_cols, self.use_tc, x_pair=pair, flags=flags)
        if self.route != "rows":
            wp, bias, _ = spline_operands(chain[-1][0], chain[-1][1], self.num_bins, self.tails, self.d_t)
            with K.timed("rq_coupling_final", x.shape[0]):
                K.rq_coupling_final(self.desc, inverse, state.pair, wp, bias, x, t_cols, y, lad, flags, y_pair=y_pair)
            return
        if isinstance(t_cols, tuple):
            first, count = t_cols
            t_cols = derived(self, "_t_cols", [], lambda: torch.arange(first, first + count, dtype=torch.int32, device=x.device),
                             extra=(first, count, x.device))
        m = N.spline_param_count(self.num_bins, self.tails == "linear")
        run_last_chunks(chain, state, self.use_tc, x.shape[0], self.d_t * m, flags, lambda params, q0, q1: K.rqs_rows(
            self.desc, inverse, x[q0:q1], params, t_cols, id_cols, None if lad is None else lad[q0:q1], flags, out=y[q0:q1]))

    def step(self, plan, pair, wp, bias, x, t_cols, y, lad, flags, inverse, y_pair=None, terms=None):
        """One launch of the step kernel with this spline: `plan` (StepPlan) and the packed last layer (wp, bias) may be
        sub-networks of the chain's (the autoregressive inverse runs one per feature).  terms: None, or per trunk layer an fp32
        tensor (or None) added to that layer's pre-activation row by row -- a sub-network reads a column prefix of it."""
        if terms is None:
            K.rq_coupling_step(plan, pair, self.desc, inverse, wp, bias, x, t_cols, y, lad, flags, y_pair=y_pair)
        else:
            K.rq_coupling_step(plan, pair, self.desc, inverse, wp, bias, x, t_cols, y, lad, flags, y_pair=y_pair, terms=terms)


def made_step_ready(chain, in_features):
    """True when the coupling-step kernel runs a MADE chain in one launch with the epilogue of the model that owns it (the affine
    map of MaskedAffineAutoregressiveTransform, the mixture of MixtureOfGaussiansMADE): a tensor-core chain on an input pair of
    in_features columns (the features zero padded to a multiple of 8), its last layer fusable, its trunk as the step kernel
    takes it.  Otherwise the model keeps its torch formulation."""
    return chain_uses_tc(chain, in_features) and fused_last_layer_ok(chain) and step_kernel_ready(chain, in_features)


def mog_operands(weight, bias, num_components):
    """(Pair16 of a MADE final layer with its 3C rows per feature packed to kernels.mog_made_padded_rows(C) rows (zero padded),
    the bias packed the same way, rows per feature) for nfk_mog_made_step_f16x3.  Cached on the weight until it changes."""
    m = 3 * num_components
    mp = K.mog_made_padded_rows(num_components)
    wp_pair, bias_packed = pack_final_spline(weight, bias, weight.shape[0] // m, m, mp)
    return wp_pair, bias_packed, mp


def ar_affine_operands(weight, bias):
    """(Pair16 of a MADE final layer as it stands -- rows 2j, 2j + 1 = (u_j, shift_j), no padding --, its fp32 bias, 2 rows per
    feature) for nfk_affine_ar_step_f16x3.  Cached on the weight until weight or bias is modified."""
    def build():
        w = weight.detach().contiguous()
        return K.split_f16(w, K.weight_exp(w)), bias.detach().float().contiguous()
    return derived(weight, "_ar_affine", [weight, bias], build) + (2,)


def spline_head(chain, spline, divisor, d_t, in_features):
    """SplineHead of (chain, spline), cached on the spline until a chain weight, the spline settings or a route option change."""
    from . import config
    layers = [] if chain is None else list(chain)
    structure = None if chain is None else (type(chain), tuple((l[1] is None,) + tuple(l[2:]) for l in layers))
    return derived(spline, "_spline_head", [l[0] for l in layers], lambda: SplineHead(chain, spline, divisor, d_t, in_features),
                   extra=(structure, spline.num_bins, spline.tails, spline.tail_bound, spline.min_bin_width,
                          spline.min_bin_height, spline.min_derivative, divisor, d_t, in_features, config.fuse_coupling,
                          config.coupling_step_kernel, backend(), current_geometry() is None))


def step_plan(chain):
    """StepPlan of a chain, cached on its initial weight until a trunk parameter or the activation exponent changes."""
    body = chain[:-1]
    return derived(body[0][0], "_step_plan", [t for layer in body for t in layer[:2]],
                   lambda: StepPlan(body).set_flags(plan_step_kernel(chain)), extra=(act_exp(),))


class Chain(list):
    """A dense chain whose layers also see a context tensor (ResidualNet with context_features, nn/nets/resnet.py:36-100):
    layer 0 carries residual token "ctx_init" (add W0[:, d_id:] context + b0: the reference concatenates [inputs, context] in
    front of the initial layer), the second layer of every block "glu_skip" (inputs + t * sigmoid(context_layer(context))).
    ctx_init = (weight padded to a multiple of 8 columns, bias, unpadded weight); ctx_gates[i] likewise for layer i."""

    def __init__(self, layers, context, ctx_init, ctx_gates, ctx_pad):
        super().__init__(layers)
        self.context, self.ctx_init, self.ctx_gates, self.ctx_pad = context, ctx_init, ctx_gates, ctx_pad
        self._pair = None

    def context_pair(self, flags=None):
        """Pair16 of the context, zero padded to ctx_pad columns (TMA rows are multiples of 16 bytes); split once per call."""
        if self._pair is None:
            n, c = self.context.shape
            self._pair = K.Pair16.zeros(n, self.ctx_pad, act_exp(), self.context.device) if c != self.ctx_pad else \
                K.Pair16.empty(n, c, act_exp(), self.context.device)
            K.split_f16(self.context, act_exp(), out=self._pair.cols(0, c), flags=flags)
        return self._pair

    def rows(self, r0, r1):
        part = Chain(list(self), self.context[r0:r1], self.ctx_init, self.ctx_gates, self.ctx_pad)
        if self._pair is not None:
            part._pair = self._pair.rows(r0, r1)
        return part


_IMAGE_GEOMETRY = [None]


class image_geometry:
    """`with image_geometry(b, h, w)`: the 2-D rows flowing through the native chain are the pixels of b images of h x w (channels
    last).  3x3 convolutions of a ConvChain need it; row blocks are kept to whole images while it is set."""

    def __init__(self, b, h, w):
        self.geom = (int(b), int(h), int(w))

    def __enter__(self):
        self.prev, _IMAGE_GEOMETRY[0] = _IMAGE_GEOMETRY[0], self.geom
        return self

    def __exit__(self, *exc):
        _IMAGE_GEOMETRY[0] = self.prev


def current_geometry():
    return _IMAGE_GEOMETRY[0]


def whole_images(rows):
    """`rows` rounded down to a multiple of the pixels per image (row blocks of an image chain), at least one image."""
    g = _IMAGE_GEOMETRY[0]
    if g is None:
        return rows
    hw = g[1] * g[2]
    return max(hw, rows // hw * hw)


class ConvChain(list):
    """Dense chain of a ConvResidualNet (nn/nets/resnet.py:103-205 of the reference) on pixel rows: 1x1 convolutions are dense
    layers as they stand; the layers listed in `conv3x3` are 3x3 / padding-1 convolutions whose weight is stored reshaped to
    [out, 9*in] in (ky, kx, c) order and whose operand is the im2col of the incoming pair (kernels.im2col3x3).  `in_pad`: the
    initial layer's weight is zero padded to this many columns (a TMA row is a multiple of 16 bytes; cfg 5 has 6 and 12 identity
    channels)."""

    def __init__(self, layers, conv3x3, in_features, in_pad):
        super().__init__(layers)
        self.conv3x3, self.in_features, self.in_pad = frozenset(conv3x3), in_features, in_pad


def chain_rows(chain, r0, r1):
    return chain.rows(r0, r1) if isinstance(chain, Chain) else chain


class ChainState:
    """Activation between two layers: fp32 tensor (`raw`, FFMA path) or the Pair16 a tensor-core layer consumes."""

    def __init__(self, raw=None, pair=None):
        self.raw, self.pair = raw, pair


def run_trunk(chain, x, id_cols, use_tc, x_pair=None, flags=None):
    """All layers of `chain` but the last, on the identity columns of x.  Returns the ChainState feeding the last layer
    (tensor-core path: the Pair16 of its pre-activated input).
    x_pair: Pair16 of the identity columns when the caller already has it (no gather / split pass then).
    The tensor-core path walks row sub-blocks (config.trunk_block_rows)."""
    from . import config
    n = x.shape[0]
    step = whole_images(max(128, int(config.trunk_block_rows)))
    if use_tc and n > step and len(chain) > 1:
        width = chain[-2][0].shape[0]
        dst = K.Pair16.empty(n, width, act_exp(), x.device)
        for r0 in range(0, n, step):
            r1 = min(n, r0 + step)
            _run_trunk_block(chain_rows(chain, r0, r1), x[r0:r1], id_cols, True, dst.rows(r0, r1),
                             None if x_pair is None else x_pair.rows(r0, r1), flags)
        return ChainState(pair=dst)
    return _run_trunk_block(chain, x, id_cols, use_tc, None, x_pair, flags)


def _run_trunk_block(chain, x, id_cols, use_tc, last_out, x_pair, flags):
    body = chain[:-1]
    last_relu_in = chain[-1][2]
    if use_tc:
        # every layer's epilogue writes the Pair16 the next layer consumes (pre-activated for it) and, where a residual
        # block needs its input again, the fp32 tensor as well
        in_pad = getattr(chain, "in_pad", None)
        if x_pair is None:
            x_id = x if id_cols is None else K.gather_cols(x, id_cols)
            if in_pad is not None and in_pad != x_id.shape[1]:
                x_pair = K.Pair16.zeros(x_id.shape[0], in_pad, act_exp(), x_id.device)
                K.split_f16(x_id, act_exp(), relu=body[0][2] if body else last_relu_in, out=x_pair.cols(0, x_id.shape[1]), flags=flags)
            else:
                x_pair = K.split_f16(x_id, act_exp(), relu=body[0][2] if body else last_relu_in, flags=flags)
        elif in_pad is not None and in_pad != x_pair.shape[1]:
            raise ValueError("a pre-split input of {} columns cannot feed an initial layer padded to {}".format(x_pair.shape[1], in_pad))
        elif (body[0][2] if body else last_relu_in):
            raise ValueError("a pre-split input cannot feed a layer that applies relu to its input")
        state = ChainState(pair=x_pair)
        skip_src = None
        if type(chain) is list and step_kernel_ready(chain, x_pair.shape[1]):
            # the whole trunk in ONE launch: the coupling-step kernel stopped after its last trunk layer (the activation pair
            # stays in shared memory between the layers; only the last layer's pair is written)
            out = last_out if last_out is not None else K.Pair16.empty(x_pair.shape[0], body[0][0].shape[0], act_exp(), x_pair.hi.device)
            with K.timed("trunk_step", x_pair.shape[0]):
                K.rq_coupling_step(step_plan(chain), x_pair, h_pair=out, flags=flags)
            return ChainState(pair=out)
        ctx_pair = chain.context_pair(flags) if isinstance(chain, Chain) else None
        conv = getattr(chain, "conv3x3", ())
        geom = current_geometry()
        for i, (weight, bias, relu_in, relu_out, residual) in enumerate(body):
            if i in conv:       # 3x3 convolution: dense layer on the im2col of the (already activated) incoming pair
                if geom is None or state.pair.shape[0] % (geom[1] * geom[2]):
                    raise RuntimeError("a 3x3 convolution layer needs whole images (dense.image_geometry)")
                state = ChainState(raw=state.raw, pair=K.im2col3x3(state.pair, state.pair.shape[0] // (geom[1] * geom[2]), geom[1], geom[2]))
            need_raw = i + 2 < len(chain) and chain[i + 2][4] in ("skip", "glu_skip")
            pair_out = last_out if i == len(body) - 1 else None
            b = bias.detach() if bias is not None else None
            if residual == "glu_skip":
                # inputs + (W2 a + b2) * sigmoid(Wc context + bc): two GEMMs and one elementwise pass
                wg, bg, _ = chain.ctx_gates[i]
                gate = K.linear_f16x3(ctx_pair, split_weight(wg), bg.detach(), want_y=True, flags=flags)[0]
                t = K.linear_f16x3(state.pair, split_weight(weight), b, relu_out=relu_out, want_y=True, flags=flags)[0]
                y, pair = K.glu_skip(t, gate, skip_src, want_y=need_raw, want_split=True, split_relu=chain[i + 1][2],
                                     pair_out=pair_out, flags=flags)
            else:
                res = skip_src if residual == "skip" else None
                if residual == "ctx_init":          # [inputs, context] W0^T + b0 = inputs W0a^T + (context W0b^T + b0)
                    wb, bb, _ = chain.ctx_init
                    res = K.linear_f16x3(ctx_pair, split_weight(wb), bb.detach() if bb is not None else None, want_y=True,
                                         flags=flags)[0]
                y, pair = K.linear_f16x3(state.pair, split_weight(weight), b, residual=res, relu_out=relu_out, want_y=need_raw,
                                         want_split=True, split_relu=chain[i + 1][2], pair_out=pair_out, flags=flags)
            if need_raw:
                skip_src = y
            state = ChainState(raw=y, pair=pair)
        return state
    hidden = x if id_cols is None else K.gather_cols(x, id_cols)
    branch = None
    ctx = chain.context.contiguous() if isinstance(chain, Chain) else None
    for i, (weight, bias, relu_in, relu_out, residual) in enumerate(body):
        b = bias.detach() if bias is not None else None
        if residual == "ctx_init":
            _, bb, wb = chain.ctx_init
            c0 = K.linear(ctx, wb, bb.detach() if bb is not None else None)
            hidden = K.linear(hidden, weight.detach(), None, residual=c0, relu_in=relu_in, relu_out=relu_out)
        elif residual == "glu_skip":
            _, bg, wg = chain.ctx_gates[i]
            t = K.linear(branch, weight.detach(), b, relu_in=relu_in, relu_out=relu_out)
            hidden = K.glu_skip(t, K.linear(ctx, wg, bg.detach()), hidden, want_y=True)[0]
        elif residual == "skip":
            hidden = K.linear(branch, weight.detach(), b, residual=hidden, relu_in=relu_in, relu_out=relu_out, out=hidden)
        elif relu_in:   # first layer of a residual block: keep its input for the skip connection
            branch = K.linear(hidden, weight.detach(), b, relu_in=relu_in, relu_out=relu_out)
        else:
            hidden = K.linear(hidden, weight.detach(), b, relu_in=relu_in, relu_out=relu_out)
    return ChainState(raw=hidden)


def run_last_chunks(chain, state, use_tc, n, n_params, flags, epilogue):
    """The last layer into HBM in row chunks small enough to stay L2-resident (config.param_chunk_mib), each followed by
    epilogue(params, r0, r1)."""
    from . import config
    rows = int(max(256, min(1 << 16, (config.param_chunk_mib << 20) // (4 * max(1, n_params)) // 128 * 128)))
    for q0 in range(0, n, rows):
        q1 = min(n, q0 + rows)
        with K.timed("final_linear", q1 - q0):
            params = run_last(chain, state, q0, q1, use_tc, flags=flags)
        with K.timed("spline_epilogue", q1 - q0):
            epilogue(params, q0, q1)


def run_last(chain, state, r0, r1, use_tc, flags=None):
    """Last layer of the chain on rows [r0, r1) of the trunk output -> fp32 conditioner output."""
    weight, bias, relu_in, relu_out, _ = chain[-1]
    b = bias.detach() if bias is not None else None
    if use_tc:
        return K.linear_f16x3(state.pair.rows(r0, r1), split_weight(weight), b, relu_out=relu_out, want_y=True, flags=flags)[0]
    return K.linear(state.raw[r0:r1], weight.detach(), b, relu_in=relu_in, relu_out=relu_out)


def affine_map(x, weight, bias, x_pair=None, pair_cols=0, flags=None, y_first_col=0):
    """y = x @ weight.T + bias for a folded ActNorm/Permutation/LU run: one tensor-core GEMM.  x_pair: Pair16 of x when the
    producer already wrote it (else one split pass).  pair_cols > 0: also return the Pair16 of y, filled for its first
    pair_cols columns (what the coupling behind this run feeds to its conditioner).  y_first_col > 0: nobody reads the fp32
    values of the columns before it (the consumer multiplies their pair), so they are not written.  Returns (y, pair or None)."""
    from . import config
    n, k = x.shape
    if backend() == "tc" and k % 8 == 0 and K.f16x3_supported(k, weight.stride(0), k):
        w_pair = split_weight(weight)
        o = weight.shape[0]
        y = torch.empty(n, o, dtype=torch.float32, device=x.device)
        if x_pair is None:
            x_pair = K.split_f16(x, act_exp(), flags=flags)
        y_pair = K.Pair16.empty(n, o, act_exp(), x.device) if (pair_cols and o % 8 == 0) else None
        step = max(128, int(config.affine_block_rows))
        for r0 in range(0, n, step):
            r1 = min(n, r0 + step)
            K.linear_f16x3(x_pair.rows(r0, r1), w_pair, bias, want_y=True, y_out=y[r0:r1], want_split=y_pair is not None,
                           split_cols=pair_cols, pair_out=None if y_pair is None else y_pair.rows(r0, r1), flags=flags,
                           y_first_col=y_first_col if y_pair is not None else 0)
        return y, y_pair
    return K.linear(x, weight, bias), None


def pack_final_affine(weight, bias, d_t, mult):
    """Operands of nfk_affine_coupling_final_f16x3: the last conditioner layer with its rows INTERLEAVED (shift_j, raw scale_j)
    instead of the reference's blocked [shifts | scales] (coupling.py:229-232), as a Pair16, plus the bias in the same order.
    Cached on the weight until weight or bias is modified."""
    def build():
        w, b = weight.detach(), bias.detach()
        if mult == 2:
            wi = torch.stack([w[:d_t], w[d_t:]], dim=1).reshape(2 * d_t, w.shape[1]).contiguous()
            bi = torch.stack([b[:d_t], b[d_t:]], dim=1).reshape(-1).contiguous()
        else:
            wi, bi = w.contiguous(), b.contiguous()
        return K.split_f16(wi, K.weight_exp(wi)), bi.float()
    return derived(weight, "_pack_affine", [weight, bias], build, extra=(d_t, mult))


def spline_operands(weight, bias, num_bins, tails, d_t):
    """(Pair16 of the packed last-layer weight, packed bias, padded parameters per feature MP) of the fused final layer / step
    kernels for a spline of num_bins bins on d_t features."""
    m = N.spline_param_count(num_bins, tails == "linear")
    mp = K.rq_coupling_final_padded_params(num_bins, tails)
    wp_pair, bias_packed = pack_final_spline(weight, bias, d_t, m, mp)
    return wp_pair, bias_packed, mp


def pack_final_spline(weight, bias, d_t, m, mp):
    """Packed operands of the fused coupling kernel: rows regrouped to `mp` per transformed feature (zero padded), split
    into a Pair16; bias packed the same way (fp32).  Cached on the weight until weight or bias is modified."""
    def build():
        w, b = weight.detach(), bias.detach()
        k = w.shape[1]
        wp = w.new_zeros(d_t, mp, k)
        wp[:, :m, :] = w.reshape(d_t, m, k)
        bp = b.new_zeros(d_t, mp)
        bp[:d_t, :m] = b.reshape(d_t, m)
        wp2 = wp.reshape(d_t * mp, k)
        return K.split_f16(wp2, K.weight_exp(wp2)), bp.reshape(-1).contiguous()
    return derived(weight, "_pack_spline", [weight, bias], build, extra=(d_t, m, mp))


# ---- training: a conditioner chain under autograd on the tensor cores (config.native_training) ---------------------------
def split_weight_t(weight, cols_pad):
    """Pair16 of weight^T [in, cols_pad] (the weight's rows zero padded to cols_pad, a multiple of 8): the operand that turns the
    gradient of a layer's output into the gradient of its input on nfk_linear_f16x3.  Cached on the weight until it is modified."""
    def build():
        w = weight.detach()
        wt = w.new_zeros(w.shape[1], cols_pad)
        wt[:, :w.shape[0]] = w.t()
        return K.split_f16(wt, split_weight(weight).exp)        # same absmax as the weight: no second host read
    return derived(weight, "_split_t", [weight], build, extra=(cols_pad,))


def _pad8(n):
    return (n + 7) // 8 * 8


def _chain_forward(layers, x, exp, flags):
    """Every layer on nfk_linear_f16x3 (one launch per layer).  Returns (the Pair16 each layer multiplied -- its input, activated as
    the layer takes it --, the fp32 output of the last layer)."""
    pairs = [K.split_f16(x, exp, relu=layers[0][2], flags=flags)]
    skip_src, y = None, None
    for i, (weight, bias, _, act_out, residual) in enumerate(layers):
        last = i == len(layers) - 1
        need_raw = i + 2 < len(layers) and layers[i + 2][4] == "skip"
        y, pair = K.linear_f16x3(pairs[i], split_weight(weight), bias.detach(), residual=skip_src if residual == "skip" else None,
                                 relu_out=act_out, want_y=need_raw or last, want_split=not last,
                                 split_relu=0 if last else layers[i + 1][2], split_exp=exp, flags=flags)
        if need_raw:
            skip_src = y
        if not last:
            pairs.append(pair)
    return pairs, y


class DenseChainTraining(torch.autograd.Function):
    """Output [B, out] of a conditioner chain (the list of ResidualNet / MLP dense_chain(): relu or no activations, skip adds
    into layers without an output activation, a last layer without one) on input x [B, in], with its backward on the tensor
    cores.  `structure` holds (act_in, act_out, residual) per layer, `params` (weight, bias) per layer.

    Forward: per layer nfk_linear_f16x3 at the activation exponent (lowered and repeated when a value leaves the fp16 range, as
    the inference path does); the pair each layer multiplied is saved -- the relu masks are read back from these pairs.
    Backward, per layer in reverse: dW, db from nfk_linear_f16x3_wgrad on (gradient pair, saved input pair); the gradient of the
    layer's input as nfk_linear_f16x3 of the gradient pair with the pair of W^T (split_weight_t); then nfk_mask_split_f16 applies
    the relu mask, adds the gradient a skip connection carries around the block (after the mask: the block's relu sits between
    the skip and the branch, so it cannot enter through the dense layer's residual input) and splits the result for the next
    layer.  Each gradient pair takes its exponent from the absmax of its tensor (kernels.gradient_exp): one host read per layer,
    waited for while the layer's weight-gradient kernel runs."""

    @staticmethod
    def forward(ctx, x, structure, *params):
        from . import config
        ctx.set_materialize_grads(False)
        layers = [(params[2 * i], params[2 * i + 1]) + tuple(s) for i, s in enumerate(structure)]
        exp = act_exp()
        with K.on_device_of(x):
            while True:
                flags = torch.zeros(1, dtype=torch.int32, device=x.device)
                pairs, y = _chain_forward(layers, x, exp, flags)
                if not config.check_domain:
                    break
                v = int(flags.item())
                if (v & 4) and config.auto_activation_exp and exp > -24:
                    exp = max(-24, exp - 5)
                    continue
                K.raise_for_flag_value(v)
                break
        ctx.save_for_backward(*[t for p in pairs for t in (p.hi, p.lo)], *params)
        ctx.structure, ctx.exp = structure, exp
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_y):
        from . import config
        want = ctx.needs_input_grad
        grads = [None] * len(want)
        if grad_y is None:
            return tuple(grads)
        n_layers = len(ctx.structure)
        saved = ctx.saved_tensors
        pairs = [K.Pair16(saved[2 * i], saved[2 * i + 1], ctx.exp) for i in range(n_layers)]
        params = saved[2 * n_layers:]
        layers = [(params[2 * i], params[2 * i + 1]) + tuple(s) for i, s in enumerate(ctx.structure)]
        with K.on_device_of(grad_y):
            flags = torch.zeros(1, dtype=torch.int32, device=grad_y.device)
            g32 = grad_y.contiguous()
            bound = K.absmax(g32)
            out = layers[-1][0].shape[0]
            g, _ = K.mask_split(g32, K.gradient_exp(bound), cols_pad=_pad8(out), want_y=False, flags=flags)
            dy = {}                     # layer -> (fp32 gradient of its output, absmax bound): the skip adds still to come
            for i in reversed(range(n_layers)):
                weight, bias = layers[i][:2]
                out = weight.shape[0]
                d_op = read_amax = None
                if i > 0 or want[0]:
                    d_op = K.linear_f16x3(g, split_weight_t(weight, g.shape[1]), want_y=True, flags=flags)[0]
                    if i > 0:
                        read_amax = K.absmax_start(d_op)         # read after the weight gradient is enqueued: it hides the wait
                if want[2 + 2 * i] or want[3 + 2 * i]:
                    dw, db = K.linear_wgrad(g.cols(0, out), pairs[i], want_bias=True)
                    grads[2 + 2 * i] = dw if want[2 + 2 * i] else None
                    grads[3 + 2 * i] = db if want[3 + 2 * i] else None
                if i == 0:
                    grads[0] = d_op
                    break
                # the gradient of layer i - 1's pre-activation: its output feeds layer i (through act_in) and, when layer i + 1 is
                # a skip layer, that layer's sum as well
                skip = dy.pop(i + 1) if i + 1 < n_layers and layers[i + 1][4] == "skip" else None
                relu = layers[i][2] or layers[i - 1][3]
                b = read_amax() + (skip[1] if skip is not None else 0.0)
                keep = layers[i - 1][4] == "skip"            # its output gradient flows on to layer i - 3's output
                g, g_raw = K.mask_split(d_op, K.gradient_exp(b), mask=pairs[i] if relu else None,
                                        skip=skip[0] if skip is not None else None, cols_pad=pairs[i].shape[1], want_y=keep, flags=flags)
                if keep:
                    dy[i - 1] = (g_raw, b)
            if config.check_domain:
                v = int(flags.item())
                if v & 4:
                    raise K.Float16RangeError("a conditioner gradient is not finite (the fp16 split of a gradient overflowed)")
        return tuple(grads)


def train_chain(chain, x):
    """Conditioner output of the dense chain `chain` (splines.training.routed_conditioner accepted it) on x, differentiable."""
    structure = tuple((int(l[2]), int(l[3]), l[4]) for l in chain)
    return DenseChainTraining.apply(x.contiguous(), structure, *[t for l in chain for t in l[:2]])
