"""MADE: masked autoregressive network (reference nflows/transforms/made.py:17-283), the conditioner of the
autoregressive transforms.  Masks are fixed 0/1 buffers; a masked layer is a dense layer with weight * mask, so on the
native path it runs on the same tensor-core dense kernels as the coupling conditioners (`dense_chain`)."""
import torch
from torch import nn
from torch.nn import functional as F
from torch.nn import init

from .. import dense as D
from .. import kernels as K
from ..utils import torchutils


def _get_input_degrees(in_features):
    """Degrees 1..D of the D inputs."""
    return torch.arange(1, in_features + 1)


class MaskedLinear(nn.Linear):
    """nn.Linear whose weight is multiplied by a fixed autoregressive mask.  Hidden units get degrees
    `arange(H) % (D-1) + 1` (or random ones) and may see inputs of degree <= their own; the output layer repeats each
    input degree `multiplier` times CONSECUTIVELY (row j*multiplier + k belongs to feature j) and may only see hidden
    units of strictly smaller degree."""

    def __init__(self, in_degrees, out_features, autoregressive_features, random_mask, is_output, bias=True):
        super().__init__(in_features=len(in_degrees), out_features=out_features, bias=bias)
        mask, degrees = self._get_mask_and_degrees(in_degrees=in_degrees, out_features=out_features,
                                                   autoregressive_features=autoregressive_features,
                                                   random_mask=random_mask, is_output=is_output)
        self.register_buffer("mask", mask)
        self.register_buffer("degrees", degrees)

    @classmethod
    def _get_mask_and_degrees(cls, in_degrees, out_features, autoregressive_features, random_mask, is_output):
        if is_output:
            out_degrees = torchutils.tile(_get_input_degrees(autoregressive_features), out_features // autoregressive_features)
            mask = (out_degrees[..., None] > in_degrees).float()
        else:
            if random_mask:
                low = min(torch.min(in_degrees).item(), autoregressive_features - 1)
                out_degrees = torch.randint(low=low, high=autoregressive_features, size=[out_features], dtype=torch.long)
            else:
                max_ = max(1, autoregressive_features - 1)
                min_ = min(1, autoregressive_features - 1)
                out_degrees = torch.arange(out_features) % max_ + min_
            mask = (out_degrees[..., None] >= in_degrees).float()
        return mask, out_degrees

    def forward(self, x):
        return F.linear(x, self.weight * self.mask, self.bias)

    def masked_weight(self):
        """weight * mask as a tensor object that stays the same until the weight changes (the operands derived from it are
        cached on it and freed with it)."""
        return D.derived(self, "_masked_weight", [self.weight, self.mask], lambda: (self.weight.detach() * self.mask).contiguous())


class MaskedFeedforwardBlock(nn.Module):
    """bn? -> masked linear -> activation -> dropout (same width in and out)."""

    def __init__(self, in_degrees, autoregressive_features, context_features=None, random_mask=False, activation=F.relu,
                 dropout_probability=0.0, use_batch_norm=False):
        super().__init__()
        features = len(in_degrees)
        self.batch_norm = nn.BatchNorm1d(features, eps=1e-3) if use_batch_norm else None
        self.linear = MaskedLinear(in_degrees=in_degrees, out_features=features,
                                   autoregressive_features=autoregressive_features, random_mask=random_mask, is_output=False)
        self.degrees = self.linear.degrees
        self.activation = activation
        self.dropout = nn.Dropout(p=dropout_probability)

    def forward(self, inputs, context=None):
        t = self.batch_norm(inputs) if self.batch_norm else inputs
        return self.dropout(self.activation(self.linear(t)))


class MaskedResidualBlock(nn.Module):
    """Pre-activation residual block of two masked linears; degrees are preserved so the skip connection is legal."""

    def __init__(self, in_degrees, autoregressive_features, context_features=None, random_mask=False, activation=F.relu,
                 dropout_probability=0.0, use_batch_norm=False, zero_initialization=True):
        if random_mask:
            raise ValueError("Masked residual block can't be used with random masks.")
        super().__init__()
        features = len(in_degrees)
        if context_features is not None:
            self.context_layer = nn.Linear(context_features, features)
        self.use_batch_norm = use_batch_norm
        if use_batch_norm:
            self.batch_norm_layers = nn.ModuleList([nn.BatchNorm1d(features, eps=1e-3) for _ in range(2)])
        linear_0 = MaskedLinear(in_degrees=in_degrees, out_features=features, autoregressive_features=autoregressive_features,
                                random_mask=False, is_output=False)
        linear_1 = MaskedLinear(in_degrees=linear_0.degrees, out_features=features,
                                autoregressive_features=autoregressive_features, random_mask=False, is_output=False)
        self.linear_layers = nn.ModuleList([linear_0, linear_1])
        self.degrees = linear_1.degrees
        if torch.all(self.degrees >= in_degrees).item() != 1:
            raise RuntimeError("In a masked residual block, the output degrees can't be less than the corresponding input degrees.")
        self.activation = activation
        self.dropout = nn.Dropout(p=dropout_probability)
        if zero_initialization:
            init.uniform_(self.linear_layers[-1].weight, a=-1e-3, b=1e-3)
            init.uniform_(self.linear_layers[-1].bias, a=-1e-3, b=1e-3)

    def forward(self, inputs, context=None):
        t = inputs
        if self.use_batch_norm:
            t = self.batch_norm_layers[0](t)
        t = self.linear_layers[0](self.activation(t))
        if context is not None:
            t = t + self.context_layer(context)
        if self.use_batch_norm:
            t = self.batch_norm_layers[1](t)
        t = self.linear_layers[1](self.dropout(self.activation(t)))
        return inputs + t


class MADE(nn.Module):
    """Masked initial layer -> residual (default) or feedforward masked blocks -> masked output layer producing
    `output_multiplier` values per feature, feature-major.  NOTE: like the reference class it does NOT expose
    `hidden_features`, so spline transforms built on it do not rescale their softmax logits."""

    def __init__(self, features, hidden_features, context_features=None, num_blocks=2, output_multiplier=1,
                 use_residual_blocks=True, random_mask=False, activation=F.relu, dropout_probability=0.0,
                 use_batch_norm=False):
        if use_residual_blocks and random_mask:
            raise ValueError("Residual blocks can't be used with random masks.")
        super().__init__()
        self.initial_layer = MaskedLinear(in_degrees=_get_input_degrees(features), out_features=hidden_features,
                                          autoregressive_features=features, random_mask=random_mask, is_output=False)
        if context_features is not None:
            self.context_layer = nn.Linear(context_features, hidden_features)
        self.use_residual_blocks = use_residual_blocks
        self.random_mask = random_mask
        self.activation = activation
        block_cls = MaskedResidualBlock if use_residual_blocks else MaskedFeedforwardBlock
        blocks = []
        degrees = self.initial_layer.degrees
        for _ in range(num_blocks):
            blocks.append(block_cls(in_degrees=degrees, autoregressive_features=features, context_features=context_features,
                                    random_mask=random_mask, activation=activation, dropout_probability=dropout_probability,
                                    use_batch_norm=use_batch_norm))
            degrees = blocks[-1].degrees
        self.blocks = nn.ModuleList(blocks)
        self.final_layer = MaskedLinear(in_degrees=degrees, out_features=features * output_multiplier,
                                        autoregressive_features=features, random_mask=random_mask, is_output=True)

    def forward(self, inputs, context=None):
        t = self.initial_layer(inputs)
        if context is not None:
            t = t + self.activation(self.context_layer(context))
        if not self.use_residual_blocks:
            t = self.activation(t)
        for block in self.blocks:
            t = block(t, context)
        return self.final_layer(t)

    def dense_chain(self, context=None):
        """[(weight*mask, bias, act_in, act_out, residual)] for the no-BN case with an activation the native kernels run
        (dense.activation_code; the act slots hold its code, 0 for none).  Residual blocks: the initial layer, then per block
        (l0 with the activation on its input and output, l1 adding the skip), then the final layer.  Feed-forward blocks: an MLP
        -- the initial layer (with the activation on its output unless `_activate_initial` is off) and every block's linear with
        the activation on its output -- which with non-random masks keeps the initial layer's degrees in every hidden layer.
        The context terms are not layers of the chain: with a context, `context_projection` computes them and the coupling-step
        kernel adds them to the trunk layers.  None with a context the net has no context layers for (the reference fails there
        as well).  A net WITH context layers called without a context is the plain chain, as the reference then skips the terms."""
        from .. import config
        act = D.native_activation(self.activation)
        if act is None or (context is not None and not self._has_context_layers()):
            return None
        for block in self.blocks:
            if (getattr(block, "use_batch_norm", False) or getattr(block, "batch_norm", None) is not None
                    or D.activation_code(block.activation) != act or (block.dropout.p > 0.0 and block.training)):
                return None
        if not self.use_residual_blocks:
            if self.random_mask or not config.native_activations:
                return None
            chain = [(self.initial_layer.masked_weight(), self.initial_layer.bias, 0, act if self._activate_initial else 0, None)]
            chain += [(b.linear.masked_weight(), b.linear.bias, 0, act, None) for b in self.blocks]
            chain.append((self.final_layer.masked_weight(), self.final_layer.bias, 0, 0, None))
            return chain
        chain = [(self.initial_layer.masked_weight(), self.initial_layer.bias, 0, 0, None)]
        for block in self.blocks:
            l0, l1 = block.linear_layers
            chain.append((l0.masked_weight(), l0.bias, act, act, None))
            chain.append((l1.masked_weight(), l1.bias, 0, 0, "skip"))
        chain.append((self.final_layer.masked_weight(), self.final_layer.bias, 0, 0, None))
        return chain

    def _has_context_layers(self):
        """The context layer of the initial layer and, with residual blocks, of every block (feed-forward blocks have none)."""
        return hasattr(self, "context_layer") and (not self.use_residual_blocks
                                                   or all(hasattr(block, "context_layer") for block in self.blocks))

    #: the initial layer's context term is act(Wc c + bc), and on the feed-forward path its output is activated, here;
    #: nflows.nn.nde's MADE adds the term without the activation and leaves the initial layer's output as it is
    _activate_initial = True

    def context_projection(self, sort=False, width=None):
        """ContextProjection of this net's context layers (None without them), its weight rows in the degree-sorted hidden order
        of the autoregressive inverse when `sort`, each term zero padded to `width` columns when given.  Cached until a
        context-layer parameter changes."""
        if not self._has_context_layers():
            return None
        layers = [self.context_layer] + [block.context_layer for block in self.blocks if hasattr(block, "context_layer")]

        def build():
            perm = None
            if sort:
                perm = torch.argsort(self.initial_layer.degrees.to(self.context_layer.weight.device), stable=True)
            act = D.activation_code(self.activation) if self._activate_initial else 0
            return ContextProjection(self, perm, initial_act=act, width=width)
        return D.derived(self, "_sorted_context_projection" if sort else "_context_projection",
                         [t for l in layers for t in (l.weight, l.bias)], build, extra=(width, D.activation_code(self.activation)))

    # ---- native: what the models that run a MADE on the coupling-step kernel share ----------------------------------------
    def in_pad(self):
        """Columns of the input pair: the features rounded up to 8 (TMA rows are multiples of 16 bytes)."""
        return (self.initial_layer.in_features + 7) // 8 * 8

    def hidden_pad(self):
        """The hidden width rounded up to 32, the step kernel's granularity (sbi's H = 50 runs as 64)."""
        return (self.initial_layer.out_features + 31) // 32 * 32

    def padded_chain(self, context):
        """dense_chain(context) with the initial layer's columns zero padded to in_pad() and the hidden units to hidden_pad()
        (rows of the trunk weights and biases, columns of the square and final weights), cached per parameter version; the chain
        itself when nothing needs padding, and only W0 copied when only its columns do.  Exact: every activation the kernels run
        maps 0 to 0, so a zero hidden unit stays zero through it and the skips."""
        chain = self.dense_chain(context)
        d, dp, hp = self.initial_layer.in_features, self.in_pad(), self.hidden_pad()
        if chain is None or (dp == d and hp == chain[0][0].shape[0]):
            return chain

        def padded():
            if hp == chain[0][0].shape[0]:
                w0 = chain[0][0].new_zeros(hp, dp)
                w0[:, :d] = chain[0][0]
                return [(w0,) + tuple(chain[0][1:])] + list(chain[1:])
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

    def degrees_kept(self):
        """Every block keeps the initial layer's hidden degrees, so the units a feature sees are a prefix once sorted."""
        degrees = [self.initial_layer.degrees] + [block.degrees for block in self.blocks]
        return D.derived(self, "_degrees_kept", degrees, lambda: all(torch.equal(d.cpu(), degrees[0].cpu()) for d in degrees[1:]))

    def sorted_subnets(self, chain, pack_final):
        """Degree-sorted copies of `chain`'s weights for the D sequential passes (an autoregressive inverse, a sampler); only
        when degrees_kept().  Feature i (degree i + 1) only sees hidden units of degree <= i; with the hidden units sorted by
        degree (one permutation for every hidden layer) those are a PREFIX, so pass i runs the sub-network of the first h_i units
        (rounded up to 32) and the final layer of feature i alone -- the total work of the D passes is ~1/8 of D full passes.
        Hidden units the chain pads take degree D, so they sort last and no feature's prefix needs them.
        pack_final(weight, bias) -> (Pair16, bias, rows per feature).  Returns (plans by width, h_i per feature, packed final
        layer, its bias, rows per feature), cached per parameter version."""
        features = self.initial_layer.in_features

        def build():
            deg = self.initial_layer.degrees.to(chain[0][0].device)
            hidden = chain[0][0].shape[0]
            deg = torch.cat([deg, deg.new_full((hidden - deg.numel(),), features)])
            perm = torch.argsort(deg, stable=True)
            sorted_deg = deg[perm].cpu()
            body = []
            for li, (w, b, act_in, act_out, res) in enumerate(chain[:-1]):
                w = w.detach()
                w = w[perm] if li == 0 else w[perm][:, perm]
                body.append((w.contiguous(), b.detach()[perm].contiguous(), act_in, act_out, res))
            wf = chain[-1][0].detach()[:, perm].contiguous()
            wp_pair, bias_packed, mp = pack_final(wf, chain[-1][1].detach())
            flags_l = D.plan_step_kernel(body + [chain[-1]])
            plans, widths = {}, []
            for i in range(features):
                count = int((sorted_deg <= i).sum())
                h = min(hidden, max(32, (count + 31) // 32 * 32))
                widths.append(h)
                if h not in plans:
                    sub = [((w[:h] if li == 0 else w[:h, :h]).contiguous(), b[:h].contiguous(), ai, ao, rs)
                           for li, (w, b, ai, ao, rs) in enumerate(body)]
                    plans[h] = D.StepPlan(sub).set_flags(flags_l)
            return plans, widths, wp_pair, bias_packed, mp
        return D.derived(self, "_subnets", [t for layer in chain for t in layer[:2]], build, extra=(D.act_exp(),))

    def native_context_ok(self, rows, context):
        """No context, or one the step kernel takes beside `rows`: a native-ok 2-D tensor on rows' device with rows' row count,
        for a net with context layers of its width.  Any other context stays on the torch path, which broadcasts or raises as the
        reference does."""
        if context is None:
            return True
        return (torch.is_tensor(context) and K.native_ok(context) and context.dim() == 2 and context.device == rows.device
                and context.shape[0] == rows.shape[0] and self._has_context_layers()
                and context.shape[1] == self.context_layer.in_features)

    def row_blocks(self, n, context):
        """(r0, r1) of a call's row blocks: the whole batch without a context, else config.coupling_block_rows rows (their context
        terms are projected once and read by every launch of the block)."""
        from .. import config
        block = n if context is None else max(128, int(config.coupling_block_rows))
        return [(r0, min(n, r0 + block)) for r0 in range(0, n, max(1, block))]

    def input_pair(self, x, flags):
        """Pair16 of x, zero padded to in_pad() columns."""
        n, d = x.shape
        if self.in_pad() == d:
            return K.split_f16(x, D.act_exp(), flags=flags)
        pair = K.Pair16.zeros(n, self.in_pad(), D.act_exp(), x.device)
        K.split_f16(x, D.act_exp(), out=pair.cols(0, d), flags=flags)
        return pair

    def sequential_passes(self, sub, ys, flags, launch):
        """The D passes of one row block on the sorted sub-networks `sub` (sorted_subnets): pass i calls
        launch(plan of width h_i, input pair, feature i's final rows, their bias, i), which writes feature i into ys[:, i], then
        splits that column into the input pair of pass i + 1."""
        plans, widths, wf, bias, mp = sub
        d = self.initial_layer.in_features
        pair = K.Pair16.zeros(ys.shape[0], self.in_pad(), D.act_exp(), ys.device)
        for i in range(d):
            h = widths[i]
            launch(plans[h], pair, K.Pair16(wf.hi[i * mp:(i + 1) * mp, :h], wf.lo[i * mp:(i + 1) * mp, :h], wf.exp),
                   bias[i * mp:(i + 1) * mp], i)
            if i + 1 < d:
                K.split_f16(ys[:, i:i + 1], pair.exp, out=pair.cols(i, i + 1), flags=flags)


class ContextProjection:
    """The context terms of a conditional MADE (reference made.py:187-202, 274-283).  Context only ever enters as a per-row
    additive term on a hidden layer -- relu(Wc c + bc) on the initial layer, Wc_b c + bc_b on the first linear of residual block
    b -- so the terms are two tensor-core GEMMs on the context's fp16 pair (the block projections stacked into one), and they do
    not depend on the inputs: the D passes of the inverse share them.  Feed-forward blocks have no context layers: the initial
    layer's term is then the only one.  `perm`: hidden units in this order (the degree sort of the autoregressive inverse; a
    sub-network of the first h units then reads the first h columns of every term).  `initial_act`: the activation code
    (include/nfk.h: NFK_ACT_*) of the initial layer's term, act(Wc c + bc); 0 for Wc c + bc.  `width`: every term has this many
    columns, the ones past the hidden width zero (a trunk zero padded to a wider hidden layer)."""

    def __init__(self, net, perm, initial_act=1, width=None):
        from .. import kernels as K
        h = net.initial_layer.out_features
        c = net.context_layer.in_features
        blocks = [block for block in net.blocks if hasattr(block, "context_layer")]
        self.hidden, self.context_features, self.num_blocks = h, c, len(blocks)
        self.initial_act = int(initial_act)
        self.width = h if width is None else int(width)
        self.pad = (c + 7) // 8 * 8                  # TMA rows are multiples of 16 bytes: zero padded like dense.Chain

        def operands(layers):
            w = torch.cat([layer.weight.detach() for layer in layers])
            b = torch.cat([layer.bias.detach() for layer in layers])
            if perm is not None:
                rows = torch.cat([perm + i * h for i in range(len(layers))])
                w, b = w[rows], b[rows]
            if self.width != h:
                k = len(layers)
                w = F.pad(w.reshape(k, h, c), (0, 0, 0, self.width - h)).reshape(k * self.width, c)
                b = F.pad(b.reshape(k, h), (0, self.width - h)).reshape(-1)
            if self.pad != c:
                w = F.pad(w, (0, self.pad - c))
            w = w.float().contiguous()
            return K.split_f16(w, K.weight_exp(w)), b.float().contiguous()

        self.initial = operands([net.context_layer])
        self.blocks = operands([block.context_layer for block in blocks]) if blocks else None

    def terms(self, context, flags=None):
        """Per trunk layer of the step kernel (initial layer, then the two linears of every block) the fp32 term of the rows of
        `context` [n, context_features], or None: [act(Wc c + bc), Wc_0 c + bc_0, None, Wc_1 c + bc_1, None, ...] (the first
        without the activation when initial_act is 0; just the first with feed-forward blocks)."""
        from .. import dense as D
        from .. import kernels as K
        n, c = context.shape
        exp = D.act_exp()
        pair = K.Pair16.zeros(n, self.pad, exp, context.device) if c != self.pad else K.Pair16.empty(n, c, exp, context.device)
        K.split_f16(context, exp, out=pair.cols(0, c), flags=flags)
        with K.timed("ar_context_terms", n):
            out = [K.linear_f16x3(pair, self.initial[0], self.initial[1], relu_out=self.initial_act, flags=flags)[0]]
            if self.blocks is not None:
                stacked = K.linear_f16x3(pair, self.blocks[0], self.blocks[1], flags=flags)[0]
                h = self.width
                for b in range(self.num_blocks):
                    out += [stacked[:, b * h:(b + 1) * h], None]
        return out
