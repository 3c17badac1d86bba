"""MADE as a density estimator (reference nflows/nn/nde/made.py:208-427): the nde MADE and MixtureOfGaussiansMADE.

The nde MADE is the MADE of transforms/made.py with one difference in its forward pass: the initial layer's context term is
added WITHOUT an activation, and no activation follows the initial layer on the feed-forward path either (reference :274-283);
`_activate_initial = False` tells the shared dense chain and context projection so.
Masked layers, blocks, masks, degrees, state_dict keys and the torch CPU RNG consumption order are those of transforms/made.py
(whose residual blocks are zero initialised as well), so a seed re-creates the reference's weights.

MixtureOfGaussiansMADE runs on the coupling-step kernel with its mixture epilogue (nfk_mog_made_step_f16x3): log_prob is one
launch per row block, sample one launch per feature on the degree-sorted sub-networks of the autoregressive inverse."""
import numpy as np
import torch
from torch import distributions
from torch.nn import functional as F

from ... import dense as D
from ... import kernels as K
from ...transforms import made as made_module
from ...transforms.autoregressive import sorted_subnets
from ...transforms.base import params_frozen
from ...utils import torchutils


class MADE(made_module.MADE):
    """MADE of reference nn/nde/made.py:208-283: residual (default) or feed-forward masked blocks; the context enters the
    initial layer as `+ context_layer(context)` with no activation."""

    _activate_initial = False

    def __init__(self, features, hidden_features, context_features=None, num_blocks=2, output_multiplier=1,
                 use_residual_blocks=True, random_mask=False, activation=F.relu, dropout_probability=0.0,
                 use_batch_norm=False):
        super().__init__(features, hidden_features, context_features=context_features, num_blocks=num_blocks,
                         output_multiplier=output_multiplier, use_residual_blocks=use_residual_blocks, random_mask=random_mask,
                         activation=activation, dropout_probability=dropout_probability, use_batch_norm=use_batch_norm)

    def forward(self, inputs, context=None):
        temps = self.initial_layer(inputs)
        if context is not None:
            temps = temps + self.context_layer(context)
        for block in self.blocks:
            temps = block(temps, context)
        return self.final_layer(temps)


class MixtureOfGaussiansMADE(MADE):
    """MADE whose outputs parametrise, per feature, a mixture of `num_mixture_components` Gaussians conditioned on the
    features before it (reference nn/nde/made.py:284-427).  Feature j's parameters are outputs.reshape(B, D, C, 3)[:, j]:
    (logit, mean, unconstrained std) per component, std = softplus(unconstrained) + epsilon.

    Native path (CUDA fp32, no autograd, residual blocks (at most 4) or non-random feed-forward blocks (at most 8) without batch
    norm or active dropout, an activation of dense.activation_code, C <= kernels' NFK_MOG_MAX_COMPONENTS): `log_prob` is one
    launch of the coupling-step kernel per row block, `sample` D launches per row block.  Features that are not a multiple of 8
    and hidden widths that are not a multiple of 32 run with the operands zero padded (exact: every activation the kernels run
    maps 0 to 0, so a zero hidden unit stays zero through it and the skips).  Everything else runs the torch formulation, line
    for line the reference's.

    sample(num_samples, context) returns (context rows, num_samples, D) like the reference and fails like it without a context.
    The one difference: the samples live on the context's device (the reference allocates them on the CPU, so it fails for a
    CUDA model).  On the native path u ~ U[0, 1) and e ~ N(0, 1) of shape [rows, D] are drawn on the device with the default
    generator (torch.manual_seed reproduces the samples) and component c* is the first whose cumulative softmax weight
    exceeds u."""

    def __init__(self, features, hidden_features, context_features=None, num_blocks=2, num_mixture_components=5,
                 use_residual_blocks=True, random_mask=False, activation=F.relu, dropout_probability=0.0, use_batch_norm=False,
                 epsilon=1e-2, custom_initialization=True):
        if use_residual_blocks and random_mask:
            raise ValueError("Residual blocks can't be used with random masks.")
        super().__init__(features, hidden_features, context_features=context_features, num_blocks=num_blocks,
                         output_multiplier=3 * num_mixture_components, use_residual_blocks=use_residual_blocks,
                         random_mask=random_mask, activation=activation, dropout_probability=dropout_probability,
                         use_batch_norm=use_batch_norm)
        self.num_mixture_components = num_mixture_components
        self.features = features
        self.hidden_features = hidden_features
        self.epsilon = epsilon
        if custom_initialization:
            self._initialize()

    def forward(self, inputs, context=None):
        return super().forward(inputs, context=context)

    def log_prob(self, inputs, context=None):
        if torch.is_tensor(inputs) and self._native_ready(inputs, context):
            with K.on_device_of(inputs):
                x = inputs if inputs.stride(-1) == 1 else inputs.contiguous()

                def attempt():
                    lp = K.zeros_lad(x)
                    flags = K.new_flags(x.device)
                    self._native_log_prob(x, context, lp, flags)
                    return None, lp, flags
                return K.run_with_activation_rescale(attempt)[1]
        K.warn_eager_cuda(inputs, self)
        return self._torch_log_prob(inputs, context)

    def _torch_log_prob(self, inputs, context=None):
        outputs = self.forward(inputs, context=context)
        outputs = outputs.reshape(*inputs.shape, self.num_mixture_components, 3)
        logits, means, unconstrained_stds = outputs[..., 0], outputs[..., 1], outputs[..., 2]
        log_mixture_coefficients = torch.log_softmax(logits, dim=-1)
        stds = F.softplus(unconstrained_stds) + self.epsilon
        log_prob = torch.sum(
            torch.logsumexp(
                log_mixture_coefficients
                - 0.5 * (np.log(2 * np.pi) + 2 * torch.log(stds) + ((inputs[..., None] - means) / stds) ** 2),
                dim=-1,
            ),
            dim=-1,
        )
        return log_prob

    def sample(self, num_samples, context=None):
        if context is not None:
            context = torchutils.repeat_rows(context, num_samples)
        with torch.no_grad():
            if context is not None and self._native_sample_ready(context):
                with K.on_device_of(context):
                    ctx = context if context.stride(-1) == 1 else context.contiguous()
                    u = torch.rand(ctx.shape[0], self.features, device=ctx.device)
                    e = torch.randn(ctx.shape[0], self.features, device=ctx.device)

                    def attempt():
                        flags = K.new_flags(ctx.device)
                        return self._native_sample(ctx, u, e, flags), None, flags
                    samples = K.run_with_activation_rescale(attempt)[0]
                return samples.reshape(-1, num_samples, self.features)
            samples = torch.zeros(context.shape[0], self.features, device=context.device)
            for feature in range(self.features):
                outputs = self.forward(samples, context)
                outputs = outputs.reshape(*samples.shape, self.num_mixture_components, 3)
                logits, means, unconstrained_stds = (outputs[:, feature, :, 0], outputs[:, feature, :, 1],
                                                     outputs[:, feature, :, 2])
                logits = torch.log_softmax(logits, dim=-1)
                stds = F.softplus(unconstrained_stds) + self.epsilon
                component_distribution = distributions.Categorical(logits=logits)
                components = component_distribution.sample((1,)).reshape(-1, 1)
                means, stds = means.gather(1, components).reshape(-1), stds.gather(1, components).reshape(-1)
                samples[:, feature] = (means + torch.randn(context.shape[0], device=context.device) * stds).detach()
        return samples.reshape(-1, num_samples, self.features)

    def _initialize(self):
        # mixture logits near zero (coefficients about uniform), unconstrained stds near the inverse softplus of 1 - epsilon
        self.final_layer.weight.data[::3, :] = self.epsilon * torch.randn(self.features * self.num_mixture_components,
                                                                          self.hidden_features)
        self.final_layer.bias.data[::3] = self.epsilon * torch.randn(self.features * self.num_mixture_components)
        self.final_layer.weight.data[2::3] = self.epsilon * torch.randn(self.features * self.num_mixture_components,
                                                                        self.hidden_features)
        self.final_layer.bias.data[2::3] = torch.log(torch.exp(torch.Tensor([1 - self.epsilon])) - 1) * torch.ones(
            self.features * self.num_mixture_components) + self.epsilon * torch.randn(self.features * self.num_mixture_components)

    # ---- native ----------------------------------------------------------------------------------------------------
    def _in_pad(self):
        return (self.features + 7) // 8 * 8

    def _hidden_pad(self):
        return (self.hidden_features + 31) // 32 * 32

    def _native_chain(self, context):
        """The dense chain with the initial layer's columns zero padded to _in_pad() and the hidden units to _hidden_pad() (rows
        of the trunk weights and biases, columns of the square and final weights), cached per parameter version; None when the
        net has no chain the step kernel takes."""
        chain = self.dense_chain(context)
        if chain is None:
            return None
        d, dp, h, hp = self.features, self._in_pad(), self.hidden_features, self._hidden_pad()
        if dp == d and hp == h:
            return chain

        def padded():
            out = []
            for li, (w, b, relu_in, relu_out, res) in enumerate(chain):
                last = li == len(chain) - 1
                wp = w.new_zeros(w.shape[0] if last else hp, dp if li == 0 else hp)
                wp[:w.shape[0], :w.shape[1]] = w.detach()
                bp = b.detach().new_zeros(w.shape[0] if last else hp)
                bp[:b.numel()] = b.detach()
                out.append((wp, bp, relu_in, relu_out, res))
            return out
        return D.derived(self, "_mog_chain", [t for layer in chain for t in layer[:2]], padded)

    def _native_context_ok(self, rows, context):
        if context is None:
            return True
        return (torch.is_tensor(context) and K.native_ok(context) and context.dim() == 2 and context.device == rows.device
                and context.shape[0] == rows.shape[0] and self._has_context_layers()
                and context.shape[1] == self.context_layer.in_features)

    def _native_head(self, context):
        chain = self._native_chain(context)
        if chain is None:
            return None, None
        return chain, D.MogHead(chain, self._in_pad(), self.num_mixture_components)

    def _native_ready(self, inputs, context):
        if not (K.native_ok(inputs, context) and inputs.dim() == 2 and inputs.shape[1] == self.features and params_frozen(self)
                and self._native_context_ok(inputs, context)):
            return False
        _, head = self._native_head(context)
        return head is not None and head.route == "step"

    def _native_sample_ready(self, context):
        if not (K.native_ok(context) and self._native_context_ok(context, context)):
            return False
        _, head = self._native_head(context)
        return head is not None and head.route == "step" and self._subnets_of(self._native_chain(context)) is not None

    def _subnets_of(self, chain):
        """The degree-sorted sub-networks of the sampler (transforms.autoregressive.sorted_subnets); padded hidden units take
        degree D, so they sort last and no feature's prefix needs them."""
        deg = self.initial_layer.degrees
        hp = self._hidden_pad()
        pad = lambda dg: torch.cat([dg, dg.new_full((hp - dg.numel(),), self.features)]) if hp != dg.numel() else dg
        degrees = [pad(deg)] + [pad(block.degrees) for block in self.blocks]
        return sorted_subnets(self, chain, degrees, self.features,
                              lambda w, b: D.mog_operands(w, b, self.num_mixture_components))

    def _input_pair(self, x, flags):
        n, d = x.shape
        if self._in_pad() == d:
            return K.split_f16(x, D.act_exp(), flags=flags)
        pair = K.Pair16.zeros(n, self._in_pad(), D.act_exp(), x.device)
        K.split_f16(x, D.act_exp(), out=pair.cols(0, d), flags=flags)
        return pair

    def _row_blocks(self, n, context):
        """Row blocks of a call: the whole batch without a context, else config.coupling_block_rows rows (their context terms
        are projected once and read by every launch of the block)."""
        from ... import config
        block = n if context is None else max(128, int(config.coupling_block_rows))
        return [(r0, min(n, r0 + block)) for r0 in range(0, n, max(1, block))]

    def _native_log_prob(self, x, context, lp, flags):
        """lp += log p(x | context): one launch per row block."""
        chain, head = self._native_head(context)
        proj = None if context is None else self.context_projection(width=self._hidden_pad())
        ctx = None if context is None else (context if context.stride(1) == 1 else context.contiguous())
        wf, bias, _ = D.mog_operands(chain[-1][0], chain[-1][1], self.num_mixture_components)
        plan = D.step_plan(chain)
        for r0, r1 in self._row_blocks(x.shape[0], context):
            terms = None if proj is None else proj.terms(ctx[r0:r1], flags)
            xs = x[r0:r1]
            head.step(plan, self._input_pair(xs, flags), wf, bias, self.epsilon, (0, self.features), x=xs, lad=lp[r0:r1],
                      flags=flags, terms=terms)
        return lp

    def _native_sample(self, context, u, e, flags):
        """Per row block, D launches on the degree-sorted sub-networks: pass i draws feature i from (u[:, i], e[:, i]) and
        splits it into the input pair of pass i + 1."""
        chain, head = self._native_head(context)
        plans, widths, wf, bias, mp = self._subnets_of(chain)
        proj = self.context_projection(sort=True, width=self._hidden_pad())
        n, d = context.shape[0], self.features
        samples = torch.empty(n, d, dtype=torch.float32, device=context.device)
        for r0, r1 in self._row_blocks(n, context):
            terms = proj.terms(context[r0:r1], flags)
            ys = samples[r0:r1]
            pair = K.Pair16.zeros(r1 - r0, self._in_pad(), D.act_exp(), context.device)
            for i in range(d):
                h = widths[i]
                wf_i = K.Pair16(wf.hi[i * mp:(i + 1) * mp, :h], wf.lo[i * mp:(i + 1) * mp, :h], wf.exp)
                head.step(plans[h], pair, wf_i, bias[i * mp:(i + 1) * mp], self.epsilon, (i, 1), y=ys,
                          noise=(u[r0:r1, i:], e[r0:r1, i:]), flags=flags, terms=terms)
                if i + 1 < d:
                    K.split_f16(ys[:, i:i + 1], pair.exp, out=pair.cols(i, i + 1), flags=flags)
        return samples
