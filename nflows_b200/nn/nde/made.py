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
    def _step_ready(self, context):
        """The mixture step kernel runs the padded chain: a component count with an instance and the MADE step route."""
        chain = self.padded_chain(context)
        return (chain is not None and K.mog_made_padded_rows(self.num_mixture_components) > 0
                and D.made_step_ready(chain, self.in_pad()))

    def _native_ready(self, inputs, context):
        return (K.native_ok(inputs, context) and inputs.dim() == 2 and inputs.shape[1] == self.features and params_frozen(self)
                and self.native_context_ok(inputs, context) and self._step_ready(context))

    def _native_sample_ready(self, context):
        return (K.native_ok(context) and self.native_context_ok(context, context) and self._step_ready(context)
                and self.degrees_kept())

    def _native_log_prob(self, x, context, lp, flags):
        """lp += log p(x | context): one launch per row block."""
        chain = self.padded_chain(context)
        proj = None if context is None else self.context_projection(width=self.hidden_pad())
        ctx = None if context is None else (context if context.stride(1) == 1 else context.contiguous())
        wf, bias, _ = D.mog_operands(chain[-1][0], chain[-1][1], self.num_mixture_components)
        plan = D.step_plan(chain)
        for r0, r1 in self.row_blocks(x.shape[0], context):
            terms = None if proj is None else proj.terms(ctx[r0:r1], flags)
            xs = x[r0:r1]
            K.mog_made_step(plan, self.input_pair(xs, flags), wf, bias, self.num_mixture_components, self.epsilon,
                            (0, self.features), x=xs, lad_accum=lp[r0:r1], flags=flags, terms=terms)
        return lp

    def _native_sample(self, context, u, e, flags):
        """Per row block, the D passes of sequential_passes on the degree-sorted sub-networks: pass i draws feature i from
        (u[:, i], e[:, i])."""
        c = self.num_mixture_components
        sub = self.sorted_subnets(self.padded_chain(context), lambda w, b: D.mog_operands(w, b, c))
        proj = self.context_projection(sort=True, width=self.hidden_pad())
        n = context.shape[0]
        samples = torch.empty(n, self.features, dtype=torch.float32, device=context.device)
        for r0, r1 in self.row_blocks(n, context):
            terms = proj.terms(context[r0:r1], flags)
            ys = samples[r0:r1]
            self.sequential_passes(sub, ys, flags, lambda plan, pair, wf, bias, i: K.mog_made_step(
                plan, pair, wf, bias, c, self.epsilon, (i, 1), y=ys, noise=(u[r0:r1, i:], e[r0:r1, i:]), flags=flags,
                terms=terms))
        return samples
