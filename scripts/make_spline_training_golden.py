"""Generate tests/golden/spline_training_grads.pt by running the UNMODIFIED reference (a checkout of bayesiains/nflows) on the CPU.

    NFLOWS_REFERENCE_SRC=<path of the reference checkout> python scripts/make_spline_training_golden.py

Training losses and the gradient of every parameter of RQ-spline flows whose splines train on nfk_rqs_planes_backward and
nfk_rqs_shared_backward (config.native_training), each in an fp32 and an fp64 run of the same weights:
  "glow_rq":         Glow-RQ on 3 x 8 x 8 images, 2 levels x 2 steps, 16 hidden channels, K = 8, linear tails (bound 3), the
                     perturbation of oracle/make_golden.py; loss -log_prob(x).mean();
  "nsf_uncond_linear": 2 x [RQ coupling with apply_unconditional_transform=True (ResidualNet, 16 hidden, K = 5, linear tails,
                     bound 3), ReversePermutation] on 6 features, x ~ N(0, 1.5^2);
  "nsf_uncond_sample": the same flow in the sampling direction: samples, lad = inverse(noise) and the loss
                     mean(0.5 |samples|^2 - (log N(noise) - lad)) that reaches both the samples and the log-density;
  "nsf_uncond_none": the same with tails=None on inputs in [0, 1];
  "image_uncond":    one image coupling with apply_unconditional_transform=True and img_shape=[8, 8] on 4 x 8 x 8 images
                     (ConvResidualNet, 16 hidden channels, K = 8, linear tails).
Every case stores the seed, the weight checksum after the perturbation, the inputs (the noise of the sampling case), and per
dtype the loss and the gradients by parameter name; the fp64 run's gradients are stored rounded to fp32 (a relative 6e-8, far
below any fp32 error bar), which keeps the file at about 0.7 MB.  No weights: nflows_b200's constructors consume the torch CPU
RNG in the reference's order, so the tests re-create them from the seed and check the checksum."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from oracle import make_golden as MG  # noqa: E402  (exits with a message when NFLOWS_REFERENCE_SRC is not set)

from nflows.nn.nets import ConvResidualNet  # noqa: E402

torch, T, Flow, np, torchutils, ResidualNet = MG.torch, MG.T, MG.Flow, MG.np, MG.torchutils, MG.ResidualNet
StandardNormal = MG.StandardNormal
BATCH = 4


def glow_rq():
    return MG.glow_multiscale(image_shape=(3, 8, 8), levels=2, steps=2, hidden_channels=16)


def nsf_uncond(tails):
    steps = []
    for i in range(2):
        steps.append(T.PiecewiseRationalQuadraticCouplingTransform(
            mask=torchutils.create_alternating_binary_mask(6, even=(i % 2 == 0)),
            transform_net_create_fn=lambda a, b: ResidualNet(a, b, hidden_features=16, num_blocks=1),
            num_bins=5, tails=tails, tail_bound=3.0, apply_unconditional_transform=True))
        steps.append(T.ReversePermutation(6))
    return Flow(T.CompositeTransform(steps), StandardNormal([6]))


def image_uncond():
    coupling = T.PiecewiseRationalQuadraticCouplingTransform(
        mask=torchutils.create_mid_split_binary_mask(4),
        transform_net_create_fn=lambda a, b: ConvResidualNet(a, b, hidden_channels=16, num_blocks=2),
        num_bins=8, tails="linear", tail_bound=3.0, apply_unconditional_transform=True, img_shape=[8, 8])
    return Flow(T.CompositeTransform([coupling]), StandardNormal([4, 8, 8]))


def sample_loss(flow, noise):
    samples, lad = flow._transform.inverse(noise.reshape(-1, *flow._distribution._shape))
    log_base = -0.5 * noise.square().sum(1) - 0.5 * noise.shape[1] * np.log(2 * np.pi)
    return (0.5 * samples.reshape(samples.shape[0], -1).square().sum(1) - (log_base - lad)).mean()


def case(seed, build, x, sample=False):
    torch.manual_seed(seed)
    flow = build().eval()
    MG.perturb(flow, seed + 1)
    rec = dict(seed=seed, perturb_seed=seed + 1, checksum=MG.weight_checksum(flow.state_dict()), x=x)
    for suffix, dtype in (("", torch.float32), ("_fp64", torch.float64)):
        flow.to(dtype)
        flow.zero_grad()
        loss = sample_loss(flow, x.to(dtype)) if sample else -flow.log_prob(x.to(dtype)).mean()
        loss.backward()
        rec["loss" + suffix] = loss.detach()
        rec["grads" + suffix] = {n: p.grad.detach().float() for n, p in flow.named_parameters() if p.grad is not None}
    return rec


def main():
    g = torch.Generator().manual_seed(7)
    rec = {
        "glow_rq": case(110, glow_rq, torch.randn(BATCH, 3, 8, 8, generator=g)),
        "nsf_uncond_linear": case(112, lambda: nsf_uncond("linear"), 1.5 * torch.randn(16, 6, generator=g)),
        "nsf_uncond_sample": case(112, lambda: nsf_uncond("linear"), torch.randn(16, 6, generator=g), sample=True),
        "nsf_uncond_none": case(114, lambda: nsf_uncond(None), torch.rand(16, 6, generator=g)),
        "image_uncond": case(116, image_uncond, torch.randn(BATCH, 4, 8, 8, generator=g)),
    }
    MG.save("spline_training_grads", rec)


if __name__ == "__main__":
    main()
