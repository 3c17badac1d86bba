"""Training of image RQ couplings and of PiecewiseRationalQuadraticCDF with the spline on the kernels (config.native_training) on
an H100: nfk_rqs_planes, nfk_rqs_planes_backward and nfk_rqs_shared_backward against fp64 autograd at every instance, their
shape, NULL and determinism contract, whole-model gradients and an SGD run against fp64 copies, and the evidence that the kernels
ran (or, with the switch off, that nothing launched)."""
import copy

import pytest
import torch

import _spline_cases as S
import _spline_training_models as MODELS
from conftest import load_golden
from nflows_b200 import _native as N
from nflows_b200 import config
from nflows_b200 import kernels as K
from nflows_b200 import transforms as T
from oracle import flow_oracle as O
from test_spline_training_gpu import _sandwich
from test_spline_training_host import assert_statistically_as_accurate, autograd_vjp, near_knot

pytestmark = pytest.mark.gpu

# every instance branch: < 8, 8 exact, < 16, 16 exact, <= 32, <= 64
KERNEL_BINS = (3, 8, 12, 16, 24, 64)


def _m(bins, tails):
    return 3 * bins - 1 if tails == "linear" else 3 * bins + 1


def _away_from_knots(x, uw, uh, tails, inverse):
    """x with the inputs within rounding of an fp64 knot (near_knot) moved 5e-5 of the interval inward: at a knot the gradient
    jumps (the spline's second derivative is not continuous) and fp32 knots may take either bin, so a batch sum of parameter
    gradients would measure which side a handful of knot inputs fell on, not the arithmetic or the reduction."""
    near = near_knot(x, uw, uh, tails, inverse, S.DIVISOR).to(x.device)
    step = 5e-5 * (2 * S.TAIL_BOUND if tails == "linear" else 1.0)
    return torch.where(near, x - torch.sign(x - (0.0 if tails == "linear" else 0.5)) * step, x)


def _planes_case(n, c, pixels, bins, tails, dev, seed, inverse=False):
    """x [n, c, 1, pixels], params [n, c*M, 1, pixels] and the same parameters as element rows (uw, uh, ud [n*c*pixels, .])."""
    g = torch.Generator(device=dev).manual_seed(seed)
    m = _m(bins, tails)
    uw, uh, ud = S.params(n * c * pixels, bins, tails, g, scale=1.5)
    rows = torch.cat([uw, uh, ud], -1)                                          # element (b, j, p) in row order
    params = rows.reshape(n, c, pixels, m).permute(0, 1, 3, 2).reshape(n, c * m, 1, pixels).contiguous()
    x = _away_from_knots(S.inputs(n * c * pixels, tails, g) * 0.999, uw, uh, tails, inverse).reshape(n, c, 1, pixels)
    return x, params, (uw, uh, ud)


def _rows_of(gp, n, c, pixels, m):
    return gp.reshape(n, c, m, pixels).permute(0, 1, 3, 2).reshape(-1, m)


@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("tails", ["linear", None])
@pytest.mark.parametrize("bins", KERNEL_BINS)
def test_planes_kernels_against_fp64(cuda_device, bins, tails, inverse, monkeypatch):
    monkeypatch.setattr(O, "F32_CUMSUM", True)
    for n, c, pixels in ((40, 6, 16), (13, 3, 64), (500, 1, 4)):              # >= 2000 elements per shape
        x, params, (uw, uh, ud) = _planes_case(n, c, pixels, bins, tails, cuda_device, bins * 7 + c + inverse,
                                                  inverse)
        desc = S.desc(bins, tails)
        m = _m(bins, tails)
        what = (bins, tails, inverse, n, c, pixels)
        # forward: y and the per-sample log|det|
        lad = torch.zeros(n, device=cuda_device)
        y = K.rqs_planes(desc, inverse, x, params, lad, None)
        (ty, tl), (ry, rl) = S.truth_and_yardstick(x.reshape(-1), uw, uh, ud, tails, inverse)
        assert_statistically_as_accurate(y.reshape(-1).cpu(), ry, ty, what + ("y",))
        assert_statistically_as_accurate(lad.cpu(), rl.reshape(n, -1).sum(1), tl.reshape(n, -1).sum(1), what + ("lad",))
        # backward
        g = torch.Generator(device=cuda_device).manual_seed(bins)
        gy, gl = torch.randn(x.shape, generator=g, device=cuda_device), torch.randn(n, generator=g, device=cuda_device)
        gx, gp = K.rqs_planes_backward(desc, inverse, x, params, gy, gl)
        glx = gl[:, None].expand(n, c * pixels).reshape(-1)
        args = (x.reshape(-1), uw, uh, ud, gy.reshape(-1), glx, tails, inverse)
        tx, tp = autograd_vjp(*args, torch.float64, S.DIVISOR)
        rx, rp = autograd_vjp(*args, torch.float32, S.DIVISOR)
        skip = near_knot(x.reshape(-1), uw, uh, tails, inverse, S.DIVISOR)
        assert_statistically_as_accurate(gx.reshape(-1).cpu(), rx.cpu(), tx, what + ("g_x",), skip)
        assert_statistically_as_accurate(_rows_of(gp, n, c, pixels, m).cpu(), rp.cpu(), tp, what + ("g_params",), skip)


@pytest.mark.parametrize("pixels", [1, 4, 16, 64, 256, 1024])
def test_planes_shapes_nulls_and_determinism(cuda_device, pixels):
    """C_t from 1 to 48, batches of 1 to past one launch round, NULL cotangents and grad_x, bitwise-identical repeats, and a
    forward log|det| that is bitwise identical across batch splits."""
    bins, tails = 8, "linear"
    desc = S.desc(bins, tails)
    sms = torch.cuda.get_device_properties(cuda_device).multi_processor_count
    for c in (1, 3, 6, 12, 48):
        threads = min(256, max(32, (c * pixels + 31) // 32 * 32))
        fwd_round = sms * (2048 // threads)                                      # samples of one forward launch round
        for n in sorted({1, 7, min(fwd_round + 3, max(8, (1 << 22) // (c * pixels * 23)))}):
            x, params, _ = _planes_case(n, c, pixels, bins, tails, cuda_device, c + pixels + n)
            lad = torch.zeros(n, device=cuda_device)
            y = K.rqs_planes(desc, False, x, params, lad, None)
            lad2 = torch.zeros(n, device=cuda_device)
            assert torch.equal(K.rqs_planes(desc, False, x, params, lad2, None), y) and torch.equal(lad, lad2)
            if n > 1:
                h = n // 2
                la, lb = torch.zeros(h, device=cuda_device), torch.zeros(n - h, device=cuda_device)
                ya = K.rqs_planes(desc, False, x[:h].contiguous(), params[:h].contiguous(), la, None)
                yb = K.rqs_planes(desc, False, x[h:].contiguous(), params[h:].contiguous(), lb, None)
                assert torch.equal(torch.cat([la, lb]), lad) and torch.equal(torch.cat([ya, yb]), y)
            gy, gl = torch.randn_like(x), torch.randn(n, device=cuda_device)
            gx, gp = K.rqs_planes_backward(desc, False, x, params, gy, gl)
            gx2, gp2 = K.rqs_planes_backward(desc, False, x, params, gy, gl)
            assert torch.equal(gx, gx2) and torch.equal(gp, gp2)
            gx_y, gp_y = K.rqs_planes_backward(desc, False, x, params, gy, None)
            gx_l, gp_l = K.rqs_planes_backward(desc, False, x, params, None, gl)
            assert float((gx_y + gx_l - gx).abs().max()) <= 1e-4 * max(1.0, float(gx.abs().max()))
            assert float((gp_y + gp_l - gp).abs().max()) <= 1e-4 * max(1.0, float(gp.abs().max()))
            none_x, gp_n = K.rqs_planes_backward(desc, False, x, params, gy, gl, want_grad_x=False)
            assert none_x is None and torch.equal(gp_n, gp)


def _shared_case(n, f, bins, tails, dev, seed, inverse=False):
    g = torch.Generator(device=dev).manual_seed(seed)
    uw, uh, ud = S.params(f, bins, tails, g, scale=1.5)
    x = S.inputs(n * f, tails, g) * 0.999
    x = _away_from_knots(x, uw.repeat(n, 1), uh.repeat(n, 1), tails, inverse).reshape(n, f)
    return x, uw, uh, ud


def _sums_ok(got, truth, ref32):
    """The batch-summed parameter gradients: within 4x the norm-relative error of torch's fp32 formulation (and its reduction of
    the expanded per-row gradient) from fp64, or 2e-5.  4x and not 3x: the per-element arithmetic of the kernels' spline (MUFU
    exponentials and reciprocals) is held to 4x at the percentiles by the existing training tests, and at a few rows the sums
    are no more than that arithmetic."""
    return _rel(got, truth) <= max(2e-5, 4 * _rel(ref32, truth))


def _shared_truth(x, uw, uh, ud, gy, gl, tails, inverse, dtype):
    n, f = x.shape
    rows = lambda p: p[None].expand(n, *p.shape).reshape(n * f, -1)
    gx, gp = autograd_vjp(x.reshape(-1), rows(uw), rows(uh), rows(ud), gy.reshape(-1), gl[:, None].expand(n, f).reshape(-1),
                          tails, inverse, dtype, S.DIVISOR)
    return gx, gp.reshape(n, f, -1).sum(0)


def _rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).norm()) / max(float(b.double().cpu().norm()), 1e-30)


@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("tails", ["linear", None])
@pytest.mark.parametrize("bins", KERNEL_BINS)
def test_shared_backward_against_fp64(cuda_device, bins, tails, inverse, monkeypatch):
    """Per element (one row per launch: a sum of one term is exact) against fp64 autograd with the spline bar of the training
    tests; the batch sum against the fp64 sum of those same per-element values, which isolates the two-pass reduction (every row
    of a feature shares its knots, so against fp64 autograd a sum would carry each feature's knot rounding coherently)."""
    monkeypatch.setattr(O, "F32_CUMSUM", True)
    desc = S.desc(bins, tails)
    for n, f in ((150, 24), (40, 64), (9, 192)):
        x, uw, uh, ud = _shared_case(n, f, bins, tails, cuda_device, bins + f + inverse, inverse)
        g = torch.Generator(device=cuda_device).manual_seed(f)
        gy, gl = torch.randn(n, f, generator=g, device=cuda_device), torch.randn(n, generator=g, device=cuda_device)
        gx, guw, guh, gud = K.rqs_shared_backward(desc, inverse, x, uw, uh, ud, gy, gl)
        rows = [K.rqs_shared_backward(desc, inverse, x[r:r + 1], uw, uh, ud, gy[r:r + 1], gl[r:r + 1]) for r in range(n)]
        per_el = torch.stack([torch.cat(o[1:], -1) for o in rows])                 # [n, f, MT]
        assert torch.equal(torch.cat([o[0] for o in rows]), gx)
        what = (bins, tails, inverse, n, f)
        rr = lambda p: p[None].expand(n, *p.shape).reshape(n * f, -1)
        args = (x.reshape(-1), rr(uw), rr(uh), rr(ud), gy.reshape(-1), gl[:, None].expand(n, f).reshape(-1), tails, inverse)
        tx, tp = autograd_vjp(*args, torch.float64, S.DIVISOR)
        rx, rp = autograd_vjp(*args, torch.float32, S.DIVISOR)
        skip = near_knot(x.reshape(-1), rr(uw), rr(uh), tails, inverse, S.DIVISOR)
        assert_statistically_as_accurate(gx.reshape(-1).cpu(), rx.cpu(), tx, what + ("g_x",), skip)
        assert_statistically_as_accurate(per_el.reshape(n * f, -1).cpu(), rp.cpu(), tp, what + ("g_params",), skip)
        got = torch.cat([guw, guh, gud], -1)
        assert _rel(got, per_el.double().sum(0)) <= 1e-5, what + (_rel(got, per_el.double().sum(0)),)


@pytest.mark.parametrize("f", [1, 5, 64, 192, 784])
def test_shared_backward_batches_nulls_and_determinism(cuda_device, f):
    """B from 1 to 2^20 elements' worth of rows: the fp32 parameter sums against fp64 with the torch fp32 bar, bitwise repeats,
    NULL cotangents and NULL grad_x."""
    bins, tails = 8, "linear"
    desc = S.desc(bins, tails)
    for n in sorted({1, 3, 255, 4097, max(1, (1 << 20) // f)}):
        x, uw, uh, ud = _shared_case(n, f, bins, tails, cuda_device, n + f)
        g = torch.Generator(device=cuda_device).manual_seed(n)
        gy, gl = torch.randn(n, f, generator=g, device=cuda_device), torch.randn(n, generator=g, device=cuda_device)
        out = K.rqs_shared_backward(desc, False, x, uw, uh, ud, gy, gl)
        again = K.rqs_shared_backward(desc, False, x, uw, uh, ud, gy, gl)
        assert all(torch.equal(a, b) for a, b in zip(out, again))
        got = torch.cat(out[1:], -1)
        # torch's own fp32 reduction of the expanded per-row gradient against fp64
        from nflows_b200.transforms.splines import unconstrained_rational_quadratic_spline as spline
        for dtype in (torch.float32, torch.float64):
            leaves = [p.detach().to(dtype).requires_grad_(True) for p in (uw, uh, ud)]
            ex = lambda p: p[None].expand(n, *p.shape)
            y, lad = spline(x.to(dtype), ex(leaves[0]) / S.DIVISOR, ex(leaves[1]) / S.DIVISOR, ex(leaves[2]), tails=tails,
                            tail_bound=S.TAIL_BOUND)
            ((y * gy.to(dtype)).sum() + (lad.sum(1) * gl.to(dtype)).sum()).backward()
            grad = torch.cat([p.grad for p in leaves], -1)
            if dtype == torch.float32:
                ref32 = grad
            else:
                truth = grad
        assert _sums_ok(got, truth, ref32), (f, n, _rel(got, truth), _rel(ref32, truth))
        gx_y = K.rqs_shared_backward(desc, False, x, uw, uh, ud, gy, None)
        gx_l = K.rqs_shared_backward(desc, False, x, uw, uh, ud, None, gl)
        for a, b, c in zip(gx_y, gx_l, out):
            assert float((a + b - c).abs().max()) <= 1e-4 * max(1.0, float(c.abs().max()))
        none_x = K.rqs_shared_backward(desc, False, x, uw, uh, ud, gy, gl, want_grad_x=False)
        assert none_x[0] is None and all(torch.equal(a, b) for a, b in zip(none_x[1:], out[1:]))


# ---- whole models against fp64 copies ---------------------------------------------------------------------------------------
def _model_grads(model, x, sample, native, monkeypatch):
    monkeypatch.setattr(config, "native_training", native)
    g, _ = MODELS.grads(model, x, sample)
    return [g.get(n) for n, _ in model.named_parameters()]


def _check_model(model, x, sample, tags_wanted, monkeypatch):
    model = model.eval()
    model64 = copy.deepcopy(model).double()
    g_torch = [None if t is None else t.double() for t in _model_grads(model, x, sample, False, monkeypatch)]
    before = N.launch_count()
    K.TIMELINE = []
    try:
        g_native = [None if t is None else t.double() for t in _model_grads(model, x, sample, True, monkeypatch)]
        torch.cuda.synchronize()
        tags = {t[0] for t in K.TIMELINE}
    finally:
        K.TIMELINE = None
    assert N.launch_count() > before and tags_wanted <= tags, tags
    g64 = [None if t is None else t.double() for t in _model_grads(model64, x.double(), sample, False, monkeypatch)]
    _sandwich(g_native, g_torch, g64, tags_wanted)


PLANES = {"rqs_planes", "rqs_planes_backward"}
SHARED = {"rqs_shared_backward"}

MODEL_CASES = {
    "glow_rq": (lambda: MODELS.glow_rq(image_shape=(3, 16, 16)), (3, 16, 16), False, PLANES),
    "glow_rq_sample": (lambda: MODELS.glow_rq(image_shape=(3, 16, 16)), (3 * 16 * 16,), True, PLANES),
    "nsf_uncond_linear": (lambda: MODELS.nsf_uncond("linear", features=16, hidden=32, bins=8), (16,), False, SHARED),
    "nsf_uncond_none": (lambda: MODELS.nsf_uncond(None, features=16, hidden=32, bins=8), (16,), False, SHARED),
    "image_uncond": (lambda: MODELS.image_uncond(channels=4, size=8), (4, 8, 8), False, PLANES | SHARED),
}


@pytest.mark.parametrize("name", sorted(MODEL_CASES))
def test_model_gradients_against_fp64(cuda_device, name, monkeypatch):
    make, shape, sample, tags = MODEL_CASES[name]
    torch.manual_seed(3)
    model = make()
    from nflows_b200.flows import recipes
    recipes.perturb_(model)
    model = model.to(cuda_device)
    torch.manual_seed(1)
    x = torch.randn(64, *shape) if name != "nsf_uncond_none" else torch.rand(64, *shape)
    _check_model(model, x.to(cuda_device), sample, tags, monkeypatch)


@pytest.mark.parametrize("key", ["glow_rq", "image_uncond", "nsf_uncond_linear", "nsf_uncond_none", "nsf_uncond_sample"])
def test_golden_models_against_fp64(cuda_device, key, monkeypatch):
    rec = load_golden("spline_training_grads")[key]
    model = MODELS.golden_flow(key, rec).to(cuda_device)
    sample = MODELS.GOLDEN_BUILDERS[key][1]
    tags = (PLANES if key.startswith(("glow", "image")) else set()) | (SHARED if "uncond" in key else set())
    _check_model(model, rec["x"].to(cuda_device), sample, tags, monkeypatch)


def test_sgd_run_against_fp64(cuda_device, monkeypatch):
    """20 SGD steps of the small Glow-RQ from one initialisation on the same batches: the parameter changes pass the sandwich.
    Convolutions in exact fp32, the recipe's own initialisation and a step small enough that 20 steps stay near the linear regime:
    with cuDNN's default TF32, the perturbed weights and lr 1e-3 (the loss sums 768 dimensions) the trajectories are chaotic, and
    even the two torch-only runs (fp32 against fp64) end 4e-2 apart, so the comparison measured the chaos, not the spline."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    torch.manual_seed(4)
    base = MODELS.glow_rq(image_shape=(3, 16, 16)).eval()
    runs = {}
    for key, dtype, native in (("native", torch.float32, True), ("torch", torch.float32, False), ("fp64", torch.float64, False)):
        monkeypatch.setattr(config, "native_training", native)
        model = copy.deepcopy(base).to(device=cuda_device, dtype=dtype)
        opt = torch.optim.SGD(model.parameters(), lr=1e-4)
        g = torch.Generator().manual_seed(0)
        for _ in range(20):
            x = torch.randn(64, 3, 16, 16, generator=g).to(device=cuda_device, dtype=dtype)
            opt.zero_grad()
            (-model.log_prob(x).mean()).backward()
            opt.step()
        runs[key] = [p.detach().double().clone() for p in model.parameters()]
    init = [p.detach().double().to(cuda_device) for p in base.parameters()]
    delta = lambda r: [a - b for a, b in zip(r, init)]
    _sandwich(delta(runs["native"]), delta(runs["torch"]), delta(runs["fp64"]), "sgd")


def test_switch_off_launches_nothing(cuda_device, monkeypatch):
    monkeypatch.setattr(config, "native_training", False)
    for make, shape, sample, _ in MODEL_CASES.values():
        model = make().to(cuda_device)
        x = torch.rand(8, *shape, device=cuda_device)
        before = N.launch_count()
        MODELS.grads(model, x, sample)
        torch.cuda.synchronize()
        assert N.launch_count() == before
    cdf = T.PiecewiseRationalQuadraticCDF(shape=[3, 4], num_bins=8, tails="linear", tail_bound=3.0).to(cuda_device)
    before = N.launch_count()
    cdf(torch.randn(5, 3, 4, device=cuda_device))[1].sum().backward()
    assert N.launch_count() == before
