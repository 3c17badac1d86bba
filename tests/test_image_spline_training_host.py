"""Training of image RQ couplings and of PiecewiseRationalQuadraticCDF with the spline on the kernels, without a GPU: the package's
torch path against the reference's gradients (tests/golden/spline_training_grads.pt); RQSplinePlanes and RQSplineShared with CPU
stand-ins of nfk_rqs_planes, nfk_rqs_planes_backward, nfk_rqs_elementwise and nfk_rqs_shared_backward that restate their
contracts on the host build of the per-element spline source (tests/rqs_vjp_host.cpp) against fp64 autograd; the routing; and the
argument checks of the new entry points."""
import ctypes

import pytest
import torch

import _spline_cases as S
import _spline_training_models as MODELS
from conftest import load_golden
from nflows_b200 import _native as N
from nflows_b200 import config
from nflows_b200 import kernels as K
from nflows_b200 import transforms as T
from nflows_b200.transforms.splines import training
from oracle import flow_oracle as O
from test_spline_training_host import _null, autograd_vjp, host_forward, host_lib, host_vjp  # noqa: F401  (host_lib: fixture)


@pytest.fixture(scope="module")
def gold():
    return load_golden("spline_training_grads")


# ---- the torch path against the reference ---------------------------------------------------------------------------------
@pytest.mark.parametrize("key", sorted(MODELS.GOLDEN_BUILDERS))
def test_torch_path_reproduces_the_reference_gradients(gold, key):
    rec = gold[key]
    flow = MODELS.golden_flow(key, rec)
    assert abs(MODELS.weight_checksum(flow.state_dict()) - rec["checksum"]) <= 1e-9 * rec["checksum"]
    got, value = MODELS.grads(flow, rec["x"], MODELS.GOLDEN_BUILDERS[key][1])
    assert abs(float(value) - float(rec["loss"])) <= 1e-5 * max(1.0, abs(float(rec["loss"])))
    assert sorted(got) == sorted(rec["grads"])
    for name, g in got.items():
        want = rec["grads"][name]
        assert float((g - want).norm()) <= 1e-4 * max(float(want.norm()), 1e-6), (key, name)


# ---- CPU stand-ins of the kernels -----------------------------------------------------------------------------------------
def _to_rows(x, params, m):
    """Plane layout -> one element per row: x [n, c, h, w] -> [n*c*h*w], params [n, c*m, h, w] -> [n*c*h*w, m]."""
    n, c, h, w = x.shape
    return x.reshape(-1), params.reshape(n, c, m, h * w).permute(0, 1, 3, 2).reshape(-1, m)


def _from_rows(gp, n, c, h, w, m):
    return gp.reshape(n, c, h * w, m).permute(0, 1, 3, 2).reshape(n, c * m, h, w)


def _m(desc):
    return 3 * desc.num_bins - 1 if desc.linear_tails else 3 * desc.num_bins + 1


def _shared_params(uw, uh, ud, rows, desc):
    """Per-element parameter rows [rows * F, M] of batch-shared uw, uh [F, K], ud [F, nd]."""
    p = torch.cat([uw, uh, ud], -1)
    return p[None].expand(rows, *p.shape).reshape(-1, p.shape[-1])


@pytest.fixture
def stand_ins(host_lib, monkeypatch):
    calls = {"rqs_planes": 0, "rqs_planes_backward": 0, "rqs_elementwise": 0, "rqs_shared_backward": 0, "grad_x": [],
             "cotangents": []}

    def rqs_planes(desc, inverse, x, params, lad_accum, flags):
        assert x.is_contiguous() and params.is_contiguous()
        calls["rqs_planes"] += 1
        n, c, h, w = x.shape
        xr, pr = _to_rows(x, params, _m(desc))
        y, lad, f = host_forward(host_lib, desc, inverse, xr, pr)
        flags |= f
        lad_accum += lad.reshape(n, -1).sum(1)
        return y.reshape(x.shape)

    def rqs_planes_backward(desc, inverse, x, params, grad_y, grad_lad, want_grad_x=True):
        calls["rqs_planes_backward"] += 1
        calls["grad_x"].append(want_grad_x)
        calls["cotangents"].append((grad_y is not None, grad_lad is not None))
        n, c, h, w = x.shape
        gy = torch.zeros_like(x) if grad_y is None else grad_y
        gl = torch.zeros(n) if grad_lad is None else grad_lad
        xr, pr = _to_rows(x, params, _m(desc))
        gx, gp = host_vjp(host_lib, desc, inverse, xr, pr, gy.reshape(-1), gl[:, None].expand(n, c * h * w).reshape(-1))
        return (gx.reshape(x.shape) if want_grad_x else None), _from_rows(gp, n, c, h, w, _m(desc))

    def rqs_elementwise(desc, inverse, x, uw, uh, ud, param_period=0, flags=None):
        calls["rqs_elementwise"] += 1
        n, f = x.shape
        assert param_period == f
        y, lad, fl = host_forward(host_lib, desc, inverse, x.reshape(-1), _shared_params(uw, uh, ud, n, desc))
        flags |= fl
        return y.reshape(n, f), lad.reshape(n, f)

    def segment_sum_(values, out_accum, segment_len):
        out_accum += values.reshape(-1, segment_len).sum(1)
        return out_accum

    def rqs_shared_backward(desc, inverse, x, uw, uh, ud, grad_y, grad_lad, want_grad_x=True):
        calls["rqs_shared_backward"] += 1
        calls["grad_x"].append(want_grad_x)
        calls["cotangents"].append((grad_y is not None, grad_lad is not None))
        n, f = x.shape
        k = desc.num_bins
        gy = torch.zeros_like(x) if grad_y is None else grad_y
        gl = torch.zeros(n) if grad_lad is None else grad_lad
        gx, gp = host_vjp(host_lib, desc, inverse, x.reshape(-1), _shared_params(uw, uh, ud, n, desc), gy.reshape(-1),
                          gl[:, None].expand(n, f).reshape(-1))
        gp = gp.double().reshape(n, f, -1).sum(0).float()                 # the batch sum the kernel's two passes form
        return (gx.reshape(n, f) if want_grad_x else None), gp[:, :k], gp[:, k:2 * k], gp[:, 2 * k:]

    for name, fn in dict(rqs_planes=rqs_planes, rqs_planes_backward=rqs_planes_backward, rqs_elementwise=rqs_elementwise,
                         segment_sum_=segment_sum_, rqs_shared_backward=rqs_shared_backward, on_device_of=lambda t: _null(),
                         new_flags=lambda device: torch.zeros(1, dtype=torch.int32), zeros_lad=lambda x: torch.zeros(x.shape[0]),
                         raise_for_flags=lambda flags: K.raise_for_flag_value(int(flags))).items():
        monkeypatch.setattr(K, name, fn)
    monkeypatch.setattr(training, "_cuda_fp32", lambda t: t.dtype == torch.float32)
    monkeypatch.setattr(config, "native_training", True)
    return calls


def _planes_case(n=6, c=3, h=2, w=5, bins=8, tails="linear", seed=0):
    g = torch.Generator().manual_seed(seed)
    m = 3 * bins - 1 if tails == "linear" else 3 * bins + 1
    x = torch.randn(n, c, h, w, generator=g) * 2 if tails else torch.rand(n, c, h, w, generator=g)
    params = torch.randn(n, c * m, h, w, generator=g)
    return x, params, m


def _close(got, want, what):
    assert float((got.double() - want).abs().max()) <= 1e-3 * max(1.0, float(want.abs().max())), what


@pytest.mark.parametrize("tails", ["linear", None])
@pytest.mark.parametrize("inverse", [False, True])
def test_planes_function_matches_torch_autograd(stand_ins, tails, inverse):
    bins = 5
    x, params, m = _planes_case(bins=bins, tails=tails)
    if inverse:
        x = x * 0.999
    xs, ps = x.clone().requires_grad_(True), params.clone().requires_grad_(True)
    y, lad = training.rq_spline_planes(xs, ps, inverse, bins, tails, S.TAIL_BOUND, 1e-3, 1e-3, 1e-3, 4.0)
    assert y.shape == x.shape and lad.shape == (x.shape[0],)
    n, c, h, w = x.shape
    xr, pr = _to_rows(x, params, m)
    uw, uh, ud = pr[:, :bins], pr[:, bins:2 * bins], pr[:, 2 * bins:]
    gy, gl = torch.randn_like(y), torch.randn_like(lad)
    for cot in ((gy, None), (None, gl), (gy, gl)):
        xs.grad, ps.grad = None, None
        loss = sum((t * g).sum() for t, g in ((y, cot[0]), (lad, cot[1])) if g is not None)
        loss.backward(retain_graph=True)
        cy = torch.zeros_like(y) if cot[0] is None else cot[0]
        cl = torch.zeros(n) if cot[1] is None else cot[1]
        tx, tp = autograd_vjp(xr, uw, uh, ud, cy.reshape(-1), cl[:, None].expand(n, c * h * w).reshape(-1), tails, inverse,
                              torch.float64, 4.0)
        _close(xs.grad.reshape(-1), tx, (tails, inverse, "g_x"))
        _close(ps.grad, _from_rows(tp, n, c, h, w, m), (tails, inverse, "g_params"))
    assert stand_ins["rqs_planes"] == 1 and stand_ins["rqs_planes_backward"] == 3
    assert stand_ins["cotangents"] == [(True, False), (False, True), (True, True)]   # None cotangents reach the kernel as NULL


@pytest.mark.parametrize("tails", ["linear", None])
@pytest.mark.parametrize("inverse", [False, True])
@pytest.mark.parametrize("shape", [(7,), (2, 3, 4)])
def test_shared_function_matches_torch_autograd(stand_ins, tails, inverse, shape):
    torch.manual_seed(len(shape) + 2 * inverse)
    cdf = T.PiecewiseRationalQuadraticCDF(shape=list(shape), num_bins=6, tails=tails, tail_bound=S.TAIL_BOUND)
    n = 9
    x = torch.randn(n, *shape) * 2 if tails else torch.rand(n, *shape)
    if inverse:
        x = x * 0.999
    xs = x.clone().requires_grad_(True)
    y, lad = (cdf.inverse if inverse else cdf)(xs)
    assert y.shape == x.shape and lad.shape == (n,)
    gy, gl = torch.randn_like(y), torch.randn_like(lad)
    ((y * gy).sum() + (lad * gl).sum()).backward()
    f = x[0].numel()
    flat = lambda p: p.detach().reshape(f, p.shape[-1])
    uw, uh, ud = flat(cdf.unnormalized_widths), flat(cdf.unnormalized_heights), flat(cdf.unnormalized_derivatives)
    rows = lambda p: p[None].expand(n, *p.shape).reshape(n * f, -1)
    tx, tp = autograd_vjp(x.reshape(-1), rows(uw), rows(uh), rows(ud), gy.reshape(-1), gl[:, None].expand(n, f).reshape(-1),
                          tails, inverse, torch.float64, 1.0)
    tp = tp.reshape(n, f, -1).sum(0)
    _close(xs.grad.reshape(-1), tx, "g_x")
    _close(cdf.unnormalized_widths.grad.reshape(f, -1), tp[:, :6], "g_w")
    _close(cdf.unnormalized_heights.grad.reshape(f, -1), tp[:, 6:12], "g_h")
    _close(cdf.unnormalized_derivatives.grad.reshape(f, -1), tp[:, 12:], "g_d")
    assert stand_ins["rqs_elementwise"] == 1 and stand_ins["rqs_shared_backward"] == 1


def test_functions_respect_needs_input_grad_and_refuse_double_backward(stand_ins):
    x, params, _ = _planes_case()
    ps = params.clone().requires_grad_(True)
    y, lad = training.rq_spline_planes(x, ps, False, 8, "linear", S.TAIL_BOUND, 1e-3, 1e-3, 1e-3, None)
    (y.sum() + lad.sum()).backward()
    assert stand_ins["grad_x"] == [False] and ps.grad is not None and x.grad is None
    xs = x.clone().requires_grad_(True)
    y, lad = training.rq_spline_planes(xs, params, False, 8, "linear", S.TAIL_BOUND, 1e-3, 1e-3, 1e-3, None)
    gx, = torch.autograd.grad(lad.sum(), xs, create_graph=True)
    with pytest.raises(RuntimeError):
        gx.sum().backward()                      # once_differentiable: no double backward

    cdf = T.PiecewiseRationalQuadraticCDF(shape=[4], num_bins=4, tails="linear", tail_bound=S.TAIL_BOUND)
    cdf.unnormalized_heights.requires_grad_(False)
    xc = torch.randn(5, 4)
    y, lad = cdf(xc)
    lad.sum().backward()
    assert stand_ins["grad_x"][-1] is False and cdf.unnormalized_heights.grad is None
    assert cdf.unnormalized_widths.grad is not None and cdf.unnormalized_derivatives.grad is not None
    xs = torch.randn(5, 4, requires_grad=True)
    y, lad = cdf(xs)
    gx, = torch.autograd.grad(lad.sum(), xs, create_graph=True)
    with pytest.raises(RuntimeError):
        gx.sum().backward()


def test_functions_raise_the_reference_domain_error(stand_ins):
    x, params, _ = _planes_case(tails=None)
    x[0, 0, 0, 0] = 1.5
    with pytest.raises(T.InputOutsideDomain):
        training.rq_spline_planes(x, params.requires_grad_(True), False, 8, None, 1.0, 1e-3, 1e-3, 1e-3, None)
    cdf = T.PiecewiseRationalQuadraticCDF(shape=[3], num_bins=4)
    with pytest.raises(T.InputOutsideDomain):
        cdf(torch.tensor([[0.5, 1.5, 0.2]]))


# ---- routing -----------------------------------------------------------------------------------------------------------------
def test_image_coupling_routes_and_matches_torch(stand_ins, monkeypatch):
    torch.manual_seed(0)
    flow = MODELS.image_uncond(channels=4, size=4)
    x = torch.randn(3, 4, 4, 4)
    grads_native, loss_native = MODELS.grads(flow, x, False)
    assert stand_ins["rqs_planes"] == 1 and stand_ins["rqs_planes_backward"] == 1
    assert stand_ins["rqs_elementwise"] == 1 and stand_ins["rqs_shared_backward"] == 1
    noise = torch.randn(3, 64)
    MODELS.grads(flow, noise, True)                                  # the sampling direction: the inverses route as well
    assert stand_ins["rqs_planes"] == 2 and stand_ins["rqs_elementwise"] == 2
    monkeypatch.setattr(config, "native_training", False)
    grads_torch, loss_torch = MODELS.grads(flow, x, False)
    assert stand_ins["rqs_planes"] == 2 and stand_ins["rqs_elementwise"] == 2
    assert abs(float(loss_native - loss_torch)) <= 1e-4 * max(1.0, abs(float(loss_torch)))
    for name, g in grads_torch.items():
        assert float((grads_native[name] - g).abs().max()) <= 1e-3 * max(1.0, float(g.abs().max())), name


@pytest.mark.parametrize("tails", ["linear", None])
def test_2d_coupling_with_unconditional_transform_routes(stand_ins, tails):
    torch.manual_seed(1)
    flow = MODELS.nsf_uncond(tails)
    x = torch.randn(8, 6) if tails else torch.rand(8, 6)
    MODELS.grads(flow, x, False)
    assert stand_ins["rqs_elementwise"] == 2 and stand_ins["rqs_shared_backward"] == 2
    assert stand_ins["rqs_planes"] == 0


def test_routing_gates(stand_ins, monkeypatch):
    x, params, m = _planes_case()
    p = params.clone().requires_grad_(True)
    assert training.routed_planes(x, p, 8, "linear")
    assert not training.routed(x, p, 8, "linear")                              # the row gate keeps its semantics
    assert not training.routed_planes(x, params, 8, "linear")                  # no gradient to compute
    with torch.no_grad():
        assert not training.routed_planes(x, p, 8, "linear")
    assert not training.routed_planes(x[0], p[0], 8, "linear")                 # 3-D
    assert not training.routed_planes(x, p[:, :-1], 8, "linear")               # wrong parameter width
    assert not training.routed_planes(x.double(), p.double(), 8, "linear")
    wide = torch.randn(x.shape[0], x.shape[1] * (3 * 65 - 1), *x.shape[2:], requires_grad=True)
    assert not training.routed_planes(x, wide, 65, "linear")
    assert not training.routed_planes(x, p, 8, "circular")
    cdf = T.PiecewiseRationalQuadraticCDF(shape=[2, 3], num_bins=8, tails="linear", tail_bound=3.0)
    prm = (cdf.unnormalized_widths, cdf.unnormalized_heights, cdf.unnormalized_derivatives)
    xc = torch.randn(5, 2, 3)
    assert training.routed_shared(xc, *prm, "linear")
    assert training.routed_shared(torch.randn(5, 6), *(q.reshape(6, -1) for q in prm), "linear")
    assert not training.routed_shared(torch.randn(5, 3, 2), *prm, "linear")    # shape mismatch
    assert not training.routed_shared(xc.double(), *(q.double() for q in prm), "linear")
    assert not training.routed_shared(xc, *prm, "circular")
    big = T.PiecewiseRationalQuadraticCDF(shape=[2, 3], num_bins=65, tails="linear")
    assert not training.routed_shared(xc, big.unnormalized_widths, big.unnormalized_heights, big.unnormalized_derivatives,
                                      "linear")
    with torch.no_grad():
        assert not training.routed_shared(xc, *prm, "linear")
    monkeypatch.setattr(training, "_cuda_fp32", lambda t: t.is_cuda and t.dtype == torch.float32)
    assert not training.routed_planes(x, p, 8, "linear") and not training.routed_shared(xc, *prm, "linear")   # CPU stays torch
    monkeypatch.setattr(training, "_cuda_fp32", lambda t: t.dtype == torch.float32)
    monkeypatch.setattr(config, "native_training", False)
    assert not training.routed_planes(x, p, 8, "linear") and not training.routed_shared(xc, *prm, "linear")


def test_models_that_stay_torch_launch_nothing(stand_ins, monkeypatch):
    """A mismatched CDF shape, circular tails, fp64, K = 65 and the switch off keep the torch formulation."""
    torch.manual_seed(2)
    cdf = T.PiecewiseRationalQuadraticCDF(shape=[3], num_bins=4, tails="linear", tail_bound=3.0)
    with pytest.raises(Exception):
        cdf(torch.randn(4, 5))                                                  # the torch path's own shape error
    big = T.PiecewiseRationalQuadraticCDF(shape=[3], num_bins=65, tails="linear", tail_bound=3.0, min_bin_width=1e-4,
                                          min_bin_height=1e-4)
    big(torch.randn(4, 3))[1].sum().backward()
    cdf64 = T.PiecewiseRationalQuadraticCDF(shape=[3], num_bins=4, tails="linear", tail_bound=3.0).double()
    cdf64(torch.randn(4, 3, dtype=torch.float64))[1].sum().backward()
    flow = MODELS.image_uncond(channels=4, size=4).double()
    MODELS.grads(flow, torch.randn(2, 4, 4, 4, dtype=torch.float64), False)
    monkeypatch.setattr(config, "native_training", False)
    flow = MODELS.image_uncond(channels=4, size=4)
    MODELS.grads(flow, torch.randn(2, 4, 4, 4), False)
    MODELS.grads(MODELS.nsf_uncond(None), torch.rand(4, 6), False)
    assert stand_ins["rqs_planes"] == stand_ins["rqs_elementwise"] == 0
    assert stand_ins["rqs_planes_backward"] == stand_ins["rqs_shared_backward"] == 0


# ---- argument checks of the entry points (no device needed: nothing is launched) ----------------------------------------------
def test_new_entry_points_reject_bad_arguments_before_launch():
    lib = N.load()
    desc = N.spline_desc(8, "linear", 3.0, 0, 1, 0, 1, 1e-3, 1e-3, 1e-3)
    m = 23
    # nfk_rqs_planes: desc, inv, x, ldx, params, ldp, c_t, pixels, y, ldy, lad, n, flags, stream
    f = lib.nfk_rqs_planes
    ok = [ctypes.byref(desc), 0, 16, 12, 4096, 12 * m, 3, 4, 8192, 12, 0, 10, 0, None]
    for i, v, msg in ((2, None, "NULL tensor"), (4, None, "NULL tensor"), (8, None, "NULL tensor"), (6, 0, "bad sizes"),
                      (7, 0, "bad sizes"), (11, -1, "bad sizes"), (3, 11, "strides"), (9, 11, "strides"), (5, 12 * m - 1, "strides"),
                      (8, 16, "alias"), (8, 4096, "alias"), (7, 1 << 26, "32-bit")):
        args = list(ok)
        args[i] = v
        assert f(*args) == -1 and msg.encode() in lib.nfk_last_error(), (i, v, lib.nfk_last_error())
    assert f(*ok[:11], 0, None, None) == 0                                     # no samples: nothing to do
    # nfk_rqs_planes_backward: desc, inv, x, ldx, params, ldp, gy, ldgy, gl, gx, ldgx, gp, ldgp, c_t, pixels, n, stream
    f = lib.nfk_rqs_planes_backward
    ok = [ctypes.byref(desc), 0, 16, 12, 4096, 12 * m, 64, 12, 128, 256, 12, 8192, 12 * m, 3, 4, 10, None]
    for i, v, msg in ((2, None, "NULL tensor"), (4, None, "NULL tensor"), (11, None, "NULL tensor"), (13, 0, "bad sizes"),
                      (15, -1, "bad sizes"), (3, 11, "strides"), (7, 11, "strides"), (10, 11, "strides"), (12, 12 * m - 1, "strides"),
                      (11, 4096, "alias"), (9, 16, "alias"), (9, 64, "alias")):
        args = list(ok)
        args[i] = v
        assert f(*args) == -1 and msg.encode() in lib.nfk_last_error(), (i, v, lib.nfk_last_error())
    args = list(ok)
    args[6], args[7] = None, 0                                                  # NULL grad_y: its stride is not checked
    args[15] = 0
    assert f(*args) == 0
    # nfk_rqs_shared_backward: desc, inv, x, uw, uh, ud, gy, gl, gx, guw, guh, gud, F, n, ws, ws_bytes, stream
    f = lib.nfk_rqs_shared_backward
    F, n = 5, 100
    need = lib.nfk_rqs_shared_backward_workspace(n, F, 8, 1)
    assert need == ((n + 15) // 16) * F * (2 * 8 + 7) * 4                      # 16-row slabs: far below 2^17 (slab, feature) pairs
    assert lib.nfk_rqs_shared_backward_workspace(1 << 20, 32, 8, 1) == (1 << 20) // 256 * 32 * 23 * 4
    base = 1 << 20
    ok = [ctypes.byref(desc), 0, base, base + 4096, base + 8192, base + 12288, base + 16384, base + 20480, base + 24576,
          base + 65536, base + 69632, base + 73728, F, n, base + (1 << 18), need, None]
    for i, v, msg in ((2, None, "NULL tensor"), (3, None, "NULL parameter"), (9, None, "NULL parameter"), (12, 0, "bad sizes"),
                      (13, -1, "bad sizes"), (14, None, "workspace"), (15, need - 4, "workspace"), (8, base, "alias"),
                      (9, base + 4096, "alias"), (10, base + 65536, "alias"), (11, base + (1 << 18), "alias")):
        args = list(ok)
        args[i] = v
        assert f(*args) == -1 and msg.encode() in lib.nfk_last_error(), (i, v, lib.nfk_last_error())
    bad = N.spline_desc(8, "linear", 3.0, 0, 1, 0, 1, 1e-3, 1e-3, 1e-3)
    bad.num_bins = 65
    for fn, args in ((lib.nfk_rqs_shared_backward, ok), (lib.nfk_rqs_planes_backward, None)):
        if args is not None:
            assert fn(ctypes.byref(bad), *args[1:]) == -1
    one = N.spline_desc(1, "linear", 3.0, 0, 1, 0, 1, 1e-3, 1e-3, 1e-3)      # K = 1 with tails: no derivative logits, NULL ud ok
    args = list(ok)
    args[0], args[5], args[11], args[15] = ctypes.byref(one), None, None, 1 << 30
    args[13] = -1
    assert f(*args) == -1 and b"bad sizes" in lib.nfk_last_error()
