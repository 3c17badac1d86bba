"""Pin the CPU oracle (oracle/flow_oracle.py) against outputs of the real reference.

The fixtures in tests/golden were produced by oracle/make_golden.py, which imports the unmodified
reference (a checkout of bayesiains/nflows).  Same ATen kernels, same order => expected bit-exact; asserted at
1e-6 relative (and exact equality for pure indexing)."""
import torch

from conftest import load_golden, rel_err
from oracle import flow_oracle as O

TOL = 1e-6


def test_searchsorted_known_answer():
    g = load_golden("searchsorted")
    for row, want in zip(g["inputs"], g["idx"]):
        got = O.searchsorted(g["bin_locations"].repeat(9, 1), row)
        assert torch.equal(got, want)
    # reference tests/utils/torchutils_test.py:80-90: left edges and midpoints map to arange(9)
    assert torch.equal(g["idx"][0], torch.arange(9))
    assert torch.equal(g["idx"][2], torch.arange(9))


def test_spline_function_vectors():
    g = load_golden("spline")
    for inv in (False, True):
        y, l = O.rq_spline_unconstrained(g["x_tails"].clone(), g["uw"].clone(), g["uh"].clone(), g["ud_tails"].clone(),
                                         inverse=inv, tail_bound=g["tail_bound"])
        wy, wl = g["tails_inv%d" % inv]
        assert rel_err(y, wy) <= TOL and rel_err(l, wl) <= TOL
        y, l = O.rq_spline(g["x_constrained"].clone(), g["uw"].clone(), g["uh"].clone(), g["ud_constrained"].clone(), inverse=inv)
        wy, wl = g["constrained_inv%d" % inv]
        assert rel_err(y, wy) <= TOL and rel_err(l, wl) <= TOL
        y, l = O.rq_spline(g["x_constrained"].clone() * 4 - 1, g["uw"].clone(), g["uh"].clone(), g["ud_constrained"].clone(),
                           inverse=inv, left=-1.0, right=3.0, bottom=-1.0, top=3.0, min_bin_width=1e-2, min_bin_height=2e-2,
                           min_derivative=5e-2)
        wy, wl = g["constrained_box_inv%d" % inv]
        assert rel_err(y, wy) <= TOL and rel_err(l, wl) <= TOL


def test_cfg1_affine_flow():
    g = load_golden("cfg1_affine")
    spec = [("affine_coupling", "_transform._transforms.%d." % i, {}) for i in range(2)]
    z, lad = O.composite(g["sd"], spec, g["x"])
    assert rel_err(z, g["z"]) <= TOL and rel_err(lad, g["lad"]) <= TOL
    assert rel_err(O.flow_log_prob(g["sd"], spec, g["x"]), g["log_prob"]) <= TOL
    xr, ladr = O.composite(g["sd"], spec, g["z"], inverse=True)
    assert rel_err(xr, g["x_roundtrip"]) <= TOL and rel_err(ladr, g["lad_inverse"]) <= TOL


def test_affine_variants():
    g = load_golden("affine_variants")
    y, l = O.affine_coupling(g["sd_general"], "", g["x"], scale_activation="general")
    assert rel_err(y, g["y_general"]) <= TOL and rel_err(l, g["lad_general"]) <= TOL
    y, l = O.affine_coupling(g["sd_general"], "", g["x"], inverse=True, scale_activation="general")
    assert rel_err(y, g["xinv_general"]) <= TOL and rel_err(l, g["ladinv_general"]) <= TOL
    y, l = O.affine_coupling(g["sd_additive"], "", g["x"], additive=True)
    assert rel_err(y, g["y_additive"]) <= TOL and torch.equal(l, g["lad_additive"])
    assert torch.equal(l, torch.zeros_like(l))


def test_cfg2_rq_coupling():
    g = load_golden("cfg2_rq_coupling")
    sd = {k: v.clone() for k, v in g["sd"].items()}
    kw = dict(num_bins=8, tails="linear", tail_bound=3.0)
    for suffix in ("", "_x3"):
        if suffix:
            for k in sd:
                if "final_layer" in k:
                    sd[k] = sd[k] * 3.0
        y, l = O.rq_coupling(sd, "", g["x"], **kw)
        assert rel_err(y, g["y" + suffix]) <= TOL and rel_err(l, g["lad" + suffix]) <= TOL
        # identity half is bit-exact (reference tests/transforms/coupling_test.py:50)
        idf = sd["identity_features"]
        assert torch.equal(y[:, idf], g["x"][:, idf])
        y, l = O.rq_coupling(sd, "", g["x"], inverse=True, **kw)
        assert rel_err(y, g["xinv" + suffix]) <= TOL and rel_err(l, g["ladinv" + suffix]) <= TOL


def test_rq_coupling_constrained():
    g = load_golden("rq_coupling_constrained")
    kw = dict(num_bins=5, tails=None, min_bin_width=2e-3, min_bin_height=3e-3, min_derivative=4e-3)
    y, l = O.rq_coupling(g["sd"], "", g["x"], **kw)
    assert rel_err(y, g["y"]) <= TOL and rel_err(l, g["lad"]) <= TOL
    y, l = O.rq_coupling(g["sd"], "", g["x"], inverse=True, **kw)
    assert rel_err(y, g["xinv"]) <= TOL and rel_err(l, g["ladinv"]) <= TOL


def test_linear_transforms():
    g = load_golden("linear_transforms")
    for name, fn, sd in (("actnorm", O.actnorm, g["sd_actnorm"]), ("lu", O.lu_linear, g["sd_lu"]),
                         ("perm", O.permutation, g["sd_perm"])):
        y, l = fn(sd, "", g["x"])
        assert rel_err(y, g[name + "_y"]) <= TOL and rel_err(l, g[name + "_lad"]) <= TOL
        y, l = fn(sd, "", g["x"], inverse=True)
        assert rel_err(y, g[name + "_xinv"]) <= TOL and rel_err(l, g[name + "_ladinv"]) <= TOL
    y, _ = O.permutation(g["sd_perm"], "", g["x"])
    assert torch.equal(y, g["x"][:, g["sd_perm"]["_permutation"]])
    lower, upper, diag = O.lu_factors(g["sd_lu"], "")
    assert rel_err(lower @ upper, g["lu_weight"]) <= TOL
    assert rel_err(torch.sum(torch.log(diag)), g["lu_logabsdet"]) <= TOL


def test_nsf_small_flow():
    g = load_golden("nsf_small")
    spec = O.nsf_spec(g["layers"])
    z, lad = O.composite(g["sd"], spec, g["x"], inverse=False)
    assert rel_err(z, g["z"]) <= TOL and rel_err(lad, g["lad"]) <= TOL
    assert rel_err(O.flow_log_prob(g["sd"], spec, g["x"]), g["log_prob"]) <= TOL
    xs, lads = O.composite(g["sd"], [(k, p.replace("_transform._transforms", "_transform._transforms"), kw) for k, p, kw in spec],
                           g["noise"], inverse=True)
    assert rel_err(xs, g["sample"]) <= TOL and rel_err(lads, g["lad_inverse"]) <= TOL
    assert rel_err(O.flow_log_prob_chunked(g["sd"], spec, g["x"], chunk=100), g["log_prob"]) <= TOL


def test_autoregressive_rq_small():
    g = load_golden("ar_rq_small")
    y, l = O.ar_rq(g["sd"], "", g["x"], num_bins=4, tails=None)
    assert rel_err(y, g["y"]) <= TOL and rel_err(l, g["lad"]) <= TOL
    xi, li = O.ar_rq(g["sd"], "", g["x"], num_bins=4, tails=None, inverse=True)
    assert rel_err(xi, g["xinv"]) <= TOL and rel_err(li, g["ladinv"]) <= TOL
