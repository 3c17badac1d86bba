"""Shared pieces of the coupling-kernel tests: launch counters, the fp64-sandwich tolerances, the timeline of tagged launches,
and the case table of the shapes the three fused coupling kernels accept (test_coupling_shape_envelope.py runs it on a GPU,
test_coupling_shape_routes.py checks on the CPU that each case takes the route it is meant to exercise)."""
import contextlib
import copy
from collections import namedtuple

import torch

from conftest import rel_err
from nflows_b200 import kernels as K
from nflows_b200 import transforms as T
from nflows_b200.nn.nets import MLP, ResidualNet
from nflows_b200.utils import torchutils
from oracle import flow_oracle as O

TOL = 1e-5
ROWS = (1, 129, 132 * 128 + 1000)          # one row, a ragged second tile, more rows than one launch round of 132 CTAs
SUBSET = 1024                              # rows of a large batch held to the oracle
TAIL_BOUND = 2.5


class step_launches:
    """Counts launches of the coupling-step kernel with a spline (fp32 outputs, pair outputs)."""

    def __init__(self, monkeypatch):
        self.fp32 = self.pair = 0
        inner = K.rq_coupling_step

        def wrapped(plan, a, desc=None, *args, **kw):
            if desc is not None:
                if kw.get("y_pair") is not None:
                    self.pair += 1
                else:
                    self.fp32 += 1
            return inner(plan, a, desc, *args, **kw)

        monkeypatch.setattr(K, "rq_coupling_step", wrapped)


class final_launches:
    """Counts launches of the fused final-layer spline kernel (fp32 outputs, pair outputs)."""

    def __init__(self, monkeypatch):
        self.fp32 = self.pair = 0
        inner = K.rq_coupling_final

        def wrapped(*args, **kw):
            if kw.get("y_pair") is not None:
                self.pair += 1
            else:
                self.fp32 += 1
            return inner(*args, **kw)

        monkeypatch.setattr(K, "rq_coupling_final", wrapped)


@contextlib.contextmanager
def timeline():
    """The tags of the launches kernels.timed brackets inside the block (a list, filled as they run)."""
    tags = []
    K.TIMELINE = []
    try:
        yield tags
    finally:
        tags.extend(t[0] for t in K.TIMELINE)
        K.TIMELINE = None


def sandwich(want, truth):
    """(output, log|det|) tolerances: the fp32 reference's own distance from fp64, with the floors of test_native_parity.py."""
    return max(TOL, 3 * rel_err(want[0], truth[0])), max(3e-5, 5 * rel_err(want[1], truth[1]))


# ---- the case table ---------------------------------------------------------------------------------------------------
# hidden width, conditioner ("res": ResidualNet with `depth` blocks, "mlp": MLP with `depth` hidden layers), identity features
# (first), transformed features (after them), spline instance; kind: "rq" spline, "affine" (default scale), "affine_general",
# "additive".  route / packed: what the CPU part expects of the head (dense.SplineHead / coupling._AffineHead) and of the column
# layout (identity and feature counts multiples of 8: one packed pass; else the gathered trunk input with a t_cols tensor).
Case = namedtuple("Case", "name hidden net depth d_id d_t bins tails kind route packed")


def _rq(name, hidden, net, depth, d_id, d_t, bins, tails, route="step", packed=True):
    return Case(name, hidden, net, depth, d_id, d_t, bins, tails, "rq", route, packed)


# A. the coupling-step kernel (conditioner and spline in one launch).  The bin variant is rotated so that every (bins, tails)
# instance meets a two-chunk trunk width (> 128) at least once.
STEP_CASES = [
    _rq("h32", 32, "res", 1, 8, 8, 16, "linear"),          # smallest width and input; K = 16: 4 column tiles
    _rq("h96", 96, "res", 2, 24, 16, 8, None),            # 3 K-slabs, input narrower than one slab
    _rq("h128", 128, "res", 1, 40, 24, 10, "linear"),     # exactly one full chunk
    _rq("h160a", 160, "res", 2, 16, 24, 4, "linear"),     # two chunks, the second 32 wide
    _rq("h160b", 160, "res", 2, 16, 24, 16, "linear"),
    _rq("h192a", 192, "res", 1, 264, 16, 8, "linear"),    # second chunk 64 wide; input > 256, partial last slab
    _rq("h192b", 192, "res", 1, 264, 16, 8, None),
    _rq("h224a", 224, "res", 3, 16, 8, 10, "linear"),     # second chunk 96 wide
    _rq("h224b", 224, "res", 3, 16, 8, 10, None),
    _rq("h256", 256, "res", 4, 392, 64, 16, None),        # 8 square layers at the maximum width
    _rq("mlp160", 160, "mlp", 9, 16, 16, 4, None),        # MLP layer flags (no skips), 8 square layers
    _rq("mlp64", 64, "mlp", 1, 16, 16, 4, "linear"),      # no square layer (placeholder weight maps)
]

# B. the fused final-layer kernel after the trunk: the widths the step kernel refuses, across every (bins, tails) instance,
# and partial last column tiles on the gathered route (26 and 29 features: not multiples of 8)
FINAL_CASES = [
    _rq("h288a", 288, "res", 1, 16, 24, 4, "linear", "final"),      # first width past 256: 9 slabs, partial sums 4 + 4 + 1
    _rq("h288b", 288, "res", 1, 16, 24, 4, None, "final"),
    _rq("h1000a", 1000, "res", 1, 16, 16, 16, "linear", "final"),   # partial last slab
    _rq("h1000b", 1000, "res", 1, 16, 16, 16, None, "final"),
    _rq("h40", 40, "res", 1, 16, 16, 10, "linear", "final"),        # not multiples of 32
    _rq("h72", 72, "res", 2, 16, 24, 10, None, "final"),
    _rq("h40n8", 40, "res", 1, 16, 16, 8, None, "final"),
    _rq("tile10", 64, "res", 1, 16, 10, 8, "linear", packed=False),  # TF = 4: tiles of 4, 4, 2 features
    _rq("tile13", 160, "res", 2, 16, 13, 4, None, packed=False),     # TF = 8: tiles of 8, 5; two-chunk trunk_step
]
# H = 512, 2 blocks, the cfg-3 coupling's 784 alternating features at K = 8 with tails: 98 column tiles per row block
WIDE_CASE = Case("h512", 512, "res", 2, 392, 392, 8, "linear", "rq", "final", True)

# C. the affine / additive final kernel
AFFINE_CASES = [
    Case("affine784", 256, "res", 2, 392, 392, None, None, "affine", "final", True),      # 784 columns: 7 tiles, last partial
    Case("affine257", 160, "res", 2, 128, 129, None, None, "affine_general", "final", False),   # odd d_t, gathered
    Case("additive271", 512, "res", 2, 136, 135, None, None, "additive", "final", False),      # odd N, layer-by-layer trunk
]

ALL_CASES = STEP_CASES + FINAL_CASES + [WIDE_CASE] + AFFINE_CASES


def build(case, seed):
    """The coupling of a case on the CPU: constructor weights, final layer x 2 (as test_coupling_step_schedule.py)."""
    torch.manual_seed(seed)
    if case.name in ("h512", "affine784"):
        mask = torchutils.create_alternating_binary_mask(case.d_id + case.d_t)
    else:
        mask = torch.cat([-torch.ones(case.d_id), torch.ones(case.d_t)])

    def net(i, o):
        if case.net == "mlp":
            return MLP([i], [o], [case.hidden] * case.depth)
        return ResidualNet(i, o, hidden_features=case.hidden, num_blocks=case.depth)

    if case.kind == "rq":
        t = T.PiecewiseRationalQuadraticCouplingTransform(mask, net, num_bins=case.bins, tails=case.tails,
                                                          tail_bound=TAIL_BOUND)
    elif case.kind == "additive":
        t = T.AdditiveCouplingTransform(mask, net)
    else:
        act = T.AffineCouplingTransform.GENERAL_SCALE_ACTIVATION if case.kind == "affine_general" else \
            T.AffineCouplingTransform.DEFAULT_SCALE_ACTIVATION
        t = T.AffineCouplingTransform(mask, net, scale_activation=act)
    t = t.eval()
    with torch.no_grad():
        for name, p in t.named_parameters():
            if "final_layer" in name or "_output_layer" in name:
                p.mul_(2.0)
    return t


def inputs(case, n, seed):
    g = torch.Generator().manual_seed(seed)
    d = case.d_id + case.d_t
    if case.kind == "rq" and case.tails is None:
        return torch.rand(n, d, generator=g)
    return torch.randn(n, d, generator=g) * 1.3


def reference(case, t):
    """ref(x, inverse) -> ((y, lad) in fp32, (y, lad) in fp64) on the CPU, for the coupling t (still on the CPU).
    ResidualNet conditioners: oracle/flow_oracle.py; MLP conditioners (no oracle function): the module's own torch path."""
    if case.net == "mlp":
        m32, m64 = copy.deepcopy(t).cpu(), copy.deepcopy(t).cpu().double()

        def ref(x, inverse):
            with torch.no_grad():
                return (m32.inverse(x) if inverse else m32(x)), (m64.inverse(x.double()) if inverse else m64(x.double()))
        return ref
    sd = {k: v.detach().cpu().clone() for k, v in t.state_dict().items()}
    sd64 = {k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}
    if case.kind == "rq":
        fn, kw = O.rq_coupling, dict(num_bins=case.bins, tails=case.tails, tail_bound=TAIL_BOUND)
    else:
        fn = O.affine_coupling
        kw = dict(additive=case.kind == "additive", scale_activation="general" if case.kind == "affine_general" else "default")

    def ref(x, inverse):
        return fn(sd, "", x, inverse=inverse, **kw), fn(sd64, "", x.double(), inverse=inverse, **kw)
    return ref


def head_route(t):
    """(route of the coupling's head, packed column layout) as the coupling decides them, on any device."""
    chain = t.transform_net.dense_chain(None)
    packed = t.num_identity_features % 8 == 0 and t.features % 8 == 0
    return t._native_head(chain).route, packed


def expected_tags(case):
    """(tags that must appear in the timeline of one call, tags that must not): the fused kernel the case targets, and, when
    the trunk runs before it, the one-launch trunk exactly when the step kernel takes the conditioner's width."""
    unfused = ("final_linear", "spline_epilogue")
    if case.kind == "rq" and case.route == "step" and case.packed:
        return ("rq_coupling_step",), ("rq_coupling_final", "trunk_step") + unfused
    trunk = "trunk_step" if K.rq_coupling_step_supported(8, "linear", case.hidden, case.d_id, 0) else None
    want = ("affine_coupling_final",) if case.kind != "rq" else ("rq_coupling_final",)
    forbid = ("rq_coupling_step",) + unfused
    return (want + (trunk,), forbid) if trunk else (want, forbid + ("trunk_step",))
