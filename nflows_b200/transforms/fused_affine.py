"""Folding of consecutive ActNorm / Permutation / LULinear transforms into ONE dense layer.

Each of these is an affine map of the feature vector (normalization.py:171-204, permutations.py:27-45,
lu.py:56-91), so a run of them is y = A x + c with a batch-constant log|det|.  A and c are composed on the
host in float64 from the transforms' parameters (tiny: D x D) and rounded once to fp32; the run then costs a
single `nfk_linear` launch instead of one elementwise pass + one gather pass + two GEMMs, and the operand
rounding is no worse than the reference's chain of fp32 ops.  Folded weights are cached on the run's first leaf and
rebuilt when any parameter changes (tensor version counters)."""
import numpy as np
import torch

from .. import dense as D
from .. import kernels as K


class Layout:
    """Physical column order of the tensor between two leaves: physical column j holds logical feature perm[j]."""

    def __init__(self, perm):
        self.perm = np.asarray(perm, dtype=np.int64)
        self.inv = np.argsort(self.perm, kind="stable")
        self._dev = {}

    def cols(self, device, inverse=False):
        """int32 gather index on `device`: logical -> physical (x_phys = x[:, cols]) or, inverse, physical -> logical."""
        key = (str(device), inverse)
        t = self._dev.get(key)
        if t is None:
            t = torch.from_numpy((self.inv if inverse else self.perm).astype(np.int32)).to(device)
            self._dev[key] = t
        return t


def is_affine_leaf(leaf, x):
    from .conv import OneByOneConvolution
    from .lu import LULinear
    from .normalization import ActNorm
    from .permutations import Permutation, RandomPermutation, ReversePermutation

    # exact types (and RandomPermutation / ReversePermutation, which only choose the index vector): a subclass that overrides
    # forward / inverse -- OneByOneConvolution(LULinear) with its own permutation and 4-D check, user subclasses -- is not
    # the plain affine map that gets folded
    if type(leaf) is ActNorm:
        return x.dim() == 2 and not (leaf.training and not bool(leaf.initialized))
    if type(leaf) in (Permutation, RandomPermutation, ReversePermutation):
        return leaf._dim == 1
    if type(leaf) is OneByOneConvolution:
        # on pixel rows (native image chain, dense.image_geometry) Glow's 1x1 convolution IS a channel permutation followed by
        # an LULinear of every row (conv.py:17-29 of the reference)
        return D.current_geometry() is not None and x.dim() == 2
    return type(leaf) is LULinear


class AffineRun:
    def __init__(self, leaves, device, conv_pixels=False):
        """conv_pixels: an OneByOneConvolution leaf stands for the whole 1x1 convolution on pixel rows (its channel
        permutation AND its LU map -- native image chains); otherwise it is the bare LULinear it inherits from (its own
        forward applies the permutation around the call, conv.py)."""
        from .lu import LULinear
        from .normalization import ActNorm

        d = None
        for leaf, _ in leaves:
            d = getattr(leaf, "features", None) or d
            if isinstance(leaf, ActNorm):
                d = leaf.log_scale.numel()
        if d is None:
            d = leaves[0][0]._permutation.numel()
        A = np.eye(d, dtype=np.float64)
        c = np.zeros(d, dtype=np.float64)
        lad = 0.0
        from .conv import OneByOneConvolution

        def permute(A, c, leaf, inv):
            perm = leaf._permutation.detach().cpu().numpy()
            if inv:
                perm = np.argsort(perm, kind="stable")
            return A[perm, :], c[perm]

        for leaf, inv in leaves:
            if conv_pixels and isinstance(leaf, OneByOneConvolution) and not inv:      # forward: its own permutation first
                A, c = permute(A, c, leaf.permutation, False)
            if isinstance(leaf, ActNorm):
                log_s = leaf.log_scale.detach().double().cpu().numpy()
                t = leaf.shift.detach().double().cpu().numpy()
                s = np.exp(log_s)
                if inv:
                    A = A / s[:, None]
                    c = (c - t) / s
                    lad -= log_s.sum()
                else:
                    A = A * s[:, None]
                    c = s * c + t
                    lad += log_s.sum()
            elif isinstance(leaf, LULinear):
                lower, upper, diag = leaf._dense_factors_f64()
                b = leaf.bias.detach().double().cpu().numpy()
                if inv:
                    import scipy.linalg as sl
                    rhs = np.concatenate([A, (c - b)[:, None]], axis=1)
                    rhs = sl.solve_triangular(lower, rhs, lower=True, unit_diagonal=True)
                    rhs = sl.solve_triangular(upper, rhs, lower=False)
                    A, c = rhs[:, :-1], rhs[:, -1]
                    lad -= np.log(diag).sum()
                else:
                    A = lower @ (upper @ A)
                    c = lower @ (upper @ c) + b
                    lad += np.log(diag).sum()
            else:  # Permutation
                A, c = permute(A, c, leaf, inv)
            if conv_pixels and isinstance(leaf, OneByOneConvolution) and inv:          # inverse: LU^-1, then the permutation's inverse
                A, c = permute(A, c, leaf.permutation, True)
        self._A, self._c, self._device = A, c, device
        self._operands = {}
        self.weight, self.bias = self.operands(None, None)
        self.lad_const = float(lad)

    def operands(self, in_layout, out_layout):
        """(weight, bias) acting on a tensor stored in `in_layout` and producing `out_layout`: rows of A follow the output
        order, columns the input order (entries are only moved, so the rounding to fp32 is the same as unpermuted)."""
        key = (id(in_layout), id(out_layout))
        hit = self._operands.get(key)
        if hit is None:
            A, c = self._A, self._c
            if out_layout is not None:
                A, c = A[out_layout.perm, :], c[out_layout.perm]
            if in_layout is not None:
                A = A[:, in_layout.perm]
            hit = (torch.from_numpy(np.ascontiguousarray(A)).float().to(self._device),
                   torch.from_numpy(np.ascontiguousarray(c)).float().to(self._device), in_layout, out_layout)
            self._operands[key] = hit
        return hit[0], hit[1]

    @classmethod
    def cached(cls, leaves, device, conv_pixels=False):
        """The run of `leaves` [(leaf, inverse)], cached on its first leaf until a parameter or buffer of a leaf changes."""
        first, inv = leaves[0]
        return D.derived(first, "_inverse_affine_run" if inv else "_affine_run",
                         [t for leaf, _ in leaves for t in (*leaf.parameters(), *leaf.buffers())],
                         lambda: cls(leaves, device, conv_pixels),
                         extra=(tuple((id(leaf), i) for leaf, i in leaves[1:]), device, conv_pixels))

    def apply(self, x, lad, in_layout=None, out_layout=None, x_pair=None, pair_cols=0, flags=None, y_first_col=0):
        """Returns (y, Pair16 of y's first pair_cols columns or None).  y_first_col: see dense.affine_map."""
        weight, bias = self.operands(in_layout, out_layout)
        y, y_pair = D.affine_map(x, weight, bias, x_pair=x_pair, pair_cols=pair_cols, flags=flags, y_first_col=y_first_col)
        if self.lad_const != 0.0:
            K.add_const_(lad, self.lad_const)
        return y, y_pair
