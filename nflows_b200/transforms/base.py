"""Transform protocol, composition and the native execution chain.

Public contract = reference nflows/transforms/base.py:10-60, 215-231: a Transform maps
``(inputs, context) -> (outputs, logabsdet[B])`` and has an ``inverse`` with the same signature.

H100-native addition: transforms that own CUDA kernels implement ``_native_apply(x, lad, flags, inverse)``
which enqueues kernels on the current stream, read-modify-writes the running ``lad`` buffer (so
``CompositeTransform`` never materialises per-transform log-dets, unlike ``_cascade`` at base.py:44-52) and
returns the output tensor.  Inputs that are not (CUDA, fp32, 2-D, no autograd) take the differentiable
torch path ``_eager`` -- that is the device-agnostic/training path of the API, never a substitute for the
kernels on CUDA inference."""
import numpy as np
import torch
from torch import nn

from .. import config
from .. import kernels as K
from ..utils import typechecks as check


class InverseNotAvailable(Exception):
    """Raised by transforms that have no inverse."""


class InputOutsideDomain(Exception):
    """Raised when an input is outside the domain of a transform (e.g. a constrained spline)."""


def params_frozen(module):
    """True when running `module` cannot need a backward pass."""
    return not torch.is_grad_enabled() or not any(p.requires_grad for p in module.parameters())


class Transform(nn.Module):
    """Base class of all transforms."""

    def forward(self, inputs, context=None):
        return self._run(inputs, context, inverse=False)

    def inverse(self, inputs, context=None):
        return self._run(inputs, context, inverse=True)

    def train(self, mode=True):
        # derived-weight caches are keyed on tensor versions, which writes through `.data` do not bump: a mode switch (what
        # follows an EMA weight swap) invalidates them (see nflows_b200.invalidate_native_caches)
        config.cache_epoch += 1
        return super().train(mode)

    # -- subclass hooks ---------------------------------------------------------------------------------
    def _eager(self, inputs, context, inverse):
        if inverse:
            raise InverseNotAvailable()
        raise NotImplementedError()

    def _native_ready(self, inputs, context):
        return False

    def _native_apply(self, inputs, lad, flags, inverse, context=None):
        raise NotImplementedError()

    # -- dispatch ---------------------------------------------------------------------------------------
    def _run(self, inputs, context, inverse):
        if torch.is_tensor(inputs) and self._native_ready(inputs, context):
            with K.on_device_of(inputs):
                x = inputs if inputs.stride(-1) == 1 else inputs.contiguous()

                def attempt():
                    lad = K.zeros_lad(x)
                    flags = K.new_flags(x.device)
                    return self._native_apply(x, lad, flags, inverse, context), lad, flags

                out, lad = K.run_with_activation_rescale(attempt)
            return out, lad
        K.warn_eager_cuda(inputs)
        return self._eager(inputs, context, inverse)


def _pixel_row_head(coupling):
    """True when a coupling over channels runs on pixel rows: no unconditional transform, a ConvResidualNet that gives a
    dense.ConvChain, and a head on a fused final-layer route (RQ: the spline kernels; affine / additive:
    nfk_affine_coupling_final_f16x3).  Route "rows" -- hidden channels not a multiple of 8, config.fuse_coupling off, an
    affine scale activation without a code -- keeps the torch path."""
    from .. import dense as D
    net = coupling.transform_net
    with D.image_geometry(1, 2, 2):
        chain = net.dense_chain(None) if (coupling.unconditional_transform is None and hasattr(net, "dense_chain")) else None
        return isinstance(chain, D.ConvChain) and coupling._native_head(chain).route != "rows"


def _flatten(transform, inverse, out):
    """Leaves of nested CompositeTransforms / InverseTransforms in execution order, as (leaf, inverse)."""
    if isinstance(transform, CompositeTransform):
        children = list(transform._transforms)
        for child in (reversed(children) if inverse else children):
            _flatten(child, inverse, out)
    elif isinstance(transform, InverseTransform):
        _flatten(transform._transform, not inverse, out)
    else:
        out.append((transform, inverse))
    return out


class CompositeTransform(Transform):
    """Applies transforms in the order given (reference base.py:32-60)."""

    def __init__(self, transforms):
        super().__init__()
        self._transforms = nn.ModuleList(transforms)

    def _eager(self, inputs, context, inverse):
        children = list(self._transforms)
        outputs = inputs
        total = inputs.new_zeros(inputs.shape[0])
        for t in (reversed(children) if inverse else children):
            outputs, lad = t.inverse(outputs, context) if inverse else t(outputs, context)
            total += lad
        return outputs, total

    def _native_ready(self, inputs, context):
        if not (K.native_ok(inputs, context) and params_frozen(self)):
            return False
        return inputs.dim() == 2 or (inputs.dim() == 4 and self._image_ready(inputs, context))

    # ---- image chains: [B, C, H, W] inputs run as PIXEL ROWS [B*H*W, C] through the 2-D machinery ---------------------------
    def _image_ready(self, inputs, context):
        """Every leaf has a per-pixel form: ActNorm, OneByOneConvolution, SqueezeTransform(2) and RQ, affine or additive couplings
        over channels with a ConvResidualNet the dense path can run (SURVEY.md section 8 row f3, BASELINE cfg 5).  Anything else:
        torch path for the whole chain."""
        from .. import dense as D
        from .conv import OneByOneConvolution
        from .coupling import AdditiveCouplingTransform, AffineCouplingTransform, PiecewiseRationalQuadraticCouplingTransform
        from .normalization import ActNorm
        from .reshape import SqueezeTransform
        if context is not None or D.backend() != "tc":
            return False
        b, c, h, w = inputs.shape
        for leaf, _ in _flatten(self, False, []):
            if type(leaf) is SqueezeTransform:
                if leaf.factor != 2:
                    return False
            elif type(leaf) is ActNorm:
                if leaf.training and not bool(leaf.initialized):
                    return False
            elif type(leaf) is OneByOneConvolution:
                pass
            elif type(leaf) is PiecewiseRationalQuadraticCouplingTransform:
                if not _pixel_row_head(leaf):
                    return False
            elif type(leaf) in (AffineCouplingTransform, AdditiveCouplingTransform):
                # a scale activation the kernel computes (additive: none), at least one transformed channel (the fused final
                # kernel takes d_t >= 1)
                if not (leaf._native_epilogue_supported() and leaf.num_transform_features > 0 and _pixel_row_head(leaf)):
                    return False
            else:
                return False
        return True

    def _native_apply_image(self, inputs, lad, flags, inverse):
        """Layout change at the ends, SqueezeTransforms as row gathers, everything between them as a 2-D chain on the pixel rows
        with a per-PIXEL log|det| buffer that is folded into the per-sample one (sum over H, W) whenever the pixel grid changes."""
        from .. import dense as D
        from .reshape import SqueezeTransform
        b, c, h, w = inputs.shape
        rows = K.nchw_to_rows(inputs)
        segment = []

        def flush(rows):
            if not segment:
                return rows
            lad_pix = K.fill_(torch.empty(b * h * w, dtype=torch.float32, device=rows.device), 0.0)
            with D.image_geometry(b, h, w):
                rows = self._run_leaves(list(segment), rows, lad_pix, flags, None)
            K.segment_sum_(lad_pix, lad, h * w)
            segment.clear()
            return rows

        for leaf, inv in _flatten(self, inverse, []):
            if type(leaf) is SqueezeTransform:
                rows = flush(rows)
                rows, (c, h, w) = K.squeeze_rows(rows, b, c, h, w, inverse=inv)
            else:
                segment.append((leaf, inv))
        rows = flush(rows)
        return K.rows_to_nchw(rows, b, c, h, w)

    def _native_apply(self, inputs, lad, flags, inverse, context=None):
        if inputs.dim() == 4:
            return self._native_apply_image(inputs, lad, flags, inverse)
        return self._run_leaves(_flatten(self, inverse, []), inputs, lad, flags, context)

    def _run_leaves(self, leaves, inputs, lad, flags, context=None):
        """Walks the flattened leaves.  Between leaves the tensor may live in a permuted COLUMN LAYOUT (fused_affine.Layout):
        a coupling that runs on the fused tensor-core path asks for its identity features first / transformed features
        last; the folded affine run in front of it emits that order for free (a row permutation of its weight matrix) and
        the run behind it absorbs it (a column permutation), so the flow state is never gathered, scattered or copied
        between layers.  Leaves that know nothing about layouts always see the logical column order."""
        from .fused_affine import AffineRun, is_affine_leaf

        x = inputs
        layout = None            # None = logical column order
        owned = False            # x is a temporary of this chain (may be overwritten in place)
        carry = {"pair": None}   # fp16 split pair of x (kernels.Pair16) when the producing kernel wrote one
        i = 0

        def wanted(k):
            if k >= len(leaves):
                return None
            fn = getattr(leaves[k][0], "_native_layout", None)
            return fn(x, context) if fn is not None else None

        def affine_run(k):
            """(end, holds an LU-type leaf) of the run of per-feature affine / permutation / LU leaves starting at k."""
            j, has_lu = k, False
            while j < len(leaves) and is_affine_leaf(leaves[j][0], x):
                has_lu = has_lu or leaves[j][0].__class__.__name__ in ("LULinear", "OneByOneConvolution")
                j += 1
            return j, has_lu

        while i < len(leaves):
            leaf, inv = leaves[i]
            # fold a run of per-feature affine / permutation / LU transforms into ONE dense layer
            j, has_lu = affine_run(i)
            if has_lu:
                from .. import dense as D
                run = AffineRun.cached(leaves[i:j], x.device, conv_pixels=D.current_geometry() is not None)
                out_layout = wanted(j)
                pair_cols = leaves[j][0].num_identity_features if out_layout is not None else 0
                # the fp32 values of the identity block are never read when the coupling behind this run hands ONLY the fp16 pair
                # of its output to another folded affine run (coupling._native_packed: pair_only) -- then they are not written
                y_first_col = pair_cols if out_layout is not None and pair_cols % 8 == 0 and affine_run(j + 1)[1] else 0
                x, pair = run.apply(x, lad, layout, out_layout, x_pair=carry["pair"], pair_cols=pair_cols, flags=flags,
                                    y_first_col=y_first_col)
                carry["pair"] = pair
                layout, owned = out_layout, True
                i = j
                continue
            want = wanted(i) if leaf._native_ready(x, context) else None
            if layout is not None and layout is not want:
                x = K.gather_cols(x, layout.cols(x.device, inverse=True))       # back to the logical order
                layout, owned, carry["pair"] = None, True, None
            if want is not None and layout is None:
                x = K.gather_cols(x, want.cols(x.device))
                layout, owned, carry["pair"] = want, True, None
            if layout is not None:
                # does a folded affine run consume this leaf's output?  Then only the fp16 pair of it is ever read.
                carry["pair_only"] = affine_run(i + 1)[1]
                x = leaf._native_apply(x, lad, flags, inv, context, layout=layout, owned=owned, carry=carry)
                carry["pair_only"] = False
                owned = True
            elif leaf._native_ready(x, context):
                x = leaf._native_apply(x, lad, flags, inv, context)
                owned, carry["pair"] = True, None
            else:
                carry["pair"] = None
                x, l = leaf.inverse(x, context) if inv else leaf(x, context)
                lad += l
                if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 2):
                    raise RuntimeError("{} changed the tensor layout inside a native chain".format(type(leaf).__name__))
                x = x.contiguous()
                owned = True
            i += 1
        if layout is not None:
            x = K.gather_cols(x, layout.cols(x.device, inverse=True))
        return x


class InverseTransform(Transform):
    """Swaps forward and inverse of a transform (reference base.py:215-231)."""

    def __init__(self, transform):
        super().__init__()
        self._transform = transform

    def forward(self, inputs, context=None):
        return self._transform.inverse(inputs, context)

    def inverse(self, inputs, context=None):
        return self._transform(inputs, context)


class MultiscaleCompositeTransform(Transform):
    """Multiscale architecture of RealNVP (reference base.py:63-212): after every transform but the last,
    half of the current tensor (along ``split_dim``) is emitted and the other half carried on.  Forward
    returns the flat concatenation of everything emitted.  Executed with torch views around the child
    transforms (which run natively where they can)."""

    def __init__(self, num_transforms, split_dim=1):
        if not check.is_positive_int(num_transforms):
            raise TypeError("Number of transforms must be a positive integer.")
        if not check.is_positive_int(split_dim):
            raise TypeError("Split dimension must be a positive integer.")
        super().__init__()
        self._transforms = nn.ModuleList()
        self._output_shapes = []
        self._num_transforms = num_transforms
        self._split_dim = split_dim

    def add_transform(self, transform, transform_output_shape):
        """Registers the next transform; returns the shape its carried-on half will have, or None for the last."""
        assert len(self._transforms) <= self._num_transforms
        if len(self._transforms) == self._num_transforms:
            raise RuntimeError("Adding more than {} transforms is not allowed.".format(self._num_transforms))
        if (self._split_dim - 1) >= len(transform_output_shape):
            raise ValueError("No split_dim in output shape")
        if transform_output_shape[self._split_dim - 1] < 2:
            raise ValueError("Size of dimension {} must be at least 2.".format(self._split_dim))
        self._transforms.append(transform)
        if len(self._transforms) == self._num_transforms:
            self._output_shapes.append(tuple(transform_output_shape))
            return None
        shape = list(transform_output_shape)
        emitted = list(shape)
        emitted[self._split_dim - 1] = (shape[self._split_dim - 1] + 1) // 2
        carried = list(shape)
        carried[self._split_dim - 1] = shape[self._split_dim - 1] // 2
        self._output_shapes.append(tuple(emitted))
        return tuple(carried)

    def forward(self, inputs, context=None):
        if self._split_dim >= inputs.dim():
            raise ValueError("No split_dim in inputs.")
        if self._num_transforms != len(self._transforms):
            raise RuntimeError("Expecting exactly {} transform(s) to be added.".format(self._num_transforms))
        batch = inputs.shape[0]
        total = inputs.new_zeros(batch)
        pieces = []
        carried = inputs
        for k, t in enumerate(self._transforms):
            out, lad = t(carried, context)
            total += lad
            if k < self._num_transforms - 1:
                emitted, carried = torch.chunk(out, chunks=2, dim=self._split_dim)
                assert emitted.shape[1:] == self._output_shapes[k]
            else:
                emitted = out
            pieces.append(emitted.reshape(batch, -1))
        return torch.cat(pieces, dim=-1), total

    def inverse(self, inputs, context=None):
        if inputs.dim() != 2:
            raise ValueError("Expecting NxD inputs")
        if self._num_transforms != len(self._transforms):
            raise RuntimeError("Expecting exactly {} transform(s) to be added.".format(self._num_transforms))
        batch = inputs.shape[0]
        sizes = [int(np.prod(s)) for s in self._output_shapes]
        chunks = torch.split(inputs, sizes, dim=1)
        pieces = [c.reshape(batch, *s) for c, s in zip(chunks, self._output_shapes)]
        total = inputs.new_zeros(batch)
        carried, lad = self._transforms[-1].inverse(pieces[-1], context)
        total += lad
        for t, piece in zip(reversed(list(self._transforms)[:-1]), reversed(pieces[:-1])):
            carried, lad = t.inverse(torch.cat([piece, carried], dim=self._split_dim), context)
            total += lad
        return carried, total
