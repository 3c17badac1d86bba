"""Permutation transforms (reference nflows/transforms/permutations.py:9-63).  Indexing is bit-exact."""
import torch

from .. import dense as D
from .. import kernels as K
from ..utils import typechecks as check
from .base import Transform


class Permutation(Transform):
    """outputs = inputs.index_select(dim, permutation); inverse uses argsort(permutation)."""

    def __init__(self, permutation, dim=1):
        if permutation.ndimension() != 1:
            raise ValueError("Permutation must be a 1D tensor.")
        if not check.is_positive_int(dim):
            raise ValueError("dim must be a positive integer.")
        super().__init__()
        self._dim = dim
        self.register_buffer("_permutation", permutation)

    @property
    def _inverse_permutation(self):
        return torch.argsort(self._permutation)

    def _index_i32(self, inverse, device):
        return D.derived(self, "_inverse_index" if inverse else "_index", [self._permutation],
                         lambda: K.index_tensor(self._inverse_permutation if inverse else self._permutation, device),
                         extra=(device,))

    def _check(self, inputs):
        if self._dim >= inputs.ndimension():
            raise ValueError("No dimension {} in inputs.".format(self._dim))
        if inputs.shape[self._dim] != len(self._permutation):
            raise ValueError("Dimension {} in inputs must be of size {}.".format(self._dim, len(self._permutation)))

    def _native_ready(self, inputs, context):
        return K.native_ok(inputs, context) and inputs.dim() == 2 and self._dim == 1

    def _native_apply(self, inputs, lad, flags, inverse, context=None):
        self._check(inputs)
        return K.gather_cols(inputs, self._index_i32(inverse, inputs.device))

    def _eager(self, inputs, context, inverse):
        self._check(inputs)
        perm = self._inverse_permutation if inverse else self._permutation
        return torch.index_select(inputs, self._dim, perm), inputs.new_zeros(inputs.shape[0])


class RandomPermutation(Permutation):
    """A fixed permutation drawn with torch.randperm at construction."""

    def __init__(self, features, dim=1):
        if not check.is_positive_int(features):
            raise ValueError("Number of features must be a positive integer.")
        super().__init__(torch.randperm(features), dim)


class ReversePermutation(Permutation):
    """Reverses the order of the features."""

    def __init__(self, features, dim=1):
        if not check.is_positive_int(features):
            raise ValueError("Number of features must be a positive integer.")
        super().__init__(torch.arange(features - 1, -1, -1), dim)
