"""LULinear (reference nflows/transforms/lu.py:10-129): W = L U with unit-lower L and upper U whose diagonal is
softplus(unconstrained) + eps, so log|det W| = sum(log diag U) costs O(D)."""
import numpy as np
import torch
from torch import nn
from torch.nn import functional as F
from torch.nn import init

from .. import kernels as K
from .base import params_frozen
from .linear import Linear


class LULinear(Linear):
    def __init__(self, features, using_cache=False, identity_init=True, eps=1e-3):
        super().__init__(features, using_cache)
        self.eps = eps
        self.lower_indices = np.tril_indices(features, k=-1)
        self.upper_indices = np.triu_indices(features, k=1)
        self.diag_indices = np.diag_indices(features)
        n_tri = ((features - 1) * features) // 2
        self.lower_entries = nn.Parameter(torch.zeros(n_tri))
        self.upper_entries = nn.Parameter(torch.zeros(n_tri))
        self.unconstrained_upper_diag = nn.Parameter(torch.zeros(features))
        self._initialize(identity_init)

    def _initialize(self, identity_init):
        init.zeros_(self.bias)
        if identity_init:
            init.zeros_(self.lower_entries)
            init.zeros_(self.upper_entries)
            init.constant_(self.unconstrained_upper_diag, np.log(np.exp(1 - self.eps) - 1))
        else:
            stdv = 1.0 / np.sqrt(self.features)
            init.uniform_(self.lower_entries, -stdv, stdv)
            init.uniform_(self.upper_entries, -stdv, stdv)
            init.uniform_(self.unconstrained_upper_diag, -stdv, stdv)

    # ---- dense factors ------------------------------------------------------------------------------------
    def _create_lower_upper(self):
        n = self.features
        lower = self.lower_entries.new_zeros(n, n)
        lower[self.lower_indices[0], self.lower_indices[1]] = self.lower_entries
        lower[self.diag_indices[0], self.diag_indices[1]] = 1.0
        upper = self.upper_entries.new_zeros(n, n)
        upper[self.upper_indices[0], self.upper_indices[1]] = self.upper_entries
        upper[self.diag_indices[0], self.diag_indices[1]] = self.upper_diag
        return lower, upper

    def _dense_factors_f64(self):
        """(L, U, diag U) as float64 numpy arrays, for host-side weight folding."""
        n = self.features
        lower = np.eye(n, dtype=np.float64)
        lower[self.lower_indices] = self.lower_entries.detach().double().cpu().numpy()
        upper = np.zeros((n, n), dtype=np.float64)
        upper[self.upper_indices] = self.upper_entries.detach().double().cpu().numpy()
        diag = F.softplus(self.unconstrained_upper_diag.detach()).double().cpu().numpy() + self.eps
        upper[self.diag_indices] = diag
        return lower, upper, diag

    @property
    def upper_diag(self):
        return F.softplus(self.unconstrained_upper_diag) + self.eps

    # ---- native: one dense layer with the folded weight (see fused_affine.py) -----------------------------
    def _native_ready(self, inputs, context):
        return K.native_ok(inputs, context) and inputs.dim() == 2 and params_frozen(self)

    def _native_apply(self, inputs, lad, flags, inverse, context=None):
        from .fused_affine import AffineRun
        if inputs.shape[1] != self.features:
            raise ValueError("Expected features = {}, got {}.".format(self.features, inputs.shape[1]))
        return AffineRun.cached([(self, inverse)], inputs.device).apply(inputs, lad, flags=flags)[0]

    # ---- torch path ---------------------------------------------------------------------------------------
    def forward_no_cache(self, inputs):
        lower, upper = self._create_lower_upper()
        outputs = F.linear(F.linear(inputs, upper), lower, self.bias)
        return outputs, self.logabsdet() * inputs.new_ones(outputs.shape[0])

    def inverse_no_cache(self, inputs):
        lower, upper = self._create_lower_upper()
        rhs = (inputs - self.bias).t()
        rhs = torch.linalg.solve_triangular(lower, rhs, upper=False, unitriangular=True)
        outputs = torch.linalg.solve_triangular(upper, rhs, upper=True, unitriangular=False).t()
        return outputs, -self.logabsdet() * inputs.new_ones(outputs.shape[0])

    def weight(self):
        lower, upper = self._create_lower_upper()
        return lower @ upper

    def weight_inverse(self):
        lower, upper = self._create_lower_upper()
        eye = torch.eye(self.features, self.features, device=self.lower_entries.device)
        lower_inv = torch.linalg.solve_triangular(lower, eye, upper=False, unitriangular=True)
        return torch.linalg.solve_triangular(upper, lower_inv, upper=True, unitriangular=False)

    def logabsdet(self):
        return torch.sum(torch.log(self.upper_diag))
