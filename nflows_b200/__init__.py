"""nflows_b200: H100-native (sm_90a) implementation of the nflows coupling-flow hot path.

Drop-in for `nflows.transforms.Transform / CompositeTransform`, the coupling / ActNorm / LULinear /
Permutation transforms, `Flow.log_prob / sample` and `StandardNormal` -- same class names, constructor
kwargs, state_dict keys and exceptions -- with CUDA fp32 inference executed by hand-written kernels in
libnfk_sm90.so (C ABI: include/nfk.h)."""
__version__ = "0.1.0"

import os as _os


class _Config:
    #: read the device flag word after each public call and raise the reference's exceptions
    #: (InputOutsideDomain / AssertionError).  Costs one device->host sync per call.
    check_domain = True
    #: upper bound (MiB) for the conditioner-output chunk a coupling keeps in flight; bounds the temporaries
    param_chunk_mib = 64
    #: run the final conditioner layer and the spline as ONE tensor-core kernel when an instance exists
    fuse_coupling = True
    #: run conditioner trunk + final layer + spline of an RQ coupling as ONE kernel (nfk_rq_coupling_step_f16x3);
    #: NFLOWS_B200_STEP_KERNEL=0 falls back to the round-1 launch sequence (one GEMM per trunk layer + fused final layer)
    coupling_step_kernel = _os.environ.get("NFLOWS_B200_STEP_KERNEL", "1") == "1"
    #: power-of-two exponent applied to activations before they are split into fp16 (hi, lo) pairs for the tensor-core
    #: dense layers: |a| * 2^exp must stay below 65000 (an overflow raises kernels.Float16RangeError) and |a| >= 2^-(3+exp)
    #: keeps the full 22-bit precision; 6 covers 2e-3 .. 1000
    activation_exp = 6
    #: when a call trips the fp16 range flag, run it again with a smaller activation exponent (steps of 5, down to -24:
    #: |a| up to 1e12) instead of raising -- the reference accepts any finite fp32 input; needs check_domain (the flag read)
    auto_activation_exp = True
    #: rows per sub-block of a dense-layer chain: bounds the temporaries of a sub-block (split pairs, hidden activations);
    #: small sub-blocks pay prologue and launch overhead per one-wave launch
    trunk_block_rows = 1 << 19
    affine_block_rows = 1 << 19
    #: rows per (trunk, fused final layer + spline) round of a coupling on the fused path
    coupling_block_rows = 1 << 19
    #: run the conditioners added to the native path on top of the relu ones on the kernels: the activations tanh, ELU,
    #: leaky-ReLU, GELU and SiLU (dense.activation_code), feed-forward MADE blocks (use_residual_blocks=False) and masked affine
    #: autoregressive transforms whose hidden width is zero padded to a multiple of 32 (sbi's 50).  Off, they keep the torch
    #: formulation, the reference's line for line, as they always have; NFLOWS_B200_NATIVE_ACTIVATIONS=1 turns it on
    native_activations = _os.environ.get("NFLOWS_B200_NATIVE_ACTIVATIONS", "0") == "1"


    #: bumped by invalidate_native_caches(); part of every derived-weight cache signature
    cache_epoch = 0


config = _Config()


def invalidate_native_caches():
    """Rebuild every operand the native path derives from parameters on its next use (fp16 split pairs, packed final layers,
    step plans, masked, padded and degree-sorted MADE weights, folded ActNorm/Permutation/LU operands, index tensors).  Each is
    cached on the module or tensor it comes from (dense.derived) and validated by the (data_ptr, version, device, shape) of its
    source tensors: writes through `param.data` (EMA swaps, old-style optimisers) do not bump the version counter, so call this
    after such writes -- `module.train()` / `.eval()` on any transform does it for you."""
    config.cache_epoch += 1
