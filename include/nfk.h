/*
 * nfk.h -- C ABI of libnfk_sm90.so: the H100 (sm_90a) kernels behind the nflows coupling-flow hot path.
 *
 * The reference (bayesiains/nflows) has NO native/FFI layer: its operator API is the Python protocol
 * `Transform.forward/inverse(inputs, context) -> (outputs, logabsdet)` (nflows/transforms/base.py:22-29).
 * This header is the boundary a binding for that protocol needs; every entry point cites the reference
 * code it replaces (paths relative to the reference's nflows/ package).  INTEGRATION.md shows the ctypes stub.
 *
 * Conventions
 *   - return 0 on success, a negative NFK_E_* code on failure; nfk_last_error() gives a thread-local message.
 *   - no allocation, no synchronisation, no stream creation inside: every pointer is caller-owned DEVICE
 *     memory (fp32, row-major), kernels are enqueued on `stream` (a cudaStream_t passed as void*).
 *   - `ld*` are row strides in ELEMENTS.  `lad_accum` ([n_rows] fp32) is read-modify-written: the running
 *     sum of log|det J| that CompositeTransform._cascade (transforms/base.py:44-52) keeps, here on device.
 *   - `flags` (device int32, may be NULL) is OR-ed with NFK_FLAG_* bits; the host reads it when it wants the
 *     reference's exceptions (InputOutsideDomain, rational_quadratic.py:81-82; AssertionError, :142).
 *   - column index lists are int32 device arrays.
 */
#ifndef NFK_H_
#define NFK_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NFK_ABI_VERSION 5

#define NFK_OK 0
#define NFK_E_INVALID (-1)   /* bad argument (shape, alignment, unsupported size) */
#define NFK_E_CUDA (-2)      /* CUDA runtime error at launch */
#define NFK_E_UNSUPPORTED (-3)

#define NFK_FLAG_OUTSIDE_DOMAIN 1  /* constrained spline input outside [left,right] */
#define NFK_FLAG_NEG_DISCRIMINANT 2 /* inverse spline: b^2-4ac < 0 */
#define NFK_FLAG_F16_RANGE 4        /* a value left the fp16 range while a split pair was formed (see nfk_linear_f16x3) */

#define NFK_MAX_BINS 64

/* Activation codes of the conditioner layers: the `relu*` arguments of the dense-layer entry points and the activation field
 * of the coupling-step layer flags take one of these (0 and 1 keep their old meaning, "none" and "relu").  Every code maps 0
 * to exactly 0, so zero-padded hidden units stay zero.  fp32, accurate libdevice functions (the library is built without
 * --use_fast_math).  Any other value is NFK_E_INVALID before anything is launched. */
#define NFK_ACT_NONE 0          /* x */
#define NFK_ACT_RELU 1          /* max(x, 0) */
#define NFK_ACT_TANH 2          /* tanhf(x) */
#define NFK_ACT_ELU 3           /* x > 0 ? x : expm1f(x)            (alpha = 1) */
#define NFK_ACT_LEAKY_RELU 4    /* x > 0 ? x : 0.01 x              (negative slope 0.01) */
#define NFK_ACT_GELU 5          /* 0.5 x (1 + erff(x / sqrt(2)))    (exact, not the tanh approximation) */
#define NFK_ACT_SILU 6          /* x / (1 + expf(-x)) */
#define NFK_ACT_COUNT 7

/* Spline hyper-parameters: kwargs of rational_quadratic_spline / unconstrained_rational_quadratic_spline
 * (transforms/splines/rational_quadratic.py:13-25, 66-80). */
typedef struct NfkSplineDesc {
    int32_t num_bins;        /* K */
    int32_t linear_tails;    /* 1: tails="linear" (identity outside [-B,B], boundary derivatives padded, ud has K-1
                                entries); 0: constrained (ud has K+1 entries, domain flag raised outside) */
    double left, right, bottom, top; /* linear_tails: (-B, B, -B, B) */
    double min_bin_width, min_bin_height, min_derivative;
    double softplus_beta;    /* 1.0, or log(2)/(1-min_derivative) when enable_identity_init (:100-104) */
    double wh_divisor;       /* sqrt(hidden_features) applied to widths/heights (coupling.py:554-559); 1.0 = none */
} NfkSplineDesc;

/* ---- library ------------------------------------------------------------------------------------------- */
int nfk_version(void);
const char* nfk_last_error(void);
/* number of kernels this library has enqueued since load (all threads); evidence for bench.py's gpu_launches */
int64_t nfk_launch_count(void);
/* 0 if the current device is compute capability 9.x (sm_90a), else NFK_E_UNSUPPORTED */
int nfk_check_device(void);

/* ---- rational-quadratic spline ------------------------------------------------------------------------- */
/* Elementwise spline = rational_quadratic_spline / unconstrained_... (rational_quadratic.py:13-181) incl.
 * torchutils.searchsorted (utils/torchutils.py:134-136).  Element e reads x[e] and parameter row
 * r = (param_period ? e % param_period : e): uw[r*stride_w + k], uh[r*stride_h + k], ud[r*stride_d + k].
 * Writes y[e], lad[e].  param_period > 0 gives the batch-shared parameters of PiecewiseRationalQuadraticCDF
 * (transforms/nonlinearities.py:386-467). */
int nfk_rqs_elementwise(const NfkSplineDesc* desc, int inverse, const float* x, const float* uw, const float* uh,
                        const float* ud, int64_t stride_w, int64_t stride_h, int64_t stride_d, int64_t param_period,
                        float* y, float* lad, int64_t n_elem, int32_t* flags, void* stream);

/* Coupling epilogue with the conditioner output in HBM = PiecewiseCouplingTransform._coupling_transform +
 * _piecewise_cdf + sum_except_batch + the scatter of CouplingTransform.forward (coupling.py:96-98, 279-293,
 * 549-582).  params is [n_rows, d_t*M] contiguous, column j*M+k = parameter k of transformed feature j,
 * M = 3K-1 (tails) or 3K+1.  Feature j is read from x[n*ldx + t_cols[j]] and written to y[n*ldy + t_cols[j]];
 * the d_id identity columns id_cols are copied bit-exactly.  lad_accum[n] += sum_j lad(n, j). */
int nfk_rqs_rows(const NfkSplineDesc* desc, int inverse, const float* x, int64_t ldx, const float* params,
                 const int32_t* t_cols, int32_t d_t, const int32_t* id_cols, int32_t d_id, float* y, int64_t ldy,
                 float* lad_accum, int64_t n_rows, int32_t* flags, void* stream);

/* ---- dense layers (conditioner ResidualNet/MLP, LULinear, folded ActNorm+Permutation+LU) ------------------ */
/* Y[n, o] = post( sum_k pre(X[n, k]) * W[o, k] + bias[o] ) + R[n, o]
 * with pre = the activation of code relu_in, post = that of relu_out (NFK_ACT_*; 0 none, 1 relu), R optional (NULL).  W is [out, in] row-major exactly as
 * torch.nn.Linear stores it (F.linear: nn/nets/resnet.py:44-49,94-99; transforms/lu.py:65-66).  fp32 accumulate
 * with fp32-equivalent operand precision (see DESIGN.md: SIMT FFMA path, or split-fp16 wgmma path). */
int nfk_linear(const float* X, int64_t ldx, const float* W, int64_t ldw, const float* bias, const float* R,
               int64_t ldr, float* Y, int64_t ldy, int64_t n_rows, int32_t in_features, int32_t out_features,
               int relu_in, int relu_out, void* stream);

/* Tensor-core version of nfk_linear (wgmma f16, TMA-fed, fp32 accumulators in registers) with fp32-equivalent
 * operand precision.  Every operand is a SPLIT PAIR of fp16 tensors with a per-tensor power-of-two scale:
 *     v * 2^exp = v_hi + v_lo,  v_hi = nearest fp16 of v * 2^exp,  v_lo = nearest fp16 of the exact remainder
 * (22 mantissa bits; 4 bytes per element for the pair), and each K-step accumulates a_lo*w_hi + a_hi*w_lo + a_hi*w_hi in
 * fp32; the epilogue multiplies by 2^-(a_exp + w_exp).  Pick exp so that max |v| * 2^exp stays below 65000 and typical
 * values sit well above 2^-3 (weights: max |w| -> 2^14; activations: a fixed exponent such as 6).
 * The epilogue can emit the fp32 result Y and/or, for the first split_cols columns (0 = all), the split pair of Y (of
 * act(Y) when split_relu is an activation code other than 0) with exponent y_exp that the next layer consumes.  y_first_col > 0 says the fp32 result is only needed
 * for columns >= y_first_col (the rest of Y may be left unwritten: a consumer that multiplies the pair never reads it).
 * A pair element that leaves the fp16 range
 * raises NFK_FLAG_F16_RANGE in `flags`.  hi/lo pointers are fp16 device arrays, ld* in ELEMENTS; TMA needs in_features, lda,
 * ldw multiples of 8 and 16-byte aligned bases (nfk_linear_f16x3_supported). */
int nfk_linear_f16x3_supported(int64_t lda, int64_t ldw, int32_t in_features);
int nfk_linear_f16x3(const void* a_hi, const void* a_lo, int64_t lda, int32_t a_exp, const void* w_hi, const void* w_lo,
                     int64_t ldw, int32_t w_exp, const float* bias, const float* R, int64_t ldr, float* Y, int64_t ldy,
                     void* y_hi, void* y_lo, int64_t lds, int32_t y_exp, int32_t split_cols, int32_t y_first_col, int relu_out,
                     int split_relu, int64_t n_rows, int32_t in_features, int32_t out_features, int32_t* flags, void* stream);
/* hi[n, j], lo[n, j] = fp16 split pair of pre(x[n*ldx + j]) * 2^scale_exp, pre = the activation of code `relu` (NFK_ACT_*): weights (once per parameter
 * update), tensors entering a tensor-core chain from outside, the transformed half of a coupling output. */
/* *out = max(*out, max |x[n, j]|) over an n_rows x n_cols matrix (NaNs skipped); *out must be >= 0 on entry.  Used to pick the
 * power-of-two exponent of a weight's split pair. */
int nfk_absmax(const float* x, int64_t ldx, int64_t n_rows, int32_t n_cols, float* out, void* stream);
int nfk_split_f16(const float* x, int64_t ldx, int32_t n_cols, int relu, int32_t scale_exp, void* hi, void* lo, int64_t ldo,
                  int64_t n_rows, int32_t* flags, void* stream);

/* Affine / additive coupling with the LAST conditioner layer fused in (coupling.py:212-269 + the final nn.Linear of the
 * conditioner, nn/nets/resnet.py:99): params = a W^T + bias is formed on the tensor cores (operands as for nfk_linear_f16x3)
 * and consumed in the epilogue's registers -- y_j = x_j * s_j + t_j (inverse: (x_j - t_j) / s_j), lad_accum[n] += +-sum log s_j
 * -- the [n_rows, mult*d_t] parameter tensor is never written.  The weight rows / bias entries must be INTERLEAVED when
 * mult == 2: row 2j = shift of feature j, row 2j+1 = its unconstrained scale (the reference's BLOCKED order is rows j and
 * d_t + j).  scale_activation as nfk_affine_coupling_rows.  Only the transformed columns of y are written (y may alias x).
 * lad_accum is updated with atomicAdd (a row's columns are spread over several threads): the sum order is not fixed. */
int nfk_affine_coupling_final_f16x3(const void* a_hi, const void* a_lo, int64_t lda, int32_t a_exp, const void* w_hi,
                                    const void* w_lo, int64_t ldw, int32_t w_exp, const float* bias, int32_t hidden_features,
                                    const float* x, int64_t ldx, const int32_t* t_cols, int32_t t_col0, int32_t d_t, int32_t mult,
                                    int32_t scale_activation, int inverse, float* y, int64_t ldy, float* lad_accum, int64_t n_rows,
                                    int32_t* flags, void* stream);

/* Context gate + skip connection of a residual block (nn/nets/resnet.py:50-53: `F.glu(cat(temps, context_layer(context)))`
 * then `inputs + temps`):  v = skip + t * sigmoid(gate)  (skip may be NULL).  Writes v as fp32 (y, may be NULL) and / or as the
 * fp16 pair of pre(v) * 2^y_exp (pre = the activation of code split_relu, NFK_ACT_*) that the next dense layer multiplies. */
int nfk_glu_skip_rows(const float* t, int64_t ldt, const float* gate, int64_t ldg, const float* skip, int64_t ldsk, float* y,
                      int64_t ldy, void* y_hi, void* y_lo, int64_t lds, int32_t y_exp, int split_relu, int64_t n_rows,
                      int32_t n_cols, int32_t* flags, void* stream);


/* ---- fused RQ-coupling step ------------------------------------------------------------------------------------ */
/* Final conditioner layer + spline + scatter + log|det| in ONE wgmma kernel: replaces the last F.linear of the
 * conditioner (nn/nets/resnet.py:99), PiecewiseCouplingTransform._coupling_transform / _piecewise_cdf (coupling.py:279-293,
 * 549-582), the spline (splines/rational_quadratic.py:13-181) and the transform-half scatter (coupling.py:98).
 *   a_hi/a_lo  : fp16 split pair (exponent a_exp) of the last hidden activation [n_rows, hidden_features]
 *   wp_hi/wp_lo: fp16 split pair (exponent w_exp) of the PACKED final weight [d_t * MP, hidden_features]: row j*MP + k =
 *                reference row j*M + k for k < M, zero rows for M <= k < MP, MP = nfk_rq_coupling_final_padded_params
 *   bias_packed: fp32, packed the same way, [d_t * MP]
 * Transformed feature j lives in column t_cols[j], or, when t_cols is NULL, in column t_col0 + j (the layout
 * CompositeTransform arranges: no index load in front of every x load).
 * Writes y[n, t_cols[j]] for every transformed feature and adds the row's log|det| to lad_accum.  y may be x itself
 * (in place: the identity columns then need no copy); otherwise the caller fills the identity columns of y.
 * Output: EITHER y (fp32; y_hi = y_lo = NULL) OR, with y = NULL, the fp16 split pair y_hi / y_lo (row pitch lds, exponent y_exp)
 * of the same columns -- what the tensor-core layer that consumes the coupling output next reads (needs t_cols = NULL,
 * t_col0 a multiple of 8); x is left untouched in that mode.
 * nfk_rq_coupling_final_supported says whether an instance exists for (num_bins, tails, hidden_features, lda); otherwise
 * use nfk_linear* + nfk_rqs_rows. */
int nfk_rq_coupling_final_supported(int32_t num_bins, int32_t linear_tails, int32_t hidden_features, int64_t lda);
int32_t nfk_rq_coupling_final_padded_params(int32_t num_bins, int32_t linear_tails);
int nfk_rq_coupling_final_f16x3(const NfkSplineDesc* desc, int inverse, const void* a_hi, const void* a_lo, int64_t lda,
                               int32_t a_exp, const void* wp_hi, const void* wp_lo, int64_t ldw, int32_t w_exp,
                               const float* bias_packed, int32_t hidden_features, const float* x, int64_t ldx,
                               const int32_t* t_cols, int32_t t_col0, int32_t d_t, float* y, int64_t ldy, void* y_hi,
                               void* y_lo, int64_t lds, int32_t y_exp, float* lad_accum, int64_t n_rows, int32_t* flags,
                               void* stream);

/* ---- the whole RQ-coupling step in ONE kernel ----------------------------------------------------------------------- */
/* Conditioner (initial layer, square layers of the residual blocks, final layer) + spline + scatter + log|det| of
 * PiecewiseRationalQuadraticCouplingTransform.forward / inverse (coupling.py:73-99, 105-130, 279-293, 549-582) with a
 * ResidualNet / MLP conditioner (nn/nets/resnet.py:39-55, 92-100; nn/nets/mlp.py) -- one wgmma kernel, no intermediate
 * tensor in global memory but the skip tensor: a CTA keeps the hidden activation of a 128-row tile in shared memory as the
 * fp16 split pair the next layer multiplies and streams only weights.  Same arithmetic as nfk_linear_f16x3 / nfk_rq_coupling_final_f16x3.
 *   a_hi/a_lo   : fp16 split pair (exponent a_exp) of the conditioner input [n_rows, in_features] (the identity features,
 *                 pre-activated if the first layer applies an activation to its input)
 *   w0_hi/w0_lo : pair (w0_exp) of the initial layer's weight [hidden, in_features]
 *   wt_hi/wt_lo : pairs of the num_square_layers hidden x hidden weights stacked row-wise, layer l with exponent wt_exps[l]
 *                 (HOST array); may be NULL when num_square_layers == 0
 *   bias_trunk  : fp32 [(1 + num_square_layers) * hidden]
 *   layer_flags : HOST array [1 + num_square_layers], bits: 1 the activation on the output (acc + bias), 2 add the
 *                 saved skip tensor, 4 save the fp32 output as the skip tensor, 8 the next layer takes the activation of this
 *                 output; bits [8, 12): the activation code (NFK_ACT_*) of bits 1 and 8, where 0 reads as relu (so a word
 *                 without the field means relu); a field above NFK_ACT_SILU is NFK_E_INVALID
 *   act_exp     : exponent of every hidden activation pair
 *   wp_hi/wp_lo, bias_packed, x, t_cols, t_col0, d_t, y | (y_hi, y_lo, y_exp), lad_accum: as nfk_rq_coupling_final_f16x3
 *   h_hi/h_lo   : when non-NULL the kernel stops after the last trunk layer and writes that layer's output pair (exponent
 *                 act_exp, pre-activated per its flag bit 8) here instead of running the final layer + spline
 *   workspace   : nfk_rq_coupling_step_workspace_bytes(hidden) bytes of device scratch (skip tensors, one 128-row tile per CTA) */
typedef struct NfkCouplingStep {
    const NfkSplineDesc* spline;
    int32_t inverse;
    const void* a_hi; const void* a_lo; int64_t lda; int32_t a_exp; int32_t in_features;
    const void* w0_hi; const void* w0_lo; int64_t ldw0; int32_t w0_exp;
    const void* wt_hi; const void* wt_lo; int64_t ldwt; const int32_t* wt_exps;
    const float* bias_trunk; const int32_t* layer_flags; int32_t num_square_layers; int32_t act_exp;
    const void* wp_hi; const void* wp_lo; int64_t ldwp; int32_t wp_exp; const float* bias_packed; int32_t hidden_features;
    const float* x; int64_t ldx; const int32_t* t_cols; int32_t t_col0; int32_t d_t;
    float* y; int64_t ldy; void* y_hi; void* y_lo; int64_t lds; int32_t y_exp;
    void* h_hi; void* h_lo; int64_t ldh;
    float* lad_accum; int64_t n_rows;
    void* workspace; size_t workspace_bytes;
    int32_t* flags;
} NfkCouplingStep;
int nfk_rq_coupling_step_supported(int32_t num_bins, int32_t linear_tails, int32_t hidden_features, int32_t in_features,
                                   int32_t num_square_layers);
size_t nfk_rq_coupling_step_workspace_bytes(int32_t hidden_features);
int nfk_rq_coupling_step_f16x3(const NfkCouplingStep* step, void* stream);

/* nfk_rq_coupling_step_f16x3 with per-row additive terms on trunk layers (the context projections of a conditional MADE,
 * reference transforms/made.py:187-202, 274-283): trunk layer l (0 = initial layer) computes
 *     post(acc + bias + layer[l].add[row * layer[l].ld + col]) (+ skip)
 * i.e. the term enters before the layer's relu, like the bias.  layer[l].add == NULL: no term on layer l.
 *   add : fp32 device memory [n_rows, ld], 8-byte aligned; only rows < n_rows and columns < hidden_features are read
 *   ld  : row pitch in elements, even and >= hidden_features (a sub-network of a wider net may read a column prefix)
 * A term on a layer the descriptor does not have, or together with the trunk-only output (h_hi), is NFK_E_INVALID.
 * nfk_rq_coupling_step_f16x3(step, stream) is this entry point with no terms. */
#define NFK_STEP_MAX_LAYERS 9
typedef struct NfkRowTerm {
    const float* add;
    int64_t ld;
} NfkRowTerm;
typedef struct NfkStepRowTerms {
    NfkRowTerm layer[NFK_STEP_MAX_LAYERS];
} NfkStepRowTerms;
int nfk_rq_coupling_step_terms_f16x3(const NfkCouplingStep* step, const NfkStepRowTerms* terms, void* stream);

/* ---- masked affine autoregressive step ------------------------------------------------------------------------------ */
/* The coupling-step kernel with the affine map of MaskedAffineAutoregressiveTransform in place of the spline (reference
 * transforms/autoregressive.py:96-128; MADE trunk made.py:17-283): for the d_t consecutive features j = t_col0 .. t_col0 + d_t - 1,
 *     (u_j, shift_j) = rows 2j, 2j + 1 of the final layer   (params.view(B, D, 2)[..., 0] and [..., 1]: MADE's order)
 *     scale_j = softplus(u_j) + 1e-3                          (F.softplus, threshold 20)
 *     forward: y_j = scale_j * x_j + shift_j,   lad_accum[n] += sum_j log(scale_j)
 *     inverse: y_j = (x_j - shift_j) / scale_j, lad_accum[n] -= sum_j log(scale_j)
 * Same trunk, row terms (NULL: none) and workspace as nfk_rq_coupling_step_terms_f16x3; step->spline is ignored.
 *   wp_hi/wp_lo, wp_exp : fp16 split pair of the final layer [2 d_t, hidden] exactly in MADE's row order, no padding rows
 *   bias_packed         : its bias [2 d_t], 8-byte aligned
 *   t_cols must be NULL; x and y are fp32 (no pair output, no trunk-only output: h_hi must be NULL); y may not alias x.
 * The autoregressive inverse calls it once per feature i with d_t = 1, t_col0 = i, the two rows of feature i and a trunk of the
 * degree-sorted sub-network feature i sees.  Shapes: those of nfk_rq_coupling_step_supported. */
int nfk_affine_ar_step_f16x3(const NfkCouplingStep* step, const NfkStepRowTerms* terms, void* stream);

/* ---- mixture-of-Gaussians MADE step ------------------------------------------------------------------------------------- */
/* The coupling-step kernel with the mixture density of MixtureOfGaussiansMADE / MADEMoG in place of the spline (reference
 * nn/nde/made.py:284-427, distributions/mixture.py).  Feature j's parameters are rows (j C + c) 3 + k of MADE's final layer
 * (outputs.reshape(B, D, C, 3)), k = 0 logit l_c, 1 mean mu_c, 2 unconstrained std u_c, and sigma_c = softplus(u_c) + epsilon
 * (F.softplus, threshold 20).  For the d_t consecutive features j = t_col0 .. t_col0 + d_t - 1:
 *   NFK_MOG_LOG_PROB (made.py:333-360):  lad_accum[n] += sum_j LSE_c( log_softmax(l)_c
 *                                                         - 0.5 (log 2 pi + 2 log sigma_c + ((x_j - mu_c) / sigma_c)^2) )
 *       log-softmax and logsumexp max-subtracted; the features summed in a fixed order (the same for any row-block split).
 *       Needs x and lad_accum; y, u and e must be NULL.
 *   NFK_MOG_SAMPLE (made.py:362-401, with the draw made explicit):  c* = the smallest c with u_j < sum_{c' <= c} softmax(l)_{c'}
 *       (C - 1 when rounding leaves u_j above the total), y_j = mu_{c*} + sigma_{c*} e_j, fp32.  u_j in [0, 1) and e_j are
 *       read at u[n * ld_noise + j - t_col0] (likewise e).  x is not read (may be NULL); lad_accum must be NULL.  The sampler
 *       calls it once per feature i with d_t = 1, t_col0 = i and a trunk of the degree-sorted sub-network feature i sees.
 * Same trunk, row terms (NULL: none) and workspace as nfk_rq_coupling_step_terms_f16x3; step->spline is ignored.
 *   wp_hi/wp_lo, wp_exp : fp16 split pair of the final layer packed to MP = nfk_mog_made_padded_rows(C) rows per feature (rows
 *                         3C .. MP - 1 zero), [d_t MP, hidden]; 16-byte aligned
 *   bias_packed         : its bias packed the same way [d_t MP], 16-byte aligned
 *   t_cols must be NULL; no pair output and no trunk-only output (y_hi, h_hi NULL).
 * num_components C is 1 .. NFK_MOG_MAX_COMPONENTS: 3C rows per feature fit a 64-row packing, and every packed row count has
 * its own kernel instance (the ptxas register, stack and spill lines of each are in DESIGN.md, section 5.3).
 * nfk_mog_made_padded_rows(C) is roundup(3C, 8), 48 for C = 11 .. 13 (a 96-row column tile), 0 for an unsupported C.
 * Shapes: those of nfk_rq_coupling_step_supported.  Bad arguments return NFK_E_INVALID before anything is launched. */
#define NFK_MOG_MAX_COMPONENTS 21
#define NFK_MOG_LOG_PROB 0
#define NFK_MOG_SAMPLE 1
typedef struct NfkMogArgs {
    int32_t num_components;
    int32_t mode;               /* NFK_MOG_LOG_PROB or NFK_MOG_SAMPLE */
    float epsilon;              /* > 0 */
    const float* u;             /* sample mode: [n_rows, ld_noise] fp32 uniforms in [0, 1) */
    const float* e;             /* sample mode: [n_rows, ld_noise] fp32 standard normals */
    int64_t ld_noise;
} NfkMogArgs;
int32_t nfk_mog_made_padded_rows(int32_t num_components);
int nfk_mog_made_step_f16x3(const NfkCouplingStep* step, const NfkStepRowTerms* terms, const NfkMogArgs* mog, void* stream);

/* ---- row-wise elementwise transforms -------------------------------------------------------------------- */
/* out[n, j] = x[n*ldx + cols[j]] (identity_split gather, coupling.py:82; Permutation._permute,
 * permutations.py:27-39).  Bit-exact copy. */
int nfk_gather_cols(const float* x, int64_t ldx, const int32_t* cols, int32_t n_cols, float* out, int64_t ldo,
                    int64_t n_rows, void* stream);

/* ActNorm (transforms/normalization.py:171-204): forward y = scale[j]*x + shift[j]; inverse y = (x - shift[j]) /
 * scale[j]; scale = exp(log_scale) is computed by the caller.  lad_accum[n] += lad_const (may be NULL/0). */
int nfk_actnorm(const float* x, int64_t ldx, const float* scale, const float* shift, float* y, int64_t ldy,
                float* lad_accum, float lad_const, int64_t n_rows, int32_t d, int inverse, void* stream);

/* lad_accum[n] += c for every row (constant log|det| of LULinear / ActNorm, lu.py:123-129). */
int nfk_add_const(float* lad_accum, float c, int64_t n_rows, void* stream);
int nfk_fill(float* dst, float value, int64_t n, void* stream);

/* Affine / additive coupling epilogue (coupling.py:212-269).  params is [n_rows, mult*d_t] contiguous with the
 * BLOCKED layout shift = params[:, :d_t], raw scale = params[:, d_t:] (mult = 2), or shift only (mult = 1,
 * additive).  scale_activation: 0 = sigmoid(u+2)+1e-3 (DEFAULT), 1 = clamp(softplus(u)+1e-3, 0, 3) (GENERAL). */
int nfk_affine_coupling_rows(const float* x, int64_t ldx, const float* params, int32_t mult, int32_t scale_activation,
                             int inverse, const int32_t* t_cols, int32_t d_t, const int32_t* id_cols, int32_t d_id,
                             float* y, int64_t ldy, float* lad_accum, int64_t n_rows, void* stream);

/* StandardNormal._log_prob + Flow._log_prob's final add (distributions/normal.py:23-33, flows/base.py:49):
 * out[n] = (-0.5 * sum_j z[n, j]^2 - log_z) + (lad ? lad[n] : 0). */
int nfk_std_normal_log_prob(const float* z, int64_t ldz, int32_t d, float log_z, const float* lad, float* out,
                            int64_t n_rows, void* stream);

/* ---- image path: per-pixel form of the 4-D transforms (SURVEY.md section 8 row f3) ------------------------ */
/* Inside a native image chain the tensor is PIXEL ROWS [n_images*H*W, C] fp32 (channels last); the 4-D ActNorm,
 * OneByOneConvolution and channel-wise coupling (normalization.py:178-186, conv.py:17-29, coupling.py:280-285) are then
 * the 2-D entry points above applied to those rows.
 * nfk_nchw_to_rows: x [n_images, channels, pixels] <-> rows [n_images*pixels, channels] (to_nchw = 0: x -> rows, reads
 * `x`, writes `rows`; to_nchw = 1: reads `x` as rows, writes `rows` as NCHW -- the first pointer is always the source). */
int nfk_nchw_to_rows(const float* src, float* dst, int64_t n_images, int32_t channels, int32_t pixels, int to_nchw, void* stream);
/* SqueezeTransform (reshape.py:7-68, factor 2) on pixel rows.  h2 x w2 is the SQUEEZED grid, channels the UNSQUEEZED channel
 * count: forward reads [n*2h2*2w2, channels] and writes [n*h2*w2, 4*channels] with channel c*4 + dy*2 + dx = pixel (dy, dx)
 * of the 2x2 window of channel c; inverse the other way round. */
int nfk_squeeze_rows(const float* in, float* out, int64_t n_images, int32_t h2, int32_t w2, int32_t channels, int inverse,
                     void* stream);
/* K-major operand of a 3x3, padding-1 convolution (nn.Conv2d in ConvResidualBlock, nn/nets/resnet.py:103-160) from the fp16
 * pair of its (already activated) input: out[(b,y,x), (ky*3+kx)*channels + c] = in[(b, y+ky-1, x+kx-1), c], 0 outside the image.
 * The convolution is then nfk_linear_f16x3 with the weight reshaped to [out_channels, 9*channels] in (ky, kx, c) order. */
int nfk_im2col3x3_f16(const void* hi, const void* lo, int64_t lds, void* out_hi, void* out_lo, int64_t ldo, int64_t n_images,
                      int32_t h, int32_t w, int32_t channels, void* stream);
/* out_accum[s] += sum of values[s*segment_len .. +segment_len): per-pixel log|det| -> per-sample (sum_except_batch over H, W). */
int nfk_segment_sum(const float* values, float* out_accum, int64_t n_segments, int32_t segment_len, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NFK_H_ */
