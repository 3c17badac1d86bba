"""The case table of the split-fp16 dense layer (nfk_linear_f16x3, nfk_linear_tc.cu) and the branches each case lands in.

test_dense_cases.py checks on the CPU that every branch of BRANCHES is hit at 132 and 114 SMs (the H100 SXM and PCIe counts);
test_dense_layer_gpu.py runs every case on a GPU against fp64 and re-checks the plan with the device's own SM count.  plan()
uses the launcher's formulas (linear_f16x3_launch: tiles of BM x BN, K-slabs of BK, one persistent CTA per SM up to the tile
count; the kernel's fold_residual / vec_y / vec_s conditions), so a case whose shape silently lands elsewhere fails here first.

Destination layouts.  Every output buffer has 2 sentinel rows above and 3 below the rows the launch writes, and a layout:
  "vec"      row pitch even, first column at offset 0 -> the vector stores (float2 / half2)
  "odd_ld"   row pitch odd                            -> scalar stores
  "odd_col"  a view starting at column 1 of an even pitch: misaligned for the vector stores -> scalar stores
Buffers come from the CUDA caching allocator (512-byte aligned), so the alignment follows from the offset alone; the GPU test
asserts the pointers it builds agree with the plan."""
from collections import namedtuple

BM = BN = 128
BK = 32
STAGES = 6
DRAIN = 2

ACT_CODES = range(7)        # include/nfk.h: NFK_ACT_NONE, RELU, TANH, ELU, LEAKY_RELU, GELU, SILU
ROWS_ABOVE, ROWS_BELOW = 2, 3

Case = namedtuple("Case", "id n k o out split_cols y_first_col relu_out split_relu residual bias data a_exp w_max "
                          "a_layout w_layout y_layout s_layout")


def case(id, n, k, o, out="y", split_cols=0, y_first_col=0, relu_out=0, split_relu=0, residual=False, bias=True, data="randn",
         a_exp=6, w_max=None, a_layout="dense", w_layout="dense", y_layout="vec", s_layout="vec"):
    """out: "y" (fp32 only), "pair" (fp16 pair only), "both".  data: "randn", or "nonneg" (|randn| activations times |randn|
    weights: the tensor core's round-toward-zero accumulation grows with K instead of cancelling).  a_exp: the activation pair's
    exponent; w_max: p to scale the weights to max |w| = 2^p (weight_exp then clamps at +-40); None: randn / sqrt(K)."""
    return Case(id, n, k, o, out, split_cols, y_first_col, relu_out, split_relu, residual, bias, data, a_exp, w_max, a_layout,
                w_layout, y_layout, s_layout)


CASES = [
    case("row1_o1_k8", 1, 8, 1),                                                             # one row, one column, one slab
    case("n63_o2_k16_pair_only", 63, 16, 2, out="pair", split_relu=1),
    case("n64_o8_k24_split_odd_relu", 64, 24, 8, out="both", split_cols=3, relu_out=1, split_relu=1),     # partial slab
    case("n65_o127_k40_residual_separate", 65, 40, 127, out="both", split_cols=64, relu_out=1, residual=True,
         y_layout="odd_ld", s_layout="odd_col"),
    case("n127_o128_k192_ring_folded_first_col_even", 127, 192, 128, out="both", split_cols=64, y_first_col=64, residual=True,
         bias=False, y_layout="odd_col", s_layout="odd_ld"),                                  # num_k = ring depth
    case("n256_o129_k200_views_first_col_odd", 256, 200, 129, out="both", split_cols=33, y_first_col=33, a_layout="col_view",
         w_layout="col_view"),                                                                # num_k = 7: past the ring, odd
    case("n300_o255_k2304_same_sign", 300, 2304, 255, out="both", data="nonneg", a_layout="row_slice"),
    case("n200_o9016_k4608_same_sign", 200, 4608, 9016, data="nonneg"),                     # 142 tiles: more than CTAs
    case("n20000_o8_k200_ring_phase", 20000, 200, 8, out="both", split_cols=8, residual=True),  # 157 tiles, num_k = 7
    case("n129_o40_k64_first_col_even_vec", 129, 64, 40, out="both", split_cols=16, y_first_col=16),
    # the ACT instance: every code as relu_out and as split_relu, with a residual (separate, and folded)
    case("act_tanh_elu", 100, 32, 48, out="both", relu_out=2, split_relu=3, residual=True),
    case("act_elu_tanh", 100, 48, 40, out="both", relu_out=3, split_relu=2),
    case("act_leaky_gelu", 70, 64, 24, out="both", relu_out=4, split_relu=5, s_layout="odd_col"),
    case("act_gelu_leaky", 70, 96, 24, out="both", relu_out=5, split_relu=4, y_layout="odd_ld"),
    case("act_silu_silu", 90, 40, 33, out="both", relu_out=6, split_relu=6),
    case("act_split_only_folded", 90, 40, 32, out="both", split_relu=2, residual=True),
    # exponents at the ends of what the callers produce
    case("a_exp_m24", 150, 72, 64, a_exp=-24),
    case("w_max_2m26", 150, 72, 64, w_max=-26, bias=False),
    case("w_max_2p54", 150, 72, 64, w_max=54),
]

# the branches every case table must reach (test_dense_cases.py)
BRANCHES = (
    {"rows%%128=%d" % r for r in (1, 63, 64, 65, 127, 0)} | {"one_row", "tiles>ctas"}
    | {"o=%d" % o for o in (1, 2, 8, 127, 128, 129, 255, 9016)}
    | {"k=%d" % k for k in (8, 16, 24, 40, 192, 200, 2304, 4608)}
    | {"num_k=1", "num_k_odd>1", "num_k=ring", "num_k>ring", "num_k>=64", "partial_slab", "partial_drain", "ring_phase_across_tiles"}
    | {"y_only", "pair_only", "both", "split_odd", "split_even", "split=o", "y_first_col_odd", "y_first_col_even_scalar",
       "y_first_col_even_vec", "instance_relu", "instance_act", "residual_folded", "residual_separate", "residual_act_instance",
       "bias_none"}
    | {"relu_out=%d" % c for c in ACT_CODES} | {"split_relu=%d" % c for c in ACT_CODES}
    | {"y_vec", "y_scalar", "y_tail", "pair_vec", "pair_scalar", "pair_tail"}
    | {"a_col_view", "a_row_slice", "w_col_view", "a_exp=6", "a_exp=-24", "w_max=2^-26", "w_max=2^54", "same_sign_k=2304",
       "same_sign_k=4608"}
)


def want_y(c):
    return c.out in ("y", "both")


def want_pair(c):
    return c.out in ("pair", "both")


def split_n(c):
    return c.split_cols if c.split_cols > 0 else c.o


def dest_geometry(layout, o, itemsize):
    """(row pitch, first column, byte offset of the first column) of a destination buffer of a layout."""
    if layout == "vec":
        ld, col0 = o + o % 2, 0
    elif layout == "odd_ld":
        ld, col0 = o + 1 - o % 2, 0
    else:
        ld, col0 = o + 2 + o % 2, 1
    return ld, col0, col0 * itemsize


def plan(c, sm_count):
    """The set of BRANCHES case c lands in on a device with sm_count SMs."""
    hit = set()
    num_k = (c.k + BK - 1) // BK
    tiles = ((c.n + BM - 1) // BM) * ((c.o + BN - 1) // BN)
    grid = min(tiles, sm_count)
    hit.add("rows%%128=%d" % (c.n % BM))
    if c.n == 1:
        hit.add("one_row")
    if tiles > grid:
        hit.add("tiles>ctas")
        if num_k % STAGES:
            hit.add("ring_phase_across_tiles")          # a CTA's second tile starts mid-ring
    hit.add("o=%d" % c.o)
    hit.add("k=%d" % c.k)
    if num_k == 1:
        hit.add("num_k=1")
    elif num_k % 2:
        hit.add("num_k_odd>1")
    if num_k == STAGES:
        hit.add("num_k=ring")
    if num_k > STAGES:
        hit.add("num_k>ring")
    if num_k >= 64:
        hit.add("num_k>=64")
    if c.k % BK:
        hit.add("partial_slab")
    if num_k % DRAIN:
        hit.add("partial_drain")
    hit.add({"y": "y_only", "pair": "pair_only", "both": "both"}[c.out])
    y, s = want_y(c), want_pair(c)
    if s:
        sn = split_n(c)
        hit.add("split=o" if sn == c.o else ("split_odd" if sn % 2 else "split_even"))
        hit.add("split_relu=%d" % c.split_relu)
    if y:
        hit.add("relu_out=%d" % c.relu_out)
    act = c.relu_out > 1 or c.split_relu > 1
    hit.add("instance_act" if act else "instance_relu")
    if c.residual:
        hit.add("residual_separate" if c.relu_out else "residual_folded")
        if act:
            hit.add("residual_act_instance")
    if not c.bias:
        hit.add("bias_none")
    if y:
        ld, _, off = dest_geometry(c.y_layout, c.o, 4)
        vec_y = ld % 2 == 0 and off % 8 == 0
        hit.add("y_vec" if vec_y and c.o - c.y_first_col >= 2 else "y_scalar")
        if c.o % 2:
            hit.add("y_tail")
        if c.y_first_col:
            if c.y_first_col % 2:
                hit.add("y_first_col_odd")
            else:
                hit.add("y_first_col_even_vec" if vec_y else "y_first_col_even_scalar")
    if s:
        ld, _, off = dest_geometry(c.s_layout, c.o, 2)
        vec_s = ld % 2 == 0 and off % 4 == 0
        hit.add("pair_vec" if vec_s and split_n(c) >= 2 else "pair_scalar")
        if split_n(c) % 2:
            hit.add("pair_tail")
    if c.a_layout != "dense":
        hit.add("a_" + c.a_layout)
    if c.w_layout != "dense":
        hit.add("w_" + c.w_layout)
    hit.add("a_exp=%d" % c.a_exp)
    if c.w_max is not None:
        hit.add("w_max=2^%d" % c.w_max)
    if c.data == "nonneg":
        hit.add("same_sign_k=%d" % c.k)
    return hit
