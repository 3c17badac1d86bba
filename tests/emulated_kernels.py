"""CPU stand-ins for the Python kernel wrappers of nflows_b200.kernels, for tests of the HOST logic of the native chain
(column layouts, row blocking, context / image chains) where there is no GPU.

Each stand-in restates the CONTRACT of the wrapper it replaces (include/nfk.h) with torch CPU ops, including the fp16 split-pair
operand format, so a flow can be pushed through `_native_apply` on CPU tensors.  Test infrastructure only: nothing in the
package imports this, and the kernels themselves are checked on hardware by the `-m gpu` tests."""
import contextlib
import math

import torch
import torch.nn.functional as F

from nflows_b200 import _native as N
from nflows_b200 import kernels as K
from nflows_b200.transforms import splines

#: the activations of include/nfk.h's codes NFK_ACT_*; True and False read as relu and none
_ACTS = {N.ACT_RELU: F.relu, N.ACT_TANH: torch.tanh, N.ACT_ELU: F.elu, N.ACT_LEAKY_RELU: F.leaky_relu, N.ACT_GELU: F.gelu,
         N.ACT_SILU: F.silu}


def _act(code, x):
    """The activation of `code` on x, computed in fp64 and returned in x's dtype."""
    return _ACTS[int(code)](x.double()).to(x.dtype) if code else x


def _pair(x, exp, act=0, out=None):
    v = _act(act, x).double() * 2.0 ** exp
    hi = v.to(torch.float16)
    lo = (v - hi.double()).to(torch.float16)
    if out is None:
        return K.Pair16(hi, lo, exp)
    out.hi.copy_(hi)
    out.lo.copy_(lo)
    return out


def _value(pair):
    return ((pair.hi.double() + pair.lo.double()) * 2.0 ** -pair.exp)


def _spline(desc, x, params, inverse):
    """x: [n, d_t]; params: [n, d_t, M] with the reference's (widths, heights, derivatives) order."""
    k = desc.num_bins
    w, h, d = params[..., :k] / desc.wh_divisor, params[..., k:2 * k] / desc.wh_divisor, params[..., 2 * k:]
    common = dict(inputs=x, unnormalized_widths=w, unnormalized_heights=h, unnormalized_derivatives=d, inverse=bool(inverse),
                  min_bin_width=desc.min_bin_width, min_bin_height=desc.min_bin_height, min_derivative=desc.min_derivative)
    if desc.linear_tails:
        return splines.unconstrained_rational_quadratic_spline(tails="linear", tail_bound=desc.right, **common)
    return splines.rational_quadratic_spline(left=desc.left, right=desc.right, bottom=desc.bottom, top=desc.top, **common)


def _cols(t_cols, width):
    if isinstance(t_cols, tuple):
        return torch.arange(t_cols[0], t_cols[0] + t_cols[1])
    return t_cols.long()


class Calls(dict):
    """Calls per wrapper name; `trace` is the ordered list of (wrapper, rows) of every call."""

    def __init__(self):
        super().__init__()
        self.trace = []


def install(monkeypatch):
    calls = Calls()

    def count(name, rows):
        calls[name] = calls.get(name, 0) + 1
        calls.trace.append((name, int(rows)))

    def native_ok(t, context=None):
        return t.dtype == torch.float32 and not (torch.is_grad_enabled() and t.requires_grad)

    def linear(x, weight, bias=None, residual=None, relu_in=0, relu_out=0, out=None):
        count("linear", x.shape[0])
        y = _act(relu_out, F.linear(_act(relu_in, x), weight, bias))
        if residual is not None:
            y = y + residual
        if out is not None:
            out.copy_(y)
            return out
        return y

    def gather_cols(x, cols, out=None):
        count("gather_cols", x.shape[0])
        y = x[:, cols.long()]
        if out is not None:
            out.copy_(y)
            return out
        return y.contiguous()

    def actnorm(x, scale, shift, lad_accum, lad_const, inverse):
        count("actnorm", x.shape[0])
        if lad_accum is not None:
            lad_accum += lad_const
        return (x - shift) / scale if inverse else x * scale + shift

    def rqs_rows(desc, inverse, x, params, t_cols, id_cols, lad_accum, flags, out=None):
        count("rqs_rows", x.shape[0])
        y = torch.empty_like(x) if out is None else out
        t = t_cols.long()
        m = params.shape[1] // t.numel()
        yt, lad = _spline(desc, x[:, t], params.reshape(x.shape[0], t.numel(), m), inverse)
        if id_cols is not None:
            y[:, id_cols.long()] = x[:, id_cols.long()]
        y[:, t] = yt
        if lad_accum is not None:
            lad_accum += lad.sum(dim=1)
        return y

    def rqs_elementwise(desc, inverse, x, uw, uh, ud, param_period=0, flags=None):
        count("rqs_elementwise", x.shape[0])
        flat = x.reshape(-1)
        idx = torch.arange(flat.numel()) % param_period if param_period else torch.arange(flat.numel())
        params = torch.cat([p.reshape(-1, p.shape[-1])[idx] for p in (uw, uh, ud)], dim=-1)
        y, lad = _spline(desc, flat[:, None], params[:, None, :], inverse)
        return y.reshape(x.shape), lad.reshape(x.shape)

    def std_normal_log_prob(z, log_z, lad=None):
        lp = -0.5 * (z * z).sum(dim=1) - log_z
        return lp + lad if lad is not None else lp

    def run_with_activation_rescale(fn):
        out, lad, _ = fn()
        return out, lad

    def weight_exp(w):
        amax = float(w.detach().abs().max())
        if not (amax > 0.0) or not math.isfinite(amax):
            return 0
        return max(-40, min(40, 14 - math.ceil(math.log2(amax))))

    def split_f16(x, exp, relu=0, out=None, flags=None):
        count("split_f16", x.shape[0])
        if out is not None and out.exp != exp:
            raise ValueError("exponent mismatch")
        return _pair(x, exp, relu, out)

    def glu_skip(t, gate, skip=None, want_y=True, want_split=False, split_relu=0, split_exp=None, pair_out=None, flags=None):
        count("glu_skip", t.shape[0])
        from nflows_b200 import config
        v = t * torch.sigmoid(gate)
        if skip is not None:
            v = v + skip
        pair = _pair(v, config.activation_exp if split_exp is None else split_exp, split_relu, pair_out) if want_split else None
        return (v if want_y else None), pair

    def nchw_to_rows(x):
        count("nchw_to_rows", x.shape[0] * x.shape[2] * x.shape[3])
        b, c, h, w = x.shape
        return x.permute(0, 2, 3, 1).reshape(b * h * w, c).contiguous()

    def rows_to_nchw(rows, b, c, h, w):
        count("rows_to_nchw", rows.shape[0])
        return rows.reshape(b, h, w, c).permute(0, 3, 1, 2).contiguous()

    def squeeze_rows(rows, b, c, h, w, inverse=False):
        count("squeeze_rows", rows.shape[0])
        from nflows_b200.transforms.reshape import SqueezeTransform
        img = rows.reshape(b, h, w, c).permute(0, 3, 1, 2)
        out = (SqueezeTransform().inverse(img) if inverse else SqueezeTransform()(img))[0]
        return out.permute(0, 2, 3, 1).reshape(-1, out.shape[1]).contiguous(), tuple(out.shape[1:])

    def im2col3x3(pair, n_images, h, w):
        count("im2col3x3", pair.shape[0])
        n, c = pair.shape
        assert n == n_images * h * w

        def one(t):
            img = F.pad(t.reshape(n_images, h, w, c), (0, 0, 1, 1, 1, 1))
            taps = [img[:, ky:ky + h, kx:kx + w, :] for ky in range(3) for kx in range(3)]
            return torch.cat(taps, dim=-1).reshape(n, 9 * c).contiguous()
        return K.Pair16(one(pair.hi), one(pair.lo), pair.exp)

    def segment_sum_(values, out_accum, segment_len):
        count("segment_sum", values.numel())
        out_accum += values.reshape(out_accum.numel(), segment_len).sum(dim=1)
        return out_accum

    def f16x3_supported(lda, ldw, k):
        return k >= 8 and k % 8 == 0 and lda % 8 == 0 and ldw % 8 == 0

    def linear_f16x3(a, w, bias=None, residual=None, relu_out=0, want_y=True, want_split=False, split_relu=0,
                     split_exp=None, split_cols=0, y_out=None, pair_out=None, flags=None, y_first_col=0):
        count("linear_f16x3", a.shape[0])
        from nflows_b200 import config
        assert f16x3_supported(a.hi.stride(0), w.hi.stride(0), a.shape[1]) and a.shape[1] == w.shape[1], (a.shape, w.shape)
        v = _value(a) @ _value(w).t()
        if bias is not None:
            v = v + bias.double()
        v = _act(relu_out, v)
        if residual is not None:
            v = v + residual.double()
        v = v.float()
        y = None
        if want_y:
            y = y_out if y_out is not None else torch.empty_like(v)
            y[:, y_first_col:] = v[:, y_first_col:]
            if y_first_col:
                y[:, :y_first_col] = float("nan")        # the kernel leaves these unwritten: nobody may read them
        pair = None
        if want_split:
            exp = config.activation_exp if split_exp is None else split_exp
            cols = split_cols or v.shape[1]
            pair = pair_out if pair_out is not None else K.Pair16.empty(v.shape[0], v.shape[1], exp, v.device)
            _pair(v[:, :cols], exp, split_relu, pair.cols(0, cols))
        return y, pair

    def rq_coupling_final_supported(num_bins, tails, hidden, lda):
        return num_bins in (4, 8, 10, 16) and hidden >= 8 and hidden % 8 == 0 and lda % 8 == 0

    def rq_coupling_final_padded_params(num_bins, tails):
        m = 3 * num_bins - 1 if tails == "linear" else 3 * num_bins + 1
        return (m + 7) // 8 * 8

    def rq_coupling_final(desc, inverse, a, wp, bias_packed, x, t_cols, y, lad_accum, flags, y_pair=None):
        count("rq_coupling_final", x.shape[0])
        return final_layer_spline(desc, inverse, a, wp, bias_packed, x, t_cols, y, lad_accum, y_pair)

    def final_layer_spline(desc, inverse, a, wp, bias_packed, x, t_cols, y, lad_accum, y_pair):
        t = _cols(t_cols, x.shape[1])
        d_t = t.numel()
        mp = wp.shape[0] // d_t
        m = 3 * desc.num_bins - 1 if desc.linear_tails else 3 * desc.num_bins + 1
        params = (_value(a) @ _value(wp).t() + bias_packed.double()).float().reshape(x.shape[0], d_t, mp)[:, :, :m]
        yt, lad = _spline(desc, x[:, t], params, inverse)
        if lad_accum is not None:
            lad_accum += lad.sum(dim=1)
        if y_pair is not None:
            _pair(yt, y_pair.exp, False, K.Pair16(y_pair.hi[:, t], y_pair.lo[:, t], y_pair.exp))
            y_pair.hi[:, t], y_pair.lo[:, t] = _pair(yt, y_pair.exp).hi, _pair(yt, y_pair.exp).lo
            return None
        y[:, t] = yt
        return y

    def rq_coupling_step_supported(num_bins, tails, hidden, in_features, num_square_layers):
        # the predicate of nfk_rq_coupling_step_supported (csrc/nfk_coupling_step_tc.cu)
        return (num_bins in (4, 8, 10, 16) and 32 <= hidden <= 256 and hidden % 32 == 0 and in_features >= 8 and in_features % 8 == 0
                and 0 <= num_square_layers < 9)

    def trunk(plan, a, terms):
        """The layer recursion of include/nfk.h (nfk_rq_coupling_step_f16x3 and its _terms_ form) on the operands a dense.StepPlan
        packs: flag bit 0 the activation on (acc + bias + row term), bit 1 add the current skip tensor, bit 2 the fp32 result
        becomes the skip tensor, bit 3 the next consumer sees the activation of it; bits [8, 12) the activation code, 0 meaning
        relu.  Every hidden activation goes through the fp16 pair at the plan's exponent.  terms: None, or per trunk layer None or
        an fp32 [>= n, >= hidden] tensor.  Returns the pair of the last trunk layer's output."""
        n, hdim = a.shape[0], plan.hidden
        assert hdim % 32 == 0 and a.shape[1] % 8 == 0, (hdim, a.shape)
        assert terms is None or len(terms) <= len(plan.layer_flags)
        cur, skip = _value(a), None
        for l, f in enumerate(plan.layer_flags):
            if l == 0:
                w = _value(plan.w0)
            else:
                blk = slice((l - 1) * hdim, l * hdim)
                w = _value(K.Pair16(plan.wt_hi[blk], plan.wt_lo[blk], int(plan.wt_exps_c[l - 1])))
            v = cur @ w.t() + plan.bias[l * hdim:(l + 1) * hdim].double()
            if terms is not None and l < len(terms) and terms[l] is not None:
                assert terms[l].shape[0] >= n and terms[l].shape[1] >= hdim
                v = v + terms[l][:n, :hdim].double()
            code = (f >> N.STEP_ACT_SHIFT) & 15 or N.ACT_RELU
            if f & 1:
                v = _act(code, v)
            if f & 2:
                v = v + skip
            v = v.float().double()                      # the kernel's sums are fp32
            if f & 4:
                skip = v
            cur = _value(_pair(v.float(), plan.act_exp, code if f & 8 else 0))
        return _pair(cur.float(), plan.act_exp)

    def rq_coupling_step(plan, a, desc=None, inverse=False, wp=None, bias_packed=None, x=None, t_cols=None, y=None, lad_accum=None,
                         flags=None, y_pair=None, h_pair=None, terms=None):
        count("rq_coupling_step" if h_pair is None else "trunk_step", a.shape[0])
        assert terms is None or (h_pair is None and y_pair is None)
        h = trunk(plan, a, terms)
        if h_pair is not None:
            h_pair.hi.copy_(h.hi)
            h_pair.lo.copy_(h.lo)
            return None
        return final_layer_spline(desc, inverse, h, wp, bias_packed, x, t_cols, y, lad_accum, y_pair)

    def affine_ar_step(plan, a, wf, bias, x, cols, y, lad_accum, flags, inverse, terms=None):
        """include/nfk.h: nfk_affine_ar_step_f16x3 -- the trunk, then the final rows [u_j, shift_j] and scale = softplus(u) + 1e-3
        in fp32."""
        count("affine_ar_step", a.shape[0])
        c0, d_t = cols
        assert wf.shape[0] == 2 * d_t and bias.numel() == 2 * d_t
        params = (_value(trunk(plan, a, terms)) @ _value(wf).t() + bias.double()).float()
        scale, shift = F.softplus(params[:, 0::2]) + 1e-3, params[:, 1::2]
        xt = x[:, c0:c0 + d_t]
        y[:, c0:c0 + d_t] = (xt - shift) / scale if inverse else scale * xt + shift
        if lad_accum is not None:
            lad = torch.log(scale).sum(dim=1)
            lad_accum += -lad if inverse else lad
        return y

    def mog_made_step(plan, a, wf, bias, num_components, epsilon, cols, x=None, lad_accum=None, y=None, noise=None, flags=None,
                      terms=None):
        """include/nfk.h: nfk_mog_made_step_f16x3 -- the trunk, then the packed final rows and the mixture log-density or draw in
        fp64.  Records every launch's hidden width and input pair width in calls["hidden"] and calls["in_features"]."""
        count("mog_made_step", a.shape[0])
        calls.setdefault("hidden", []).append(plan.hidden)
        calls.setdefault("in_features", []).append(a.shape[1])
        n = a.shape[0]
        c0, d_t = cols
        mp = K.mog_made_padded_rows(num_components)
        assert wf.shape[0] == mp * d_t and bias.numel() == mp * d_t
        params = _value(trunk(plan, a, terms)) @ _value(wf).t() + bias.double()
        params = params.reshape(n, d_t, mp)[..., :3 * num_components].reshape(n, d_t, num_components, 3)
        logits, means, stds = params[..., 0], params[..., 1], F.softplus(params[..., 2]) + epsilon
        if noise is None:
            xt = x[:, c0:c0 + d_t].double()
            t = torch.log_softmax(logits, -1) - 0.5 * (math.log(2 * math.pi) + 2 * torch.log(stds)
                                                       + ((xt[..., None] - means) / stds) ** 2)
            lad_accum += torch.logsumexp(t, -1).sum(-1).float()
            return lad_accum
        u, e = noise
        cdf = torch.cumsum(torch.softmax(logits, -1), -1)
        c = torch.clamp((u[:, :d_t].double()[..., None] >= cdf).sum(-1), max=num_components - 1)
        pick = lambda t: t.gather(-1, c[..., None])[..., 0]
        y[:, c0:c0 + d_t] = (pick(means) + pick(stds) * e[:, :d_t].double()).float()
        return y

    def affine_coupling_rows(x, params, mult, scale_activation, inverse, t_cols, id_cols, lad_accum, out=None):
        count("affine_coupling_rows", x.shape[0])
        y = torch.empty_like(x) if out is None else out
        t, d_t = t_cols.long(), t_cols.numel()
        y[:, id_cols.long()] = x[:, id_cols.long()]
        shift = params[:, :d_t]
        if mult == 2:
            raw = params[:, d_t:]
            scale = torch.sigmoid(raw + 2) + 1e-3 if scale_activation == 0 else (F.softplus(raw) + 1e-3).clamp(0, 3)
            y[:, t] = (x[:, t] - shift) / scale if inverse else x[:, t] * scale + shift
            lad_accum += -torch.log(scale).sum(dim=1) if inverse else torch.log(scale).sum(dim=1)
        else:
            y[:, t] = x[:, t] - shift if inverse else x[:, t] + shift
        return y

    def affine_coupling_final(a, w, bias, x, t_cols, mult, scale_activation, inverse, y, lad_accum, flags=None):
        count("affine_coupling_final", x.shape[0])
        t = _cols(t_cols, x.shape[1])
        params = (_value(a) @ _value(w).t() + bias.double()).float()
        xt = x[:, t]
        if mult == 2:
            shift, raw = params[:, 0::2], params[:, 1::2]
            scale = torch.sigmoid(raw + 2) + 1e-3 if scale_activation == 0 else (F.softplus(raw) + 1e-3).clamp(0, 3)
            lad = torch.log(scale).sum(dim=1)
            y[:, t] = (xt - shift) / scale if inverse else xt * scale + shift
            if lad_accum is not None:
                lad_accum += -lad if inverse else lad
        else:
            y[:, t] = xt - params if inverse else xt + params
        return y

    # the functional spline API keeps its torch formulation (it is what the stand-ins of the spline kernels call)
    monkeypatch.setattr(splines.rational_quadratic, "_use_native", lambda inputs, *params: False)
    for name, fn in dict(
            native_ok=native_ok, on_device_of=lambda t: contextlib.nullcontext(), warn_eager_cuda=lambda *a, **k: None,
            new_flags=lambda device: torch.zeros(1, dtype=torch.int32), index_tensor=lambda idx, device: idx.to(torch.int32),
            fill_=lambda t, v: t.fill_(v), add_const_=lambda lad, c: lad.add_(c),
            zeros_lad=lambda x: torch.zeros(x.shape[0]), linear=linear, gather_cols=gather_cols, actnorm=actnorm, rqs_rows=rqs_rows,
            rqs_elementwise=rqs_elementwise,
            std_normal_log_prob=std_normal_log_prob, raise_for_flags=lambda flags: None,
            run_with_activation_rescale=run_with_activation_rescale, weight_exp=weight_exp, split_f16=split_f16, glu_skip=glu_skip,
            nchw_to_rows=nchw_to_rows, rows_to_nchw=rows_to_nchw, squeeze_rows=squeeze_rows, im2col3x3=im2col3x3,
            segment_sum_=segment_sum_, f16x3_supported=f16x3_supported, linear_f16x3=linear_f16x3,
            rq_coupling_final_supported=rq_coupling_final_supported, rq_coupling_final_padded_params=rq_coupling_final_padded_params,
            rq_coupling_final=rq_coupling_final, affine_coupling_final=affine_coupling_final, affine_coupling_rows=affine_coupling_rows,
            rq_coupling_step_supported=rq_coupling_step_supported, rq_coupling_step=rq_coupling_step,
            affine_ar_step=affine_ar_step, mog_made_step=mog_made_step).items():
        monkeypatch.setattr(K, name, fn)
    return calls
