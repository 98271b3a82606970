"""Element-by-element tests of the dense-head, part-head and camera-head kernels against float64 statements of the same
operations, computed from the exact 16-bit / fp32 inputs each kernel received.  fp16 and bf16 throughout.

Every allowance is derived next to its assert from the kernel's arithmetic:
  * fp32 rounding: 2^-24 relative per operation, so a sequential sum of n terms is off by at most n 2^-24 of the sum of
    the magnitudes, a tree level adds 2^-24;
  * tensor-core products (mma.sync, wgmma) accumulate in fp32 with an order the PTX manual leaves open: 2^-20 of the
    magnitude sum, as in tests/ulp_bounds.py;
  * expf / expm1f / erff / rsqrtf: at most 2 ulp (2^-22 relative), __expf: ex2.approx (2^-22) of an fp32 argument
    x log2(e) (2^-24 |x|);
  * the window attentions split P into 16-bit hi + lo: |P - hi - lo| <= 2^-22 P (fp16; plus 2^-25 absolute where lo or
    hi is subnormal) and 2^-16 P (bf16).
16-bit outputs go through `check16` (the fp32-reachable interval where derived), fp32 outputs through `check32`.  The
worst error / bound and the share of elements that are not RN16 of the reference are printed (run with -s).
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from launch_refs import U24
from launch_refs import check_tail as _check_tail
from launch_refs import conf64 as _conf64
from launch_refs import tail_act64 as _tail_act64
from ulp_bounds import check16, check32, ulp16, ulp_distance

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
U_SPLIT_P = {torch.float16: 2.0 ** -22, torch.bfloat16: 2.0 ** -16}      # what the hi + lo split of P leaves


@pytest.fixture(scope="module")
def ops():
    from iggt_official_b200 import ops as _ops
    return _ops


def _report(what, *values):
    print(f"[bound] {what}: " + " ".join(f"{v:.3g}" if isinstance(v, float) else str(v) for v in values))


def _frac_off(out, ref64, dtype):
    return float((ulp_distance(out, ref64, dtype) != 0).double().mean())


def _check_attn(out, o64, bound, dtype, max_frac_off, what):
    """|O - O64| <= bound per element, and at most `max_frac_off` of the elements off RN16(O64).  Returns (worst
    error / bound, fraction off)."""
    o = out.double()
    assert torch.isfinite(o).all(), f"{what}: non-finite outputs"
    ratio = (o - o64).abs() / bound
    worst = ratio.max().item()
    i = int(ratio.view(-1).argmax())
    assert worst <= 1.0, (f"{what}: {int((ratio > 1).sum())} of {o.numel()} elements beyond the bound; worst "
                          f"{worst:.3g} x bound at flat {i}: out {o.view(-1)[i].item()!r} ref {o64.view(-1)[i].item()!r}")
    frac = _frac_off(out, o64, dtype)
    assert frac <= max_frac_off, f"{what}: {frac:.2%} of the elements are not RN16(ref) (limit {max_frac_off:.2%})"
    return worst, frac


def _attn_bound(q, k, v, s64, scale, dtype, score_abs):
    """float64 softmax attention of [..., Lq, d] x [..., Lk, d] and its per-element bound (window attentions, tensor-core
    path).  s64: exact scores; score_abs: per-score allowance of the fp32 score arithmetic (besides the __expf terms).
      weight error d_ij = score_abs + 2^-24 |s - m| (fp32 argument of ex2 after the max subtraction) + 2^-22 (ex2.approx)
      O error <= ulp16(O)                         (final RN16 + the fp32 1 / l and the product by it)
               + (u_P + 2^-20) (P @ |V|)          (hi + lo split of P, fp32 accumulation of P V on the tensor cores)
               + (P d) @ |V| + |O| (sum_j P d + 2^-20)   (weight errors: O = sum p (1 + d) v / sum p (1 + d); l's sum)
               + fp16: 2^-25 sum_j |V_j|          (hi / lo below 2^-14 are subnormal: 2^-25 absolute per weight)"""
    p = torch.softmax(s64, -1)
    o64 = p @ v
    m = s64.amax(-1, keepdim=True)
    d = score_abs + U24 * (s64 - m).abs() + 2.0 ** -22
    pd = p * d
    va = v.abs()
    bound = (ulp16(o64, dtype) + (U_SPLIT_P[dtype] + 2.0 ** -20) * (p @ va) + pd @ va
             + o64.abs() * (pd.sum(-1, keepdim=True) + 2.0 ** -20))
    if dtype == torch.float16:
        bound = bound + 2.0 ** -25 * va.sum(-2, keepdim=True)
    return o64, bound


# ------------------------------------------------------------------------------------- HAB window attention (8x8, d 32)
def _hab_ref(qkv, dtype):
    NB, H, W, _ = qkv.shape
    x = qkv.double().view(NB, H // 8, 8, W // 8, 8, 3, 4, 32).permute(5, 0, 1, 3, 6, 2, 4, 7)
    x = x.reshape(3, NB, H // 8, W // 8, 4, 64, 32)
    q, k, v = x[0], x[1], x[2]
    scale = 32 ** -0.5
    s64 = q @ k.transpose(-1, -2) * scale
    # fp32 S = Q K^T on the tensor cores (2^-20 of sum |q||k|), times the fp32 constant RN(32^-0.5) (2^-24 relative)
    # and the rounding of that product (2^-24): 2^-23 |s|
    score_abs = 2.0 ** -20 * scale * (q.abs() @ k.abs().transpose(-1, -2)) + 2.0 ** -23 * s64.abs()
    o64, bound = _attn_bound(q, k, v, s64, scale, dtype, score_abs)

    def back(t):                                   # [NB, nh, nw, head, 64, 32] -> [NB, H, W, 128]
        return t.view(NB, H // 8, W // 8, 4, 8, 8, 32).permute(0, 1, 4, 2, 5, 3, 6).reshape(NB, H, W, 128)

    return back(o64), back(bound)


# Logits of standard deviation ~8: q.k * d^-0.5 over d dims of N(0, sd^2) products has standard deviation sd^2.
SD8 = math.sqrt(8.0)
GRIDS = [(1, 36, 36), (2, 36, 26)]                 # (NB, gh, gw): the largest square grid, a non-square one with 2 images


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("NB,gh,gw", GRIDS)
def test_window_attention_hab(ops, dtype, NB, gh, gw):
    H, W = 8 * gh, 8 * gw
    g = torch.Generator(device="cuda").manual_seed(gh * 100 + gw)
    qkv = torch.randn(NB, H, W, 384, device="cuda", generator=g) * SD8
    qkv[..., 256:] = torch.randn(NB, H, W, 128, device="cuda", generator=g)
    qkv = qkv.to(dtype)
    out = ops.window_attention(qkv)
    torch.cuda.synchronize()
    o64, bound = _hab_ref(qkv, dtype)
    # a correct kernel's fp32 error is far below half an ulp of the output except at a few RN16 midpoints
    _report(f"HAB {dtype} {NB}x{H}x{W}", *_check_attn(out, o64, bound, dtype, 0.02, f"HAB {NB}x{H}x{W}"))


# --------------------------------------------------------------------------- OCAB (8x8 queries, 12x12 keys, d 64, bias)
def _ocab_ref(q, k, v, table, rpi, dtype):
    """oracle.ref_model's partition / unfold / bias (the scrambled query windows included) in float64, with the bound."""
    from oracle import ref_model
    b, h, w, c = q.shape
    ws, heads, d = 8, 4, 64
    qf, kf, vf = (t.double().permute(0, 3, 1, 2) for t in (q, k, v))
    q_win = ref_model.window_partition(qf, ws).view(-1, ws * ws, c)
    kvw = F.unfold(torch.cat([kf, vf], 1), kernel_size=(12, 12), stride=ws, padding=2)
    nw = kvw.shape[-1]
    kvw = kvw.view(b, 2, c, 144, nw).permute(1, 0, 4, 3, 2).reshape(2, b * nw, 144, c)
    qh = q_win.reshape(-1, 64, heads, d).permute(0, 2, 1, 3)
    kh = kvw[0].reshape(-1, 144, heads, d).permute(0, 2, 1, 3)
    vh = kvw[1].reshape(-1, 144, heads, d).permute(0, 2, 1, 3)
    bias = table.double()[rpi.long().view(-1)].view(64, 144, -1).permute(2, 0, 1).unsqueeze(0)
    s64 = (qh @ kh.transpose(-2, -1)) * 0.125 + bias
    # fp32 S = Q K^T on the tensor cores (2^-20 of 0.125 sum |q||k|); fmaf(S, 0.125, bias) rounds once (2^-24 |s|);
    # zero-padded border keys give Q K^T = 0 exactly (score = bias)
    score_abs = 2.0 ** -20 * 0.125 * (qh.abs() @ kh.abs().transpose(-2, -1)) + U24 * s64.abs()
    o64, bound = _attn_bound(qh, kh, vh, s64, 0.125, dtype, score_abs)

    def back(t):
        t = t.transpose(1, 2).reshape(-1, 64, c).view(-1, ws, ws, c)
        return ref_model.window_reverse(t, ws, h, w)

    return back(o64), back(bound)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("NB,gh,gw", GRIDS)
def test_window_attention_ocab(ops, dtype, NB, gh, gw):
    from oracle import ref_model
    h, w = 4 * gh, 4 * gw
    g = torch.Generator(device="cuda").manual_seed(7 * gh + gw)
    q = (torch.randn(NB, h, w, 256, device="cuda", generator=g) * SD8).to(dtype)
    k = (torch.randn(NB, h, w, 256, device="cuda", generator=g) * SD8).to(dtype)
    v = torch.randn(NB, h, w, 256, device="cuda", generator=g).to(dtype)
    table = torch.randn(361, 4, device="cuda", generator=g) * 2.0
    rpi = (ref_model.calculate_rpi_oca(8).cuda() % 361).int().contiguous()      # the python-style wrap of part_head.py
    out = ops.ocab_attention(q, k, v, table, rpi)
    torch.cuda.synchronize()
    o64, bound = _ocab_ref(q, k, v, table, rpi, dtype)
    wy = torch.arange(h, device="cuda") // 8
    wx = torch.arange(w, device="cuda") // 8
    by = (wy == 0) | (wy == h // 8 - 1)
    bx = (wx == 0) | (wx == w // 8 - 1)
    kinds = {"corner": by[:, None] & bx[None, :], "edge": by[:, None] ^ bx[None, :], "interior": ~by[:, None] & ~bx[None, :]}
    for name, sel in kinds.items():
        sel = sel[None].expand(NB, h, w)
        assert sel.any()
        _report(f"OCAB {dtype} {NB}x{h}x{w} {name}",
                *_check_attn(out[sel], o64[sel], bound[sel], dtype, 0.02, f"OCAB {NB}x{h}x{w} {name} windows"))


# ------------------------------------------------------------------------------------------------ bilinear upsample
def _bilinear64(x, H, W, tabx, taby):
    """align_corners=True bilinear in float64 at exact source positions, plus the fp32-reachable slack.
    The kernel's position fy = RN(RN((h-1)/(H-1)) * oy) is off the exact one by <= 2^-23 (h-1); ly = fy - y0 is exact
    and hy = 1 - ly rounds once (2^-25).  A position error moves the value by at most that error times the difference of
    two neighbouring taps - which can be rows y0 - 1 .. y0 + 2 when fy crosses an integer - so <= 2 dpos max|x| there.
    Each interpolated axis rounds twice in the blend hy (hx a + lx b) + ly (hx c + lx d) (<= 2^-23 of the tap maximum),
    the table add once.  An axis with n_out == n_in (the scale is exactly 1), n_out == 1 or n_in == 1 (the scale is 0)
    is exact: fy = oy (or 0), ly = 0, hy = 1, so hy * t + 0 * b = t - that axis is a copy, with no slack and no window."""
    NB, h, w, C = x.shape
    xd = x.double()
    exact_y, exact_x = H in (h, 1) or h == 1, W in (w, 1) or w == 1

    def axis(n_in, n_out):
        pos = torch.arange(n_out, device=x.device, dtype=torch.float64) * ((n_in - 1) / (n_out - 1) if n_out > 1 else 0.0)
        i0 = pos.floor().long().clamp(max=n_in - 1)
        i1 = (i0 + 1).clamp(max=n_in - 1)
        return i0, i1, pos - i0

    y0, y1, ly = axis(h, H)
    x0, x1, lx = axis(w, W)
    lyv, lxv = ly.view(1, H, 1, 1), lx.view(1, 1, W, 1)
    rows = xd[:, y0] * (1 - lyv) + xd[:, y1] * lyv
    ref = rows[:, :, x0] * (1 - lxv) + rows[:, :, x1] * lxv
    # max |x| over rows y0-1 .. y0+2 and columns x0-1 .. x0+2 of each output element (only the tap on an exact axis)
    py, px = (0, 0) if exact_y else (1, 2), (0, 0) if exact_x else (1, 2)
    a = F.pad(xd.abs().permute(0, 3, 1, 2), px + py)
    mloc = F.max_pool2d(a, (1 if exact_y else 4, 1 if exact_x else 4), stride=1).permute(0, 2, 3, 1)[:, y0][:, :, x0]
    dy = 0.0 if exact_y else 2.0 ** -23 * (h - 1) + 2.0 ** -25
    dx = 0.0 if exact_x else 2.0 ** -23 * (w - 1) + 2.0 ** -25
    rounds = 2.0 ** -23 * ((not exact_y) + (not exact_x))
    slack = (2 * dy + 2 * dx + rounds) * mloc
    if tabx is not None:
        t = torch.cat([tabx.double()[None, None].expand(NB, H, W, C // 2), taby.double()[None, :, None].expand(NB, H, W, C // 2)], -1)
        ref = ref + t
        slack = slack + U24 * (ref.abs() + t.abs() + mloc)
    return ref, slack


def _pe_tables(H, W, C, g):
    return (torch.randn(W, C // 2, device="cuda", generator=g), torch.randn(H, C // 2, device="cuda", generator=g))


# the heads' ladders (g / 2 -> g -> 2g -> 4g -> 8g, then 8g -> 14g at full resolution) for g = 36 x 26
LADDER = [((18, 13), (36, 26), 256), ((36, 26), (72, 52), 256), ((72, 52), (144, 104), 256), ((144, 104), (288, 208), 256),
          ((288, 208), (504, 364), 128), ((36, 36), (72, 72), 256), ((144, 144), (288, 288), 128)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("src,dst,C", LADDER)
@pytest.mark.parametrize("with_pe", [False, True])
def test_upsample_bilinear_ladder(ops, dtype, src, dst, C, with_pe):
    (h, w), (H, W) = src, dst
    g = torch.Generator(device="cuda").manual_seed(h * 1000 + W)
    x = torch.randn(1, h, w, C, device="cuda", generator=g).to(dtype)
    tx, ty = _pe_tables(H, W, C, g) if with_pe else (None, None)
    out = ops.upsample_bilinear(x, H, W, tx, ty)
    torch.cuda.synchronize()
    ref, slack = _bilinear64(x, H, W, tx, ty)
    lo, hi = ref - slack, ref + slack
    # every element is RN16 of a value the fp32 arithmetic can reach (0 steps outside the interval); the position
    # error (up to 2^-14.8 of a tap at h = 288) flips a minority of roundings
    worst, frac = check16(out, ref, dtype, 0, 1.0, lo, hi, what=f"upsample {src}->{dst}")
    _report(f"upsample {dtype} {src}->{dst} C={C} pe={with_pe}", worst, frac)
    assert frac <= 0.05, f"{frac:.2%} of the elements are not RN16(ref)"


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("h,w,H,W", [(19, 23, 19, 23), (7, 1, 7, 1), (1, 9, 1, 9), (12, 16, 12, 40), (12, 16, 30, 16)])
def test_upsample_bilinear_same_size_axis_is_a_copy(ops, dtype, h, w, H, W):
    """An axis with H == h has sy = 1, ly = 0: that axis is an exact copy, so the output is the float64 1-D
    interpolation along the other axis with that axis's slack only (`_bilinear64` gives the copied axis no slack).  With
    both, the output is the input, bit for bit."""
    g = torch.Generator(device="cuda").manual_seed(h * 31 + W)
    x = torch.randn(2, h, w, 32, device="cuda", generator=g).to(dtype)
    out = ops.upsample_bilinear(x, H, W)
    torch.cuda.synchronize()
    if (H, W) == (h, w):
        assert torch.equal(out.view(torch.int16), x.view(torch.int16))
    ref, slack = _bilinear64(x, H, W, None, None)
    worst, frac = check16(out, ref, dtype, 0, 1.0, ref - slack, ref + slack, what=f"upsample {h}x{w}->{H}x{W}")
    _report(f"upsample {dtype} {h}x{w}->{H}x{W}", worst, frac)


# (n_in, n_out) whose fp32 position of the last output, RN(RN((n_in - 1) / (n_out - 1)) * (n_out - 1)), is one ulp below
# n_in - 1
LANDS_BELOW = {(97, 149), (72, 278), (2, 42), (5, 42)}


def _fp32_last_pos(n_in, n_out):
    return float(np.float32(np.float32(n_in - 1) / np.float32(n_out - 1)) * np.float32(n_out - 1))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("h,w,H,W", [(1, 1, 5, 7), (1, 6, 4, 11), (6, 1, 11, 4), (5, 6, 1, 9), (5, 6, 9, 1), (5, 6, 1, 1),
                                     (97, 3, 149, 3), (72, 5, 278, 5), (2, 6, 42, 6), (2, 5, 42, 42)])
@pytest.mark.parametrize("with_pe", [False, True])
def test_upsample_bilinear_edges(ops, dtype, h, w, H, W, with_pe):
    """Axes of length 1 in or out, and sizes whose last row (last column) the kernel's fp32 position RN(RN((h-1)/(H-1))
    * (H-1)) puts one ulp below h - 1: it then blends rows h - 2 and h - 1 with ly = 1 - 2^-k instead of copying row
    h - 1."""
    g = torch.Generator(device="cuda").manual_seed(h * 7 + w * 5 + H * 3 + W)
    C = 32
    x = torch.randn(2, h, w, C, device="cuda", generator=g).to(dtype)
    tx, ty = _pe_tables(H, W, C, g) if with_pe else (None, None)
    out = ops.upsample_bilinear(x, H, W, tx, ty)
    torch.cuda.synchronize()
    ref, slack = _bilinear64(x, H, W, tx, ty)
    worst, frac = check16(out, ref, dtype, 0, 1.0, ref - slack, ref + slack, what=f"upsample {h}x{w}->{H}x{W}")
    _report(f"upsample edge {dtype} {h}x{w}->{H}x{W} pe={with_pe}", worst, frac)
    for n_in, n_out in ((h, H), (w, W)):          # the cases meant to land below the last input row still do
        if (n_in, n_out) in LANDS_BELOW:
            assert _fp32_last_pos(n_in, n_out) < n_in - 1, (n_in, n_out)
    if h > 1 and H > h and W == w:
        # the last output row is input row h - 1 (+ the table row).  With W == w the horizontal blend is a copy, so the
        # output is hy x[h-2] + ly x[h-1] (+ t), 2 (3) roundings: off x[h-1] (+ t) by <= dy |x[h-2] - x[h-1]| (dy as in
        # `_bilinear64`) + 2^-23 (|x[h-2]| + |x[h-1]|) (+ 2^-24 of the sum)
        last = x[:, h - 1].double()
        if tx is not None:
            last = last + torch.cat([tx.double()[None].expand(2, W, C // 2), ty.double()[H - 1].expand(2, W, C // 2)], -1)
        dy = 2.0 ** -23 * (h - 1) + 2.0 ** -25
        sl = (2 * dy + 2.0 ** -23) * (x[:, h - 2].double().abs() + x[:, h - 1].double().abs()) + U24 * last.abs()
        check16(out[:, -1], last, dtype, 0, 1.0, last - sl, last + sl, what="last row = input row h - 1")


# ------------------------------------------------------------------------------------------------- dpt tails (fp32 out)
TAIL_SHAPES = [(2, 37, 50), (1, 16, 8), (3, 5, 3), (1, 100, 131), (1, 518, 518)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("NB,H,W", TAIL_SHAPES)
@pytest.mark.parametrize("OC,mode", [(2, 0), (4, 1), (8, 2)])
def test_dpt_tail_fused(ops, dtype, NB, H, W, OC, mode):
    """conv3x3 128 -> 32 on the tensor cores (2^-20 of its magnitude sum Sz), + bias, ReLU, then the fp32 1x1: 32 fmaf
    (32 * 2^-24 = 2^-19 of |f| @ |w2| + |b2|) -> |o - o64| <= (2^-19 + 2^-20) A <= 2^-18 A with A = |w2| @ Sz + |b2|."""
    g = torch.Generator(device="cuda").manual_seed(H * W + OC)
    x = torch.randn(NB, H, W, 128, device="cuda", generator=g).to(dtype)
    wt = (torch.randn(32, 128, 3, 3, device="cuda", generator=g) / math.sqrt(128 * 9)).to(dtype)
    b = torch.randn(32, device="cuda", generator=g) * 0.1
    w2 = torch.randn(OC, 32, device="cuda", generator=g) / math.sqrt(32) * 3
    b2 = torch.randn(OC, device="cuda", generator=g) * 0.5
    wp = wt.permute(0, 2, 3, 1).reshape(32, 9 * 128).contiguous()
    main, conf = ops.dpt_tail_fused(x, wp, b, w2, b2, mode)
    torch.cuda.synchronize()
    xd = x.double().permute(0, 3, 1, 2)
    z = F.conv2d(xd, wt.double(), b.double(), padding=1)
    sz = F.conv2d(xd.abs(), wt.double().abs(), b.double().abs(), padding=1)
    f = F.relu(z).permute(0, 2, 3, 1)
    o64 = f @ w2.double().t() + b2.double()
    A = sz.permute(0, 2, 3, 1) @ w2.double().abs().t() + b2.double().abs()
    _report(f"dpt_tail_fused {dtype} {NB}x{H}x{W} mode {mode}",
            _check_tail(main, conf, o64, A, mode, 2.0 ** -18, f"fused tail {NB}x{H}x{W} mode {mode}"))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("NB,H,W", [(2, 9, 11), (1, 518, 518)])
@pytest.mark.parametrize("OC,mode", [(2, 0), (4, 1), (8, 2)])
def test_dpt_tail(ops, dtype, NB, H, W, OC, mode):
    """1x1 32 -> OC in fp32: 32 sequential fmaf from the bias -> |o - o64| <= 32 * 2^-24 A = 2^-19 A."""
    g = torch.Generator(device="cuda").manual_seed(29 + H)
    x = (torch.randn(NB, H, W, 32, device="cuda", generator=g) * 2).to(dtype)
    w = torch.randn(OC, 32, device="cuda", generator=g) / 2
    b = torch.randn(OC, device="cuda", generator=g) * 0.5
    main, conf = ops.dpt_tail(x, w, b, mode)
    torch.cuda.synchronize()
    o64 = x.double() @ w.double().t() + b.double()
    A = x.double().abs() @ w.double().abs().t() + b.double().abs()
    _report(f"dpt_tail {dtype} {NB}x{H}x{W} mode {mode}",
            _check_tail(main, conf, o64, A, mode, 2.0 ** -19, f"tail {NB}x{H}x{W} mode {mode}"))


def _one_hot_tail_inputs(dtype, vals):
    """Inputs for which o is exact: channel 0 of x carries `vals`, the 1x1 (and conv) weights pick it with weight 1, every
    other weight and bias is 0 - the sums then add exact zeros."""
    n = vals.numel()
    x = torch.zeros(1, 1, n, 128, device="cuda", dtype=dtype)
    x[0, 0, :, 0] = vals.to(dtype)
    return x


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fused", [False, True])
def test_dpt_tail_expm1_near_zero_and_overflow(ops, dtype, fused):
    """sign * expm1(|o|) keeps its relative accuracy near 0 (expm1f: <= 2 ulp, 2^-22 |r|; exp(o) - 1 would be off by
    2^-24 absolute, thousands of ulp at o = 2^-20), exp(o) and 1 + exp(o) within 2^-22 relative, and o above
    log(FLT_MAX) = 88.72 gives inf at exactly those positions."""
    vals = torch.cat([2.0 ** -torch.arange(1, 24, dtype=torch.float64, device="cuda"),
                      torch.tensor([0.0, 3.0, 40.0, 88.0, 89.0, 100.0, 65000.0 if dtype == torch.float16 else 1e30],
                                   dtype=torch.float64, device="cuda")])
    for mode, OC in ((0, 2), (1, 4)):
        x = _one_hot_tail_inputs(dtype, vals)
        o_exact = x[0, 0, :, 0].double()
        w2 = torch.zeros(OC, 32, device="cuda")
        w2[:, 0] = 1.0
        b2 = torch.zeros(OC, device="cuda")
        if fused:
            wp = torch.zeros(32, 9 * 128, device="cuda", dtype=dtype)
            wp[0, 4 * 128] = 1.0                   # centre tap, channel 0 -> conv channel 0
            main, conf = ops.dpt_tail_fused(x, wp, torch.zeros(32, device="cuda"), w2, b2, mode)
        else:
            main, conf = ops.dpt_tail(x[..., :32].contiguous(), w2, b2, mode)
        torch.cuda.synchronize()
        o = o_exact.view(1, 1, -1, 1).expand(1, 1, o_exact.numel(), OC - 1)
        ref = torch.exp(o) if mode == 0 else torch.expm1(o)
        fin = torch.isfinite(ref) & (ref < 3.0e38)
        assert torch.equal(torch.isinf(main), ~fin), f"mode {mode}: inf positions differ"
        w = check32(main[fin], ref[fin], ref[fin].abs(), 2.0 ** -22, what=f"mode {mode} activation")
        cref = 1 + torch.exp(o_exact.view(1, 1, -1))
        cfin = cref < 3.0e38
        assert torch.equal(torch.isinf(conf), ~cfin)
        wc = check32(conf[cfin], cref[cfin], cref[cfin], 2.0 ** -22 + U24, what=f"mode {mode} conf")
        _report(f"tail exact-o {dtype} fused={fused} mode {mode}", w, wc)


# -------------------------------------------------------------------------------------------- pure permutation kernels
def _random_bits(shape, dtype, g):
    """Random 16-bit patterns (NaN and inf encodings included) as `dtype`."""
    b = torch.randint(-32768, 32768, shape, device="cuda", generator=g, dtype=torch.int32).to(torch.int16)
    flat = b.view(-1)
    specials = [0x7C00, 0xFC00, 0x7E00, 0x7F80, 0xFF80, 0x7FC0, 0x0001, 0x8000]
    for i, s in enumerate(specials):
        if i < flat.numel():
            flat[(i * 7919) % flat.numel()] = s - 65536 if s >= 32768 else s
    return b.view(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("k", [2, 4])
@pytest.mark.parametrize("NB,h,w,C", [(2, 5, 7, 64), (1, 1, 1, 8), (1, 2, 3, 16), (3, 37, 26, 256)])
def test_deconv_shuffle_bit_exact(ops, dtype, k, NB, h, w, C):
    g = torch.Generator(device="cuda").manual_seed(NB * h * w + C + k)
    y = _random_bits((NB * h * w, k * k * C), dtype, g)
    out = ops.deconv_shuffle(y, NB, h, w, C, k)
    torch.cuda.synchronize()
    # y[(n, yy, xx), (dy k + dx) C + c] -> out[n, k yy + dy, k xx + dx, c]
    ref = y.view(torch.int16).view(NB, h, w, k, k, C).permute(0, 1, 3, 2, 4, 5).reshape(NB, h * k, w * k, C)
    assert torch.equal(out.view(torch.int16), ref)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("NB,h,w,C", [(2, 37, 37, 64), (2, 6, 8, 64), (1, 1, 1, 64), (1, 2, 3, 64), (2, 5, 4, 8),
                                      (1, 36, 26, 128)])
def test_im2col3x3_s2_bit_exact(ops, dtype, NB, h, w, C):
    g = torch.Generator(device="cuda").manual_seed(NB + h * 100 + w + C)
    x = _random_bits((NB, h, w, C), dtype, g)
    A, ho, wo = ops.im2col3x3_s2(x)
    torch.cuda.synchronize()
    assert (ho, wo) == ((h - 1) // 2 + 1, (w - 1) // 2 + 1)
    # A[(n, oy, ox), (ky 3 + kx) C + c] = x[n, 2 oy + ky - 1, 2 ox + kx - 1, c], +0 outside
    xp = F.pad(x.view(torch.int16), (0, 0, 1, 1, 1, 1))
    iy = (2 * torch.arange(ho, device="cuda"))[:, None] + torch.arange(3, device="cuda")[None]
    ix = (2 * torch.arange(wo, device="cuda"))[:, None] + torch.arange(3, device="cuda")[None]
    ref = xp[:, iy][:, :, :, ix]                   # [NB, ho, 3, wo, 3, C]
    ref = ref.permute(0, 1, 3, 2, 4, 5).reshape(NB * ho * wo, 9 * C)
    assert torch.equal(A.view(torch.int16), ref)


# ---------------------------------------------------------------------------------------------------------- col2im
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("NB,h,w,C", [(2, 5, 6, 64), (1, 36, 26, 256), (1, 72, 52, 128), (2, 1, 7, 64), (2, 6, 1, 64),
                                      (1, 1, 1, 64), (3, 4, 5, 8)])
def test_col2im_k4s2p1(ops, dtype, NB, h, w, C):
    """out = bias + (<= 4 taps) in fp32: 4 roundings of partial sums <= 4 2^-24 of the magnitude sum - the output must be
    RN16 of a point of that interval (0 steps outside it)."""
    g = torch.Generator(device="cuda").manual_seed(43 + h * w + C)
    Y = torch.randn(NB * h * w, 16 * C, device="cuda", generator=g).to(dtype)
    bias = torch.randn(C, device="cuda", generator=g)
    out = ops.col2im_k4s2p1(Y, bias, NB, h, w, C)
    torch.cuda.synchronize()
    Yd = Y.double().view(NB, h, w, 4, 4, C)
    full = torch.zeros(NB, 2 * h + 2, 2 * w + 2, C, dtype=torch.float64, device="cuda")
    mag = torch.zeros_like(full)
    for ky in range(4):                            # out[2 iy - 1 + ky, 2 ix - 1 + kx] += Y[iy, ix, ky, kx]
        for kx in range(4):
            full[:, ky:ky + 2 * h:2, kx:kx + 2 * w:2] += Yd[:, :, :, ky, kx]
            mag[:, ky:ky + 2 * h:2, kx:kx + 2 * w:2] += Yd[:, :, :, ky, kx].abs()
    ref = full[:, 1:2 * h + 1, 1:2 * w + 1] + bias.double()
    mag = mag[:, 1:2 * h + 1, 1:2 * w + 1] + bias.double().abs()
    slack = 4 * U24 * mag
    worst, frac = check16(out, ref, dtype, 0, 0.01, ref - slack, ref + slack, what=f"col2im {NB}x{h}x{w}x{C}")
    _report(f"col2im {dtype} {NB}x{h}x{w}x{C}", worst, frac)


# ----------------------------------------------------------------------------------------------------- layernorm16
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C", [64, 128, 256])
@pytest.mark.parametrize("rows", [1, 7, 1001])
@pytest.mark.parametrize("offset", [0.0, 300.0])
def test_layernorm16(ops, dtype, C, rows, offset):
    """One warp per row, PER = C / 32 values per lane.
      mean: PER - 1 sequential adds + 5 shuffle levels, / C exact (a power of 2): |dm| <= (PER + 4) 2^-24 mean|x|
      var:  d = x - m rounds (2^-24), squares (2^-24), PER - 1 + 5 adds of positive terms; + eps (2^-24); rsqrtf
            (2^-22): |drstd| / rstd <= (PER + 8) 2^-25 + 2^-22  (the error dm only enters var at second order)
      y = (x - m) rstd w + b: 3 roundings of the product chain + 1 of the add
      |y - y64| <= |w| rstd (|dm| + |x - m| (drstd + 3 2^-24)) + 2^-24 (|y| + |b|)
    With the +300 offset dm is ~2^-14.6 of a standard deviation of 2: the kernel's mean is the first thing to go."""
    PER = C // 32
    g = torch.Generator(device="cuda").manual_seed(41 + C + rows)
    x = (torch.randn(rows, C, device="cuda", generator=g) * 2 + offset + 0.5).to(dtype)
    w = torch.rand(C, device="cuda", generator=g) + 0.5
    b = torch.randn(C, device="cuda", generator=g)
    out = ops.layernorm16(x, w, b)
    torch.cuda.synchronize()
    xd = x.double()
    m = xd.mean(-1, keepdim=True)
    d = xd - m
    rstd = 1.0 / torch.sqrt((d * d).mean(-1, keepdim=True) + 1e-5)
    ref = d * rstd * w.double() + b.double()
    dm = (PER + 4) * U24 * xd.abs().mean(-1, keepdim=True)
    drstd = (PER + 8) * 2.0 ** -25 + 2.0 ** -22
    slack = w.double().abs() * rstd * (dm + d.abs() * (drstd + 3 * U24)) + U24 * (ref.abs() + b.double().abs())
    worst, frac = check16(out, ref, dtype, 0, 1.0, ref - slack, ref + slack, what=f"layernorm16 C={C} rows={rows}")
    _report(f"layernorm16 {dtype} C={C} rows={rows} offset={offset}", worst, frac)
    if offset == 0.0:                              # without the cancellation the fp32 value sits within ~2^-20 of y
        assert frac <= 0.05, f"{frac:.2%} of the elements are not RN16(ref)"


# --------------------------------------------------------------------------------------- channel_mean, se_scale_add
SE_SHAPES = [(1, 288, 288), (2, 288, 208), (3, 24, 16)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("NB,h,w", SE_SHAPES)
def test_channel_mean(ops, dtype, NB, h, w):
    """Grid (G = min(max(hw / 64, 1), 296), NB), 256 / C = 2 threads per channel per CTA: each thread sums
    n_t = ceil(hw / (2 G)) values sequentially (n_t 2^-24 of its magnitude sum), scales by RN(1 / hw) (2 roundings), and
    2 G atomic adds meet in the output (each <= 2^-24 of the running sum <= mean|x|):
    |mean - mean64| <= (n_t + 2 + 2 G) 2^-24 mean|x|."""
    C = 128
    hw = h * w
    G = min(max(hw // 64, 1), 296)
    n_t = -(-hw // (2 * G))
    g = torch.Generator(device="cuda").manual_seed(59 + hw)
    x = (torch.randn(NB, h, w, C, device="cuda", generator=g) + 0.3).to(dtype)
    mean = ops.channel_mean(x)
    torch.cuda.synchronize()
    xd = x.double().view(NB, hw, C)
    worst = check32(mean, xd.mean(1), xd.abs().mean(1), (n_t + 2 + 2 * G) * U24, what=f"channel_mean {NB}x{h}x{w}")
    _report(f"channel_mean {dtype} {NB}x{h}x{w}", worst)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("NB,h,w", SE_SHAPES)
@pytest.mark.parametrize("R", [4, 16])
@pytest.mark.parametrize("alpha", [0.01, 1.0])
def test_se_scale_add(ops, dtype, NB, h, w, R, alpha):
    """hid = relu(b1 + w1 @ mean): C = 128 fmaf (C 2^-24 of |w1| @ |mean| + |b1|); a = b2 + w2 @ hid: R fmaf
    (R 2^-24 of its magnitude sum) + |w2| @ (the hidden error); s = alpha / (1 + expf(-a)): sigmoid' <= 1/4, expf 2^-22,
    the add and the division 2^-24 each -> |ds| <= alpha (da / 4 + 2^-21 sigmoid); y = y0 + cx s: 2 roundings.
    |y - y64| <= |cx| |ds| + 2^-23 (|cx s| + |y|), as an interval around the float64 value."""
    C = 128
    g = torch.Generator(device="cuda").manual_seed(61 + h * w + R)
    y0 = torch.randn(NB, h, w, C, device="cuda", generator=g).to(dtype)
    cx = torch.randn(NB, h, w, C, device="cuda", generator=g).to(dtype)
    mean = torch.randn(NB, C, device="cuda", generator=g) * 0.5
    w1 = torch.randn(R, C, device="cuda", generator=g) / 8
    b1 = torch.randn(R, device="cuda", generator=g)
    w2 = torch.randn(C, R, device="cuda", generator=g)
    b2 = torch.randn(C, device="cuda", generator=g)
    out = ops.se_scale_add(y0, cx, mean, w1, b1, w2, b2, alpha)
    torch.cuda.synchronize()
    md, w1d, b1d, w2d, b2d = (t.double() for t in (mean, w1, b1, w2, b2))
    a1 = md @ w1d.t() + b1d
    e1 = C * U24 * (md.abs() @ w1d.abs().t() + b1d.abs())
    hid = F.relu(a1)
    a2 = hid @ w2d.t() + b2d
    e2 = R * U24 * (hid.abs() @ w2d.abs().t() + b2d.abs()) + e1 @ w2d.abs().t()
    sig = torch.sigmoid(a2)
    s = (alpha * sig)[:, None, None, :]
    ds = (alpha * (e2 / 4 + 2.0 ** -21 * sig))[:, None, None, :]
    cxd = cx.double()
    ref = y0.double() + cxd * s
    slack = cxd.abs() * ds + 2.0 ** -23 * ((cxd * s).abs() + ref.abs())
    worst, frac = check16(out, ref, dtype, 0, 1.0, ref - slack, ref + slack, what=f"se_scale_add {NB}x{h}x{w} R={R}")
    _report(f"se_scale_add {dtype} {NB}x{h}x{w} R={R} alpha={alpha}", worst, frac)
    assert frac <= 0.01, f"{frac:.2%} of the elements are not RN16(ref)"


# ---------------------------------------------------------------------------------------------------------- skinny GEMM
def _act64(z, act):
    return {0: lambda t: t, 1: F.gelu, 2: F.relu, 4: F.silu}[act](z)


SKINNY = [(1, 9, 8), (7, 1000, 264), (8, 6144, 16), (9, 1000, 2048), (17, 9, 8192), (32, 6144, 2048), (20, 1000, 16),
          (32, 9, 264)]
OPTS = [(True, True, True), (False, False, False), (True, False, True), (False, True, False)]     # bias, gamma, resid


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,N,K", SKINNY)
@pytest.mark.parametrize("act", [0, 1, 2, 4])
def test_skinny_gemm(ops, dtype, M, N, K, act):
    """Lane l of a warp accumulates 8 k of every 256-k stage (8 ceil(K / 256) sequential fmaf), 5 shuffle levels reduce
    the 32 lanes: |z - z64| <= (8 ceil(K / 256) + 6) 2^-24 S, S = |x| @ |W|^T + |b|.  GELU / SiLU: slope <= 1.13 and their
    own erff / expf error (<= 2^-21 |z|); ReLU exact; gamma and resid one rounding each.
    |out - ref| <= (u + 2^-20) (1.13 |gamma| S + |resid|),  u = (8 ceil(K / 256) + 6) 2^-24."""
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N + K + act)
    u = (8 * -(-K // 256) + 6) * U24
    worst = 0.0
    for use_b, use_g, use_r in OPTS:
        xfull = torch.randn(M, K + 12, device="cuda", generator=g) * 2
        x = xfull[:, 4:4 + K]                                  # ldx = K + 12 > K, 16-byte aligned start
        w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(dtype)
        b = torch.randn(N, device="cuda", generator=g) if use_b else None
        gam = torch.rand(N, device="cuda", generator=g) + 0.5 if use_g else None
        rfull = torch.randn(M, N + 5, device="cuda", generator=g)
        res = rfull[:, 3:3 + N] if use_r else None            # strided resid (ldr = N + 5)
        out = ops.skinny_gemm(x, w, b, act=act, gamma=gam, resid=res)
        torch.cuda.synchronize()
        xd, wd = x.double(), w.double()
        z = xd @ wd.t() + (b.double() if use_b else 0.0)
        S = xd.abs() @ wd.abs().t() + (b.double().abs() if use_b else 0.0)
        ref = _act64(z, act)
        gd = gam.double() if use_g else torch.ones(N, dtype=torch.float64, device="cuda")
        ref = ref * gd
        scale = 1.13 * gd.abs() * S
        if use_r:
            ref = ref + res.double()
            scale = scale + res.double().abs()
        worst = max(worst, check32(out, ref, scale, u + 2.0 ** -20,
                                   what=f"skinny M={M} N={N} K={K} act={act} b/g/r={use_b}/{use_g}/{use_r}"))
    _report(f"skinny_gemm {dtype} M={M} N={N} K={K} act={act}", worst)


# -------------------------------------------------------------------------------------------------- small attention
@pytest.mark.parametrize("N", [1, 2, 31, 32, 33, 64, 196])
def test_small_attention(ops, N):
    """fp32 throughout, one warp per query row, lane j takes keys j, j + 32, ...:
      s = fmaf chain over d = 128 (2^-17 of scale sum |q||k|), * RN(scale) (2 roundings: 2^-23 |s|), expf(s - m) (the
      subtraction 2^-24 |s - m|, expf 2^-22) -> weight error d_ij;
      l: ceil(N / 32) sequential adds + 5 levels; P V: N sequential fmaf (N 2^-24 of P @ |V|); acc * (1 / l): 2 roundings.
      |O - O64| <= (P d) @ |V| + |O| (sum P d + (ceil(N / 32) + 8) 2^-24) + N 2^-24 P @ |V|."""
    B, H, d = 3, 16, 128
    g = torch.Generator(device="cuda").manual_seed(37 + N)
    sd = math.sqrt(8.0)                         # logits q.k / sqrt(128) of standard deviation ~8
    qkv = torch.randn(B * N, 3 * H * d, device="cuda", generator=g)
    qkv[:, :2 * H * d] *= sd
    out = ops.small_attention(qkv, B, N, H, d)
    torch.cuda.synchronize()
    q, k, v = qkv.double().view(B, N, 3, H, d).permute(2, 0, 3, 1, 4)
    scale = d ** -0.5
    s = q @ k.transpose(-1, -2) * scale
    p = torch.softmax(s, -1)
    o64 = p @ v
    dd = (d * U24 * scale * (q.abs() @ k.abs().transpose(-1, -2)) + 2.0 ** -23 * s.abs()
          + U24 * (s - s.amax(-1, keepdim=True)).abs() + 2.0 ** -22)
    pd = p * dd
    va = v.abs()
    bound = pd @ va + o64.abs() * (pd.sum(-1, keepdim=True) + (-(-N // 32) + 8) * U24) + N * U24 * (p @ va)

    def flat(t):
        return t.transpose(1, 2).reshape(B * N, H * d)

    o64, bound = flat(o64), flat(bound)
    err = (out.double() - o64).abs()
    ratio = (err / bound).max().item()
    assert torch.isfinite(out).all() and ratio <= 1.0, f"N={N}: worst {ratio:.3g} x bound"
    _report(f"small_attention N={N}", ratio)


def test_small_attention_rejects_more_keys_than_shared_memory_holds(ops):
    qkv = torch.zeros(197, 3 * 16 * 128, device="cuda")
    with pytest.raises(ValueError):
        ops.small_attention(qkv, 1, 197, 16, 128)


# -------------------------------------------------------------------------------- one-launch camera head, by phases
# The hi + lo split of an fp32 activation (cam_split) leaves |x - hi - lo| <= 2^-22 |x| (+ 2^-25 absolute where lo is an
# fp16 subnormal) / 2^-16 |x| (bf16); the products with the 16-bit weights are exact, the tensor cores accumulate in
# fp32 (2^-20), the 8 warps' partial tiles meet in 8 sequential fp32 adds (2^-21) and the bias adds once:
#   |z - z64| <= (u_split + 2^-19) (|x| @ |W|^T + |b|)  (+ fp16: 2^-25 sum_k |W|)
# SiLU / GELU: slope <= 1.13 and their own expf / erff error (<= 2^-21 |z|): rel u_split + 2^-18 on 1.13 x that scale.
U_SPLIT_X = {torch.float16: 2.0 ** -22, torch.bfloat16: 2.0 ** -16}


@pytest.fixture(scope="module")
def camera():
    from oracle import weights
    from iggt_official_b200.models.vggt import VGGT
    sd = weights.make_state_dict(3, "stress", prefixes=("camera_head.",))
    m = VGGT()
    m.load_state_dict(sd, strict=False)
    m.eval().to("cuda")
    return m.camera_head


def _ln64(x, w, b, eps):
    """float64 LayerNorm over the last dim and the scale of the kernel's fp32 one (one warp per 2048-row: 16 iterations
    of 4-term partial sums + 5 shuffle levels for the mean and the variance, rsqrtf 2^-22, 4 roundings of the output):
    |y - y64| <= 2^-19 (|w| rstd (mean|x| + |x - m|) + |y| + |b|)."""
    m = x.mean(-1, keepdim=True)
    d = x - m
    rstd = 1.0 / torch.sqrt((d * d).mean(-1, keepdim=True) + eps)
    wa = w.abs() if w is not None else 1.0
    y = d * rstd * (w if w is not None else 1.0) + (b if b is not None else 0.0)
    scale = wa * rstd * (x.abs().mean(-1, keepdim=True) + d.abs()) + y.abs() + (b.abs() if b is not None else 0.0)
    return y, scale


def _gemm64(x, xs, W, b, dtype):
    """z64 = x @ W^T + b, and the scale of its allowance: |x| @ |W|^T + |b| + (the input's own error scale xs) @ |W|^T."""
    Wd = W.double()
    z = x @ Wd.t() + (b.double() if b is not None else 0.0)
    s = x.abs() @ Wd.abs().t() + (b.double().abs() if b is not None else 0.0)
    if xs is not None:
        s = s + xs @ Wd.abs().t()
    if dtype == torch.float16:                     # 2^-25 absolute per subnormal lo, relative to u_split = 2^-22
        s = s + 2.0 ** -3 * Wd.abs().sum(1)
    return z, s


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,S", [(1, 1), (1, 8), (1, 9), (2, 8)])       # M = 1, 8 (8-row kernel), 9, 16 (16-row kernel)
def test_camera_head_phases(ops, camera, dtype, B, S):
    M = B * S
    g = torch.Generator(device="cuda").manual_seed(M * 3 + S)
    tok = torch.randn(M, 2048, device="cuda", generator=g) * 1.5 + 0.2
    pk = camera._packed(dtype, tok.device)
    out, ws = ops.camera_head(pk["cstruct"], pk, tok, B, S, 1, dtype, return_workspace=True)
    torch.cuda.synchronize()
    D = 2048
    f = ws[:M * (15 * D + 1024 + 16) * 4].view(torch.float32)
    parts, o = {}, 0
    for name, n in (("pt", D), ("ptn", D), ("e", D), ("x", D), ("o", D), ("mod", 3 * D), ("qkv", 3 * D), ("f", 4 * D),
                    ("hdn", 1024), ("pred", 16)):
        parts[name] = f[o:o + M * n].view(M, n)
        o += M * n
    u = U_SPLIT_X[dtype]
    rel_ln, rel_mm, rel_act = 2.0 ** -19, u + 2.0 ** -19, u + 2.0 ** -18
    dbl = lambda t: t.double()
    res = {}
    # pt = token_norm(tokens), ptn = adaln_norm(pt) (no affine, eps 1e-6), each from its exact fp32 input
    ref, sc = _ln64(dbl(tok), dbl(pk["tok_w"]), dbl(pk["tok_b"]), 1e-5)
    res["pt"] = check32(parts["pt"], ref, sc, rel_ln, what="pt")
    ref, sc = _ln64(dbl(parts["pt"]), None, None, 1e-6)
    res["ptn"] = check32(parts["ptn"], ref, sc, rel_ln, what="ptn")
    # e = SiLU(embed_pose(empty)): K = 16 (9 weights + zero padding), the first iteration reads the empty token
    z, sc = _gemm64(dbl(pk["empty16"]).expand(M, 16), None, pk["emb_w"], pk["emb_b"], dtype)
    res["e"] = check32(parts["e"], F.silu(z), 1.13 * sc, rel_act, what="e")
    # mod = Linear(e): N = 6144, no LayerNorm
    z, sc = _gemm64(dbl(parts["e"]), None, pk["mod_w"], pk["mod_b"], dtype)
    res["mod"] = check32(parts["mod"], z, sc, rel_mm, what="mod")
    # o = the last block's token attention from the surviving qkv: one warp per (row, head), lane = 4 dims: q.k in 4
    # products + 5 levels (9 2^-24 of scale sum |q||k|), * RN(128^-0.5) (2^-23 |s|), expf(s - m) (2^-24 |s - m| + 2^-22);
    # S sequential adds of l and of o (fmaf), o * (1 / l)
    qkv = dbl(parts["qkv"]).view(B, S, 3, 16, 128).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    scale = 128 ** -0.5
    s = q @ k.transpose(-1, -2) * scale
    p = torch.softmax(s, -1)
    o64 = p @ v
    dd = 9 * U24 * scale * (q.abs() @ k.abs().transpose(-1, -2)) + 2.0 ** -23 * s.abs() \
        + U24 * (s - s.amax(-1, keepdim=True)).abs() + 2.0 ** -22
    pd = p * dd
    bound = pd @ v.abs() + o64.abs() * (pd.sum(-1, keepdim=True) + (S + 3) * U24) + S * U24 * (p @ v.abs())
    flat = lambda t: t.transpose(1, 2).reshape(M, D)
    ratio = ((dbl(parts["o"]) - flat(o64)).abs() / flat(bound)).max().item()
    assert ratio <= 1.0, f"attention phase: worst {ratio:.3g} x bound"
    res["o"] = ratio
    # hdn = GELU(pose_branch.fc1(trunk_norm(x))) from the final x: the LayerNorm runs in the kernel's staging (2^-19 of
    # its scale per input element, carried through |W|)
    y, ysc = _ln64(dbl(parts["x"]), dbl(pk["trk_w"]), dbl(pk["trk_b"]), 1e-5)
    z, sc = _gemm64(y, ysc, pk["pb1_w"], pk["pb1_b"], dtype)
    res["hdn"] = check32(parts["hdn"], F.gelu(z), 1.13 * sc, rel_act, what="hdn")
    # pred = pose_branch.fc2(hdn): N = 9, one ragged 16-column tile; columns 9..15 stay the zeroed padding
    z, sc = _gemm64(dbl(parts["hdn"]), None, pk["pb2_w"], pk["pb2_b"], dtype)
    res["pred"] = check32(parts["pred"][:, :9], z, sc, rel_mm, what="pred")
    assert torch.equal(parts["pred"][:, 9:], torch.zeros_like(parts["pred"][:, 9:]))
    # out = activate_pose(pred) of the (only) iteration: ReLU on the FoV columns, bit for bit
    pred = parts["pred"][:, :9]
    assert torch.equal(out[-1], torch.cat([pred[:, :7], torch.relu(pred[:, 7:])], -1))
    _report(f"camera phases {dtype} M={M}", *(f"{k}={v:.3g}" for k, v in res.items()))
