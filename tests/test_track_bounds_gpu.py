"""Element-by-element tests of the track-head kernels (csrc/track.cu) against float64 statements of the same operations,
computed from the exact 16-bit / fp32 inputs each kernel received, fp16 and bf16: avgpool2_nhwc, sample_bilinear_nhwc,
corr_sample, track_input, layernorm_rows, and the flash-attention kernel at the update transformer's shapes.

Every allowance is derived next to its assert from the kernel's arithmetic.  The library is built without
--use_fast_math, so every fp32 operation rounds once (u = 2^-24 relative; a * b + c may contract to one fma, which only
removes a rounding), division is IEEE, and sinf / cosf (2 ulp), tanf (4 ulp) and rsqrtf (2 ulp) keep the maximum
errors of the CUDA C Programming Guide's single-precision function table.  A sequential fp32 sum of n terms is within
n u of the sum of its partial sums' magnitudes; each level of a shuffle tree adds u of the sum of the magnitudes.
16-bit outputs go through `check16` against the interval a correct kernel's fp32 arithmetic can reach, fp32 outputs
through `check32` (tests/ulp_bounds.py).  The worst error / bound and the share of elements that are not RN16 of the
float64 value are printed (run with -s).

Two CPU tests pin the float64 statements of sample_bilinear_nhwc and corr_sample to the plain-PyTorch statements of the
reference's formulation in tests/emu_ops.py (grid_sample, the full correlation volume).
"""
import math

import pytest
import torch

import emu_ops
from ulp_bounds import check16, check32, check_attn_bound1

DTYPES = [torch.float16, torch.bfloat16]
U24 = 2.0 ** -24
SECOND_ORDER = 1.0 + 2.0 ** -20          # products of two first-order rounding errors, on top of every derived slack
gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def ops():
    from iggt_official_b200 import ops as _ops
    return _ops


def _report(what, *values):
    print(f"[bound] {what}: " + " ".join(f"{v:.3g}" if isinstance(v, float) else str(v) for v in values))


# ------------------------------------------------------------------------------------------------------ avgpool2_nhwc
def _avgpool64(x):
    """Exact mean of every 2 x 2 window (floor: an odd last row / column is dropped) and the slack of the kernel's fp32
    sum ((t00 + t01) + t10) + t11: each addition rounds once, by at most u of its partial sum; x 0.25 is exact (the
    means stay far from the fp32 subnormals)."""
    NB, H, W, C = x.shape
    Ho, Wo = H // 2, W // 2
    v = x[:, :2 * Ho, :2 * Wo].double().reshape(NB, Ho, 2, Wo, 2, C)
    t = [v[:, :, dy, :, dx] for dy in (0, 1) for dx in (0, 1)]          # the kernel's order
    p1 = t[0] + t[1]
    p2 = p1 + t[2]
    p3 = p2 + t[3]
    return p3 * 0.25, SECOND_ORDER * U24 * (p1.abs() + p2.abs() + p3.abs()) * 0.25


def _pool_input(case, dtype, g):
    if case == "odd":                                  # floor drops row 34 and column 76
        return torch.randn(3, 35, 77, 128, device="cuda", generator=g).to(dtype)
    if case == "c2":
        return torch.randn(4, 11, 9, 2, device="cuda", generator=g).to(dtype)
    if case == "grid_stride":                          # level 0 of a 518^2 scene: 8.5M threads, 16x the 132*16 CTA cap
        return torch.randn(8, 259, 259, 128, device="cuda", generator=g).to(dtype)
    if dtype == torch.float16:                         # near 65504: the sum (~2.6e5) overflows any 16-bit accumulator
        mag = 65504.0 - torch.rand(2, 6, 8, 16, device="cuda", generator=g) * 1000.0
        sign = torch.where(torch.arange(16, device="cuda") % 2 == 0, 1.0, -1.0)
        return (mag * sign).to(dtype)
    # bf16 over 2^-100 .. 2^100: the fp32 sum absorbs the smaller taps of a window
    e = torch.randint(-100, 101, (2, 6, 8, 16), device="cuda", generator=g).double()
    return (torch.randn(2, 6, 8, 16, device="cuda", generator=g).double() * torch.exp2(e)).to(dtype)


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", ["odd", "c2", "grid_stride", "extreme"])
def test_avgpool2(ops, dtype, case):
    g = torch.Generator(device="cuda").manual_seed(11)
    x = _pool_input(case, dtype, g)
    out = ops.avgpool2_nhwc(x)
    torch.cuda.synchronize()
    ref, slack = _avgpool64(x)
    assert out.shape == ref.shape and torch.isfinite(out.float()).all()
    # every value RN16 of a point of [ref - slack, ref + slack]; fp32 holds the sum of four 16-bit values exactly unless
    # their exponents spread over more than 24 - 11 bits, so an element is off RN16(ref) only by a double rounding
    _report(f"avgpool2 {dtype} {case}",
            *check16(out, ref, dtype, 0, 0.002, ref - slack, ref + slack, what=f"avgpool2 {case}"))


# ------------------------------------------------------------------------------------------------ sample_bilinear_nhwc
def _sample64(x, coords):
    """Bilinear value in float64 at the kernel's clamped coordinate (fminf / fmaxf to [0, W-1] x [0, H-1] are exact),
    x1 = min(x0 + 1, W - 1), and the magnitude sum sum_i |w_i v_i|."""
    NB, H, W, C = x.shape
    cx = coords[..., 0].clamp(0, W - 1).double()
    cy = coords[..., 1].clamp(0, H - 1).double()
    x0, y0 = cx.floor(), cy.floor()
    fx, fy = (cx - x0)[..., None], (cy - y0)[..., None]
    x0, y0 = x0.long(), y0.long()
    x1, y1 = (x0 + 1).clamp(max=W - 1), (y0 + 1).clamp(max=H - 1)
    n = torch.arange(NB, device=x.device)[:, None]
    xd = x.double()
    terms = [xd[n, y0, x0] * ((1 - fx) * (1 - fy)), xd[n, y0, x1] * (fx * (1 - fy)),
             xd[n, y1, x0] * ((1 - fx) * fy), xd[n, y1, x1] * (fx * fy)]
    return sum(terms), sum(t.abs() for t in terms)


def _sample_case(case, g, dev):
    NB, H, W, C = {"c128": (2, 30, 41, 128), "c72": (2, 30, 41, 72), "h1": (2, 1, 37, 128),
                   "w1": (2, 29, 1, 128)}[case]
    x = torch.randn(NB, H, W, C, device=dev, generator=g)
    R = 64
    coords = torch.rand(NB, R, 2, device=dev, generator=g) * torch.tensor([W + 5.0, H + 5.0], device=dev) - 3.0
    coords[:, 8:16] = coords[:, 8:16].round()                            # integer positions: fx = fy = 0
    special = torch.tensor([[0.0, 0.0], [W - 1.0, H - 1.0], [W - 1.0, 0.5], [0.25, H - 1.0], [-2.5, -0.75],
                            [W + 1.25, H + 3.5], [-7.0, H - 1.5], [W - 1.5, -0.125]], device=dev)
    coords[:, :8] = special
    return x, coords


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", ["c128", "c72", "h1", "w1"])
def test_sample_bilinear(ops, dtype, case):
    g = torch.Generator(device="cuda").manual_seed(21)
    x, coords = _sample_case(case, g, "cuda")
    x = x.to(dtype)
    out = ops.sample_bilinear_nhwc(x, coords)
    torch.cuda.synchronize()
    ref, mag = _sample64(x, coords)
    # 1 - fx and 1 - fy round once each, and (v00 (1-fx) + v01 fx) (1-fy) + (v10 (1-fx) + v11 fx) fy puts at most four
    # more roundings (products, fmas, sums) on any term's path: 6 u of sum |w_i v_i|, 8 u allowed
    _report(f"sample_bilinear {dtype} {case}", check32(out, ref, mag, 8 * U24, what=f"sample_bilinear {case}"))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", ["c128", "h1", "w1"])
def test_sample_reference_matches_grid_sample(dtype, case):
    """CPU: the float64 statement above is grid_sample(align_corners=True, padding_mode="border") at the same points,
    which is what emu_ops.sample_bilinear_nhwc (the reference's formulation) computes.  grid_sample gets there through
    a normalised coordinate x * RN(2 / max(W - 1, 1)) - 1 and back, in fp32: four roundings of values up to
    max(W - 1, 1), so a position error of <= 4 u max(W, H) pixels, which moves the value by at most that times the
    difference of two taps (<= 2 max|x|); the interpolation itself is within 8 u of sum |w_i v_i| as above."""
    g = torch.Generator().manual_seed(22)
    x, coords = _sample_case(case, g, "cpu")
    x = x.to(dtype)
    got = emu_ops.sample_bilinear_nhwc(x, coords)
    ref, mag = _sample64(x, coords)
    H, W = x.shape[1:3]
    scale = mag + max(H, W) * x.double().abs().max()                   # 8 u max(H, W) max|x| = 4 u max(H, W) 2 max|x|
    _report(f"grid_sample vs fp64 {dtype} {case}", check32(got, ref, scale, 8 * U24, what=f"grid_sample {case}"))


# -------------------------------------------------------------------------------------------------------- corr_sample
S32 = float(torch.tensor(1 / math.sqrt(128), dtype=torch.float32))       # the kernel's constant, RN32(1/sqrt(128))


def _corr64(levels, targets, coords, B, N, S):
    """The reference's formulation in float64: per level, the full correlation volume <target, fmap> / sqrt(128) of each
    row (b, n, s) with image b * S + s, sampled bilinearly with zero padding at coords / 2^l + (i - 4, j - 4), output
    index i * 9 + j (i moves along x).  An axis of size 1 samples pixel 0 at every offset: the reference normalises
    with 2 / max(size - 1, 1) and grid_sample(align_corners=True) maps every coordinate of a size-1 axis back to 0.
    Returns the values [rows, 567] and the slack of the kernel's fp32 arithmetic:
      * <t, f>: four products per lane (an fma chain, 4 roundings) and a 5-level shuffle tree: 9 u sum |t f| (A);
      * x RN32(1/sqrt(128)): the constant's relative error |S32 sqrt(128) - 1| and the product's rounding u;
      * the bilinear combination: 1 - fx, 1 - fy and at most four more roundings on each tap's path, 6 u.
    Also returns max |corr| over each row's level volume (per output), which bounds a sampling-position error's effect."""
    rows = B * N * S
    dev = targets.device
    r = torch.arange(rows, device=dev)
    img = (r // (N * S)) * S + r % S
    t = targets.double()
    d = torch.arange(-4, 5, device=dev, dtype=torch.float64)
    s = 1 / math.sqrt(128)
    ds = abs(S32 * math.sqrt(128) - 1.0)
    vals, slacks, vmaxs = [], [], []
    for lvl, fm in enumerate(levels):
        NI, H, W, C = fm.shape
        f = fm.double().reshape(NI, H * W, C)
        vol = (f @ t.T)[img, :, r]                                      # [rows, H*W]: row r against its own image
        avol = (f.abs() @ t.abs().T)[img, :, r]
        cx = coords[:, 0].double() / 2 ** lvl                          # exact, like the kernel's product by 2^-l
        cy = coords[:, 1].double() / 2 ** lvl
        X = torch.zeros(rows, 9, 1, device=dev, dtype=torch.float64) if W == 1 else cx[:, None, None] + d[None, :, None]
        Y = torch.zeros(rows, 1, 9, device=dev, dtype=torch.float64) if H == 1 else cy[:, None, None] + d[None, None, :]
        X, Y = X.expand(rows, 9, 9).reshape(rows, 81), Y.expand(rows, 9, 9).reshape(rows, 81)
        x0, y0 = X.floor(), Y.floor()
        fx, fy = X - x0, Y - y0
        val = torch.zeros(rows, 81, device=dev, dtype=torch.float64)
        slack = torch.zeros_like(val)
        for dx, dy, w in ((0, 0, (1 - fx) * (1 - fy)), (1, 0, fx * (1 - fy)), (0, 1, (1 - fx) * fy), (1, 1, fx * fy)):
            xi, yi = (x0 + dx).long(), (y0 + dy).long()
            ok = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
            p = yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)
            c = torch.where(ok, vol.gather(1, p), 0.0)
            a = torch.where(ok, avol.gather(1, p), 0.0)
            val += w * c * s
            slack += w * (9 * U24 * a * S32 + c.abs() * s * (ds + U24 + 6 * U24))
        vals.append(val)
        slacks.append(slack * SECOND_ORDER)
        vmaxs.append((vol.abs().amax(1, keepdim=True) * s).expand(rows, 81))
    return torch.cat(vals, 1), torch.cat(slacks, 1), torch.cat(vmaxs, 1)


def _corr_coords(rows, H, W, g, dev):
    """Level-0 pixels: windows over every border of every level, integer and half-integer positions, the corners."""
    c = torch.rand(rows, 2, device=dev, generator=g) * torch.tensor([W + 12.0, H + 12.0], device=dev) - 6.0
    c[1::3] = c[1::3].round()
    c[2::3] = c[2::3].floor() + 0.5
    c[0] = torch.tensor([0.0, 0.0])
    c[1] = torch.tensor([W - 1.0, H - 1.0])
    c[2] = torch.tensor([-4.5, H + 3.5])
    return c


def _pyramid(ops, fm0, g):
    """The track head's pyramid: LayerNorm(128) of the 16-bit maps, then six 2 x 2 average pools."""
    w = torch.rand(128, device="cuda", generator=g) + 0.5
    b = torch.randn(128, device="cuda", generator=g) * 0.1
    levels = [ops.layernorm16(fm0, w, b, eps=1e-5)]
    for _ in range(6):
        levels.append(ops.avgpool2_nhwc(levels[-1]))
    return levels


# (H, W) of level 0 and ldo: 64 x 64 ends at 1 x 1, 64 x 130 at 1 x 2 and 130 x 64 at 2 x 1 (one flat axis),
# 259 x 196 at 4 x 3; ldo 567 has no padding, 576 nine zero columns
CORR_CASES = [(64, 64, 576), (64, 130, 567), (130, 64, 576), (259, 196, 567), (70, 77, 576)]


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,W,ldo", CORR_CASES)
def test_corr_sample(ops, dtype, H, W, ldo):
    g = torch.Generator(device="cuda").manual_seed(H * 1000 + W)
    B, N, S = 2, 5, 3                                   # a wrong (b, n, s) -> image b * S + s mapping reads another map
    rows = B * N * S
    fm0 = (torch.randn(B * S, H, W, 128, device="cuda", generator=g) * 3 + 1).to(dtype)
    levels = _pyramid(ops, fm0, g)
    assert [tuple(l.shape[1:3]) for l in levels][-1] == (H >> 6, W >> 6)
    targets = torch.randn(rows, 128, device="cuda", generator=g)
    coords = _corr_coords(rows, H, W, g, "cuda")
    out = ops.corr_sample(levels, targets, coords, B, N, S, ldo)
    torch.cuda.synchronize()
    assert out.shape == (rows, ldo) and not out[:, 567:].any()
    ref, slack, _ = _corr64(levels, targets, coords, B, N, S)
    # the slack covers every correct fp32 evaluation order; the fp32 error is ~2^-20 of |corr| where a 16-bit step is
    # 2^-11 (fp16) / 2^-8 (bf16), so only a few elements round differently from RN16(ref)
    _report(f"corr_sample {dtype} {H}x{W} ldo={ldo}",
            *check16(out[:, :567], ref, dtype, 0, 0.01, ref - slack, ref + slack, what=f"corr {H}x{W}"))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,W", [(64, 64), (64, 130), (130, 64)])
def test_corr_reference_matches_emu_flat_axes(dtype, H, W):
    """CPU: the float64 statement above against emu_ops.corr_sample (the reference's formulation: the full volume in
    fp32 and grid_sample with zero padding) on pyramids whose coarsest level has one or two axes of size 1.  emu works
    in fp32: its einsum may sum in any order (127 u of sum |t f| instead of 9 u: one 16-bit step at most), and
    grid_sample's coordinate normalisation moves a sampling position by up to 4 u max(H, W) pixels, which changes the
    value by at most that times the difference of two taps (2 max|corr|).  A wrong size-1 rule would zero-pad or shift
    whole windows."""
    g = torch.Generator().manual_seed(H + W)
    B, N, S = 1, 4, 2
    rows = B * N * S
    lv = [torch.randn(B * S, H, W, 128, generator=g).to(dtype)]
    for _ in range(6):
        lv.append(emu_ops.avgpool2_nhwc(lv[-1]))
    targets = torch.randn(rows, 128, generator=g)
    coords = _corr_coords(rows, H, W, g, "cpu")
    got = emu_ops.corr_sample(lv, targets, coords, B, N, S, 567)
    ref, slack, vmax = _corr64(lv, targets, coords, B, N, S)
    slack = slack + 8 * U24 * max(H, W) * vmax
    _report(f"emu corr vs fp64 {dtype} {H}x{W}",
            *check16(got, ref, dtype, 1, 0.05, ref - slack, ref + slack, what=f"emu corr {H}x{W}"))


# -------------------------------------------------------------------------------------------------------- track_input
def _track_input_case(BN, S, g):
    rows = BN * S
    base = torch.rand(BN, 1, 2, generator=g) * 60
    flow = torch.rand(BN, S, 2, generator=g) * 300 - 150               # +-150 feature pixels: arguments up to 1.5e5 rad
    flow[:, 0] = 0
    coords = (base + flow).reshape(rows, 2)
    fcorr, tfeat = torch.randn(rows, 128, generator=g), torch.randn(rows, 128, generator=g)
    pos, ref = torch.randn(BN, 388, generator=g), torch.randn(2, 388, generator=g)
    w, b = torch.rand(388, generator=g) + 0.5, torch.randn(388, generator=g) * 0.1
    return coords, fcorr, tfeat, pos, ref, w, b


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("BN,S,ldo", [(7, 4, 392), (13, 1, 388), (5, 3, 416), (64, 8, 392)])
def test_track_input(ops, dtype, BN, S, ldo):
    g = torch.Generator().manual_seed(BN * 10 + S)
    coords, fcorr, tfeat, pos, ref, w, b = _track_input_case(BN, S, g)
    rows = BN * S
    out, raw = ops.track_input(*(t.cuda() for t in (coords, fcorr, tfeat, pos, ref, w, b)), S, dtype, ldo, want_raw=True)
    torch.cuda.synchronize()
    out, raw = out.cpu(), raw.cpu()
    assert out.shape == (rows, ldo) and not out[:, 388:].any()
    # the reference's fp32 statement (base_track_predictor.py:135-160): flows, argument flow * div_term, (x + pos) + ref
    fl = coords - coords.view(BN, S, 2)[:, :1].expand(BN, S, 2).reshape(rows, 2)
    div = torch.arange(0, 64, 2, dtype=torch.float32) * (1000.0 / 64)
    s = torch.arange(rows) % S
    pos_r, ref_r = pos.repeat_interleave(S, 0), ref[(s > 0).long()]
    # channels 128..387: flow / 518 (x2), the correlation and track features - the same fp32 operations in the same order
    tail = torch.cat([fl / 518.0, fl / 518.0, fcorr, tfeat], 1)
    assert torch.equal(raw[:, 128:], (tail + pos_r[:, 128:]) + ref_r[:, 128:])
    # channels 0..127: sin / cos of the SAME fp32 argument (the kernel forms flow * (float(2m) * 15.625f), exact factor)
    emb = torch.zeros(rows, 128, dtype=torch.float64)
    for axis in (0, 1):
        arg = (fl[:, axis:axis + 1] * div).double()
        emb[:, 64 * axis:64 * axis + 64:2], emb[:, 64 * axis + 1:64 * axis + 64:2] = torch.sin(arg), torch.cos(arg)
    p1 = emb + pos_r[:, :128].double()
    want = p1 + ref_r[:, :128].double()
    # sinf / cosf within 2 ulp (<= 2^-22 |sin|), then two fp32 additions (u of each partial sum)
    slack = SECOND_ORDER * (2.0 ** -22 * emb.abs() + U24 * (p1.abs() + want.abs()))
    worst_emb = check32(raw[:, :128], want, slack, 1.0, what="flow embedding")
    # zero flow (s = 0): sin 0 = 0 and cos 0 = 1 exactly
    e0 = torch.zeros(rows, 128)
    e0[:, 1::2] = 1.0
    first = s == 0
    assert torch.equal(raw[first, :128], ((e0 + pos_r[:, :128]) + ref_r[:, :128])[first])
    # LayerNorm(388) of the kernel's own raw rows
    y, slk = _ln64_slack(raw, w, b, 1e-5, lane_terms=13)
    worst, frac = check16(out[:, :388], y, dtype, 0, 0.01, y - slk, y + slk, what="track_input LayerNorm")
    _report(f"track_input {dtype} {BN}x{S} ldo={ldo}", worst_emb, worst, frac)


# ----------------------------------------------------------------------------------------------------- layernorm_rows
def _ln64_slack(x, w, b, eps, lane_terms):
    """float64 LayerNorm of the fp32 rows x and the slack of a one-warp fp32 evaluation (per lane a sequential sum of
    `lane_terms` values, a 5-level shuffle tree):
      mean: lane_terms + 5 roundings, and the division (or the product by RN(1/C)) <= 2: dmu = (lane_terms + 7) u mean|x|;
      variance: d = x - mean32 (2 u on d^2), lane_terms + 5 roundings of the sum of d^2 >= 0, / C and + eps (2 u):
        relative (lane_terms + 9) u of var + eps; mean32 adds at most dmu^2 to it;
      rsqrtf: 2 ulp (2^-22), so r32 = r (1 +- dr), dr = (lane_terms + 9) u / 2 + 2^-22 + dmu^2 / (2 (var + eps));
      y = (x - mean32) r32 w + b: |w| r dmu from the mean, and 3 more roundings (u of |x - mean32|, the two products,
        the final fma / add u |y| + u |b|)."""
    xd = x.double()
    w, b = w.double().to(x.device), b.double().to(x.device)
    eps32 = float(torch.tensor(eps, dtype=torch.float32))             # the kernel adds the fp32 eps
    mu = xd.mean(1, keepdim=True)
    xc = xd - mu
    var = (xc * xc).mean(1, keepdim=True)
    r = 1 / torch.sqrt(var + eps32)
    y = xc * r * w + b
    dmu = (lane_terms + 7) * U24 * xd.abs().mean(1, keepdim=True)
    dr = (lane_terms + 9) * U24 / 2 + 2.0 ** -22 + dmu * dmu / (2 * (var + eps32))
    slack = w.abs() * r * (dmu + (xc.abs() + dmu) * (dr + 3 * U24)) + U24 * (y.abs() + b.abs())
    return y, slack * SECOND_ORDER


def _ln_rows(C, g, dev):
    """37 rows (not a multiple of 8), pitch C + 8: 25 rows of N(0.3, 2^2); 6 rows at a common offset of 1e4 with
    standard deviation 1 (a one-pass E[x^2] - mean^2 loses the variance there); 6 constant rows whose sums are exact."""
    big = torch.randn(37, C + 8, device=dev, generator=g) * 2 + 0.3
    big[25:31] = 1e4 + torch.randn(6, C + 8, device=dev, generator=g)
    big[31:37] = torch.tensor([3.25, -0.5, 0.0, 17.0, -1024.0, 0.125], device=dev)[:, None]
    return big


LN_WIDTHS = [1, 31, 32, 33, 128, 384, 388, 2047, 2048]


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C", LN_WIDTHS)
def test_layernorm_rows(ops, dtype, C):
    g = torch.Generator(device="cuda").manual_seed(C)
    big = _ln_rows(C, g, "cuda")
    x = big[:, 2:C + 2]                                 # an offset view with a row pitch, like delta[:, 2:C+2]
    w = torch.rand(C, device="cuda", generator=g) + 0.5
    b = torch.randn(C, device="cuda", generator=g)
    y, slack = _ln64_slack(x, w, b, 1e-5, lane_terms=-(-C // 32))
    offset = slice(25, 31)
    steady = torch.cat([torch.arange(0, 25), torch.arange(31, 37)]).cuda()
    report = []
    for mode in ("16", "32", "both"):
        ld16 = C + 3 if mode == "16" else C
        o32 = torch.full((37, C), 7.0, device="cuda") if mode != "16" else None
        o16 = torch.full((37, ld16), 7.0, dtype=dtype, device="cuda") if mode != "32" else None
        ops.layernorm_rows(x, w, b, 1e-5, out32=o32, out16=o16)
        torch.cuda.synchronize()
        if o32 is not None:
            report.append(check32(o32, y, slack, 1.0, what=f"out32 C={C} mode={mode}"))
        if o16 is not None:
            assert not o16[:, C:].any()
            # rows of N(0.3, 4) and constant rows: the fp32 error is far below a 16-bit step; the rows at 1e4 carry the
            # fp32 mean's rounding (~1e-3 of their spread), a legitimate shift that is only held to the interval
            report += list(check16(o16[steady, :C], y[steady], dtype, 0, 0.01, (y - slack)[steady],
                                   (y + slack)[steady], what=f"out16 C={C} mode={mode}"))
            report += list(check16(o16[offset, :C], y[offset], dtype, 0, 1.0, (y - slack)[offset],
                                   (y + slack)[offset], what=f"out16 C={C} mode={mode} offset rows"))
    _report(f"layernorm_rows {dtype} C={C}", *report)


# ------------------------------------------------------------------------------- attention, update-transformer shapes
HEADS, HD = 8, 48                                       # 8 heads of 48 columns, zero-padded to 64 (heads/track_head.py)


def _padded(g, rows, dtype, sd=1.0):
    t = torch.randn(rows, HEADS, 64, device="cuda", generator=g) * sd
    t[:, :, HD:] = 0
    return t.reshape(rows, HEADS * 64).to(dtype)


# (kind, num_seq, Lq, Lk) of _attn_block / _cross_block with B = 2, N = 18 (time: B * (N + 64) sequences of L = S) and
# B * S = 6 (v2p: 64 virtual queries over N points; p2v: N queries over 64 virtual tokens; sv: 64 x 64)
ATTN_CASES = ([("time", 164, L, L) for L in (1, 2, 8, 24)] + [("v2p", 6, 64, N) for N in (1, 63, 65, 300, 1024)]
              + [("p2v", 6, N, 64) for N in (1, 63, 65, 300, 1024)] + [("sv", 6, 64, 64)])


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("kind,num_seq,Lq,Lk", ATTN_CASES)
def test_attention_update_transformer(ops, dtype, split, kind, num_seq, Lq, Lk):
    if split and Lk <= 128:
        pytest.skip("one kv tile: nothing to split")
    g = torch.Generator(device="cuda").manual_seed(num_seq * 7 + Lq * 3 + Lk)
    sd = math.sqrt(8.0)                                 # logits q.k / sqrt(48) over 48 products: standard deviation 8
    W = HEADS * 64
    if Lq == Lk and kind in ("time", "sv"):            # self attention: column slices of one packed qkv, like the module
        qkv = torch.cat([_padded(g, num_seq * Lq, dtype, sd), _padded(g, num_seq * Lq, dtype, sd),
                         _padded(g, num_seq * Lq, dtype)], 1)
        q, k, v = qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:]
    else:                                               # cross attention: q alone, k and v slices of one packed kv
        q = _padded(g, num_seq * Lq, dtype, sd)
        kv = torch.cat([_padded(g, num_seq * Lk, dtype, sd), _padded(g, num_seq * Lk, dtype)], 1)
        k, v = kv[:, :W], kv[:, W:]
    out = ops.attention(q, k, v, num_seq, Lq, Lk, HEADS, scale=1.0 / math.sqrt(HD), splits=2 if split else None)
    torch.cuda.synchronize()
    assert not out.view(-1, HEADS, 64)[..., HD:].any(), "padding columns 48..63 of a head are not zero"
    # bound 1 (tests/ulp_bounds.py); the fp32 rounding of 1/sqrt(48) moves a logit by 2^-24 of itself, like the fp32
    # logits' own error, which the 2^-20 max|V| term covers
    _report(f"attention {dtype} {kind} {num_seq}x{Lq}x{Lk} split={split}",
            check_attn_bound1(out, q, k, v, num_seq, Lq, Lk, HEADS, dtype, scale=1.0 / math.sqrt(HD),
                              what=f"{kind} {num_seq}x{Lq}x{Lk}"))
