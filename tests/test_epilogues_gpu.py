"""Element-by-element tests of the GEMM, implicit-GEMM convolution and LayerNorm epilogues (GPU), including every
epilogue option the model calls, against float64 statements computed from the same 16-bit operands.

Every element is held to its own scale (tests/ulp_bounds.py), not to the tensor's maximum.  The common allowance:

ACC = 2^-20 of the element's magnitude sum (|A| @ |W|^T + |b|).  A correct fp32-accumulating kernel can differ from
the exact sum by its rounding errors; each add rounds by at most 2^-24 of a partial sum, and the partial sums are
bounded by the magnitude sum.  Summed over K terms of random sign these errors stay near 2^-24 of the magnitude sum
whatever K is, so 2^-20 leaves a factor 16 for the order the tensor cores and the stream-K reduce-adds choose.  16-bit
outputs may be RN16 of any value inside that interval (`around`); on top of that they are allowed 1 ulp, and only a
small share of the elements may differ from RN16 of the exact value (FRAC): the reordered fp32 sum flips a rounding
only for the elements that lie within its error of a 16-bit rounding midpoint.  Rounding toward zero, or a lost
rounding point, is off in tens of percent of the elements.

Measured on an H100 80GB HBM3 (400 W power limit): no element beyond its interval (0 ulp) in any case; the largest error
/ bound of an fp32 output 0.70 (stream-K, K = 4096); the largest shares off RN16, at K = 1024: fp16 0.52 %, bf16 0.06 %
(GELU epilogue: fp16 1.05 %, bf16 0.17 %, where a flip of the 16-bit GELU input also moves the output).  FRAC is about
twice those.

The worst value of each check (ulps, share off RN, error / bound) is printed, so a run with -s reports the margins.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from launch_refs import ACC, FRAC, FRAC_GELU, GELU_ERR
from launch_refs import act_interval as _act_interval
from launch_refs import gelu64 as _gelu64
from launch_refs import gemm64 as _gemm64
from launch_refs import gemm_plan as _plan
from ulp_bounds import around, check16, check32, rn16, ulp16

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


@pytest.fixture(scope="module")
def ops():
    from iggt_official_b200 import ops as _ops
    return _ops


def _report(what, value):
    print(f"[bound] {what}: {value}")


def _operands(g, M, N, K, dtype, lda_pad=0, ldw_pad=0):
    """A [M,K] and W [N,K] 16-bit, as column slices of wider tensors when a pad is given (offset 8 columns: TMA wants
    16-byte aligned bases)."""
    a_full = torch.randn(M, K + lda_pad, device="cuda", generator=g).to(dtype)
    w_full = (torch.randn(N, K + ldw_pad, device="cuda", generator=g) / math.sqrt(K)).to(dtype)
    a = a_full[:, 8:8 + K] if lda_pad else a_full
    w = w_full[:, 8:8 + K] if ldw_pad else w_full
    return a, w


# --------------------------------------------------------------------------------------------- 1. shapes and strides
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,N,K", [(1, 8, 8), (1, 1024, 1024), (127, 72, 392), (129, 136, 72), (1102, 1024, 1024),
                                   (127, 8, 1024), (129, 1024, 8), (1102, 72, 392), (1102, 136, 1024),
                                   (127, 1024, 72)])
def test_store16_shapes_and_strides(ops, dtype, M, N, K):
    """A and W are column slices (lda > K, ldw > K), out is a column slice of a NaN-filled buffer (ldo > N); K % 64 != 0
    and M < 128 leave TMA boxes partly outside the operands, N = 8 runs the BN = 64 tile.  For fp16 one row of A is
    +-60000, so about a quarter of that row's outputs overflow: they must be +-inf exactly where RN16(ref) is."""
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    a, w = _operands(g, M, N, K, dtype, lda_pad=24, ldw_pad=16)
    big = M // 2
    if dtype == torch.float16:
        a[big] = torch.where(torch.rand(K, device="cuda", generator=g) < 0.5, -60000.0, 60000.0).to(dtype)
    bias = torch.randn(N, device="cuda", generator=g)
    buf = torch.full((M, N + 24), float("nan"), device="cuda", dtype=dtype)
    out = buf[:, 8:8 + N]
    ops.gemm_store16(a, w, bias, out=out)
    torch.cuda.synchronize()
    acc, mag = _gemm64(a, w)
    y = acc + bias.double()
    lo, hi = around(y, ACC * (mag + bias.double().abs()))
    _report(f"store16 {dtype} {M}x{N}x{K}", check16(out, y, dtype, 1, FRAC[dtype], lo, hi, what="store16"))
    assert torch.isnan(buf[:, :8]).all() and torch.isnan(buf[:, 8 + N:]).all(), "wrote outside the output slice"
    if dtype == torch.float16:
        assert torch.isinf(out[big]).sum() > N // 10, "the overflow row should overflow"


# ------------------------------------------------------------------------------------ 2. activations and the addend
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("act", [1, 2, 3])
def test_store16_activations(ops, dtype, act):
    """act 1: GELU of the 16-bit rounded Linear output (the autocast rounding point, gemm.cuh); 2 ReLU; 3 LeakyReLU(0.01).
    An fp32 flip of the 16-bit GELU input moves GELU by up to 1.13 input ulps, many output ulps where GELU is small:
    the interval admits both roundings of the input, so the GELU case keeps 1 ulp and only its share off RN is larger."""
    M, N, K = 600, 1024, 1024
    g = torch.Generator(device="cuda").manual_seed(100 + act)
    a, w = _operands(g, M, N, K, dtype)
    bias = torch.randn(N, device="cuda", generator=g)
    out = ops.gemm_store16(a, w, bias, act=act)
    torch.cuda.synchronize()
    acc, mag = _gemm64(a, w)
    y = acc + bias.double()
    ref, lo, hi = _act_interval(act, y, ACC * (mag + bias.double().abs()), dtype)
    ulps, frac = (1, FRAC_GELU[dtype]) if act == 1 else (1, FRAC[dtype])
    _report(f"store16 act={act} {dtype}", check16(out, ref, dtype, ulps, frac, lo, hi, what=f"store16 act={act}"))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("act", [0, 2])
def test_store16_addend_column_slice(ops, dtype, act):
    """out = act(A W^T + b) + addend[row % add_rows] with add_rows < M and the addend a column slice (add_ld > N), as
    the DPT and part heads call it (positional embeddings added to a projection)."""
    M, N, K, R = 3 * 361, 256, 512, 361
    g = torch.Generator(device="cuda").manual_seed(200 + act)
    a, w = _operands(g, M, N, K, dtype)
    bias = torch.randn(N, device="cuda", generator=g)
    add = torch.randn(R, N + 16, device="cuda", generator=g).to(dtype)[:, 8:8 + N]
    out = ops.gemm_store16(a, w, bias, act=act, addend=add, add_rows=R)
    torch.cuda.synchronize()
    acc, mag = _gemm64(a, w)
    y = acc + bias.double()
    ref, lo, hi = _act_interval(act, y, ACC * (mag + bias.double().abs()), dtype)
    ad = add.double().repeat(3, 1)
    # the addend joins after the activation in fp32: one more rounding of 2^-24 of |act(y) + addend|
    s2 = 2.0 ** -23 * (ref.abs() + ad.abs())
    _report(f"store16 addend act={act} {dtype}", check16(out, ref + ad, dtype, 1, FRAC[dtype], lo + ad - s2, hi + ad + s2,
                                                         what="store16 addend"))


# ------------------------------------------------------------------------------------- 3. exhaustive activations
def _all_finite(dtype):
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    x = bits.view(dtype)
    x = x[torch.isfinite(x.float())]
    pad = (-x.numel()) % 64
    x = torch.cat([x, torch.zeros(pad, dtype=dtype)])
    return torch.cat([x.view(-1, 64), torch.full((1, 64), float("nan"), dtype=dtype)]).cuda()   # last row: NaN


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("act", [2, 3])
def test_relu_leaky_exhaustive(ops, dtype, act):
    """W = I64 and zero bias, A = every finite 16-bit value (and a NaN row): each output is act(x) of one input.  It
    must be bit-identical to RN16 of torch's fp32 op (NaN kept, the sign of zero ignored)."""
    A = _all_finite(dtype)
    out = ops.gemm_store16(A, torch.eye(64, device="cuda", dtype=dtype), torch.zeros(64, device="cuda"), act=act)
    torch.cuda.synchronize()
    ref = torch.relu(A.float()) if act == 2 else F.leaky_relu(A.float(), 0.01)
    _report(f"exhaustive act={act} {dtype}", check16(out, ref.double(), dtype, 0, 0.0, what=f"exhaustive act={act}"))


@pytest.mark.parametrize("dtype", DTYPES)
def test_gelu_exhaustive(ops, dtype):
    """The gelu_fast error bound (csrc/ptx.cuh), pinned over every finite 16-bit input:
        |out - gelu64(x)| <= 0.5 ulp16 + |x| / 2 * (1.5e-7 + 2^-24 + 2^-22)
    (Abramowitz-Stegun erf, the fp32 complement 1 - erf, ex2.approx).  A future GELU has to meet the same pin.
    Known limitation, not a failure: in the negative tail (x <~ -4) bf16 outputs differ from exact-erf GELU by many bf16
    ulps while staying inside this absolute bound, because the fp32 complement 1 - erf is quantised at 2^-24."""
    A = _all_finite(dtype)
    out = ops.gemm_store16(A, torch.eye(64, device="cuda", dtype=dtype), torch.zeros(64, device="cuda"), act=1)
    torch.cuda.synchronize()
    x = A.double()
    ref = _gelu64(x)
    delta = x.abs() / 2 * GELU_ERR
    bound = 0.5 * ulp16(ref.abs() + delta, dtype) + delta
    fin = torch.isfinite(x)
    assert torch.isnan(out[~fin]).all()
    err = (out.double() - ref).abs()[fin]
    ratio = (err / bound[fin]).max().item()
    _report(f"gelu exhaustive {dtype} err/bound", ratio)
    assert ratio <= 1.0, ratio


# ------------------------------------------------------------------ 4. gemm_resid32(round_out16=True), both schedules
@pytest.mark.parametrize("dtype", DTYPES)
def test_resid32_round_out16_whole_tiles(ops, dtype):
    """Whole tiles: x + gamma * RN16(acc + b) per element, the autocast Linear output before LayerScale.  On the same
    data the unrounded statement x + gamma * (acc + b) must fail the same per-element criterion for most elements, so
    the rounding point is observable at this tolerance."""
    M, N, K = 300, 1024, 1024
    assert _plan(M, N, K)["stream_k"] == 0
    g = torch.Generator(device="cuda").manual_seed(300)
    a, w = _operands(g, M, N, K, dtype)
    bias = torch.randn(N, device="cuda", generator=g)
    gamma = torch.rand(N, device="cuda", generator=g) + 0.5
    x = torch.randn(M, N, device="cuda", generator=g)
    x0 = x.double()
    ops.gemm_resid32(a, w, x, bias, gamma, round_out16=True)
    torch.cuda.synchronize()
    acc, mag = _gemm64(a, w)
    y = acc + bias.double()
    s = ACC * (mag + bias.double().abs())
    _, lo, hi = _act_interval(0, y, s, dtype)
    r, r_lo, r_hi = (rn16(t, dtype).double() for t in (y, lo, hi))
    g64 = gamma.double()
    ref = x0 + g64 * r
    # after the rounding only two fp32 operations remain (gamma multiply, reduce-add): 2^-23 of |x| + gamma |r|
    scale = x0.abs() + g64 * r.abs()
    _report(f"resid32 round16 {dtype}", check32(x, ref, scale, 2.0 ** -22, x0 + g64 * r_lo, x0 + g64 * r_hi,
                                               what="resid32 round_out16"))
    unrounded = x0 + g64 * y
    frac_bad = ((x.double() - unrounded).abs() > ACC * (x0.abs() + g64 * (mag + bias.double().abs()))).double().mean()
    _report(f"resid32 round16 {dtype}: share failing the unrounded statement", float(frac_bad))
    assert frac_bad > 0.5, float(frac_bad)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,N,K", [(34 * 128, 1024, 128), (2 * 1374, 1024, 4096)])   # 2nd: the C2 fc2 shape (2 views)
def test_resid32_round_out16_stream_k(ops, dtype, M, N, K):
    """Stream-K: partial tiles are reduce-added without the 16-bit rounding (the deviation DESIGN.md §2 documents), so
    the statement is the unrounded x + gamma * (acc + b)."""
    assert _plan(M, N, K)["stream_k"] == 1
    g = torch.Generator(device="cuda").manual_seed(400)
    a, w = _operands(g, M, N, K, dtype)
    bias = torch.randn(N, device="cuda", generator=g)
    gamma = torch.rand(N, device="cuda", generator=g) + 0.5
    x = torch.randn(M, N, device="cuda", generator=g)
    x0 = x.double()
    ops.gemm_resid32(a, w, x, bias, gamma, round_out16=True)
    torch.cuda.synchronize()
    acc, mag = _gemm64(a, w)
    g64 = gamma.double()
    ref = x0 + g64 * (acc + bias.double())
    scale = x0.abs() + g64 * (mag + bias.double().abs())
    _report(f"resid32 stream-K {dtype} {M}x{N}x{K}", check32(x, ref, scale, ACC, what="resid32 stream-K"))


# ------------------------------------------------------------------------- 5. gamma / bias absent, store32 with GELU
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("with_bias", [False, True])
def test_resid32_without_gamma(ops, dtype, with_bias):
    """The track head's residual GEMMs: gamma=None (= 1), bias given or not."""
    M, N, K = 257, 384, 392
    g = torch.Generator(device="cuda").manual_seed(500)
    a, w = _operands(g, M, N, K, dtype)
    bias = torch.randn(N, device="cuda", generator=g) if with_bias else None
    x = torch.randn(M, N, device="cuda", generator=g)
    x0 = x.double()
    ops.gemm_resid32(a, w, x, bias=bias)
    torch.cuda.synchronize()
    acc, mag = _gemm64(a, w)
    b64 = bias.double() if with_bias else torch.zeros(N, device="cuda", dtype=torch.float64)
    _report(f"resid32 no gamma bias={with_bias} {dtype}",
            check32(x, x0 + acc + b64, x0.abs() + mag + b64.abs(), ACC, what="resid32 gamma=None"))


@pytest.mark.parametrize("dtype", DTYPES)
def test_store32_gelu(ops, dtype):
    """gemm_store32(act=1): GELU of the fp32 value, with no 16-bit rounding before it (track head ffeat)."""
    M, N, K = 300, 520, 392
    g = torch.Generator(device="cuda").manual_seed(600)
    a, w = _operands(g, M, N, K, dtype)
    bias = torch.randn(N, device="cuda", generator=g)
    out = ops.gemm_store32(a, w, bias, act=1)
    torch.cuda.synchronize()
    acc, mag = _gemm64(a, w)
    y = acc + bias.double()
    lo, hi = around(y, ACC * (mag + bias.double().abs()))
    g_lo, g_hi = _gelu64(lo), _gelu64(hi)
    # on top of the accumulation interval: the gelu_fast error |y| / 2 * GELU_ERR and the fp32 store, 2^-24 |y|
    rel = GELU_ERR / 2 + 2.0 ** -24
    _report(f"store32 gelu {dtype}", check32(out, _gelu64(y), y.abs(), rel, torch.minimum(g_lo, g_hi),
                                             torch.maximum(g_lo, g_hi), what="store32 act=1"))


# ------------------------------------------------------------------------------------------ 6. conv_nhwc epilogues
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Cout", [64, 192])
@pytest.mark.parametrize("taps", [1, 9])
@pytest.mark.parametrize("case", ["gelu", "leaky", "resid2_relu"])
def test_conv_epilogues(ops, dtype, Cout, taps, case):
    """act=1 (GELU of the 16-bit rounded conv output, the same code path as the GEMM), act=3 (LeakyReLU 0.01), and
    resid + resid2 + act_post=2: relu(conv + b + resid + resid2) rounded once, the DPT fusion block.  NB = 3 images of
    13 x 21 pixels: both spatial tile counts ragged against the 8 x 16 tile; Cout = 192 leaves half an N tile."""
    NB, H, W, Cin = 3, 13, 21, 64
    g = torch.Generator(device="cuda").manual_seed(700 + Cout + taps)
    ks = 3 if taps == 9 else 1
    x = torch.randn(NB, H, W, Cin, device="cuda", generator=g).to(dtype)
    w = (torch.randn(Cout, Cin, ks, ks, device="cuda", generator=g) / math.sqrt(Cin * taps)).to(dtype)
    bias = torch.randn(Cout, device="cuda", generator=g)
    wp = w.permute(0, 2, 3, 1).reshape(Cout, taps * Cin).contiguous()
    r1 = r2 = None
    if case == "resid2_relu":
        r1 = torch.randn(NB, H, W, Cout, device="cuda", generator=g).to(dtype)
        r2 = torch.randn(NB, H, W, Cout, device="cuda", generator=g).to(dtype)
        out = ops.conv_nhwc(x, wp, bias, resid=r1, resid2=r2, act_post=2, taps=taps)
    else:
        out = ops.conv_nhwc(x, wp, bias, act=1 if case == "gelu" else 3, taps=taps)
    torch.cuda.synchronize()
    x64 = x.double().permute(0, 3, 1, 2)
    conv = F.conv2d(x64, w.double(), padding=ks // 2).permute(0, 2, 3, 1)
    mag = F.conv2d(x64.abs(), w.double().abs(), padding=ks // 2).permute(0, 2, 3, 1)
    y = conv + bias.double()
    s = ACC * (mag + bias.double().abs())
    if case == "resid2_relu":
        y = y + r1.double() + r2.double()
        s = s + 2.0 ** -23 * (r1.double().abs() + r2.double().abs() + y.abs())   # two more fp32 adds
        ref, lo, hi = _act_interval(2, y, s, dtype)
        ulps, frac = 1, FRAC[dtype]
    else:
        ref, lo, hi = _act_interval(1 if case == "gelu" else 3, y, s, dtype)
        ulps, frac = (1, FRAC_GELU[dtype]) if case == "gelu" else (1, FRAC[dtype])
    _report(f"conv {case} {dtype} Cout={Cout} taps={taps}",
            check16(out, ref, dtype, ulps, frac, lo, hi, what=f"conv {case}"))


# ----------------------------------------------------------------------------------------------------- 7. layernorm
_OUT = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}


@pytest.mark.parametrize("out_kind", ["f16", "bf16", "f32"])
@pytest.mark.parametrize("C", [1024, 2048])
@pytest.mark.parametrize("case", ["remap_pitch", "no_affine", "offset300"])
def test_layernorm(ops, out_kind, C, case):
    """remap_pitch: rows [g*rows_in + in_off, +rows_out) of an input with row pitch ldx > C go to rows
    [g*out_rows_per_group + out_off, +rows_out) of a NaN-filled output; every other row stays NaN.
    no_affine: w = b = None, eps = 1e-6 (camera head adaln_norm).
    offset300: 300 + randn - a variance from E[x^2] - E[x]^2 would lose ~2^-24 * 300^2 / var = 5e-3 of it.
    Error allowance: the fp32 mean of values near |x| carries ~2^-24 |x| of absolute error per add, moving x - mean by
    2^-20 (|x| + |mean|) at most, which the normalisation scales by rstd |w|; the bias adds 2^-24 |b|."""
    od = _OUT[out_kind]
    g = torch.Generator(device="cuda").manual_seed(800 + C)
    G, rin, off, rout, orpg, ooff = (3, 50, 5, 45, 52, 4) if case == "remap_pitch" else (1, 300, 0, 300, 300, 0)
    pitch = C + 64 if case == "remap_pitch" else C
    xb = torch.randn(G * rin, pitch, device="cuda", generator=g) * 3 + 1
    if case == "offset300":
        xb = xb / 3 + 299
    x = xb[:, 32:32 + C] if case == "remap_pitch" else xb
    w = b = None
    eps = 1e-6 if case != "offset300" else 1e-5
    if case != "no_affine":
        w = torch.rand(C, device="cuda", generator=g) + 0.5
        b = torch.randn(C, device="cuda", generator=g)
    out = torch.full((G * orpg, C), float("nan"), device="cuda", dtype=od)
    ops.layernorm(x, w, b, eps, out, groups=G, rows_out=rout, rows_in=rin, in_off=off, out_rows_per_group=orpg,
                  out_off=ooff)
    torch.cuda.synchronize()
    src = x.view(G, rin, C)[:, off:off + rout].reshape(-1, C).double()
    mean = src.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(((src - mean) ** 2).mean(-1, keepdim=True) + eps)
    w64 = w.double() if w is not None else torch.ones(C, device="cuda", dtype=torch.float64)
    b64 = b.double() if b is not None else torch.zeros(C, device="cuda", dtype=torch.float64)
    ref = (src - mean) * rstd * w64 + b64
    s = 2.0 ** -20 * (src.abs() + mean.abs()) * rstd * w64.abs() + 2.0 ** -22 * b64.abs()
    rows = (torch.arange(G, device="cuda")[:, None] * orpg + ooff + torch.arange(rout, device="cuda")[None]).reshape(-1)
    got = out[rows]
    keep = torch.ones(G * orpg, dtype=torch.bool, device="cuda")
    keep[rows] = False
    assert torch.isnan(out[keep].float()).all(), "rows outside the remap target changed"
    if od == torch.float32:
        _report(f"layernorm {case} C={C} f32", check32(got, ref, s / 2.0 ** -20, 2.0 ** -20, what=f"layernorm {case}"))
    else:
        # offset300: the fp32 mean of values near 300 is off by a visible share of an fp16 ulp of the normalised value,
        # so RN flips are expected in a few percent of the elements (measured: fp16 4.7 %, bf16 0.83 %); the
        # per-element interval still bounds every one of them
        frac = 0.1 if case == "offset300" else FRAC[od]
        lo, hi = around(ref, s)
        _report(f"layernorm {case} C={C} {out_kind}", check16(got, ref, od, 1, frac, lo, hi, what=f"layernorm {case}"))
