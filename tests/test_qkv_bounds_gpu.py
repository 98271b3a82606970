"""Element-by-element tests of the qkv GEMM epilogue (csrc/gemm.cuh, EPI_QKV and EPI_QKV_GATHER; launcher
`iggt_gemm_qkv`) against float64 statements computed from the same 16-bit operands and fp32 vectors, fp16 and bf16.

With qk_norm the epilogue of each 64-wide q and k head is
    u = RN16(acc + b)                                  (the autocast Linear output)
    ln = (u - mean) * rstd * w + nb                    (LayerNorm(64), eps 1e-5, two-pass, q or k affine vectors)
    rope: dims [0, 32) rotate by the y position and [32, 64) by x, each in halves of 16:
          a' = a c - b s,  b' = b c + a s             (c, s = the fp32 tables at pos_yx[row % T])
and the v columns are RN16(acc + b).  Without qk_norm all 3C columns are RN16(acc + b).

Allowances.  The library is built without --use_fast_math: every fp32 operation rounds once (u = 2^-24 relative; a
product and a sum may contract to one fma, which only removes a rounding), and rsqrtf is within 2 ulp.
* LayerNorm, from the kernel's fp32 arithmetic on the exact u:
  - mean: a sequential fp32 sum of 64 terms is within 63 u of the sum of |u_j|, so the mean is off by at most
    2^-18 mean|u|; x - mean rounds by u |d|.  Both move z by rstd times that: 2^-18 rstd |w| mean|u| (this is
    test_layernorm's 2^-20 (|u| + |mean|) term, taken at its worst case for 64 terms);
  - variance: to first order the mean's error cancels in sum (d_j^2); the 64 squares and the sum of positive terms are
    off by at most 2^-18 relative, the + eps and rsqrtf by 2^-24 + 2^-22, so rstd is within 2^-18.7 relative;
  - the products by rstd and w round by u |z w| each, + nb by u |ln|.
  Slack: 2^-18 rstd |w| mean|u| + 2^-17 |z w| + 2^-23 |ln|.
* RoPE carries slacks s_a, s_b of its inputs as |c| s_a + |s| s_b, plus one rounding of each product and of the
  sum: 2^-23 (|a c| + |b s| + |a'|).
* 16-bit outputs are checked with `check16` against RN16 of the interval [ref - slack, ref + slack]: a correct kernel's
  fp32 value lies inside it and RN16 is monotonic, so the limit is 0 steps outside the interval.  FRAC bounds the share
  of elements that are not RN16 of the float64 value; it is set from the measured share, with a factor of about 2.

§1 (exact GEMM).  A holds integers in [-128, 128] and W integers in [-64, 64] times 2^-e, the bias integers times
2^-e: every product and partial sum is a multiple of 2^-e below 2^(24-e), so the fp32 accumulation is exact in any
order and acc + b is known exactly.  e is chosen so that y is about 8 in size, where most values are not
representable in 16 bits (asserted): what remains is the epilogue's own arithmetic and the rounding point.

§2 (Gaussian operands).  The kernel's fp32 y can differ from y64 by ACC (|A| |W|^T + |b|) (ACC = 2^-20, derived in
test_epilogues_gpu.py), so an input u_j is 'ambiguous' where RN16 of the two ends of that interval differ, and can
then be off by a_j = the distance to the farther end's RN16.  dz_i/du_j = rstd (delta_ij - (1 + z_i z_j) / 64), so the
first-order effect on output i is rstd |w_i| (a_i + (1/64) sum_j a_j (1 + |z_i z_j|)).  The second-order terms are
smaller than the first-order ones by a factor of about a_j rstd |z|, below 2^-7 * 8 for |z| <= sqrt(63) and a
bf16 step: a factor 2 on the first-order term covers them.  No other element is excused.

§5 / §6 run the K|V gather instantiation on one GPU: W simulated ranks are W buffers in one allocation with guard
bands, each rank's maps point at plain device addresses (`ops.kv_gather_maps`), and the gather launches' outputs are
compared bit for bit with the plain launch and with one unsharded launch.

Measured on an H100 80GB HBM3 (700 W power limit, 1980 MHz maximum SM clock), all 119 cases in about 12 s:
* every 16-bit output within its interval (0 steps outside) in every check;
* §1: q/k not RN16 of the float64 value: fp16 at most 0.050 % (special-token rows 0.087 %, the +300 head 0.12 %),
  bf16 at most 0.010 % (special-token rows 0.045 %); v columns RN16(y) exactly.  With the rounding point removed from
  the statement 27-29 % of the elements fall outside their intervals, and 50-75 % with the other wrong statements
  (negative controls, §4);
* §2: share of ambiguous q/k inputs fp16 11-14 %, bf16 1.9-2.6 %; q/k not RN16: fp16 at most 0.52 %, bf16 at most
  0.054 %; v columns and qk_norm=False (store16): fp16 0.53 %, bf16 0.063 %;
* §5 / §6: the gathered K|V, the gather launches' qkv and the sharded q rows bit-identical to the plain and the
  unsharded launches in every case; attention at most 0.51 of bound 1.
FRAC is about twice the largest measured share.

The worst value of each check (steps outside the interval, share off RN16) is printed, so a run with -s reports the
margins.
"""
import math

import pytest
import torch

from launch_refs import ACC
from launch_refs import ln64 as _ln64
from launch_refs import qk64 as _qk64
from launch_refs import rope64 as _rope64
from launch_refs import y64 as _y64
from ulp_bounds import check16, check_attn_bound1, rn16

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
NUM_SPECIAL = 5                       # camera + 4 register tokens per view, RoPE position (0, 0)
NAN_ROWS = 3                          # NaN rows appended to the RoPE tables: a read past the valid rows shows
SENTINEL = -1                         # 0xFFFF: a NaN pattern the kernel's round-to-nearest stores never produce
# share of q/k elements not RN16 of the float64 value: about twice the largest measured (module docstring)
FRAC_EXACT = {torch.float16: 0.0025, torch.bfloat16: 0.001}
FRAC_GAUSS = {torch.float16: 0.01, torch.bfloat16: 0.0012}
FRAC_STORE16 = {torch.float16: 0.01, torch.bfloat16: 0.002}          # the store16 epilogue's (test_epilogues_gpu.py)


@pytest.fixture(scope="module")
def ops():
    from iggt_official_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def agg():
    from iggt_official_b200.models import aggregator
    assert aggregator.NUM_SPECIAL == NUM_SPECIAL
    return aggregator


def _report(what, value):
    print(f"[bound] {what}: {value}")


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _rope(agg, gh, gw):
    """The model's fp32 tables for max(gh, gw) + 1 positions with NAN_ROWS rows of NaN after them, and the model's
    int32 (y, x) positions of one view's tokens."""
    cos, sin = agg.rope_tables(max(gh, gw) + 1, "cuda")
    nan = torch.full((NAN_ROWS, 16), float("nan"), device="cuda")
    return (torch.cat([cos, nan]).contiguous(), torch.cat([sin, nan]).contiguous(),
            agg.token_positions(gh, gw, "cuda"))


def _norm_vectors(g):
    """q_norm w, b and k_norm w, b (fp32 [64]); the k vectors differ from the q ones in every element."""
    qn_w = torch.rand(64, device="cuda", generator=g) + 0.5
    qn_b = torch.randn(64, device="cuda", generator=g) * 0.5
    kn_w = torch.rand(64, device="cuda", generator=g) * 0.5 + 1.5
    kn_b = torch.randn(64, device="cuda", generator=g) * 0.5 + 2.0
    return qn_w, qn_b, kn_w, kn_b


def _exact_operands(g, M, C, K, dtype, lda_pad=0):
    """A [M, K] integers in [-128, 128] (a column slice at offset 8 of a wider tensor when lda_pad is given), W [3C, K]
    integers in [-64, 64] times 2^-e and the bias integers in [-4 * 2^e, 4 * 2^e] times 2^-e, with 2^-e chosen so that
    y = A W^T + b is about 8 in size.  Partial sums stay below K * 2^13 * 2^-e <= 2^(24-e): the fp32 accumulation is
    exact in any order."""
    e = round(math.log2(math.sqrt(K) * 74 * 37 / 8))
    assert K * 2 ** 13 <= 2 ** 24
    a_full = torch.randint(-128, 129, (M, K + lda_pad), device="cuda", generator=g).to(dtype)
    a = a_full[:, 8:8 + K] if lda_pad else a_full
    w = (torch.randint(-64, 65, (3 * C, K), device="cuda", generator=g).double() * 2.0 ** -e).to(dtype)
    bias = (torch.randint(-4 << e, (4 << e) + 1, (3 * C,), device="cuda", generator=g).double() * 2.0 ** -e).float()
    return a, w, bias


def _gauss_operands(g, M, C, K, dtype):
    """Gaussian A and W / sqrt(K); the bias rounded to 16 bit and kept in fp32, as pack_block stores it."""
    a = torch.randn(M, K, device="cuda", generator=g).to(dtype)
    w = (torch.randn(3 * C, K, device="cuda", generator=g) / math.sqrt(K)).to(dtype)
    bias = torch.randn(3 * C, device="cuda", generator=g).to(dtype).float()
    return a, w, bias


def _check(out, ref, slack, dtype, frac, what):
    """check16 of out against RN16 of [ref - slack, ref + slack], 0 steps outside; a non-finite reference (or slack)
    must be matched exactly (NaN for NaN, the same infinity)."""
    fin = torch.isfinite(ref) & torch.isfinite(slack)
    lo = torch.where(fin, ref - slack, ref)
    hi = torch.where(fin, ref + slack, ref)
    r = check16(out, ref, dtype, 0, frac, lo, hi, what=what)
    _report(what, r)
    return r


def _qkv(ops, a, w, bias, C, norm, cos, sin, pos, T, **kw):
    return ops.gemm_qkv(a, w, bias, C, qk_norm=True, qn_w=norm[0], qn_b=norm[1], kn_w=norm[2], kn_b=norm[3],
                        rope_cos=cos, rope_sin=sin, pos_yx=pos, T=T, **kw)


# ---------------------------------------------------------------------------------- 1. the epilogue, exact GEMM
GRIDS = [(2, 2, 15), (5, 7, 7), (37, 37, 8), (37, 28, 3)]     # (gh, gw, S): 28^2, 70x98, 518^2 (C2: M = 10992), 518x392


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C", [64, 192, 1024])
@pytest.mark.parametrize("gh,gw,S", GRIDS)
def test_qkv_exact_gemm(ops, agg, dtype, C, gh, gw, S):
    """The q/k epilogue on an exact acc + b.  M = S * T is never a multiple of 128 and row tiles straddle views
    (T = 9, 40, 1374, 1041); C = 64 puts q and k of one head pair in one 128-wide tile, C = 192 a tile holding q head 2
    and k head 0.  A is a column slice (lda > K); out is a column slice of a NaN-filled buffer (ldo > 3C) whose margins
    must stay NaN.  v columns are RN16(y) exactly; the special tokens' q/k are RN16 of the LayerNorm alone."""
    T, K = NUM_SPECIAL + gh * gw, 1024 if C == 1024 else 256
    M = S * T
    g = _gen(1000 * gh + 10 * gw + C)
    a, w, bias = _exact_operands(g, M, C, K, dtype, lda_pad=24)
    norm = _norm_vectors(g)
    cos, sin, pos = _rope(agg, gh, gw)
    buf = torch.full((M, 3 * C + 24), float("nan"), device="cuda", dtype=dtype)
    out = buf[:, 8:8 + 3 * C]
    _qkv(ops, a, w, bias, C, norm, cos, sin, pos, T, out=out)
    torch.cuda.synchronize()
    assert torch.isnan(buf[:, :8]).all() and torch.isnan(buf[:, 8 + 3 * C:]).all(), "wrote outside the output slice"
    y, _ = _y64(a, w, bias)
    u = rn16(y, dtype).double()
    share = (u[:, :2 * C] != y[:, :2 * C]).double().mean().item()
    _report(f"exact {dtype} C={C} {gh}x{gw} S={S}: share of q/k inputs not 16-bit", share)
    assert share > 0.5, "the rounding point would not be observable"
    tag = f"exact {dtype} C={C} {gh}x{gw} S={S}"
    _check(out[:, 2 * C:], y[:, 2 * C:], torch.zeros_like(y[:, 2 * C:]), dtype, 0.0, f"{tag} v")
    ln, s = _ln64(u[:, :2 * C], C, norm)
    ref, sr = _rope64(ln, s, cos, sin, pos, T)
    _check(out[:, :2 * C], ref, sr, dtype, FRAC_EXACT[dtype], f"{tag} q/k")
    # special tokens: position 0, where the tables hold cos = 1 and sin = 0 exactly, so RoPE is the identity
    assert (cos[0] == 1).all() and (sin[0] == 0).all()
    special = (torch.arange(M, device="cuda") % T) < NUM_SPECIAL
    _check(out[special, :2 * C], ln[special], s[special], dtype, FRAC_EXACT[dtype], f"{tag} special tokens = LN")


# ------------------------------------------------------------------------------------- 2. realistic operands
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C,gh,gw,S,K", [(1024, 37, 37, 2, 1024), (192, 5, 7, 7, 512), (64, 37, 28, 3, 1024)])
def test_qkv_gaussian(ops, agg, dtype, C, gh, gw, S, K):
    """Gaussian A and W, the bias rounded to 16 bit: the kernel's pre-LN value is RN16 of a point within
    ACC (|A| |W|^T + |b|) of y64, so inputs near a rounding midpoint are ambiguous and their head's outputs are widened
    by their first-order effect (module docstring).  v columns: the store16 bound."""
    T = NUM_SPECIAL + gh * gw
    M = S * T
    g = _gen(2000 + C + K)
    a, w, bias = _gauss_operands(g, M, C, K, dtype)
    norm = _norm_vectors(g)
    cos, sin, pos = _rope(agg, gh, gw)
    out = _qkv(ops, a, w, bias, C, norm, cos, sin, pos, T)
    torch.cuda.synchronize()
    y, mag = _y64(a, w, bias)
    sy = ACC * mag
    u = rn16(y, dtype).double()
    u_lo, u_hi = rn16(y - sy, dtype).double(), rn16(y + sy, dtype).double()
    amb = torch.maximum((u_hi - u).abs(), (u - u_lo).abs())
    tag = f"gauss {dtype} C={C} {gh}x{gw} S={S} K={K}"
    _report(f"{tag}: share of ambiguous q/k inputs", (amb[:, :2 * C] > 0).double().mean().item())
    _check(out[:, 2 * C:], y[:, 2 * C:], sy[:, 2 * C:], dtype, FRAC_STORE16[dtype], f"{tag} v")
    ref, sr = _qk64(u, C, T, norm, cos, sin, pos, amb)
    _check(out[:, :2 * C], ref, sr, dtype, FRAC_GAUSS[dtype], f"{tag} q/k")


# ------------------------------------------------------------------------------------------------------ 3. edges
@pytest.mark.parametrize("dtype", DTYPES)
def test_qkv_table_rows_constant_and_offset_heads(ops, agg, dtype):
    """Random (y, x) positions in [0, npos), y and x drawn independently, with the top row read for y and for x, and
    NaN rows after the valid ones (any read past them, or a swapped half, shows).  Row 60 of A is zero and the bias is
    constant over q head 1, so that head of row 60 has variance 0 and comes out as the rotated nb.  k head 2 has +300 in
    its bias, which a one-pass E[x^2] - E[x]^2 variance would lose."""
    C, K, T, S, npos = 192, 256, 50, 4, 8
    M = S * T
    g = _gen(3000)
    a, w, bias = _exact_operands(g, M, C, K, dtype)
    norm = _norm_vectors(g)
    cos, sin, _ = _rope(agg, npos - 1, npos - 1)
    pos = torch.randint(0, npos, (T, 2), device="cuda", generator=g, dtype=torch.int32)
    pos[NUM_SPECIAL] = torch.tensor([npos - 1, 0])
    pos[NUM_SPECIAL + 1] = torch.tensor([0, npos - 1])
    pos[NUM_SPECIAL + 2] = torch.tensor([npos - 1, npos - 1])
    pos = pos.contiguous()
    a[60] = 0
    bias[64:128] = 0.75
    bias[C + 128:C + 192] += 300.0
    out = _qkv(ops, a, w, bias, C, norm, cos, sin, pos, T)
    torch.cuda.synchronize()
    y, _ = _y64(a, w, bias)
    assert (y[60, 64:128] == 0.75).all()
    u = rn16(y, dtype).double()
    ln, s = _ln64(u[:, :2 * C], C, norm)
    assert (ln[60, 64:128] == norm[1].double()).all(), "the constant head should normalise to nb"
    ref, sr = _rope64(ln, s, cos, sin, pos, T)
    tag = f"edges {dtype}"
    _check(out[:, 2 * C:], y[:, 2 * C:], torch.zeros_like(y[:, 2 * C:]), dtype, 0.0, f"{tag} v")
    _check(out[:, :2 * C], ref, sr, dtype, FRAC_EXACT[dtype], f"{tag} q/k")
    # the interval alone: 64 elements are too few for a share
    _check(out[60:61, 64:128], ref[60:61, 64:128], sr[60:61, 64:128], dtype, 1.0, f"{tag} constant head")
    off = slice(C + 128, C + 192)
    _check(out[:, off], ref[:, off], sr[:, off], dtype, FRAC_EXACT[dtype], f"{tag} +300 head")


@pytest.mark.parametrize("dtype", DTYPES)
def test_qkv_nonfinite(ops, agg, dtype):
    """fp16: in rows 7 and 100, one q column, one k column and one v column overflow to inf at RN16 (A = 128 and
    W = 8 over the last 128 columns, which are 0 in every other row).  The q and k heads holding them are NaN in
    exactly those rows, the v column is +inf, and nothing else changes.  Both dtypes: an inf in row 50 of A makes every
    q/k head of that row NaN and its v columns +-inf (NaN where W is 0), and leaves every other row finite."""
    C, K, gh, gw, S = 192, 256, 5, 7, 4
    T = NUM_SPECIAL + gh * gw
    M = S * T
    g = _gen(4000)
    a, w, bias = _exact_operands(g, M, C, K, dtype)
    norm = _norm_vectors(g)
    cos, sin, pos = _rope(agg, gh, gw)
    hot, cols = [7, 100], [5, C + 64 + 3, 2 * C + 10]
    if dtype == torch.float16:
        a[:, K - 128:] = 0
        for r in hot:
            a[r, K - 128:] = 128
        for j in cols:
            w[j, K - 128:] = 8
    a[50, 3] = float("inf")
    out = _qkv(ops, a, w, bias, C, norm, cos, sin, pos, T)
    torch.cuda.synchronize()
    y, _ = _y64(a, w, bias)
    u = rn16(y, dtype).double()
    ref, sr = _qk64(u, C, T, norm, cos, sin, pos)
    tag = f"nonfinite {dtype}"
    _check(out[:, 2 * C:], y[:, 2 * C:], torch.zeros_like(y[:, 2 * C:]), dtype, 0.0, f"{tag} v")
    _check(out[:, :2 * C], ref, sr, dtype, FRAC_EXACT[dtype], f"{tag} q/k")
    o = out.float()
    assert torch.isnan(o[50, :2 * C]).all() and torch.isinf(o[50, 2 * C:][w[2 * C:, 3] != 0]).all()
    rest = torch.ones(M, dtype=torch.bool, device="cuda")
    rest[50] = False
    if dtype == torch.float16:
        rest[hot] = False
        bad = torch.zeros(3 * C, dtype=torch.bool, device="cuda")
        bad[0:64] = bad[C + 64:C + 128] = True
        for r in hot:
            assert torch.isnan(o[r, bad]).all() and o[r, 2 * C + 10] == float("inf")
            fin = ~bad
            fin[2 * C + 10] = False
            assert torch.isfinite(o[r, fin]).all()
    assert torch.isfinite(o[rest]).all()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("with_bias", [False, True])
def test_qkv_without_qk_norm(ops, dtype, with_bias):
    """The 24 DINOv2 blocks: qk_norm=False and no RoPE arguments; all 3C columns are the store16 epilogue,
    RN16 of a point within ACC (|A| |W|^T + |b|) of y64.  Two views of 1374 tokens, C = 1024."""
    C, K, M = 1024, 1024, 2 * 1374
    g = _gen(5000 + with_bias)
    a, w, bias = _gauss_operands(g, M, C, K, dtype)
    if not with_bias:
        bias = None
    out = ops.gemm_qkv(a, w, bias, C)
    torch.cuda.synchronize()
    y, mag = _y64(a, w, bias if with_bias else torch.zeros(3 * C, device="cuda"))
    _check(out, y, ACC * mag, dtype, FRAC_STORE16[dtype], f"no qk_norm {dtype} bias={with_bias}")


# -------------------------------------------------------------------------------------------- 4. negative controls
@pytest.mark.parametrize("dtype", DTYPES)
def test_qkv_negative_controls(ops, agg, dtype):
    """The §1 check passes on this launch, and fails against each deliberately wrong statement: LayerNorm of the
    unrounded y, RoPE with the y and x halves swapped, RoPE at the next token's position, and the q vectors on k."""
    C, K, gh, gw, S = 192, 256, 5, 7, 7
    T = NUM_SPECIAL + gh * gw
    M = S * T
    g = _gen(6000)
    a, w, bias = _exact_operands(g, M, C, K, dtype)
    norm = _norm_vectors(g)
    cos, sin, pos = _rope(agg, gh, gw)
    out = _qkv(ops, a, w, bias, C, norm, cos, sin, pos, T)[:, :2 * C]
    torch.cuda.synchronize()
    y, _ = _y64(a, w, bias)
    u = rn16(y, dtype).double()
    _check(out, *_qk64(u, C, T, norm, cos, sin, pos), dtype, FRAC_EXACT[dtype], f"control {dtype} correct")
    wrong = {
        "LN of the unrounded y": (y, norm, pos),
        "RoPE y/x halves swapped": (u, norm, pos[:, [1, 0]].contiguous()),
        "RoPE at the next token's position": (u, norm, pos.roll(-1, 0)),
        "q-norm vectors on k": (u, (norm[0], norm[1], norm[0], norm[1]), pos),
    }
    for name, (uu, nn, pp) in wrong.items():
        with pytest.raises(AssertionError) as e:
            _check(out, *_qk64(uu, C, T, nn, cos, sin, pp), dtype, FRAC_EXACT[dtype], name)
        _report(f"control {dtype} {name} fails", str(e.value).splitlines()[0][:160])


# ------------------------------------------------------------------- 5. the fused K|V gather on simulated ranks
GATHER_GRIDS = {"2x2": (2, 2, 2, 192, 256),          # (gh, gw, S_loc, C, K): S_loc T = 18 rows per scene
                "37x37": (37, 37, 1, 1024, 1024),    # C2 views on 8 ranks, scene boundaries inside tiles
                "37x28": (37, 28, 2, 64, 256)}       # T = 1041


def _ranks(W, B, Lk, C, dtype):
    """W gathered buffers [2 parities, B, Lk, 2C] cut from one flat allocation, with a guard band of one 128-row tile
    before, between and after them; every element holds SENTINEL.  Returns (buffers, guard bands as int16)."""
    G, size = 128 * 2 * C, 2 * B * Lk * 2 * C
    flat = torch.full((G + W * (size + G),), SENTINEL, dtype=torch.int16, device="cuda")
    bufs = [flat[G + r * (size + G):G + r * (size + G) + size].view(dtype).view(2, B, Lk, 2 * C) for r in range(W)]
    guards = [flat[r * (size + G):r * (size + G) + G] for r in range(W + 1)]
    return bufs, guards


def _sharded(ops, agg, dtype, W, B, grid, parity, seed):
    """Rank me holds views [me S_loc, (me + 1) S_loc) of each of B scenes of S = W S_loc views and launches the
    gather instantiation on its B S_loc T rows, with maps onto its row window of every rank's buffer."""
    gh, gw, S_loc, C, K = GATHER_GRIDS[grid]
    T = NUM_SPECIAL + gh * gw
    M_loc = S_loc * T                               # this rank's rows per scene
    Lk = W * M_loc                                  # keys per scene
    g = _gen(seed)
    a, w, bias = _gauss_operands(g, B * Lk, C, K, dtype)
    norm = _norm_vectors(g)
    cos, sin, pos = _rope(agg, gh, gw)
    bufs, guards = _ranks(W, B, Lk, C, dtype)
    runs = []
    for me in range(W):
        a_me = a.view(B, W, M_loc, K)[:, me].reshape(B * M_loc, K)
        maps = ops.kv_gather_maps([bufs[r][parity, 0, me * M_loc:] for r in range(W)], M_loc, 2 * C, 2 * C, B,
                                  Lk * 2 * C, dtype, torch.device("cuda"))
        out = _qkv(ops, a_me, w, bias, C, norm, cos, sin, pos, T, gather_maps=maps, n_gather=W, gather_rows=M_loc)
        runs.append((a_me, maps, out))
    torch.cuda.synchronize()
    return dict(a=a, w=w, bias=bias, norm=norm, rope=(cos, sin, pos), T=T, C=C, M_loc=M_loc, Lk=Lk, bufs=bufs,
                guards=guards, runs=runs)


def _bits(t):
    return t.contiguous().view(torch.int16)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("W", [1, 2, 4, 8])
@pytest.mark.parametrize("B", [1, 2, 3])
@pytest.mark.parametrize("grid", list(GATHER_GRIDS))
def test_fused_kv_gather(ops, agg, dtype, W, B, grid):
    """EPI_QKV_GATHER (n_gather > 0) on one GPU.  Every rank's buffer, in the written parity, holds bit for bit the
    K|V columns of the launches' own outputs in (scene, rank, view, token) order (the layout make_kv_gather produces,
    restated here without torch.distributed); the other parity and the guard bands still hold the sentinel; and each
    launch's own qkv output equals the plain EPI_QKV launch bit for bit.  The parity alternates with W + B, so both
    are written for every W.  2x2: 18 rows per scene, so most rows of a tile are stored by the later-scene path."""
    parity = (W + B) % 2
    r = _sharded(ops, agg, dtype, W, B, grid, parity, 7000 + 10 * W + B)
    C, M_loc, Lk, bufs = r["C"], r["M_loc"], r["Lk"], r["bufs"]
    cos, sin, pos = r["rope"]
    expect = torch.stack([out.view(B, M_loc, 3 * C)[:, :, C:] for _, _, out in r["runs"]], 1).reshape(B, Lk, 2 * C)
    assert not (_bits(expect) == SENTINEL).any()
    for i, buf in enumerate(bufs):
        assert torch.equal(_bits(buf[parity]), _bits(expect)), \
            f"rank {i}: {int((_bits(buf[parity]) != _bits(expect)).sum())} elements differ from the K|V outputs"
        assert (_bits(buf[1 - parity]) == SENTINEL).all(), f"rank {i}: the other parity was written"
    for i, gd in enumerate(r["guards"]):
        assert (gd == SENTINEL).all(), f"guard band {i} was written"
    for a_me, _, out in r["runs"]:
        plain = _qkv(ops, a_me, r["w"], r["bias"], C, r["norm"], cos, sin, pos, r["T"])
        assert torch.equal(_bits(plain), _bits(out)), "the gather launch's qkv differs from the plain launch"
    _report(f"gather {dtype} W={W} B={B} {grid} parity={parity}", "bit-exact")


# -------------------------------------------------------------- 6. the sharded global block equals the unsharded one
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("W,B,grid", [(2, 2, "2x2"), (8, 1, "37x37"), (4, 3, "37x28")])
def test_sharded_equals_unsharded(ops, agg, dtype, W, B, grid):
    """A row's GEMM result depends on neither M nor its place in the tile (fixed K order, no stream-K for qkv): the
    gathered K|V equals the K|V columns of one unsharded launch over all B S T rows, and each rank's q rows the
    matching unsharded q rows, bit for bit.  Each rank's attention over the gathered keys (num_seq = B,
    Lq = S_loc T, Lk = S T) and the matching rows of the unsharded attention both meet bound 1 against the same
    float64 statement (their split-KV plans differ, so they need not be bit-equal)."""
    parity = W % 2
    r = _sharded(ops, agg, dtype, W, B, grid, parity, 8000 + W)
    C, M_loc, Lk, T = r["C"], r["M_loc"], r["Lk"], r["T"]
    cos, sin, pos = r["rope"]
    full = _qkv(ops, r["a"], r["w"], r["bias"], C, r["norm"], cos, sin, pos, T)
    H = C // 64
    o_full = ops.attention(full[:, :C], full[:, C:2 * C], full[:, 2 * C:], B, Lk, Lk, H)
    torch.cuda.synchronize()
    kv = r["bufs"][0][parity].view(B * Lk, 2 * C)
    assert torch.equal(_bits(kv), _bits(full[:, C:])), "gathered K|V differs from the unsharded launch"
    full4 = full.view(B, W, M_loc, 3 * C)
    o4 = o_full.view(B, W, M_loc, C)
    worst = 0.0
    for me, (_, _, out) in enumerate(r["runs"]):
        q_me = out[:, :C]
        assert torch.equal(_bits(q_me), _bits(full4[:, me, :, :C].reshape(B * M_loc, C))), f"rank {me}: q rows differ"
        o_me = ops.attention(q_me, kv[:, :C], kv[:, C:], B, M_loc, Lk, H)
        torch.cuda.synchronize()
        worst = max(worst, check_attn_bound1(o_me, q_me, kv[:, :C], kv[:, C:], B, M_loc, Lk, H, dtype,
                                             what=f"rank {me} attention"))
        worst = max(worst, check_attn_bound1(o4[:, me].reshape(B * M_loc, C), q_me, kv[:, :C], kv[:, C:], B, M_loc,
                                             Lk, H, dtype, what=f"unsharded rows of rank {me}"))
    _report(f"sharded {dtype} W={W} B={B} {grid}: worst attention error / bound 1", worst)


# --------------------------------------------------------------------------------------------- 7. argument checks
def test_argument_checks(ops, agg):
    """Every refused argument is refused before a launch, with the launcher's status.  The allocations are real and
    large enough, so a missing check would launch on valid memory rather than on a bad address."""
    dt, C, K, M = torch.float16, 192, 128, 256
    g = _gen(9000)
    a, w, bias = _gauss_operands(g, M, C, K, dt)
    norm = _norm_vectors(g)
    cos, sin, pos = _rope(agg, 5, 7)
    T = NUM_SPECIAL + 35
    with pytest.raises(RuntimeError, match=r"status -1 "):               # C % 64 != 0
        ops.gemm_qkv(a, w[:288], bias[:288], 96)
    wide = torch.empty(M, 3 * C + 4, device="cuda", dtype=dt)
    with pytest.raises(RuntimeError, match=r"status -2 "):               # ldo % 8 != 0
        ops.gemm_qkv(a, w, bias, C, out=wide[:, :3 * C])
    args = list(norm) + [cos, sin, pos]
    names = ["qn_w", "qn_b", "kn_w", "kn_b", "rope_cos", "rope_sin", "pos_yx"]
    for i in range(7):
        kw = dict(zip(names, args))
        kw[names[i]] = None
        with pytest.raises(RuntimeError, match=r"status -5 "):
            ops.gemm_qkv(a, w, bias, C, qk_norm=True, T=T, **kw)
    for bad_T in (0, -1):
        with pytest.raises(RuntimeError, match=r"status -5 "):
            ops.gemm_qkv(a, w, bias, C, qk_norm=True, T=bad_T, **dict(zip(names, args)))
    # n_gather = 17: a device array of 17 valid maps (16 + 1 assembled in the [maps][pointers][ld, scene_ld] layout)
    dst = torch.empty(17, M, 2 * C, device="cuda", dtype=dt)
    m16 = ops.kv_gather_maps([dst[i] for i in range(16)], M, 2 * C, 2 * C, 1, M * 2 * C, dt, torch.device("cuda"))
    m1 = ops.kv_gather_maps([dst[16]], M, 2 * C, 2 * C, 1, M * 2 * C, dt, torch.device("cuda"))
    m17 = torch.cat([m16[:16 * 128], m1[:128], m16[16 * 128:16 * 136], m1[128:136], m16[16 * 136:]])
    assert m17.numel() == 17 * 136 + 16
    with pytest.raises(RuntimeError, match=r"status -1 "):
        _qkv(ops, a, w, bias, C, norm, cos, sin, pos, T, gather_maps=m17, n_gather=17, gather_rows=M)
    # M % gather_rows != 0, with maps of 3 scenes of 100 rows (room for every row the launch could reach)
    dst3 = torch.empty(3, 100, 2 * C, device="cuda", dtype=dt)
    m3 = ops.kv_gather_maps([dst3[0]], 100, 2 * C, 2 * C, 3, 100 * 2 * C, dt, torch.device("cuda"))
    with pytest.raises(RuntimeError, match=r"status -1 "):
        _qkv(ops, a, w, bias, C, norm, cos, sin, pos, T, gather_maps=m3, n_gather=1, gather_rows=100)
    # kv_gather_maps: no window, 17 windows, ld not a multiple of 8
    for wins, ld in (([], 2 * C), ([dst[i] for i in range(17)], 2 * C), ([dst[0]], 2 * C + 4)):
        with pytest.raises(RuntimeError, match=r"status -1 "):
            ops.kv_gather_maps(wins, M, 2 * C, ld, 1, M * 2 * C, dt, torch.device("cuda"))
    torch.cuda.synchronize()
