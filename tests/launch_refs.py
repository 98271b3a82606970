"""Float64 statements of the GEMM, convolution, qkv and DPT-tail launches, shared by the synthetic kernel tests
(test_epilogues_gpu.py, test_qkv_bounds_gpu.py, test_heads_bounds_gpu.py) and the launch census of the real forward
(test_launch_census_gpu.py), so that one statement holds both.  The allowances are derived in the docstrings of the
synthetic test files; they are restated here only as constants.

* ACC = 2^-20 of an element's magnitude sum (|A| @ |W|^T + |b|): what fp32 accumulation in any order can leave
  (test_epilogues_gpu.py).
* GELU_ERR: the gelu_fast error per unit of |x| / 2 (csrc/ptx.cuh), pinned exhaustively in test_epilogues_gpu.py.
* FRAC / FRAC_GELU: the share of 16-bit outputs allowed to differ from RN16 of the float64 value (the reordered fp32
  sum flips a rounding only near a midpoint), about twice the share measured at K <= 1024 on Gaussian data.
"""
import ctypes
import math

import torch

from ulp_bounds import around, check32, rn16

ACC = 2.0 ** -20
U24 = 2.0 ** -24
# gelu_fast (csrc/ptx.cuh): Abramowitz-Stegun erf (|err| <= 1.5e-7), the fp32 complement 1 - erf (quantised at
# 2^-24) and ex2.approx (2^-22 relative), each scaled by |x| / 2
GELU_ERR = 1.5e-7 + 2.0 ** -24 + 2.0 ** -22
FRAC = {torch.float16: 0.01, torch.bfloat16: 0.002}
FRAC_GELU = {torch.float16: 0.02, torch.bfloat16: 0.005}


def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def leaky64(x):
    return torch.where(x > 0, x, 0.01 * x)


def gemm64(a, w):
    """Exact (fp64) product of the 16-bit operands and its per-element magnitude sum."""
    a64, w64 = a.double(), w.double()
    return a64 @ w64.t(), a64.abs() @ w64.abs().t()


def gemm_plan(M, N, K, epi=1):
    """The schedule iggt_gemm_plan reports (epi: 0 store16, 1 resid32, 2 qkv, 3 store32)."""
    from iggt_official_b200 import _lib
    out = (ctypes.c_int * 7)()
    assert _lib.load().iggt_gemm_plan(epi, M, N, K, ctypes.cast(out, ctypes.c_void_p)) == 0
    return dict(zip(["bn", "pair", "stream_k", "m_tiles", "n_tiles", "k_blocks", "grid"], list(out)))


def act_interval(act, y, s, dtype):
    """(ref, lo, hi) of act(y) when the kernel's fp32 value lies within y -+ s.  act 1 is the autocast form: GELU of the
    16-bit Linear output (gemm.cuh: round16 before gelu_fast2), with the gelu_fast error on top."""
    lo, hi = around(y, s)
    if act == 1:
        x_lo, x_hi = rn16(lo, dtype).double(), rn16(hi, dtype).double()
        g_lo, g_hi = gelu64(x_lo), gelu64(x_hi)
        e = torch.maximum(x_lo.abs(), x_hi.abs()) / 2 * GELU_ERR
        return gelu64(rn16(y, dtype).double()), torch.minimum(g_lo, g_hi) - e, torch.maximum(g_lo, g_hi) + e
    f = {0: lambda t: t, 2: torch.relu, 3: leaky64}[act]
    return f(y), f(lo), f(hi)


def conv64(x, wp, taps, rows=None):
    """Exact (fp64) implicit-GEMM convolution of ONE image and its magnitude sum: x [H, W, Cin] 16-bit NHWC, wp [Cout,
    taps * Cin] tap-major (k = (ky * 3 + kx) * Cin + ci), zero padding 1 for taps = 9.  `rows` = (y0, y1) restricts the
    output to those rows.  Returns ([h, W, Cout], [h, W, Cout]) float64, built by im2col + one matmul per band of rows
    so that the float64 im2col stays near 2^27 elements."""
    H, W, Cin = x.shape
    y0, y1 = rows if rows is not None else (0, H)
    w64 = wp.double()
    if taps == 1:
        a = x[y0:y1].reshape(-1, Cin).double()
        return ((a @ w64.t()).view(y1 - y0, W, -1), (a.abs() @ w64.abs().t()).view(y1 - y0, W, -1))
    xp = torch.nn.functional.pad(x.double(), (0, 0, 1, 1, 1, 1))          # [H + 2, W + 2, Cin]
    band = max(1, (1 << 27) // (W * 9 * Cin))
    accs, mags = [], []
    for r0 in range(y0, y1, band):
        r1 = min(y1, r0 + band)
        a = torch.cat([xp[r0 + dy:r1 + dy, dx:dx + W] for dy in range(3) for dx in range(3)], -1).reshape(-1, 9 * Cin)
        accs.append((a @ w64.t()).view(r1 - r0, W, -1))
        mags.append((a.abs() @ w64.abs().t()).view(r1 - r0, W, -1))
        del a
    return torch.cat(accs), torch.cat(mags)


# ------------------------------------------------------------------------- the qkv epilogue (test_qkv_bounds_gpu.py)
EPS = 1e-5


def y64(a, w, bias):
    """acc + b in float64 from the 16-bit operands, and the magnitude sum |A| |W|^T + |b|."""
    a64, w64, b64 = a.double(), w.double(), bias.double()
    return a64 @ w64.t() + b64, a64.abs() @ w64.abs().t() + b64.abs()


def ln64(x, C, norm, amb=None):
    """LayerNorm(64) of every q and k head of x [M, 2C] (the 16-bit Linear output as float64), two-pass, with the q
    vectors on [0, C) and the k vectors on [C, 2C); returns (ln, slack), the slack of test_qkv_bounds_gpu.py's
    docstring, widened by 2 x the first-order effect of the ambiguous inputs `amb` (a_j per element, 0 where not
    ambiguous) when given."""
    M, H = x.shape[0], C // 64
    x = x.reshape(M, 2, H, 64)
    w = torch.stack([norm[0], norm[2]]).double().view(1, 2, 1, 64)
    b = torch.stack([norm[1], norm[3]]).double().view(1, 2, 1, 64)
    mean = x.mean(-1, keepdim=True)
    d = x - mean
    rstd = (d.square().mean(-1, keepdim=True) + EPS).rsqrt()
    z = d * rstd
    zw = z * w
    ln = zw + b
    s = 2.0 ** -18 * rstd * w.abs() * x.abs().mean(-1, keepdim=True) + 2.0 ** -17 * zw.abs() + 2.0 ** -23 * ln.abs()
    if amb is not None:
        a = amb.reshape(M, 2, H, 64)
        za = z.abs()
        first = rstd * w.abs() * (a + (a.sum(-1, keepdim=True) + za * (a * za).sum(-1, keepdim=True)) / 64)
        s = s + 2.0 * first
    return ln.reshape(M, 2 * C), s.reshape(M, 2 * C)


def rope64(ln, s, cos, sin, pos, T):
    """2-D RoPE of ln [M, 2C] at pos[row % T] with the fp32 table values, and the slack carried through it."""
    M = ln.shape[0]
    p = pos.long()[torch.arange(M, device=ln.device) % T]                  # [M, 2]: (y, x)
    c = cos.double()[p].view(M, 1, 2, 16)                                  # half 0 rotates by y, half 1 by x
    sn = sin.double()[p].view(M, 1, 2, 16)
    l4, s4 = ln.view(M, -1, 2, 32), s.view(M, -1, 2, 32)
    a, b = l4[..., :16], l4[..., 16:]
    sa, sb = s4[..., :16], s4[..., 16:]
    oa, ob = a * c - b * sn, b * c + a * sn
    ea = c.abs() * sa + sn.abs() * sb + 2.0 ** -23 * ((a * c).abs() + (b * sn).abs() + oa.abs())
    eb = c.abs() * sb + sn.abs() * sa + 2.0 ** -23 * ((b * c).abs() + (a * sn).abs() + ob.abs())
    return torch.cat([oa, ob], -1).reshape(M, -1), torch.cat([ea, eb], -1).reshape(M, -1)


def qk64(u, C, T, norm, cos, sin, pos, amb=None):
    ln, s = ln64(u[:, :2 * C], C, norm, None if amb is None else amb[:, :2 * C])
    return rope64(ln, s, cos, sin, pos, T)


# ------------------------------------------------------------------- the DPT tail (test_heads_bounds_gpu.py, fp32 out)
def tail_act64(o64, A, mode, rel):
    """Reference and bound of the head activation of o (exact o64, |o - o64| <= rel A):
      exp(o):           |d| <= e^o (e^(rel A) - 1) + expf's 2^-22 e^o
      sign expm1(|o|):  |d| <= e^|o| (e^(rel A) - 1) + expm1f's 2^-22 |expm1|
      1 + exp(o):       as exp, + the add's 2^-24 (1 + e^o)
    returned as (ref, scale) for check32(out, ref, scale, rel): the bound is rel * scale."""
    grow = torch.expm1(rel * A) / rel                       # (e^(rel A) - 1) / rel  (~A)
    if mode == 0:
        e = torch.exp(o64)
        return e, e * (grow + 2.0 ** -22 / rel)
    r = torch.sign(o64) * torch.expm1(o64.abs())
    return r, torch.exp(o64.abs()) * grow + r.abs() * 2.0 ** -22 / rel


def conf64(o64, A, rel):
    e = torch.exp(o64)
    return 1 + e, e * (torch.expm1(rel * A) / rel + 2.0 ** -22 / rel) + (1 + e) * U24 / rel


def check_tail(main, conf, o64, A, mode, rel, what):
    """o64 / A: [NB, H, W, OC] exact pre-activation and its magnitude sum."""
    if mode == 2:                                  # part features: channels-first, no confidence
        assert conf is None
        return check32(main, o64.permute(0, 3, 1, 2), A.permute(0, 3, 1, 2), rel, what=what)
    ref, scale = tail_act64(o64[..., :-1], A[..., :-1], mode, rel)
    w1 = check32(main, ref, scale, rel, what=what)
    cref, cscale = conf64(o64[..., -1], A[..., -1], rel)
    return max(w1, check32(conf, cref, cscale, rel, what=what + " conf"))
