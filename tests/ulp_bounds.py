"""Per-element error metrics for the kernel tests: distances in 16-bit steps and per-element fp32 bounds.

A bound relative to the tensor's maximum lets a one-ulp error at the largest element hide anywhere else, including on
elements a hundred times smaller.  These helpers hold every element to its own scale instead:

* `ulp_distance(out16, ref, dtype)`: the exact number of 16-bit steps between `out16` and RN16(ref).
* `check16(out, ref64, dtype, max_ulps, max_frac_off)`: every element within `max_ulps` steps of RN16(ref64), and at
  most a fraction `max_frac_off` of the elements not exactly RN16(ref64).  fp32 summation order flips a 16-bit
  rounding only rarely; rounding toward zero, or a lost rounding point, is off in tens of percent of the elements.
* `check32(out, ref64, scale64, rel)`: |out - ref64| <= rel * scale64 per element, the scale being the element's own
  magnitude sum (for a GEMM: (|A| @ |W|^T)_ij + |b_j| + |x_ij|), not the tensor's maximum.

Both checks optionally take `lo64` / `hi64`: the exact result is only known to within the error the fp32 arithmetic
of any correct kernel leaves (accumulation order), so every 16-bit value that is RN16 of some point of [lo64, hi64]
is admissible.  An activation after an accumulation maps the interval through the activation (see `around`).

The fp64 references are rounded to 16 bit through fp32 (`rn16`), one RN step as in the kernels, which round an fp32
value.  fp64 -> fp32 -> 16 bit can differ from a direct fp64 -> 16 bit rounding (double rounding) only when the fp64
value lies within 2^-25 (relative) of a 16-bit rounding midpoint; the kernel's own fp32 value is never that close to
the exact one, so those elements are within a 1-step flip either way and are absorbed by `max_frac_off`.
"""
import torch

# 16-bit formats: explicit mantissa bits, smallest subnormal spacing
_FMT = {torch.float16: (10, 2.0 ** -24), torch.bfloat16: (7, 2.0 ** -133)}
BIG = 1 << 20                     # distance reported for a NaN / inf mismatch (never admissible)


def rn16(x, dtype):
    """Round to the 16-bit format through fp32 (the one RN step the kernels take; see the module docstring)."""
    return x.to(torch.float32).to(dtype)


def ulp16(x, dtype):
    """Spacing of the 16-bit format at |x| (float64; the subnormal spacing below the smallest normal)."""
    bits, tiny = _FMT[dtype]
    x = x.to(torch.float64).abs()
    x = torch.where(torch.isfinite(x), x, torch.zeros_like(x))
    _, e = torch.frexp(x)
    u = torch.clamp(torch.ldexp(torch.ones_like(x), (e - 1 - bits).to(torch.int32)), min=tiny)
    return torch.where(x == 0, torch.full_like(x, tiny), u)


def _ordered(t16):
    """16-bit patterns -> integers in value order (+0 and -0 both 0; inf one step past the largest finite value)."""
    b = t16.contiguous().view(torch.int16).to(torch.int32) & 0xFFFF
    mag = b & 0x7FFF
    return torch.where(b >= 0x8000, -mag, mag)


def _interval_distance(out16, lo16, hi16):
    """Steps from out16 to the closest 16-bit value in [lo16, hi16] (per element); BIG where NaN or inf disagree."""
    o, a, b = _ordered(out16), _ordered(lo16), _ordered(hi16)
    lo, hi = torch.minimum(a, b), torch.maximum(a, b)
    d = torch.clamp(torch.maximum(lo - o, o - hi), min=0)
    # an infinity is admissible only where the interval itself reaches it, and a finite value is never 'close' to an
    # interval that holds nothing but one infinity
    inf_o = torch.isinf(out16)
    pinned_inf = torch.isinf(lo16) & torch.isinf(hi16) & (torch.sign(lo16) == torch.sign(hi16))
    d = torch.where((inf_o | pinned_inf) & (d != 0), torch.full_like(d, BIG), d)
    nan_o = torch.isnan(out16)
    nan_r = torch.isnan(lo16) | torch.isnan(hi16)
    d = torch.where(nan_o & nan_r, torch.zeros_like(d), d)
    return torch.where(nan_o != nan_r, torch.full_like(d, BIG), d)


def ulp_distance(out16, ref, dtype):
    """Exact distance in 16-bit steps between out16 and RN16(ref), per element (int32).  +-0 are the same point,
    subnormals count one step each, a NaN or an infinity on one side only is BIG."""
    assert out16.dtype == dtype
    r = rn16(ref, dtype)
    return _interval_distance(out16, r, r)


def around(ref64, slack64):
    """(lo, hi) = ref64 -+ slack64: the values a correct kernel's fp32 arithmetic can reach."""
    return ref64 - slack64, ref64 + slack64


def _where(idx, shape):
    return tuple(int(i) for i in torch.unravel_index(torch.as_tensor(idx), shape))


def check16(out, ref64, dtype, max_ulps, max_frac_off, lo64=None, hi64=None, what=""):
    """Asserts that every element of the 16-bit `out` is within `max_ulps` steps of RN16(ref64) (of RN16 of the
    interval [lo64, hi64] when given) and that at most `max_frac_off` of the elements differ from RN16(ref64).
    Returns (worst steps, fraction off) for the report."""
    assert out.dtype == dtype and out.shape == ref64.shape, (out.dtype, out.shape, ref64.shape)
    ref64 = ref64.to(torch.float64)
    exact = ulp_distance(out, ref64, dtype)
    if lo64 is None:
        dist = exact
    else:
        lo16 = rn16(torch.minimum(lo64, hi64).to(torch.float64), dtype)
        hi16 = rn16(torch.maximum(lo64, hi64).to(torch.float64), dtype)
        dist = torch.minimum(_interval_distance(out, lo16, hi16), exact)
    n = out.numel()
    n_off = int((exact != 0).sum())
    worst = int(dist.max()) if n else 0
    i = int(dist.view(-1).argmax()) if n else 0
    msg = (f"{what}: {int((dist > max_ulps).sum())} of {n} elements beyond {max_ulps} ulp, {n_off} not RN16(ref) "
           f"(limit {max_frac_off:.2%}); worst at {_where(i, out.shape)}: out {out.reshape(-1)[i].item()!r} "
           f"ref {ref64.reshape(-1)[i].item()!r} ({worst} ulp)")
    assert worst <= max_ulps, msg
    assert n_off <= max_frac_off * n, msg
    return worst, n_off / max(n, 1)


def check32(out, ref64, scale64, rel, lo64=None, hi64=None, what=""):
    """Asserts |out - ref64| <= rel * scale64 per element (the distance to [lo64, hi64] when given); NaN positions must
    match.  Returns the largest error / (rel * scale) for the report."""
    assert out.shape == ref64.shape == scale64.shape
    o = out.to(torch.float64)
    lo = ref64 if lo64 is None else torch.minimum(lo64, hi64)
    hi = ref64 if hi64 is None else torch.maximum(lo64, hi64)
    err = torch.clamp(torch.maximum(lo - o, o - hi), min=0)
    err = torch.where(o == ref64, torch.zeros_like(err), err)              # equal infinities
    nan_o, nan_r = torch.isnan(o), torch.isnan(ref64)
    assert torch.equal(nan_o, nan_r), f"{what}: NaN positions differ ({int((nan_o != nan_r).sum())} elements)"
    err = torch.where(nan_o, torch.zeros_like(err), err)
    bound = rel * scale64
    ratio = torch.where(err > 0, err / bound, torch.zeros_like(err))
    n_bad = int((err > bound).sum())
    i = int(ratio.view(-1).argmax()) if ratio.numel() else 0
    worst = float(ratio.view(-1)[i]) if ratio.numel() else 0.0
    assert n_bad == 0, (f"{what}: {n_bad} of {out.numel()} elements beyond rel {rel:.3g} x scale; worst at "
                        f"{_where(i, out.shape)}: out {o.reshape(-1)[i].item()!r} ref {ref64.reshape(-1)[i].item()!r} "
                        f"scale {scale64.reshape(-1)[i].item()!r} ({worst:.3g} x bound)")
    return worst


# ------------------------------------------------------------------------------------------- flash attention, bound 1
# |O - O64| <= ulp16(O64) + u_P * (P64 @ |V|) + 2^-20 * max|V| per element, derived in tests/test_attention_bounds_gpu.py
U_P = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}     # P is rounded to 16 bit before P V


def attn64(q, k, v, Lk, scale):
    """One head of one sequence in float64: q [Lq, 64], k / v [Lk, 64] -> O64 = softmax(q k^T * scale) v and P64 @ |V|."""
    k64, v64 = k.double(), v.double()
    p = torch.softmax(q.double() @ k64.t() * scale, -1)
    return p @ v64, p @ v64.abs()


def check_attn_bound1(out, q, k, v, num_seq, Lq, Lk, H, dtype, scale=0.125, what="", budget=1 << 25):
    """Asserts bound 1 on every element of the attention output; returns the worst error / bound.  The float64 softmax
    is built per sequence, head and block of queries, at most `budget` probabilities at a time (the global attention's
    whole P would not fit in memory).  max|V| is taken over the sequence and head."""
    qb = max(1, min(Lq, budget // max(Lk, 1)))
    worst, n_bad, at = 0.0, 0, None
    for s in range(num_seq):
        for h in range(H):
            cols = slice(64 * h, 64 * h + 64)
            ks, vs = k[s * Lk:(s + 1) * Lk, cols], v[s * Lk:(s + 1) * Lk, cols]
            vmax = vs.double().abs().max()
            for r0 in range(0, Lq, qb):
                rows = slice(s * Lq + r0, s * Lq + min(Lq, r0 + qb))
                o64, pv = attn64(q[rows, cols], ks, vs, Lk, scale)
                bound = ulp16(o64, dtype) + U_P[dtype] * pv + 2.0 ** -20 * vmax
                o = out[rows, cols].double()
                assert torch.isfinite(o).all(), f"{what}: non-finite outputs"
                ratio = (o - o64).abs() / bound
                n_bad += int((ratio > 1).sum())
                w = ratio.max().item()
                if w > worst:
                    i = int(ratio.view(-1).argmax())
                    worst, at = w, (rows.start + i // 64, 64 * h + i % 64, o.view(-1)[i].item(), o64.view(-1)[i].item())
    assert worst <= 1.0, (f"{what}: {n_bad} of {out.shape[0] * H * 64} elements beyond bound 1; worst {worst:.3g} x "
                          f"bound at ({at[0]}, {at[1]}): out {at[2]!r} ref {at[3]!r}")
    return worst
