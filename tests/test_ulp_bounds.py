"""CPU tests of the per-element metrics in ulp_bounds.py: they must count 16-bit steps exactly and must reject the
errors the GPU tests are meant to catch at the thresholds those tests use."""
import pytest
import torch

from ulp_bounds import BIG, around, check16, check32, rn16, ulp16, ulp_distance

DTYPES = [torch.float16, torch.bfloat16]
MAX_FINITE = {torch.float16: 65504.0, torch.bfloat16: torch.finfo(torch.bfloat16).max}


def _gemm_like(seed, n=20000):
    """fp64 values shaped like GEMM outputs: mostly O(1), some tiny, a few large, exact zeros."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, generator=g, dtype=torch.float64)
    x[: n // 10] *= 1e-3
    x[n // 10: n // 5] *= 100
    x[-5:] = 0.0
    return x


def _rtz16(x64, dtype):
    """Round toward zero: the RN result, stepped one code toward zero wherever RN rounded away from zero - the same
    as truncating the mantissa bits of the fp32 value (overflow gives the largest finite value, not inf)."""
    x32 = x64.to(torch.float32)
    r = x32.to(dtype)
    away = r.to(torch.float64).abs() > x32.to(torch.float64).abs()
    bits = r.view(torch.int16)
    stepped = torch.where(away, bits - 1, bits)        # magnitude - 1 in sign-magnitude (never crosses zero)
    return stepped.view(dtype)


def _step(t16, k):
    """Move k codes up in value order (k may be negative), crossing +-0 like the number line does."""
    b = t16.view(torch.int16).to(torch.int32) & 0xFFFF
    mag = b & 0x7FFF
    o = torch.where(b >= 0x8000, -mag, mag) + k
    nb = torch.where(o < 0, 0x8000 | (-o), o)
    return torch.where(nb >= 0x8000, nb - 0x10000, nb).to(torch.int16).view(t16.dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_rn_casts_are_zero_ulps(dtype):
    x = _gemm_like(1)
    specials = torch.tensor([0.0, -0.0, float("inf"), float("-inf"), 1e-30, -1e-30, 2.0 ** -24, 2.0 ** -14,
                             MAX_FINITE[dtype], -MAX_FINITE[dtype], 1e6, 3.0e38], dtype=torch.float64)
    x = torch.cat([x, specials])
    out = rn16(x, dtype)
    assert int(ulp_distance(out, x, dtype).max()) == 0
    assert check16(out, x, dtype, 0, 0.0) == (0, 0.0)


@pytest.mark.parametrize("dtype", DTYPES)
def test_round_toward_zero_fails_the_gpu_thresholds(dtype):
    """The thresholds of test_epilogues_gpu.py (1 ulp, at most 1 % of the elements off RN; 2 % for GELU) must reject
    RTZ stores: each element is within 1 ulp, but about half of them are off."""
    x = _gemm_like(2)
    rtz = _rtz16(x, dtype)
    d = ulp_distance(rtz, x, dtype)
    assert int(d.max()) == 1 and 0.3 < float((d != 0).double().mean()) < 0.7
    with pytest.raises(AssertionError, match="not RN16"):
        check16(rtz, x, dtype, 1, 0.01)
    with pytest.raises(AssertionError):                   # the GELU threshold too
        check16(rtz, x, dtype, 1, 0.02)
    # with a slack interval of fp32-accumulation size, RTZ is still off RN16(ref) in the same share of elements
    lo, hi = around(x, 2.0 ** -20 * x.abs())
    with pytest.raises(AssertionError, match="not RN16"):
        check16(rtz, x, dtype, 1, 0.01, lo, hi)


@pytest.mark.parametrize("dtype", DTYPES)
def test_one_ulp_nudges_are_counted_exactly(dtype):
    bits, _ = {torch.float16: (10, 0), torch.bfloat16: (7, 0)}[dtype]
    min_normal = torch.finfo(dtype).tiny
    min_sub = min_normal * 2.0 ** -bits
    pts = torch.tensor([0.0, -0.0, min_sub, -min_sub, min_normal - min_sub, min_normal, -min_normal, 1.0, -1.0,
                        0.3, MAX_FINITE[dtype] / 2, 3.0], dtype=torch.float64)
    r = rn16(pts, dtype)
    for k in (1, -1, 2, -3):
        nudged = _step(r, k)
        assert torch.equal(ulp_distance(nudged, pts, dtype), torch.full(pts.shape, abs(k), dtype=torch.int32)), k
    # across the subnormal / normal boundary and through zero, by value
    largest_sub = torch.tensor([min_normal - min_sub], dtype=torch.float64)
    assert _step(rn16(largest_sub, dtype), 1).item() == min_normal
    assert _step(rn16(torch.tensor([0.0], dtype=torch.float64), dtype), -1).item() == -min_sub
    assert _step(rn16(torch.tensor([min_sub], dtype=torch.float64), dtype), -2).item() == -min_sub
    # +0 and -0 are the same point
    assert int(ulp_distance(torch.tensor([-0.0]).to(dtype), torch.tensor([0.0], dtype=torch.float64), dtype)) == 0
    # a random set: exactly the nudged elements count, one step each
    x = _gemm_like(3, 5000)
    r = rn16(x, dtype)
    g = torch.Generator().manual_seed(4)
    pick = torch.rand(x.shape, generator=g) < 0.02
    sgn = torch.where(torch.rand(x.shape, generator=g) < 0.5, 1, -1)
    nudged = torch.where(pick, _step(r, 1), r)
    nudged = torch.where(pick & (sgn < 0), _step(r, -1), nudged)
    d = ulp_distance(nudged, x, dtype)
    assert torch.equal(d != 0, pick) and int(d.max()) == 1
    worst, frac = check16(nudged, x, dtype, 1, 0.05)
    assert worst == 1 and frac == float(pick.double().mean())
    with pytest.raises(AssertionError, match="beyond 0 ulp"):
        check16(nudged, x, dtype, 0, 1.0)


@pytest.mark.parametrize("dtype", DTYPES)
def test_nan_and_inf_positions_must_match(dtype):
    ref = torch.tensor([1.0, float("nan"), 2.0, float("inf"), -3.0], dtype=torch.float64)
    out = rn16(ref, dtype)
    assert int(ulp_distance(out, ref, dtype).max()) == 0               # NaN where the reference has NaN is fine
    moved = out.clone()
    moved[0], moved[1] = float("nan"), 1.0
    d = ulp_distance(moved, ref, dtype)
    assert int(d[0]) == BIG and int(d[1]) == BIG
    with pytest.raises(AssertionError):
        check16(moved, ref, dtype, 1000, 1.0)
    fin = out.clone()
    fin[3] = MAX_FINITE[dtype]                                         # the largest finite value is not inf
    assert int(ulp_distance(fin, ref, dtype)[3]) == BIG
    neg = out.clone()
    neg[3] = float("-inf")
    assert int(ulp_distance(neg, ref, dtype)[3]) == BIG
    # an interval that reaches past the overflow threshold admits both the largest finite value and inf
    top = torch.tensor([MAX_FINITE[dtype]], dtype=torch.float64)
    lo, hi = top, top * 2
    for o in (MAX_FINITE[dtype], float("inf")):
        check16(torch.tensor([o]).to(dtype), top, dtype, 0, 1.0, lo, hi)
    with pytest.raises(AssertionError):
        check16(torch.tensor([float("-inf")]).to(dtype), top, dtype, 1, 1.0, lo, hi)


def test_ulp16_spacing():
    x = torch.tensor([1.0, 1.5, 2.0, 0.0, 2.0 ** -20, 65504.0], dtype=torch.float64)
    assert ulp16(x, torch.float16).tolist() == [2.0 ** -10, 2.0 ** -10, 2.0 ** -9, 2.0 ** -24, 2.0 ** -24, 32.0]
    assert ulp16(x, torch.bfloat16).tolist()[:3] == [2.0 ** -7, 2.0 ** -7, 2.0 ** -6]


def test_check32_is_per_element():
    """An error of 1e-3 of the largest element on an element 1000x smaller passes a max-relative bound, not check32."""
    g = torch.Generator().manual_seed(5)
    ref = torch.randn(1000, generator=g, dtype=torch.float64)
    ref[7] = 1e-3
    scale = ref.abs() + 1e-3
    out = ref.clone().to(torch.float32)
    assert check32(out, ref, scale, 2.0 ** -20) < 1.0
    out[7] += 2e-6
    assert float((out.double() - ref).abs().max() / ref.abs().max()) < 1e-5       # invisible to the max metric
    with pytest.raises(AssertionError, match="1 of 1000"):
        check32(out, ref, scale, 2.0 ** -20)
    nan_out = ref.clone().to(torch.float32)
    nan_out[3] = float("nan")
    with pytest.raises(AssertionError, match="NaN"):
        check32(nan_out, ref, scale, 1.0)
