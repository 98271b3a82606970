"""Element-by-element tests of the flash-attention kernel (csrc/attention3.cu, GPU) against a float64 softmax, unsplit
and split-KV, fp16 and bf16.

Bound 1 (per element):  |O - O64| <= ulp16(O64) + u_P * (P64 @ |V|) + 2^-20 * max|V|
  * ulp16(O64): the final RN16 of O (half an ulp) and the fp32 normalisation 1 / l (a few 2^-24).
  * u_P (2^-11 fp16, 2^-8 bf16): P is rounded to 16 bit before P V, a relative error of at most half an ulp per weight.
  * 2^-20 max|V| (max over the sequence and head): ex2.approx (2^-22 relative per weight, in O and l alike), the fp32
    logits (~2^-24 * sum|q||k| ~ 2^-16 of a logit, times log2(e) / 8 per weight), the running-max rescales and the fp32
    sums of O and l; and where an fp16 weight falls below 2^-14 it is subnormal, rounded to within 2^-25 absolute:
    over 1374 keys of random sign ~2^-25 * sqrt(1374 / 3) = 2^-20.6 of max|V|.
The inputs scale q and k so that the logits have a standard deviation of about 8, which keeps the running max moving.
The bound-1 check is `check_attn_bound1` in tests/ulp_bounds.py (tests/test_track_bounds_gpu.py applies it at the
update transformer's shapes).  The worst error / bound of each case is printed (run with -s to see it).
"""
import math

import pytest
import torch

from ulp_bounds import check16, check_attn_bound1

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


@pytest.fixture(scope="module")
def ops():
    from iggt_official_b200 import ops as _ops
    return _ops


def _splits(Lk, want):
    """A kv split count the launcher accepts (no empty range), at most `want`."""
    n_kv = (Lk + 127) // 128
    s = min(want, n_kv)
    tps = (n_kv + s - 1) // s
    return (n_kv + tps - 1) // tps


def _qkv(g, num_seq, Lq, Lk, H, dtype, logit_std=8.0):
    """q, k with logits q.k / 8 of standard deviation ~logit_std, v ~ N(0, 1)."""
    sd = math.sqrt(logit_std)                         # q.k / 8 = sum of 64 products of N(0, sd^2) / 8: std sd^2
    q = (torch.randn(num_seq * Lq, H * 64, device="cuda", generator=g) * sd).to(dtype)
    k = (torch.randn(num_seq * Lk, H * 64, device="cuda", generator=g) * sd).to(dtype)
    v = torch.randn(num_seq * Lk, H * 64, device="cuda", generator=g).to(dtype)
    return q, k, v


def _report(what, value):
    print(f"[bound] {what}: {value}")


# --------------------------------------------------------------------------------- 1. bound 1 at ragged key counts
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("Lk", [1, 63, 64, 65, 127, 129, 300, 1374])
def test_bound_vs_fp64_softmax(ops, dtype, split, Lk):
    if split and Lk <= 128:
        pytest.skip("one kv tile: nothing to split")
    H = 2
    worst = 0.0
    for num_seq in (1, 3):
        for Lq in (1, 65, 300):
            g = torch.Generator(device="cuda").manual_seed(Lk * 1000 + Lq * 10 + num_seq)
            q, k, v = _qkv(g, num_seq, Lq, Lk, H, dtype)
            s = _splits(Lk, 3) if split else 1
            out = ops.attention(q, k, v, num_seq, Lq, Lk, H, splits=s)
            torch.cuda.synchronize()
            worst = max(worst, check_attn_bound1(out, q, k, v, num_seq, Lq, Lk, H, dtype,
                                             what=f"num_seq={num_seq} Lq={Lq} Lk={Lk} splits={s}"))
    _report(f"attention bound1 {dtype} Lk={Lk} split={split}", worst)


# ---------------------------------------------------------------------------------------------------- 2. needles
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("Lk", [65, 129, 300, 1374])
def test_needle(ops, dtype, split, Lk):
    """Each query row has one key whose logit is ~40 above the rest: its output row must be that key's V row within
    1 ulp.  Needles sit at keys 0, 63, 64, 127, 128, Lk - 1 (the ragged tile) and, split-KV, at the first key of the
    last split.  A decoy key (17, logit ~20 above the rest) comes earlier than every needle past key 63, so the running
    max (and, split-KV, the merge's max) changes late."""
    H, num_seq, Lq = 2, 2, 65
    s = _splits(Lk, 3) if split else 1
    if split and s == 1:
        pytest.skip("one kv tile: nothing to split")
    pos = [0, 63, 64, 127, 128, Lk - 1]
    if s > 1:
        n_kv = (Lk + 127) // 128
        pos.append((s - 1) * ((n_kv + s - 1) // s) * 128)
    pos = sorted({p for p in pos if p < Lk and p != 17})
    g = torch.Generator(device="cuda").manual_seed(31 + Lk)
    A, B = 18.0, 12.625                                # logits A^2 / 8 = 40.5, B^2 / 8 = 19.9
    q = torch.randn(num_seq, Lq, H, 64, device="cuda", generator=g) * 0.3
    k = torch.randn(num_seq, Lk, H, 64, device="cuda", generator=g) * 0.3
    v = torch.randn(num_seq, Lk, H, 64, device="cuda", generator=g)
    which = torch.arange(Lq, device="cuda") % len(pos)                  # needle of each query row
    for j, p in enumerate(pos):
        rows = which == j
        q[:, rows, :, 2 * j] = A
        k[:, p, :, 2 * j] = A
        if p > 63:
            q[:, rows, :, 2 * j + 1] = B
            k[:, 17, :, 2 * j + 1] = B
    q, k, v = (t.reshape(-1, H * 64).to(dtype) for t in (q, k, v))
    out = ops.attention(q, k, v, num_seq, Lq, Lk, H, splits=s)
    torch.cuda.synchronize()
    needle_key = torch.tensor(pos, device="cuda")[which]                 # [Lq]
    expect = v.view(num_seq, Lk, H * 64)[:, needle_key].reshape(-1, H * 64)
    _report(f"needle {dtype} Lk={Lk} splits={s}",
            check16(out, expect.double(), dtype, 1, 1.0, what=f"needle Lk={Lk} splits={s}"))


# --------------------------------------------------------------------------------------------------- 3. uniform
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("Lk", [1, 63, 64, 65, 127, 129, 300, 1374])
def test_uniform_keys_average_v(ops, dtype, split, Lk):
    """All keys of a (sequence, head) identical: every weight is exactly 1, so the output is mean(V) of the sequence
    within 1 ulp - any key past Lk that leaks in (a mask off by one) shifts it by ~1 / Lk."""
    H, num_seq, Lq = 2, 3, 65
    s = _splits(Lk, 3) if split else 1
    if split and s == 1:
        pytest.skip("one kv tile: nothing to split")
    g = torch.Generator(device="cuda").manual_seed(77 + Lk)
    q = (torch.randn(num_seq * Lq, H * 64, device="cuda", generator=g) * 0.7).to(dtype)
    krow = torch.randn(num_seq, 1, H * 64, device="cuda", generator=g) * 0.7
    k = krow.expand(num_seq, Lk, H * 64).reshape(-1, H * 64).to(dtype)
    v = (torch.randn(num_seq * Lk, H * 64, device="cuda", generator=g) + 1.0).to(dtype)
    out = ops.attention(q, k, v, num_seq, Lq, Lk, H, splits=s)
    torch.cuda.synchronize()
    mean = v.double().view(num_seq, 1, Lk, H * 64).mean(2).expand(num_seq, Lq, H * 64).reshape(-1, H * 64)
    _report(f"uniform {dtype} Lk={Lk} splits={s}",
            check16(out, mean, dtype, 1, 0.01, what=f"uniform Lk={Lk} splits={s}"))


# ------------------------------------------------------------------------------------------ 4. poisoned neighbour
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("Lk", [20, 300, 1374])
def test_poisoned_neighbour(ops, dtype, split, Lk):
    """The first keys of every sequence s+1 align with sequence s's queries (logit ~+40) and carry V = 1000.  Sequence s
    must not see them: all outputs still meet bound 1 against the per-sequence fp64 softmax."""
    H, num_seq, Lq = 2, 3, 65
    s = _splits(Lk, 3) if split else 1
    if split and s == 1:
        pytest.skip("one kv tile: nothing to split")
    g = torch.Generator(device="cuda").manual_seed(55 + Lk)
    q = torch.randn(num_seq, Lq, H, 64, device="cuda", generator=g) * 1.4
    k = torch.randn(num_seq, Lk, H, 64, device="cuda", generator=g) * 1.4
    v = torch.randn(num_seq, Lk, H, 64, device="cuda", generator=g)
    q[..., 0] = 18.0
    k[..., 0] = 0.0
    n_poison = min(128, Lk)
    k[1:, :n_poison, :, 0] = 18.0                      # 18 * 18 / 8 = 40.5
    v[1:, :n_poison] = 1000.0
    q, k, v = (t.reshape(-1, H * 64).to(dtype) for t in (q, k, v))
    out = ops.attention(q, k, v, num_seq, Lq, Lk, H, splits=s)
    torch.cuda.synchronize()
    _report(f"poisoned neighbour {dtype} Lk={Lk} splits={s}",
            check_attn_bound1(out, q, k, v, num_seq, Lq, Lk, H, dtype, what=f"poisoned Lk={Lk} splits={s}"))


# -------------------------------------------------------------------------------------------- 5. non-finite isolation
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("Lk", [20, 300, 1374])
@pytest.mark.parametrize("where", ["v", "k", "q"])
def test_nonfinite_neighbour_isolation(ops, dtype, split, Lk, where):
    """inf in the rows of sequence 1 that sequence 0's last (ragged) key tile or query tile covers must not reach
    sequence 0: its output stays finite and bit-identical to a run without the inf.  Each sequence's output depends on
    that sequence's q, k and v only."""
    H, num_seq, Lq = 2, 2, 65
    s = _splits(Lk, 3) if split else 1
    if split and s == 1:
        pytest.skip("one kv tile: nothing to split")
    g = torch.Generator(device="cuda").manual_seed(99 + Lk)
    q, k, v = _qkv(g, num_seq, Lq, Lk, H, dtype, logit_std=2.0)
    clean = ops.attention(q, k, v, num_seq, Lq, Lk, H, splits=s).clone()
    t = {"q": q, "k": k, "v": v}[where]
    L = Lq if where == "q" else Lk
    t[L:min(2 * L, (L + 127) // 128 * 128)] = float("inf")          # seq 1's rows inside seq 0's last 128-row tile
    out = ops.attention(q, k, v, num_seq, Lq, Lk, H, splits=s)
    torch.cuda.synchronize()
    o0, c0 = out[:Lq], clean[:Lq]
    assert torch.isfinite(o0.float()).all(), f"{int((~torch.isfinite(o0.float())).sum())} non-finite outputs in seq 0"
    assert torch.equal(o0, c0)


# --------------------------------------------------------------------------------------------------- 6. packed qkv
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("num_seq,L,H", [(3, 300, 4), (2, 1374, 16)])
def test_packed_qkv_slices(ops, dtype, num_seq, L, H):
    """q, k, v as the three column slices of one [num_seq * L, 3C] buffer (models/aggregator.py): bound 1, and the same
    bits as contiguous copies."""
    C = H * 64
    g = torch.Generator(device="cuda").manual_seed(7 * L + H)
    qkv = (torch.randn(num_seq * L, 3 * C, device="cuda", generator=g) * math.sqrt(8.0)).to(dtype)
    qkv[:, 2 * C:] = torch.randn(num_seq * L, C, device="cuda", generator=g).to(dtype)
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    out = ops.attention(q, k, v, num_seq, L, L, H, splits=1)
    ref_bits = ops.attention(q.contiguous(), k.contiguous(), v.contiguous(), num_seq, L, L, H, splits=1)
    torch.cuda.synchronize()
    assert torch.equal(out, ref_bits)
    _report(f"packed qkv {dtype} {num_seq}x{L} H={H}",
            check_attn_bound1(out, q, k, v, num_seq, L, L, H, dtype, what=f"packed qkv {num_seq}x{L}"))
