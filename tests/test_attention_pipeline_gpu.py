"""State carried between consecutive work items of one CTA in the flash-attention kernel (csrc/attention3.cu, GPU).

The kernel is persistent: a CTA runs many (sequence, head, query-tile pair, kv split) items in a row, and its consumer
warpgroups carry the K / V ring position, the Q buffer parity and their register pipeline from one item to the next.
Launched with many items per CTA, every sequence must give bit for bit the output it gives launched alone (one item per
CTA), and outputs meet bound 1 (tests/test_attention_bounds_gpu.py).  The cases cover items of both kinds
(full query-tile pairs and light-tail pairs whose tile B has no rows), items of a single kv tile (the whole item is
the pipeline's first and last tile), and split-KV launches whose every range is one kv tile.
"""
import math

import pytest
import torch

from ulp_bounds import check_attn_bound1

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


@pytest.fixture(scope="module")
def ops():
    from iggt_official_b200 import ops as _ops
    return _ops


# (num_seq, Lq, Lk, H, kv splits): 40 x 16 x 2 = 1280 mixed full / light-tail items; 200 x 16 one-tile items;
# 3 one-tile kv ranges of 40 x 16 x 2 pairs; one-tile items with a light tail
CASES = [
    (40, 300, 300, 16, 1),
    (200, 100, 100, 16, 1),
    (40, 300, 300, 16, 3),
    (40, 300, 128, 16, 1),
]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("num_seq,Lq,Lk,H,splits", CASES)
def test_many_items_per_cta_match_single_sequence(ops, dtype, num_seq, Lq, Lk, H, splits):
    g = torch.Generator(device="cuda").manual_seed(num_seq * 7 + Lq * 3 + Lk + splits)
    sd = math.sqrt(8.0)                                   # logits q.k / 8 with a standard deviation of ~8
    q = (torch.randn(num_seq * Lq, H * 64, device="cuda", generator=g) * sd).to(dtype)
    k = (torch.randn(num_seq * Lk, H * 64, device="cuda", generator=g) * sd).to(dtype)
    v = torch.randn(num_seq * Lk, H * 64, device="cuda", generator=g).to(dtype)
    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    q_pairs = ((Lq + 127) // 128 + 1) // 2
    assert num_seq * H * q_pairs * splits >= 4 * n_sms, "the launch must give every CTA several items"
    out = ops.attention(q, k, v, num_seq, Lq, Lk, H, splits=splits)
    torch.cuda.synchronize()
    for s in range(num_seq):
        alone = ops.attention(q[s * Lq:(s + 1) * Lq], k[s * Lk:(s + 1) * Lk], v[s * Lk:(s + 1) * Lk], 1, Lq, Lk, H,
                              splits=splits)
        torch.cuda.synchronize()
        assert torch.equal(out[s * Lq:(s + 1) * Lq], alone), f"sequence {s} differs from its own launch"
    # bound 1 (float64 reference) on three sequences; the bits of all of them are pinned to their own launches above
    for s in (0, num_seq // 2, num_seq - 1):
        rows, keys = slice(s * Lq, (s + 1) * Lq), slice(s * Lk, (s + 1) * Lk)
        check_attn_bound1(out[rows], q[rows], k[keys], v[keys], 1, Lq, Lk, H, dtype,
                          what=f"sequence {s} of {num_seq}x{Lq}x{Lk} H={H} splits={splits}")
