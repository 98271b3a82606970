"""Host logic behind the launchers, exercised WITHOUT a GPU through the C ABI (`iggt_gemm_plan`,
`iggt_attention_schedule`): N-tile choice, stream-K, and the attention work distribution.  These are the decisions the
C2 numbers in DESIGN.md rest on; the functions only run host code (an H100's 132 SMs assumed without a device)."""
import ctypes

import numpy as np
import pytest

from iggt_official_b200 import _lib

STORE16, RESID32, QKV, STORE32 = 0, 1, 2, 3
SMS = 132


def plan(epi, M, N, K):
    out = (ctypes.c_int * 7)()
    assert _lib.load().iggt_gemm_plan(epi, M, N, K, ctypes.cast(out, ctypes.c_void_p)) == 0
    return dict(zip(["bn", "pair", "stream_k", "m_tiles", "n_tiles", "k_blocks", "grid"], list(out)))


def schedule(num_seq, Lq, Lk, H, grid, cta):
    buf = (ctypes.c_int * (4 * 4096))()
    n = _lib.load().iggt_attention_schedule(num_seq, Lq, Lk, H, grid, cta, ctypes.cast(buf, ctypes.c_void_p), 4096)
    assert 0 <= n <= 4096
    return [tuple(buf[4 * i:4 * i + 4]) for i in range(n)]


def test_gemm_plan_c2_shapes():
    M = 8 * 1374                                            # the C2 token count
    qkv = plan(QKV, M, 3072, 1024)
    assert (qkv["bn"], qkv["pair"], qkv["stream_k"]) == (128, 0, 0)
    assert qkv["m_tiles"] == 86 and qkv["n_tiles"] == 24 and qkv["grid"] == SMS
    fc1 = plan(STORE16, M, 4096, 1024)
    assert (fc1["bn"], fc1["pair"], fc1["m_tiles"], fc1["n_tiles"], fc1["grid"]) == (128, 0, 86, 32, SMS)
    for N, K in ((1024, 1024), (1024, 4096)):               # proj / fc2: 5.2 waves of 128 x 128 tiles -> stream-K
        r = plan(RESID32, M, N, K)
        assert (r["bn"], r["pair"], r["stream_k"], r["grid"]) == (128, 0, 1, SMS)
        assert r["m_tiles"] * r["n_tiles"] * r["k_blocks"] >= 4 * SMS
    cam = plan(RESID32, 8, 2048, 2048)                      # one row tile: nothing to split
    assert cam["pair"] == 0 and cam["stream_k"] == 0 and cam["grid"] == cam["m_tiles"] * cam["n_tiles"]


@pytest.mark.parametrize("epi", [STORE16, RESID32, QKV, STORE32])
def test_gemm_plan_invariants(epi):
    g = np.random.default_rng(epi)
    for _ in range(300):
        M = int(g.integers(1, 50000))
        N = int(g.integers(1, 65)) * 64 if epi != QKV else 3 * 64 * int(g.integers(1, 33))
        K = int(g.integers(1, 129)) * 64
        p = plan(epi, M, N, K)
        rows_per_tile = 128
        assert p["pair"] == 0
        assert p["bn"] in (64, 128) and (epi not in (RESID32, QKV) or p["bn"] == 128)
        assert p["m_tiles"] * rows_per_tile >= M > (p["m_tiles"] - 1) * rows_per_tile      # rows covered, no spare tile
        assert p["n_tiles"] * p["bn"] >= N > (p["n_tiles"] - 1) * p["bn"]
        assert p["k_blocks"] * 64 >= K
        assert 0 < p["grid"] <= SMS
        assert not p["stream_k"] or (epi == RESID32 and p["bn"] == 128 and p["grid"] == SMS)
        if not p["stream_k"]:
            assert p["grid"] == min(p["m_tiles"] * p["n_tiles"], SMS)


def _check_attention(num_seq, Lq, H, grid):
    q_tiles = -(-Lq // 128)
    q_pairs = (q_tiles + 1) // 2
    light = q_tiles % 2 == 1 and q_pairs > 1
    seen, loads = set(), []
    for cta in range(grid):
        items = schedule(num_seq, Lq, Lq, H, grid, cta)
        load = 0.0
        for qp, head, seq, b_active in items:
            assert 0 <= qp < q_pairs and 0 <= head < H and 0 <= seq < num_seq
            assert (qp, head, seq) not in seen
            seen.add((qp, head, seq))
            assert b_active == (0 if (light and qp == q_pairs - 1) else 1)
            load += 1.0 if b_active else 0.5
        weights = [1.0 if b else 0.5 for *_, b in items]
        assert weights == sorted(weights, reverse=True)               # full items first, halves last
        loads.append(load)
    assert len(seen) == num_seq * H * q_pairs                           # every item exactly once
    return max(loads), sum(loads) / grid


def test_attention_schedule_frame_shape_is_balanced():
    """8 views x 16 heads x 1374 tokens: 640 full + 128 half items on 132 CTAs -> 5.5 item-times (round-robin: 6.0)."""
    worst, mean = _check_attention(8, 1374, 16, SMS)
    assert worst == 5.5 and abs(mean - 704 / SMS) < 1e-9


def test_attention_schedule_global_shape_and_small_cases():
    worst, mean = _check_attention(1, 8 * 1374, 16, SMS)                # 86 tiles -> 43 full pairs, no light tail
    assert worst == 6.0 and abs(mean - 688 / SMS) < 1e-9
    for num_seq, Lq, H in [(3, 300, 4), (1, 128, 1), (2, 129, 2), (1, 200, 2), (5, 1000, 3), (13, 405, 16), (1, 257, 1)]:
        total = num_seq * H * ((-(-Lq // 128) + 1) // 2)
        worst, mean = _check_attention(num_seq, Lq, H, min(total, SMS))
        assert worst - mean <= 1.0                                      # never more than one item above the average


def test_schedule_argument_errors():
    lib = _lib.load()
    assert lib.iggt_gemm_plan(7, 1, 1, 1, None) < 0
    assert lib.iggt_attention_schedule(1, 128, 128, 1, 4, 4, None, 0) < 0


# ---------------------------------------------------------------------------------------------------
# split-KV launches (view-sharded global attention: local queries against the gathered keys)
def _plan(num_seq, Lq, Lk, H, sms=SMS):
    import ctypes
    s, b = ctypes.c_int(0), ctypes.c_int64(0)
    assert _lib.load().iggt_attention_plan(num_seq, Lq, Lk, H, sms, ctypes.addressof(s), ctypes.addressof(b)) == 0
    return s.value, b.value


def _schedule_splits(num_seq, Lq, Lk, H, splits, grid, cta):
    import ctypes
    buf = (ctypes.c_int * (5 * 4096))()
    tps = ctypes.c_int(0)
    n = _lib.load().iggt_attention_schedule_splits(num_seq, Lq, Lk, H, splits, grid, cta, ctypes.addressof(buf), 4096,
                                                   ctypes.addressof(tps))
    assert 0 <= n <= 4096
    return [tuple(buf[5 * i:5 * i + 5]) for i in range(n)], tps.value


def test_attention_plan_splits_only_when_items_are_scarce():
    # one GPU, C2: plenty of items -> never split (the workspace traffic would cost more than the tail it balances)
    assert _plan(8, 1374, 1374, 16) == (1, 0)
    assert _plan(1, 8 * 1374, 8 * 1374, 16) == (1, 0)
    # 8 GPUs, C2: 1 view per rank = 96 items for 132 SMs, 86 kv tiles each -> split the kv range
    s, ws = _plan(1, 1374, 8 * 1374, 16)
    assert 3 <= s <= 8 and ws == s * 1374 * 16 * 66 * 4
    # 4 / 2 GPUs
    assert _plan(1, 2 * 1374, 8 * 1374, 16)[0] >= 2
    # C3 on 8 GPUs: 4 views per rank against 32 views of keys
    s3, _ = _plan(1, 4 * 1374, 32 * 1374, 16)
    assert s3 >= 1
    # a split never leaves an empty kv range
    for Lk in (128, 129, 300, 1374, 10992):
        for forced in range(1, 9):
            n_kv = -(-Lk // 128)
            tps = -(-n_kv // forced)
            assert (-(-n_kv // tps) - 1) * tps < n_kv


def test_split_schedule_covers_every_item_and_range_once():
    num_seq, Lq, Lk, H, splits = 1, 1374, 8 * 1374, 16, 3
    q_pairs = (-(-Lq // 128) + 1) // 2
    n_kv = -(-Lk // 128)
    seen, loads = set(), []
    for cta in range(SMS):
        items, tps = _schedule_splits(num_seq, Lq, Lk, H, splits, SMS, cta)
        assert tps == -(-n_kv // splits)
        load = 0.0
        for qp, head, seq, b_active, split in items:
            assert 0 <= split < splits and (qp, head, seq, split) not in seen
            seen.add((qp, head, seq, split))
            load += (1.0 if b_active else 0.5) * (min(n_kv, (split + 1) * tps) - split * tps)
        loads.append(load)
    assert len(seen) == num_seq * H * q_pairs * splits
    covered = sum(min(n_kv, (s + 1) * tps) - s * tps for s in range(splits))
    assert covered == n_kv                                             # the ranges tile [0, n_kv)
    # 96 items x 86 tiles on one GPU of eight: unsplit the busiest CTA runs 86 tile steps; split in three, 58
    assert max(loads) <= 2 * tps
