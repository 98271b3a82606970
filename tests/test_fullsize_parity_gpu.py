"""GPU: parity of the native forward against the oracle AT THE BASELINE SIZES.  `oracle.ref_model.forward` is evaluated on
the same GPU (exact-fp32 matmuls / convolutions, seconds per forward) with the trunk's autocast policy (`amp`) - the
mode pinned against real autocast by tests/test_oracle_amp.py - and the product must agree with it on identical inputs.

What "agree" can mean here (tests/parity_lib.py measures all of it, scripts/parity_fullsize.py reports it):
two correct implementations of a 72-block 16-bit-operand transformer differ by the rounding noise itself - a different
fp32 summation order flips 16-bit roundings, and ~1e-4 per block accumulates to ~7e-4 on the tokens
(scripts/parity_attribution.py).  The yardsticks are therefore the reference's own gaps on the same inputs:
  gap_amp  = oracle(amp) vs oracle(fp32)                      (autocast vs fp32)
  gap_tf32 = oracle(amp, cuDNN TF32 convs) vs oracle(amp)     (PyTorch's GPU default for the reference's fp32 heads)
Asserted, relative L2 against oracle(amp):
  fp16 trunk: depth, depth_conf, world_points_conf, pose_enc <= 1e-3 (north_star's figure);
              world_points, part_feat (amplified by sign*expm1 / 30+ conv layers; operands carry a 10-bit mantissa
              like the reference's own TF32 convolutions) <= 1.3 max(gap_amp, gap_tf32);
  bf16 trunk: every key <= 1.2 x max(gap_amp, gap_tf32) (the heads still run fp16 operands, iggt/models/vggt.py:189)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

CASES = [
    ("vggt", 1, 8, 518, 518, torch.float16),       # C2
    ("vggt", 1, 8, 518, 518, torch.bfloat16),      # C2 under bf16 autocast (C5's dtype)
    ("iggt", 1, 8, 532, 532, torch.float16),       # C2 with the part path (even patch grid, SURVEY F2)
    ("iggt", 1, 3, 336, 504, torch.float16),       # C1 shape
    ("iggt", 1, 3, 336, 504, torch.bfloat16),
]
AMPLIFIED = ("world_points", "part_feat")


def bound(row, key, dtype):
    e = row[key]
    gap = max(e["gap_amp_l2"], e.get("gap_tf32_l2", 0.0))
    if dtype == torch.float16:
        return 1.3 * gap if key in AMPLIFIED else 1e-3
    return 1.2 * max(gap, 1e-3 / 1.2)


@pytest.fixture(scope="module")
def models():
    return {}


@pytest.mark.parametrize("kind,B,S,H,W,dtype", CASES,
                         ids=[f"{c[0]}-{c[1]}x{c[2]}x{c[3]}x{c[4]}-{str(c[5])[6:]}" for c in CASES])
def test_forward_matches_oracle_at_full_size(models, kind, B, S, H, W, dtype):
    import parity_lib
    row = parity_lib.measure(kind, B, S, H, W, dtype, wkind="stress", wseed=1, models=models)
    keys = [k for k in parity_lib.KEYS + ("pose_enc",) if k in row]
    assert "depth" in keys and "pose_enc" in keys and (kind != "iggt" or "part_feat" in keys)
    report = {k: (round(row[k]["vs_amp_l2"], 6), round(bound(row, k, dtype), 6)) for k in keys}
    for k in keys:
        assert row[k]["vs_amp_l2"] <= bound(row, k, dtype), (k, report)
        assert row[k]["vs_amp_max"] <= 8 * bound(row, k, dtype), (k, row[k]["vs_amp_max"], report)
