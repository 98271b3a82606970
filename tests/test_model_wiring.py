"""Host-side graph of the native model classes WITHOUT a GPU: every C-ABI launcher of `ops` is replaced by its plain
PyTorch statement (tests/emu_ops.py) and `VGGT.forward` must then reproduce the fixture of the unmodified reference.
This pins what is NOT a kernel - weight packing, token / row layouts, the ResidualConvUnit and FeatureFusionBlock
fusions of the DPT head (skip-adds and ReLUs folded into conv epilogues, 1x1 out_conv moved below the upsample),
deconvolution as GEMM + pixel shuffle, the camera head's AdaLN loop - on every CPU test run; the kernels themselves are
compared with the same statements on the GPU (tests/test_kernels_gpu.py)."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import emu_ops                                                              # noqa: E402
from oracle import weights                                                  # noqa: E402

EMU = {"gemm_store16": emu_ops.gemm_store16_full, "gemm_store32": emu_ops.gemm_store32, "gemm_resid32": emu_ops.gemm_resid32_full,
       "gemm_qkv": emu_ops.gemm_qkv, "attention": emu_ops.attention, "layernorm": emu_ops.layernorm,
       "layernorm16": emu_ops.layernorm16, "conv_nhwc": emu_ops.conv_nhwc, "upsample_bilinear": emu_ops.upsample_bilinear,
       "deconv_shuffle": emu_ops.deconv_shuffle, "im2col3x3_s2": emu_ops.im2col3x3_s2, "dpt_tail": emu_ops.dpt_tail, "dpt_tail_fused": emu_ops.dpt_tail_fused,
       "skinny_gemm": emu_ops.skinny_gemm, "small_attention": emu_ops.small_attention, "patchify": emu_ops.patchify,
       "dino_assemble": emu_ops.dino_assemble, "special_tokens": emu_ops.special_tokens,
       "col2im_k4s2p1": emu_ops.col2im_k4s2p1, "ocab_attention": emu_ops.ocab_attention,
       "window_attention": emu_ops.window_attention, "channel_mean": emu_ops.channel_mean, "se_scale_add": emu_ops.se_scale_add}


def _l2(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


@pytest.mark.parametrize("fixture", ["vggt_s2_42x42_stress", "iggt_s2_28x56_stress", "iggt_b2s3_28x28_default"])
def test_model_graph_with_emulated_launchers_matches_reference_fixture(monkeypatch, fixture):
    from iggt_official_b200 import ops
    from iggt_official_b200.models import aggregator as agg_mod
    from iggt_official_b200.models.vggt import IGGT, VGGT
    for name, fn in EMU.items():
        monkeypatch.setattr(ops, name, fn)
    monkeypatch.setattr(agg_mod, "_require_cuda", lambda images: None)
    rec = torch.load(os.path.join(ROOT, "tests", "golden", fixture + ".pt"))
    c = rec["case"]
    m = (IGGT if c["model"] == "IGGT" else VGGT)()
    m.load_state_dict(weights.make_state_dict(c["wseed"], c["kind"]), strict=False)
    m.eval()
    m.compute_dtype = m.head_dtype = torch.float32                           # "16-bit" operands kept exact
    g = torch.Generator().manual_seed(c["iseed"])
    images = torch.rand(c["B"], c["S"], 3, c["H"], c["W"], generator=g)
    out = m(images[0] if c["B"] == 1 else images)
    assert _l2(torch.stack(out["pose_enc"]), rec["pose_enc"]) < 1e-4
    for k in ("depth", "depth_conf", "world_points", "world_points_conf") + (("part_feat",) if c["model"] == "IGGT" else ()):
        assert out[k].shape == rec[k].shape, k
        assert _l2(out[k], rec[k]) < 1e-4, (k, _l2(out[k], rec[k]))


def test_cpu_tensors_are_refused_without_the_hook():
    from iggt_official_b200.models.vggt import VGGT
    with pytest.raises(RuntimeError, match="CUDA"):
        VGGT()(torch.zeros(1, 3, 28, 28))


def _range_stress_state_dict(k=2e5):
    """Head activations k x larger than any fp16 can hold, the last 1x1 scaled back by 1 / k: the outputs stay O(1)."""
    sd = weights.make_state_dict(2, "default", prefixes=("aggregator.", "camera_head.", "depth_head.", "point_head."))
    for h in ("depth_head.", "point_head."):
        for i in range(4):
            sd[h + f"projects.{i}.weight"] = sd[h + f"projects.{i}.weight"] * k
            sd[h + f"projects.{i}.bias"] = sd[h + f"projects.{i}.bias"] * k
        sd[h + "scratch.output_conv2.2.weight"] = sd[h + "scratch.output_conv2.2.weight"] / k
    return sd


def test_head_activation_range_switches(monkeypatch):
    """ADVICE r1 (fp16 heads vs a checkpoint with large activations): with activations beyond 65504 the default fp16 heads
    return inf / nan - `check_finite` turns that into a FloatingPointError naming the remedy, and `head_dtype = bfloat16`
    (fp32's exponent range) computes the same network finitely.  Host logic on the CPU with emulated launchers; the same
    scenario runs on the real kernels in tests/test_model_gpu.py."""
    from iggt_official_b200 import ops
    from iggt_official_b200.models import aggregator as agg_mod
    from iggt_official_b200.models.vggt import VGGT
    for name, fn in EMU.items():
        monkeypatch.setattr(ops, name, fn)
    monkeypatch.setattr(agg_mod, "_require_cuda", lambda images: None)
    m = VGGT()
    m.load_state_dict(_range_stress_state_dict(), strict=False)
    m.eval()
    m.compute_dtype = torch.float32
    images = torch.rand(2, 3, 28, 42, generator=torch.Generator().manual_seed(5))
    m.head_dtype = torch.float32
    ref = m(images)
    m.head_dtype = torch.float16
    m.invalidate_packed()
    assert not torch.isfinite(m(images)["depth"]).all()
    m.check_finite = True
    with pytest.raises(FloatingPointError, match="head_dtype = torch.bfloat16"):
        m(images)
    m.head_dtype = torch.bfloat16
    m.invalidate_packed()
    out = m(images)                                           # check_finite still on: must pass
    assert _l2(out["depth"], ref["depth"]) < 3e-2 and _l2(out["world_points"], ref["world_points"]) < 6e-2
