"""GPU: end-to-end parity of the drop-in modules against (a) the committed golden outputs of the unmodified
reference (fp32) and (b) the oracle under the same precision policy (fp16 trunk operands).

Tolerances: the reference's own fp16-autocast vs fp32 gap on these weights is 4e-4 (depth) .. 1.3e-3
(world_points) relative L2 (scripts/parity_report.py); the native path additionally keeps head activations in
16 bit, so it is asserted within 2e-3 (depth, conf) / 5e-3 (points, pose) relative L2 of the fp32 reference
and within 5e-3 / 8e-3 element-wise relative to the tensor maximum."""
import glob
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = sorted(p for p in glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.pt"))
                if os.path.basename(p).startswith(("iggt_", "vggt_")))      # the whole-forward fixtures (make_golden.py)
L2_TOL = {"depth": 2e-3, "depth_conf": 2e-3, "world_points": 5e-3, "world_points_conf": 2e-3, "part_feat": 6e-3,
          "pose_enc": 5e-3}


def _l2(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


def _mx(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-12)).item()


@pytest.fixture(scope="module")
def models():
    from iggt_official_b200.models.vggt import IGGT, VGGT
    return {"IGGT": IGGT(), "VGGT": VGGT()}


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-3] for p in GOLDEN])
@pytest.mark.parametrize("dtype", [torch.float16])
def test_forward_matches_reference_golden(models, path, dtype):
    from oracle import weights
    rec = torch.load(path)
    c = rec["case"]
    sd = weights.make_state_dict(c["wseed"], c["kind"])
    m = models[c["model"]]
    m.load_state_dict(sd, strict=False)
    m.eval().to("cuda")
    m.compute_dtype = dtype
    g = torch.Generator().manual_seed(c["iseed"])
    images = torch.rand(c["B"], c["S"], 3, c["H"], c["W"], generator=g).cuda()
    out = m(images if c["B"] > 1 else images[0])
    torch.cuda.synchronize()
    assert out["images"].shape == (c["B"], c["S"], 3, c["H"], c["W"])
    pose = torch.stack(out["pose_enc"]).cpu()
    assert len(out["pose_enc"]) == 4 and _l2(pose, rec["pose_enc"]) < L2_TOL["pose_enc"]
    keys = ["depth", "depth_conf", "world_points", "world_points_conf"] + (["part_feat"] if c["model"] == "IGGT" else [])
    for k in keys:
        got = out[k].cpu()
        assert got.shape == rec[k].shape and got.dtype == torch.float32, k
        assert _l2(got, rec[k]) < L2_TOL[k], (k, _l2(got, rec[k]))
        assert _mx(got, rec[k]) < 4 * L2_TOL[k], (k, _mx(got, rec[k]))


def test_iggt_odd_grid_raises_like_reference(models):
    m = models["IGGT"].to("cuda")
    m.compute_dtype = torch.float16
    with pytest.raises(RuntimeError):          # 42/14 = 3: the reference's part head raises (SURVEY F2)
        m(torch.rand(2, 3, 42, 42, device="cuda"))


def test_aggregator_interface(models):
    m = models["VGGT"].to("cuda")
    toks, psi = m.aggregator(torch.rand(1, 2, 3, 28, 42, device="cuda"), compute_dtype=torch.float16)
    assert psi == 5 and len(toks) == 24
    for i, t in enumerate(toks):
        if i in (4, 11, 17, 23):
            assert t.shape == (1, 2, 5 + 6, 2048) and t.dtype == torch.float32
        else:
            assert t is None


def test_more_than_12_views_works(models):
    """S = 13 crashes the unmodified reference (SURVEY F3); frames are independent in every head."""
    m = models["VGGT"].to("cuda")
    m.compute_dtype = torch.float16
    out = m(torch.rand(13, 3, 28, 28, device="cuda"))
    assert out["depth"].shape == (1, 13, 28, 28, 1) and torch.isfinite(out["depth"]).all()


def test_head_activation_range_switches_on_the_kernels():
    """The activation-range scenario of tests/test_model_wiring.py on the real kernels: fp16 heads overflow, `check_finite`
    raises, bf16 heads (fp32's exponent range) stay finite and agree with the fp32 oracle to bf16 precision."""
    import sys
    sys.path.insert(0, os.path.dirname(__file__))
    from test_model_wiring import _range_stress_state_dict
    from oracle import ref_model
    from iggt_official_b200.models.vggt import VGGT
    sd = _range_stress_state_dict()
    m = VGGT()
    m.load_state_dict(sd, strict=False)
    m.eval().to("cuda")
    m.compute_dtype = torch.float16
    images = torch.rand(2, 3, 28, 42, generator=torch.Generator().manual_seed(5)).cuda()
    assert not torch.isfinite(m(images)["depth"]).all()
    m.check_finite = True
    with pytest.raises(FloatingPointError, match="head_dtype = torch.bfloat16"):
        m(images)
    m.head_dtype = torch.bfloat16
    out = m(images)
    ref = ref_model.forward({k: v.cuda() for k, v in sd.items()}, images, model="vggt", amp=torch.float16, skip_part=True)
    assert _l2(out["depth"], ref["depth"]) < 3e-2 and _l2(out["world_points"], ref["world_points"]) < 6e-2


def test_model_on_a_second_device_without_set_device():
    """ADVICE r1: launches follow the tensors' device (`model.to("cuda:1")` with device 0 current), incl. the per-device
    kernel configuration; needs two GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from oracle import weights
    from iggt_official_b200.models.vggt import VGGT
    sd = weights.make_state_dict(2, "default", prefixes=("aggregator.", "camera_head.", "depth_head.", "point_head."))
    images = torch.rand(2, 3, 42, 56, generator=torch.Generator().manual_seed(7))
    outs = []
    for dev in ("cuda:0", "cuda:1"):
        m = VGGT()
        m.load_state_dict(sd, strict=False)
        m.eval().to(dev)
        m.compute_dtype = torch.float16
        assert torch.cuda.current_device() == 0
        o = m(images.to(dev))
        assert o["depth"].device == torch.device(dev)
        outs.append({k: (torch.stack(v) if isinstance(v, list) else v).cpu() for k, v in o.items()})
    for k in ("depth", "world_points", "pose_enc"):
        assert _l2(outs[1][k], outs[0][k]) < 1e-4, k
