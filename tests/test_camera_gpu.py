"""GPU: the one-launch camera head (csrc/camera.cu, iggt_camera_head) against the layer-by-layer path it replaces (same
16-bit weights: only the fp32 summation order differs) and against the oracle's fp32 camera head."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _tokens(B, S, seed):
    g = torch.Generator().manual_seed(seed)
    T = 7
    return torch.randn(B, S, T, 2048, generator=g) * 1.5 + 0.2


@pytest.fixture(scope="module")
def setup():
    from oracle import weights
    from iggt_official_b200.models.vggt import VGGT
    sd = weights.make_state_dict(3, "stress", prefixes=("camera_head.",))
    m = VGGT()
    m.load_state_dict(sd, strict=False)
    m.eval().to("cuda")
    return m.camera_head, sd


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,S", [(1, 8), (1, 3), (2, 4), (1, 1), (1, 13), (2, 8), (4, 4), (4, 16), (5, 3)])
def test_fused_camera_head_matches_layer_path_and_oracle(setup, dtype, B, S):
    from oracle import ref_model
    head, sd = setup
    tok = _tokens(B, S, B * 100 + S).cuda()
    fused = head([None] * 23 + [tok], compute_dtype=dtype)
    layer = head._layers(tok[:, :, 0], head._packed(dtype, tok.device), 4)
    torch.cuda.synchronize()
    assert len(fused) == 4 and fused[0].shape == (B, S, 9) and fused[0].dtype == torch.float32
    f, l = torch.stack(fused).cpu(), torch.stack(layer).cpu()
    assert torch.isfinite(f).all()
    assert ((f - l).abs().max() / l.abs().max()).item() < 2e-4                  # same arithmetic, other summation order
    assert (f[:, :, :, 7:] >= 0).all()                                         # activate_pose: ReLU on the FoV dims
    # oracle: fp32 weights (the product rounds them to 16 bit: 2^-11 fp16 / 2^-8 bf16 relative per weight)
    ref = torch.stack(ref_model.camera_head({k: v.cuda() for k, v in sd.items()}, tok)).cpu()
    tol = 3e-3 if dtype == torch.float16 else 2.5e-2
    assert ((f - ref).norm() / ref.norm()).item() < tol


def test_fused_camera_head_reads_strided_camera_tokens_and_is_repeatable(setup):
    head, _ = setup
    tok = _tokens(1, 8, 5).cuda()
    a = torch.stack(head([None] * 23 + [tok], compute_dtype=torch.float16))
    b = torch.stack(head(None, compute_dtype=torch.float16, camera_tokens=tok[:, :, 0].contiguous()))
    c = torch.stack(head([None] * 23 + [tok], compute_dtype=torch.float16))
    assert torch.equal(a, b) and torch.equal(a, c)                              # static schedule: bit-reproducible


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,S", [(1, 17), (2, 24), (1, 40)])
def test_layer_path_above_16_views_matches_oracle(setup, dtype, B, S):
    """Scenes of more than 16 views run the camera head layer by layer (skinny GEMM, small attention with S keys per
    scene, LayerNorm): the path production takes for them, against the oracle's fp32 camera head."""
    from oracle import ref_model
    head, sd = setup
    tok = _tokens(B, S, B * 100 + S).cuda()
    got = torch.stack(head([None] * 23 + [tok], compute_dtype=dtype)).cpu()
    torch.cuda.synchronize()
    assert got.shape == (4, B, S, 9) and torch.isfinite(got).all()
    assert (got[:, :, :, 7:] >= 0).all()
    ref = torch.stack(ref_model.camera_head({k: v.cuda() for k, v in sd.items()}, tok)).cpu()
    tol = 3e-3 if dtype == torch.float16 else 2.5e-2                           # as for the one-launch head above
    assert ((got - ref).norm() / ref.norm()).item() < tol
