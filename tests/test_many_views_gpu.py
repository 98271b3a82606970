"""GPU: scenes of more views than the camera head's small_attention holds in shared memory (197 and up at head dim 128).
Cheapest first: the key-streaming token attention (csrc/heads.cu, `iggt_token_attention`) element by element against
float64 at small and large N, its adversarial logit orders and structure, then the camera head above the cap against
the oracle, which attention the head selects at the cap, and whole forwards of hundreds of small views.

The per-element bound is derived from the kernel's operation order in tests/token_attention_ref.py; the CPU tests
(tests/test_many_views_cpu.py) show it accepts an fp32 statement of the same tile walk at every shape used here and
rejects the walk with one rescale left out."""
import pytest
import torch

import token_attention_ref as ta

pytestmark = pytest.mark.gpu

H, D = 16, 128


@pytest.fixture(scope="module")
def ops():
    from iggt_official_b200 import ops as _ops
    return _ops


def _check(ops, qkv, B, N, what):
    out = ops.token_attention(qkv, B, N, H, D)
    torch.cuda.synchronize()
    assert out.shape == (B * N, H * D) and torch.isfinite(out).all(), what
    o64, bound = ta.reference_and_bound(qkv, B, N, H, D)
    r = ta.worst_ratio(out, o64, bound)
    print(f"[bound] token_attention {what}: {r:.3g}")
    assert r <= 1.0, f"{what}: worst {r:.3g} x bound"
    return out


# -------------------------------------------------------------------------------------------- kernel, against float64
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("N", [1, 2, 33, 63, 64, 65, 196, 197, 256, 257, 500, 1000, 2049])
def test_token_attention(ops, N, B):
    _check(ops, ta.random_qkv(B, N, H, D, seed=37 + N, device="cuda"), B, N, f"N={N} B={B}")


@pytest.mark.parametrize("N", [197, 257, 1000])
@pytest.mark.parametrize("kind", ta.ADVERSARIAL)
def test_token_attention_adversarial_logits(ops, kind, N):
    qkv = ta.logits_qkv(1, N, H, D, ta.adversarial_logits(kind, N, seed=N), seed=N, device="cuda")
    _check(ops, qkv, 1, N, f"{kind} N={N}")


# ------------------------------------------------------------------------------------------------------- structure
def test_token_attention_is_repeatable_and_scenes_are_independent(ops):
    B, N = 2, 300
    qkv = ta.random_qkv(B, N, H, D, seed=5, device="cuda")
    a = ops.token_attention(qkv, B, N, H, D)
    b = ops.token_attention(qkv, B, N, H, D)
    other = qkv.clone()
    other[N:] = ta.random_qkv(1, N, H, D, seed=6, device="cuda")             # scene 1 replaced
    c = ops.token_attention(other, B, N, H, D)
    torch.cuda.synchronize()
    assert torch.equal(a, b)                                                   # fixed tile order, no atomics
    assert torch.equal(a[:N], c[:N]) and not torch.equal(a[N:], c[N:])


@pytest.mark.parametrize("N", [2, 64, 65, 196])
def test_token_attention_agrees_with_small_attention_below_the_cap(ops, N):
    """not bit-equal (the summation orders differ), within the sum of both kernels' bounds (small_attention's as in
    tests/test_heads_bounds_gpu.py::test_small_attention)"""
    B = 3
    qkv = ta.random_qkv(B, N, H, D, seed=37 + N, device="cuda")
    t = ops.token_attention(qkv, B, N, H, D)
    s = ops.small_attention(qkv, B, N, H, D)
    torch.cuda.synchronize()
    _, bound_t = ta.reference_and_bound(qkv, B, N, H, D)
    q, k, v = ta.split(qkv.double(), B, N, H, D)
    scale = D ** -0.5
    sc = q @ k.transpose(-1, -2) * scale
    p = torch.softmax(sc, -1)
    dd = (D * ta.U24 * scale * (q.abs() @ k.abs().transpose(-1, -2)) + 2.0 ** -23 * sc.abs()
          + ta.U24 * (sc - sc.amax(-1, keepdim=True)).abs() + 2.0 ** -22)
    pd, va = p * dd, v.abs()
    bound_s = ta.flat(pd @ va + (p @ v).abs() * (pd.sum(-1, keepdim=True) + (-(-N // 32) + 8) * ta.U24)
                      + N * ta.U24 * (p @ va))
    r = ((t.double() - s.double()).abs() / (bound_t + bound_s)).max().item()
    print(f"[bound] token vs small attention N={N}: {r:.3g}")
    assert r <= 1.0


# ---------------------------------------------------------------------------------------- camera head above the cap
def _tokens(B, S, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, S, 7, 2048, generator=g) * 1.5 + 0.2


@pytest.fixture(scope="module")
def camera():
    """stress camera-head weights, as tests/test_camera_gpu.py"""
    from oracle import weights
    from iggt_official_b200.models.vggt import VGGT
    sd = weights.make_state_dict(3, "stress", prefixes=("camera_head.",))
    m = VGGT()
    m.load_state_dict(sd, strict=False)
    m.eval().to("cuda")
    return m.camera_head, sd


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,S", [(1, 197), (1, 300), (2, 256), (1, 1000)])
def test_camera_head_above_the_cap_matches_oracle(camera, dtype, B, S):
    from oracle import ref_model
    head, sd = camera
    tok = _tokens(B, S, B * 100 + S).cuda()
    got = torch.stack(head([None] * 23 + [tok], compute_dtype=dtype)).cpu()
    torch.cuda.synchronize()
    assert got.shape == (4, B, S, 9) and torch.isfinite(got).all()
    assert (got[:, :, :, 7:] >= 0).all()
    ref = torch.stack(ref_model.camera_head({k: v.cuda() for k, v in sd.items()}, tok)).cpu()
    tol = 3e-3 if dtype == torch.float16 else 2.5e-2      # test_camera_gpu.py::test_layer_path_above_16_views_matches_oracle
    err = ((got - ref).norm() / ref.norm()).item()
    print(f"[camera] B={B} S={S} {dtype}: rel-L2 vs oracle {err:.3g}")
    assert err < tol


def _refuse(*a, **k):
    raise AssertionError("this attention must not run at this view count")


def test_camera_head_selects_small_attention_up_to_the_cap(camera, monkeypatch, ops):
    head, _ = camera
    monkeypatch.setattr(ops, "token_attention", _refuse)
    got = head([None] * 23 + [_tokens(1, 196, 1).cuda()], compute_dtype=torch.float16)
    assert torch.isfinite(torch.stack(got)).all()


def test_camera_head_selects_token_attention_above_the_cap(camera, monkeypatch, ops):
    head, _ = camera
    monkeypatch.setattr(ops, "small_attention", _refuse)
    got = head([None] * 23 + [_tokens(1, 197, 1).cuda()], compute_dtype=torch.float16)
    assert torch.isfinite(torch.stack(got)).all()


# ------------------------------------------------------------------------------ whole forwards of hundreds of views
L2_TOL = {"depth": 2e-3, "depth_conf": 2e-3, "world_points": 5e-3, "world_points_conf": 2e-3, "part_feat": 6e-3,
          "pose_enc": 5e-3}                                                    # tests/test_model_gpu.py
PERM_TOL = {"depth": 4e-3, "depth_conf": 4e-3, "world_points": 1e-2, "world_points_conf": 4e-3,
            "pose_enc": 1e-2}                                                  # tests/test_fullsize_gpu.py
KEYS = ["depth", "depth_conf", "world_points", "world_points_conf"]


def _l2(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


def _mx(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-12)).item()


@pytest.fixture(scope="module")
def fp32_oracle():
    """the oracle in fp32 without TF32 (the fixtures of tests/test_model_gpu.py are fp32 reference outputs)"""
    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags


def _model(cls, seed):
    from oracle import weights
    sd = weights.make_state_dict(seed, "stress")
    m = cls()
    m.load_state_dict(sd, strict=False)
    m.eval().to("cuda")
    m.compute_dtype = torch.float16
    return m, {k: v.cuda() for k, v in sd.items()}


def _against_oracle(out, ref, keys):
    pe, rp = torch.stack(out["pose_enc"]), torch.stack(ref["pose_enc"])
    print(f"[forward] pose_enc: rel-L2 {_l2(pe, rp):.3g}")
    assert _l2(pe, rp) < L2_TOL["pose_enc"]
    for k in keys:
        assert out[k].shape == ref[k].shape, k
        print(f"[forward] {k}: rel-L2 {_l2(out[k], ref[k]):.3g} max-rel {_mx(out[k], ref[k]):.3g}")
        assert _l2(out[k], ref[k]) < L2_TOL[k], k
        assert _mx(out[k], ref[k]) < 4 * L2_TOL[k], k


@pytest.fixture(scope="module")
def vggt300(fp32_oracle):
    from iggt_official_b200.models.vggt import VGGT
    m, sd = _model(VGGT, 8)
    images = torch.rand(2, 300, 3, 28, 28, generator=torch.Generator().manual_seed(12)).cuda()
    with torch.no_grad():
        base = m(images[:1])
    torch.cuda.synchronize()
    return m, sd, images, base


def test_vggt_forward_of_300_views_matches_oracle(vggt300):
    from oracle import ref_model
    m, sd, images, base = vggt300
    assert base["depth"].shape == (1, 300, 28, 28, 1) and base["pose_enc"][0].shape == (1, 300, 9)
    with torch.no_grad():
        ref = ref_model.forward(sd, images[:1], model="vggt", amp=None, skip_part=True)
    _against_oracle(base, ref, KEYS)


def test_300_views_after_the_first_are_permutation_equivariant(vggt300):
    """the camera attention spans all views: permuting views 1..S-1 permutes every per-view output, pose included"""
    m, _, images, base = vggt300
    perm = torch.cat([torch.zeros(1, dtype=torch.long), 1 + torch.randperm(299, generator=torch.Generator().manual_seed(2))])
    perm = perm.cuda()
    with torch.no_grad():
        out = m(images[:1, perm])
    torch.cuda.synchronize()
    for k in KEYS:
        assert _l2(out[k], base[k][:, perm]) < PERM_TOL[k], (k, _l2(out[k], base[k][:, perm]))
    pe = _l2(torch.stack(out["pose_enc"]), torch.stack(base["pose_enc"])[:, :, perm])
    print(f"[forward] permuted pose_enc: rel-L2 {pe:.3g}")
    assert pe < PERM_TOL["pose_enc"]


def test_two_scenes_of_300_views_are_independent(vggt300):
    m, _, images, base = vggt300
    with torch.no_grad():
        both = m(images)
        second = m(images[1:])
    torch.cuda.synchronize()
    for k in KEYS:
        assert _l2(both[k][:1], base[k]) < PERM_TOL[k], k
        assert _l2(both[k][1:], second[k]) < PERM_TOL[k], k
    pe = torch.stack(both["pose_enc"])
    assert _l2(pe[:, :1], torch.stack(base["pose_enc"])) < PERM_TOL["pose_enc"]
    assert _l2(pe[:, 1:], torch.stack(second["pose_enc"])) < PERM_TOL["pose_enc"]


def test_iggt_forward_of_200_views_matches_oracle(fp32_oracle):
    from oracle import ref_model
    from iggt_official_b200.models.vggt import IGGT
    m, sd = _model(IGGT, 9)
    images = torch.rand(1, 200, 3, 28, 28, generator=torch.Generator().manual_seed(13)).cuda()
    with torch.no_grad():
        out = m(images)
        ref = ref_model.forward(sd, images, model="iggt", amp=None)
    torch.cuda.synchronize()
    _against_oracle(out, ref, KEYS + ["part_feat"])
