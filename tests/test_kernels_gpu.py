"""Per-kernel parity tests (GPU): every C-ABI launcher against a plain fp32 PyTorch statement of the
same operator on identical (16-bit-rounded) inputs.  Tolerances are written next to each assert."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


def _tol(dtype):
    # one ulp of the 16-bit output format relative to the tensor's magnitude, plus fp32 reorder noise
    return 2.0 ** -10 if dtype == torch.float16 else 2.0 ** -7


def _relmax(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-6)).item()


@pytest.fixture(scope="module")
def ops():
    from iggt_official_b200 import ops as _ops
    return _ops


def test_relu_epilogues_keep_nan_like_torch(ops):
    """torch.relu(nan) = nan, relu(-inf) = 0, relu(inf) = inf: an overflowed fp16 head activation must stay visible through
    the ReLU epilogues (fmaxf would turn inf - inf into 0 and hand `check_finite` finite garbage)."""
    g = torch.Generator(device="cuda").manual_seed(3)
    a = torch.randn(128, 64, device="cuda", generator=g).half()
    a[5, 0], a[5, 1] = float("inf"), float("-inf")             # row 5: inf - inf = nan where w[:, 0] > 0
    a[9, 0] = float("inf")                                     # row 9: +-inf by the sign of w[:, 0]
    w = (torch.randn(64, 64, device="cuda", generator=g) / 8).half()
    w[:, :2] = w[:, :2].abs() + 0.1
    w[::2, 0] *= -1
    out = ops.gemm_store16(a, w, torch.zeros(64, device="cuda"), act=2).float()
    ref = F.relu(a.float() @ w.float().t())
    torch.cuda.synchronize()
    assert torch.isnan(out[5, 1::2]).all() and (out[5, ::2] == 0).all()      # odd columns inf - inf, even ones -inf - inf
    assert torch.equal(torch.isnan(out), torch.isnan(ref)) and torch.equal(torch.isinf(out), torch.isinf(ref))
    assert torch.isinf(out[9, 1::2]).all() and (out[9, ::2] == 0).all()
    x = torch.randn(1, 8, 8, 64, device="cuda", generator=g).half()
    x[0, 3, 3, 0], x[0, 3, 3, 1] = float("inf"), float("-inf")
    wc = (torch.randn(64, 64, 3, 3, device="cuda", generator=g) / 24).half()
    wc[:, :2] = wc[:, :2].abs() + 0.1
    wp = wc.permute(0, 2, 3, 1).reshape(64, 9 * 64).contiguous()
    y = ops.conv_nhwc(x, wp, torch.zeros(64, device="cuda"), act=2).float()
    assert torch.isnan(y[0, 2:5, 2:5]).all() and torch.isfinite(y[0, 6:, 6:]).all()


def test_attention_plan_is_used_and_cached(ops):
    s, ws = ops.attention_plan(1, 1374, 10992, 16)
    assert s >= 1 and (ws > 0) == (s > 1) and ops.attention_plan(1, 1374, 10992, 16) == (s, ws)
    assert ops.attention_plan(8, 1374, 1374, 16)[0] == 1


@pytest.mark.parametrize("dtype", DTYPES)
def test_patchify_and_assemble(ops, dtype):
    NI, H, W, C = 2, 42, 56, 1024
    g = torch.Generator(device="cuda").manual_seed(13)
    img = torch.rand(NI, 3, H, W, device="cuda", generator=g)
    # patchify is one fp32 subtraction, one IEEE division and one RN16 per element: bit for bit against the same fp32
    # operations with the same constants (RN32 of the decimal mean / std); the KP padding is exactly zero.  The second
    # image set has 3 * 5 * 7 = 105 patches.
    mean = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    for im in (img, torch.rand(3, 3, 70, 98, device="cuda", generator=g)):
        ref = F.unfold((im.cpu() - mean) / std, kernel_size=14, stride=14).transpose(1, 2).reshape(-1, 588).to(dtype)
        for KP in (592, 640):
            A = ops.patchify(im, KP, dtype).cpu()
            assert A.shape == (ref.shape[0], KP)
            assert torch.equal(A[:, :588].view(torch.int16), ref.view(torch.int16)), \
                f"{int((A[:, :588] != ref).sum())} of {ref.numel()} elements differ (KP={KP})"
            assert not A[:, 588:].view(torch.int16).any()
    P, R = (H // 14) * (W // 14), 4
    pe = torch.randn(NI * P, C, device="cuda", generator=g).to(dtype)
    cls = torch.randn(C, device="cuda", generator=g)
    reg = torch.randn(R, C, device="cuda", generator=g)
    pos = torch.randn(1 + P, C, device="cuda", generator=g)
    x = torch.empty(NI * (1 + R + P), C, device="cuda")
    ops.dino_assemble(pe, cls, reg, pos, x, NI, P, R, C)
    torch.cuda.synchronize()
    refx = torch.cat([(cls + pos[0]).expand(NI, 1, C), reg.expand(NI, R, C), pe.float().view(NI, P, C) + pos[1:]], 1)
    assert torch.equal(x.view(NI, 1 + R + P, C), refx)
    cam = torch.randn(2, C, device="cuda", generator=g)
    regt = torch.randn(2, R, C, device="cuda", generator=g)
    T = 1 + R + P
    y = torch.zeros(NI * 2 * T, C, device="cuda")  # 2 scenes x NI views
    ops.special_tokens(cam, regt, y, NI * 2, T, R, C, NI, 0)
    torch.cuda.synchronize()
    y4 = y.view(2, NI, T, C)
    assert torch.equal(y4[:, 0, 0], cam[0].expand(2, C)) and torch.equal(y4[:, 1, 0], cam[1].expand(2, C))
    assert torch.equal(y4[:, 0, 1:1 + R], regt[0].expand(2, R, C)) and torch.equal(y4[:, 1, 1:1 + R], regt[1].expand(2, R, C))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("with_pe", [False, True])
def test_upsample_bilinear(ops, dtype, with_pe):
    g = torch.Generator(device="cuda").manual_seed(17)
    NB, h, w, H, W, C = 2, 19, 23, 37, 41, 128
    x = torch.randn(NB, h, w, C, device="cuda", generator=g).to(dtype)
    tx = torch.randn(W, C // 2, device="cuda", generator=g) if with_pe else None
    ty = torch.randn(H, C // 2, device="cuda", generator=g) if with_pe else None
    out = ops.upsample_bilinear(x, H, W, tx, ty)
    torch.cuda.synchronize()
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), size=(H, W), mode="bilinear", align_corners=True).permute(0, 2, 3, 1)
    if with_pe:
        ref = ref + torch.cat([tx[None, None].expand(NB, H, W, C // 2), ty[None, :, None].expand(NB, H, W, C // 2)], -1)
    assert _relmax(out, ref) < _tol(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("k", [2, 4])
def test_deconv_as_gemm_plus_shuffle(ops, dtype, k):
    from iggt_official_b200.heads.dpt_head import pack_deconv
    g = torch.Generator(device="cuda").manual_seed(19)
    NB, h, w, C = 2, 5, 7, 64
    x = torch.randn(NB, h, w, C, device="cuda", generator=g).to(dtype)
    wt = (torch.randn(C, C, k, k, device="cuda", generator=g) / 8).to(dtype)
    b = torch.randn(C, device="cuda", generator=g)
    wp, bp = pack_deconv(wt, b, dtype, "cuda")
    y = ops.gemm_store16(x.view(-1, C), wp, bp)
    out = ops.deconv_shuffle(y, NB, h, w, C, k)
    torch.cuda.synchronize()
    ref = F.conv_transpose2d(x.float().permute(0, 3, 1, 2), wt.float(), b, stride=k).permute(0, 2, 3, 1)
    assert out.shape == ref.shape and _relmax(out, ref) < 2 * _tol(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_stride2_conv_as_im2col_gemm(ops, dtype):
    from iggt_official_b200.heads.dpt_head import pack_conv3x3
    g = torch.Generator(device="cuda").manual_seed(23)
    for h, w in [(37, 37), (6, 8)]:
        NB, C = 2, 64
        x = torch.randn(NB, h, w, C, device="cuda", generator=g).to(dtype)
        wt = (torch.randn(128, C, 3, 3, device="cuda", generator=g) / 24).to(dtype)
        b = torch.randn(128, device="cuda", generator=g)
        A, ho, wo = ops.im2col3x3_s2(x)
        out = ops.gemm_store16(A, pack_conv3x3(wt, dtype, "cuda"), b).view(NB, ho, wo, 128)
        torch.cuda.synchronize()
        ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), b, stride=2, padding=1).permute(0, 2, 3, 1)
        assert out.shape == ref.shape and _relmax(out, ref) < 2 * _tol(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M,N,K,act", [(8, 2048, 2048, 0), (3, 9, 1024, 0), (20, 6144, 16, 4), (32, 1024, 8192, 1)])
def test_skinny_gemm(ops, dtype, M, N, K, act):
    g = torch.Generator(device="cuda").manual_seed(31)
    x = torch.randn(M, K, device="cuda", generator=g)
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(dtype)
    b = torch.randn(N, device="cuda", generator=g)
    gam = torch.rand(N, device="cuda", generator=g)
    res = torch.randn(M, N, device="cuda", generator=g)
    out = ops.skinny_gemm(x, w, b, act=act, gamma=gam, resid=res)
    torch.cuda.synchronize()
    ref = x.double() @ w.double().t() + b
    ref = {0: lambda t: t, 1: F.gelu, 4: F.silu}[act](ref)
    ref = res + gam * ref
    assert _relmax(out, ref.float()) < 2e-5       # fp32 activations, exact 16-bit weights: fp32 noise only


def test_small_attention(ops):
    g = torch.Generator(device="cuda").manual_seed(37)
    B, N, H, d = 2, 13, 16, 128
    qkv = torch.randn(B * N, 3 * H * d, device="cuda", generator=g)
    out = ops.small_attention(qkv, B, N, H, d)
    torch.cuda.synchronize()
    q, k, v = qkv.view(B, N, 3, H, d).permute(2, 0, 3, 1, 4)
    ref = (torch.softmax(q @ k.transpose(-1, -2) * d ** -0.5, -1) @ v).transpose(1, 2).reshape(B * N, H * d)
    assert _relmax(out, ref) < 1e-5


# ------------------------------------------------------------------ part-path kernels (csrc/part.cu)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("C", [64, 128, 256])
def test_layernorm16(ops, dtype, C):
    g = torch.Generator(device="cuda").manual_seed(41)
    x = (torch.randn(3, 5, 7, C, device="cuda", generator=g) * 2 + 0.5).to(dtype)
    w = torch.rand(C, device="cuda", generator=g) + 0.5
    b = torch.randn(C, device="cuda", generator=g)
    out = ops.layernorm16(x, w, b)
    torch.cuda.synchronize()
    assert _relmax(out, F.layer_norm(x.float(), (C,), w, b, 1e-5)) < _tol(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_deconv_k4s2p1_as_gemm_plus_col2im(ops, dtype):
    g = torch.Generator(device="cuda").manual_seed(43)
    NB, h, w, C = 2, 5, 6, 64
    x = torch.randn(NB, h, w, C, device="cuda", generator=g).to(dtype)
    wt = (torch.randn(C, C, 4, 4, device="cuda", generator=g) / 16).to(dtype)
    b = torch.randn(C, device="cuda", generator=g)
    wp = wt.permute(2, 3, 1, 0).reshape(16 * C, C).contiguous()
    y = ops.gemm_store16(x.view(-1, C), wp, None)
    out = ops.col2im_k4s2p1(y, b, NB, h, w, C)
    torch.cuda.synchronize()
    ref = F.conv_transpose2d(x.float().permute(0, 3, 1, 2), wt.float(), b, stride=2, padding=1).permute(0, 2, 3, 1)
    assert out.shape == ref.shape and _relmax(out, ref) < 3 * _tol(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_ocab_attention_matches_oracle_window_math(ops, dtype):
    """The kernel against the oracle's restatement of OCAB's partition / unfold / bias (oracle.ref_model._ocab
    internals), including the scrambled query windows."""
    from oracle import ref_model
    g = torch.Generator(device="cuda").manual_seed(47)
    b, h, w, c, ws, heads = 2, 16, 24, 256, 8, 4
    q = torch.randn(b, h, w, c, device="cuda", generator=g).to(dtype)
    k = torch.randn(b, h, w, c, device="cuda", generator=g).to(dtype)
    v = torch.randn(b, h, w, c, device="cuda", generator=g).to(dtype)
    table = torch.randn(361, heads, device="cuda", generator=g) * 0.5
    rpi = ref_model.calculate_rpi_oca(8).cuda()
    out = ops.ocab_attention(q, k, v, table, (rpi % 361).int().contiguous())
    torch.cuda.synchronize()
    qf, kf, vf = (t.float().permute(0, 3, 1, 2) for t in (q, k, v))
    q_win = ref_model.window_partition(qf, ws).view(-1, ws * ws, c)
    kvw = F.unfold(torch.cat([kf, vf], 1), kernel_size=(12, 12), stride=ws, padding=2)
    nw = kvw.shape[-1]
    kvw = kvw.view(b, 2, c, 144, nw).permute(1, 0, 4, 3, 2).reshape(2, b * nw, 144, c)
    d = c // heads
    qh = q_win.reshape(-1, 64, heads, d).permute(0, 2, 1, 3) * d ** -0.5
    kh = kvw[0].reshape(-1, 144, heads, d).permute(0, 2, 1, 3)
    vh = kvw[1].reshape(-1, 144, heads, d).permute(0, 2, 1, 3)
    bias = table[rpi.view(-1)].view(64, 144, -1).permute(2, 0, 1)
    att = torch.softmax(qh @ kh.transpose(-2, -1) + bias.unsqueeze(0), -1)
    o = (att @ vh).transpose(1, 2).reshape(-1, 64, c).view(-1, ws, ws, c)
    ref = ref_model.window_reverse(o, ws, h, w)
    assert _relmax(out, ref) < 2 * _tol(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
def test_window_attention(ops, dtype):
    from oracle import ref_model
    g = torch.Generator(device="cuda").manual_seed(53)
    b, h, w, c, heads = 2, 16, 8, 128, 4
    qkv = torch.randn(b, h, w, 3 * c, device="cuda", generator=g).to(dtype)
    out = ops.window_attention(qkv)
    torch.cuda.synchronize()
    xw = ref_model.window_partition(qkv.float(), 8).view(-1, 64, 3, heads, c // heads).transpose(1, 3)
    q, k, v = xw[:, :, 0], xw[:, :, 1], xw[:, :, 2]
    o = (torch.softmax(q @ k.transpose(-2, -1) * (c // heads) ** -0.5, -1) @ v).transpose(1, 2).reshape(-1, 64, c)
    ref = ref_model.window_reverse(o.view(-1, 8, 8, c), 8, h, w)
    assert _relmax(out, ref) < 2 * _tol(dtype)
