"""PCA feature colours (utils.misc.apply_pca_colormap, csrc/pca.cu) and the exact quantile launcher.

CPU: the host Jacobi eigensolver (iggt_sym_eig) against numpy's eigh, the float64 oracle (oracle/ref_pca.py) against
the unmodified reference's output (tests/golden/pca_ref.npz), import hygiene and argument errors.  GPU: the quantile
launcher against torch.quantile bit for bit, every stage against float64 or torch, and the public call end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden_pca as G                                     # noqa: E402
from oracle import ref_pca                                                  # noqa: E402

# The unmodified reference's fp32 pipeline (randomised PCA, fp32 projection, fp32 stretch) against the float64
# oracle: the stretch divides fp32 rounding of y (a few 1e-7 relative) by hi - lo, which is of the order of y's range
# here.  Measured: 4.1e-7 at 2 x 48 x 64, 2.6e-7 on the demo-shape sample.
ORACLE_VS_REFERENCE = 1e-5
# The device call against the float64 oracle on the demo features: fp32 moments-free projection error (C * 2^-24 of
# sum |x V|) and fp32 quantiles / stretch, divided by hi - lo.
DEVICE_VS_ORACLE = 1e-4
QS = (0.0, 0.02, 0.5, 0.98, 1.0)


def spd(C, seed, kind="random"):
    g = np.random.default_rng(seed)
    q, _ = np.linalg.qr(g.standard_normal((C, C)))
    if kind == "random":
        w = g.uniform(0.1, 10.0, C)
    elif kind == "rank_deficient":
        w = np.concatenate([g.uniform(1.0, 5.0, C - 2), [0.0, 0.0]])
    elif kind == "repeated":
        w = np.concatenate([[4.0, 4.0, 4.0], g.uniform(0.5, 2.0, C - 3)])
    a = (q * w) @ q.T
    return (a + a.T) / 2


def eigh_sorted(a):
    w, v = np.linalg.eigh(a)
    order = np.argsort(-w, kind="stable")
    return w[order], ref_pca.sign_convention(v[:, order])


def assert_sign_convention(v):
    for j in range(v.shape[1]):
        col = np.abs(v[:, j])
        k = int(np.flatnonzero(col == col.max())[0])              # the first of the largest-magnitude components
        assert v[k, j] > 0, (j, v[:, j])


# ------------------------------------------------------------------------------------------------ CPU

@pytest.mark.parametrize("C", [3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_sym_eig_random_spd(C, seed):
    from iggt_official_b200 import ops
    a = spd(C, 10 * C + seed)
    w, v = ops.sym_eig(a)
    want_w, want_v = eigh_sorted(a)
    assert np.abs(w - want_w).max() <= 1e-12 * np.abs(want_w).max()
    assert np.abs(v - want_v).max() <= 1e-10
    assert_sign_convention(v)


@pytest.mark.parametrize("C", [3, 8])
def test_sym_eig_diagonal_and_sorted(C):
    from iggt_official_b200 import ops
    d = np.random.default_rng(C).uniform(1, 9, C)
    w, v = ops.sym_eig(np.diag(d))
    assert np.array_equal(w, np.sort(d)[::-1])
    assert np.array_equal(v, np.eye(C)[:, np.argsort(-d, kind="stable")])
    d_sorted = np.sort(d)[::-1]
    w, v = ops.sym_eig(np.diag(d_sorted))
    assert np.array_equal(w, d_sorted) and np.array_equal(v, np.eye(C))
    w, v = ops.sym_eig(np.diag([2.0, 5.0, 5.0] + [1.0] * (C - 3)))   # a tie keeps the lower index first
    assert np.array_equal(v[:, 0], np.eye(C)[1]) and np.array_equal(v[:, 1], np.eye(C)[2])


@pytest.mark.parametrize("C", [3, 5, 8])
def test_sym_eig_rank_deficient(C):
    from iggt_official_b200 import ops
    a = spd(C, 100 + C, "rank_deficient")
    w, v = ops.sym_eig(a)
    want_w, want_v = eigh_sorted(a)
    scale = np.abs(want_w).max()
    assert np.abs(w - want_w).max() <= 1e-12 * scale
    # distinct non-zero eigenvalues: the vectors are unique; the two zero eigenvalues span a plane
    assert np.abs(v[:, : C - 2] - want_v[:, : C - 2]).max() <= 1e-10
    assert np.abs(v.T @ v - np.eye(C)).max() <= 1e-13
    assert np.abs(a @ v - v * w).max() <= 1e-12 * scale
    assert_sign_convention(v)


@pytest.mark.parametrize("C", [3, 6, 8])
def test_sym_eig_repeated_eigenvalue(C):
    from iggt_official_b200 import ops
    a = spd(C, 200 + C, "repeated")
    w, v = ops.sym_eig(a)
    want_w, _ = eigh_sorted(a)
    scale = np.abs(want_w).max()
    assert np.abs(w - want_w).max() <= 1e-12 * scale
    assert np.abs(v.T @ v - np.eye(C)).max() <= 1e-13
    assert np.abs(a @ v - v * w).max() <= 1e-12 * scale
    assert_sign_convention(v)


def test_sym_eig_sign_convention_on_exact_ties():
    """[[2, 1], [1, 2]] has the eigenvectors (1, 1) / sqrt 2 and (1, -1) / sqrt 2: both components tie on magnitude,
    and the first one is made positive."""
    from iggt_official_b200 import ops
    a = np.array([[2.0, 1.0, 0.0], [1.0, 2.0, 0.0], [0.0, 0.0, 5.0]])
    w, v = ops.sym_eig(a)
    assert np.allclose(w, [5.0, 3.0, 1.0], rtol=0, atol=1e-15)
    assert v[0, 1] == v[1, 1] > 0 and v[0, 2] == -v[1, 2] > 0
    assert np.array_equal(v[:, 0], [0.0, 0.0, 1.0])


def test_sym_eig_rejects_non_finite():
    from iggt_official_b200 import ops
    a = np.eye(3)
    a[1, 2] = np.nan
    with pytest.raises(RuntimeError, match="iggt_sym_eig"):
        ops.sym_eig(a)


def test_oracle_matches_the_reference_golden():
    gold = np.load(G.OUT)
    x = G.features(G.SMALL_SEED, G.SMALL_SHAPE)
    want = ref_pca.apply_pca_colormap(x)
    assert np.abs(gold["small"] - ref_pca.align_flips(gold["small"], want)).max() <= ORACLE_VS_REFERENCE
    x = G.features(G.DEMO_SEED, G.DEMO_SHAPE)
    want = ref_pca.apply_pca_colormap(x).reshape(-1, 3)[gold["demo_idx"]]
    assert np.abs(gold["demo_sample"] - ref_pca.align_flips(gold["demo_sample"], want)).max() <= ORACLE_VS_REFERENCE


def test_oracle_quantile_uses_the_fp32_rank():
    """n - 1 = 2^24 + 1 is not a float32: the rank of q = 1 is float32(n - 1) = 2^24 (clamped to n - 1 anyway) and
    q = 0.5 gives 2^23 exactly; a small case is checked by hand."""
    row = np.arange(5, dtype=np.float64)[::-1].copy()
    assert ref_pca.quantile(row, 0.5) == 2.0 and ref_pca.quantile(row, 0.3) == pytest.approx(1.2, abs=1e-6)
    assert np.float32(0.5) * np.float32(2 ** 24 + 1) == np.float32(2 ** 23)


def test_import_hygiene():
    code = ("import sys; import iggt_official_b200.utils.misc as m; "
            "bad = [k for k in sys.modules if k.split('.')[0] in "
            "('sklearn', 'torch_geometric', 'torch_scatter', 'hdbscan', 'cuml', 'matplotlib', 'cv2', 'evo')]; "
            "assert not bad, bad; "
            "assert all(hasattr(m, k) for k in ('apply_pca_colormap', 'cluster_features_to_masks', "
            "'cluster_features_to_masks_mv', 'knn_avg_features_pyg'))")
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, check=True)


def test_apply_pca_colormap_argument_errors():
    from iggt_official_b200.utils.misc import apply_pca_colormap
    with pytest.raises(ValueError):
        apply_pca_colormap(torch.zeros(4, 5, 8))
    with pytest.raises(ValueError):
        apply_pca_colormap(torch.zeros(1, 4, 5, 2))
    with pytest.raises(ValueError):
        apply_pca_colormap(torch.zeros(1, 4, 5, 9))
    with pytest.raises(ValueError):
        apply_pca_colormap(torch.zeros(1, 4, 5, 8, dtype=torch.int32))


# ------------------------------------------------------------------------------------------------ GPU

def sorted_formula(row, q):
    """torch.quantile's rank rule and ATen's lerp on torch.sort's order statistics (all on the device)."""
    n = row.shape[0]
    s = torch.sort(row).values
    out = []
    for qi in q:
        r = torch.tensor(qi, dtype=torch.float32, device=row.device) * (n - 1)
        lo = r.to(torch.int64).clamp(max=n - 1)
        hi = torch.ceil(r).to(torch.int64).clamp(max=n - 1)
        w = r - lo
        out.append(torch.lerp(s[lo], s[hi], w))
    return torch.stack(out)


def quantile_rows(kind, rows, n, g):
    if kind == "normal":
        return torch.randn(rows, n, generator=g).cuda()
    if kind == "equal":
        return torch.full((rows, n), -1.25).cuda()
    if kind == "duplicates":
        return torch.round(4 * torch.randn(rows, n, generator=g)).cuda()
    if kind == "zeros":                                           # mixed +0 / -0 with a few other values
        z = torch.where(torch.rand(rows, n, generator=g) < 0.5, torch.tensor(0.0), torch.tensor(-0.0))
        other = torch.rand(rows, n, generator=g) < 0.1
        return torch.where(other, torch.randn(rows, n, generator=g), z).cuda()
    if kind == "subnormal":
        return (torch.randn(rows, n, generator=g) * 1e-40).cuda()
    if kind == "negative":
        return (-torch.rand(rows, n, generator=g) - 1e-3).cuda()
    raise ValueError(kind)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3, 1000, 508032])
@pytest.mark.parametrize("kind", ["normal", "equal", "duplicates", "zeros", "subnormal", "negative"])
def test_quantile_equals_torch(n, kind):
    from iggt_official_b200 import ops
    g = torch.Generator().manual_seed(n + len(kind))
    y = quantile_rows(kind, 3, n, g)
    got = ops.quantile(y, QS)
    want = torch.stack([torch.quantile(y[r], torch.tensor(QS, device="cuda")) for r in range(3)])
    assert torch.equal(got, want), (got, want)                   # -0 == +0


@pytest.mark.gpu
def test_quantile_at_2_pow_24_and_padded_rows():
    from iggt_official_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    n = 2 ** 24
    buf = torch.randn(2, n + 5, device="cuda", generator=g)      # row pitch n + 5: unaligned second row
    y = buf[:, :n]
    got = ops.quantile(y, QS)
    for r in range(2):
        assert torch.equal(got[r], torch.quantile(y[r], torch.tensor(QS, device="cuda")))


@pytest.mark.gpu
def test_quantile_beyond_torch_limit():
    from iggt_official_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(2)
    y = torch.randn(1, 17_000_000, device="cuda", generator=g) * 3 + 1
    with pytest.raises(RuntimeError, match="too large"):
        torch.quantile(y[0], 0.5)
    got = ops.quantile(y, QS)
    assert torch.equal(got[0], sorted_formula(y[0], QS))


@pytest.mark.gpu
def test_quantile_nan_row():
    from iggt_official_b200 import ops
    y = torch.randn(2, 1000, device="cuda")
    y[1, 17] = float("nan")
    got = ops.quantile(y, (0.02, 0.98))
    assert torch.isnan(got[1]).all() and not torch.isnan(got[0]).any()


def demo_features(shape=G.DEMO_SHAPE, seed=G.DEMO_SEED):
    return torch.from_numpy(G.features(seed, shape)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("C,offset", [(8, 0.0), (3, 0.0), (5, 1000.0), (8, 300.0)])
def test_stage_moments_and_basis(C, offset):
    from iggt_official_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(C)
    n = 300_001
    x = (torch.randn(n, C, device="cuda", generator=g) @ torch.randn(C, C, device="cuda", generator=g)) + offset
    b = ops.pca_basis(x)
    torch.cuda.synchronize()
    assert int(b.nonfinite.item()) == 0
    d = x.double() - x[0].double()
    iu = torch.triu_indices(C, C)
    want = torch.cat([d.sum(0), (d.T @ d)[iu[0], iu[1]]])
    mag = torch.cat([d.abs().sum(0), (d.abs().T @ d.abs())[iu[0], iu[1]]])
    assert ((b.moments - want).abs() <= 1e-12 * mag).all()
    # the device basis is the host solver's, bit for bit, on the same covariance
    w, v = ops.sym_eig(b.cov.cpu().numpy())
    assert np.array_equal(w, b.evals.cpu().numpy()) and np.array_equal(v, b.evecs.cpu().numpy())
    assert torch.equal(b.V.cpu(), torch.from_numpy(v[:, :3]).float())
    assert torch.allclose(b.cov, torch.cov(x.double().T), rtol=1e-10, atol=1e-12 * float(x.double().var(0).max()))
    # two calls: bit-identical
    b2 = ops.pca_basis(x)
    assert torch.equal(b.moments, b2.moments) and torch.equal(b.evecs, b2.evecs)


@pytest.mark.gpu
def test_stage_nonfinite_count():
    from iggt_official_b200 import ops
    x = torch.randn(10_000, 6, device="cuda")
    x[5, 2] = float("nan")
    x[9000, 0] = float("inf")
    x[9001, 5] = -float("inf")
    assert int(ops.pca_basis(x).nonfinite.item()) == 3


@pytest.mark.gpu
@pytest.mark.parametrize("C,n", [(8, 508_032), (3, 1001), (7, 4099)])
def test_stage_projection_and_stretch(C, n):
    from iggt_official_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(n, C, device="cuda", generator=g) * torch.linspace(0.5, 3.0, C, device="cuda") + 0.7
    b = ops.pca_basis(x)
    y = ops.pca_project(x, b.V)
    V64 = b.V.double()
    want = (x.double() @ V64).T
    bound = C * 2.0 ** -24 * (x.double().abs() @ V64.abs()).T
    assert ((y.double() - want).abs() <= bound).all()
    qv = ops.quantile(y, (0.02, 0.98))
    out = ops.pca_stretch(y, qv)
    ref = torch.empty_like(out)
    for j in range(3):                                            # the reference's torch expression
        lo, hi = qv[j, 0], qv[j, 1]
        ref[:, j] = (y[j] - lo) / (hi - lo) if hi > lo else 0.5
    ref = torch.clamp(ref, 0, 1)
    assert torch.equal(out, ref)


@pytest.mark.gpu
def test_end_to_end_demo_features():
    from iggt_official_b200.utils.misc import apply_pca_colormap
    x = demo_features()
    w, _ = ref_pca.pca_basis(x.reshape(-1, 8).cpu().numpy())
    gaps = (w[:3] - w[1:4]) / w[:3]
    assert gaps.min() > 0.1, gaps                                 # well-separated axes: the oracle's basis is stable
    out = apply_pca_colormap(x)
    assert out.shape == (3, 336, 504, 3) and out.dtype == torch.float32 and out.is_cuda
    want = ref_pca.apply_pca_colormap(x.cpu().numpy())
    assert np.abs(out.cpu().numpy() - want).max() <= DEVICE_VS_ORACLE
    # the unmodified reference (golden sample), channel by channel c or 1 - c
    gold = np.load(G.OUT)
    got = out.reshape(-1, 3).cpu().numpy()[gold["demo_idx"]]
    assert np.abs(got - ref_pca.align_flips(got, gold["demo_sample"])).max() <= DEVICE_VS_ORACLE
    out2 = apply_pca_colormap(x)
    assert torch.equal(out, out2)


@pytest.mark.gpu
def test_end_to_end_small_golden_and_cpu_tensor():
    from iggt_official_b200.utils.misc import apply_pca_colormap
    x = torch.from_numpy(G.features(G.SMALL_SEED, G.SMALL_SHAPE))
    out_cpu = apply_pca_colormap(x)
    assert not out_cpu.is_cuda and out_cpu.dtype == torch.float32
    out_gpu = apply_pca_colormap(x.cuda())
    assert torch.equal(out_cpu, out_gpu.cpu())
    gold = np.load(G.OUT)["small"]
    got = out_cpu.numpy()
    assert np.abs(got - ref_pca.align_flips(got, gold)).max() <= DEVICE_VS_ORACLE
    assert np.abs(got - ref_pca.apply_pca_colormap(x.numpy())).max() <= DEVICE_VS_ORACLE
    out16 = apply_pca_colormap(x.cuda().half())                   # other float dtypes: computed in fp32
    assert out16.dtype == torch.float32
    assert torch.equal(out16, apply_pca_colormap(x.cuda().half().float()))


@pytest.mark.gpu
def test_end_to_end_constant_and_nan():
    from iggt_official_b200.utils.misc import apply_pca_colormap
    out = apply_pca_colormap(torch.full((2, 5, 7, 4), 0.3, device="cuda"))
    assert (out == 0.5).all()
    x = torch.randn(1, 8, 8, 8, device="cuda")
    x[0, 3, 3, 3] = float("nan")
    with pytest.raises(ValueError, match="non-finite"):
        apply_pca_colormap(x)


@pytest.mark.gpu
def test_end_to_end_beyond_torch_limit():
    """16 x 1036^2 x 8 (17.2 M pixels): torch.quantile refuses the reference's rows; here the call runs and its
    quantiles equal the sort-based formula."""
    from iggt_official_b200 import ops
    from iggt_official_b200.utils.misc import apply_pca_colormap
    g = torch.Generator(device="cuda").manual_seed(16)
    mix = torch.randn(8, 8, device="cuda", generator=g)
    x = (torch.randn(16 * 1036 * 1036, 8, device="cuda", generator=g) @ mix).view(16, 1036, 1036, 8)
    out = apply_pca_colormap(x)
    assert out.shape == (16, 1036, 1036, 3) and bool(((out >= 0) & (out <= 1)).all())
    flat = x.view(-1, 8)
    b = ops.pca_basis(flat)
    y = ops.pca_project(flat, b.V)
    qv = ops.quantile(y, (0.02, 0.98))
    for j in range(3):
        assert torch.equal(qv[j], sorted_formula(y[j], (0.02, 0.98)))
    assert torch.equal(out.view(-1, 3), ops.pca_stretch(y, qv))
