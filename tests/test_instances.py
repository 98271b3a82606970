"""Instance-mask evaluation (metrics.calculate_iou / evaluate_matched_instances, csrc/instances.cu).

CPU: the numpy + scipy oracle (oracle/ref_instances.py) and the port's host half (fed numpy counts) against the
unmodified reference's results (tests/golden/instances_ref.npz), value for value and type for type; the host
assignment against scipy's linear_sum_assignment pair for pair; argument errors.  GPU: the overlap kernel against
brute-force int64 counts over the masks' shapes, edge sizes and densities; repeated calls; every input form; the public
calls against the fixture and the oracle, end to end on the clustering's masks at the demo shape."""
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden_instances as G                                # noqa: E402
from oracle import ref_instances                                             # noqa: E402

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "instances_ref.npz"))


def golden(key):
    return json.loads(str(GOLDEN[key]))


def tagged(o):
    return json.loads(json.dumps(G.tagged(o)))


# ------------------------------------------------------------------------------------------------ CPU

@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_matches_fixture(name):
    g, p = G.case_masks(name)
    assert tagged(ref_instances.evaluate_matched_instances(g, p, G.CASES[name][2])) == golden(f"{name}_result")


def test_oracle_iou_matches_fixture():
    got = []
    for name, i, j in G.IOU_PAIRS:
        g, p = G.case_masks(name)
        got.append(ref_instances.calculate_iou(g[i], p[j]))
    assert tagged(got) == golden("iou_pairs")


@pytest.mark.parametrize("name", list(G.CASES))
def test_host_half_matches_fixture(name):
    from iggt_official_b200 import metrics
    g, p = G.case_masks(name)
    thr = G.CASES[name][2]
    if len(g) == 0 or len(p) == 0:
        got = metrics.evaluate_matched_instances(g, p, thr)                 # returns before any device work
    else:
        got = metrics._matched_from_counts(*ref_instances.counts(g, p), thr)
    assert tagged(got) == golden(f"{name}_result")


def lsap_cases():
    rng = np.random.default_rng(7)
    shapes = [(1, 1), (1, 9), (9, 1), (3, 8), (8, 3), (17, 17), (40, 120), (120, 40), (300, 300), (250, 300),
              (300, 250)]
    for nr, nc in shapes:
        yield f"rand_{nr}x{nc}", rng.random((nr, nc))
        yield f"equal_{nr}x{nc}", np.full((nr, nc), 0.75)
        yield f"binary_{nr}x{nc}", rng.integers(0, 2, (nr, nc)).astype(np.float64)
        c = rng.integers(0, 4, (nr, nc)).astype(np.float64)
        c[nr // 2:] = c[:nr - nr // 2]                                       # repeated rows
        c[:, nc // 2:] = c[:, :nc - nc // 2]                                 # repeated columns
        yield f"repeats_{nr}x{nc}", c
    for nr, nc in [(5, 5), (6, 11), (11, 6), (40, 64), (64, 40)]:
        g = rng.random((nr, 1, 6, 7)) < rng.random((nr, 1, 1, 1))
        p = rng.random((nc, 1, 6, 7)) < rng.random((nc, 1, 1, 1))
        inter, gs, ps = ref_instances.counts(g, p)
        union = gs[:, None] + ps[None, :] - inter
        iou = np.where(union > 0, inter / np.maximum(union, 1), 0.0)
        yield f"iou_{nr}x{nc}", 1 - iou


LSAP = dict(lsap_cases())


@pytest.mark.parametrize("name", list(LSAP))
def test_linear_sum_assignment_matches_scipy(name):
    from scipy.optimize import linear_sum_assignment
    from iggt_official_b200 import ops
    cost = LSAP[name]
    rows, cols = ops.linear_sum_assignment(cost)
    want_r, want_c = linear_sum_assignment(cost)
    assert rows.dtype == np.int64 and cols.dtype == np.int64
    assert np.array_equal(rows, want_r) and np.array_equal(cols, want_c)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_linear_sum_assignment_rejects_non_finite(bad):
    from iggt_official_b200 import _lib
    cost = np.ones((3, 4))
    cost[1, 2] = bad
    rows, cols = np.empty(3, np.int64), np.empty(3, np.int64)
    assert _lib.load().iggt_linear_sum_assignment(cost.ctypes.data, 3, 4, rows.ctypes.data, cols.ctypes.data) != 0


def test_argument_errors():
    from iggt_official_b200 import metrics
    m = np.zeros((2, 5, 6), bool)
    with pytest.raises(TypeError):
        metrics.evaluate_matched_instances(m.astype(np.uint8), m)
    with pytest.raises(TypeError):
        metrics.evaluate_matched_instances(m, [m[0], m[1].astype(np.float32)])
    with pytest.raises(TypeError):
        metrics.evaluate_matched_instances(torch.zeros(2, 5, 6, dtype=torch.uint8), m)
    with pytest.raises(TypeError):
        metrics.calculate_iou(m[0].astype(np.int64), m[1])
    with pytest.raises(ValueError):
        metrics.evaluate_matched_instances(m, np.zeros((2, 6, 5), bool))
    with pytest.raises(ValueError):
        metrics.evaluate_matched_instances([m[0], np.zeros((5, 7), bool)], m)
    with pytest.raises(ValueError):
        metrics.calculate_iou(m[0], np.zeros(30, bool))


# ------------------------------------------------------------------------------------------------ GPU

def rand_stack(K, n, seed, ld=None, ones_row=True, zero_row=True):
    """uint8 [K, ld] CUDA, 0/1 in the first n bytes of each row, zero padding: a density per row drawn uniformly, plus an
    all-ones and an all-zero row."""
    ld = ld or (n + 15) // 16 * 16
    gen = torch.Generator(device="cuda").manual_seed(seed)
    dens = torch.rand(K, generator=gen, device="cuda").tolist()
    m = torch.zeros((K, ld), dtype=torch.uint8, device="cuda")
    for i in range(K):
        m[i, :n] = torch.rand(n, generator=gen, device="cuda") < dens[i]
    if ones_row:
        m[0, :n] = 1
    if zero_row and K > 2:
        m[K // 2, :n] = 0
    return m


def brute(g, p, n, chunk=1 << 22):
    """Exact int64 counts: fp32 products of 0/1 chunks below 2^24 pixels are exact integers."""
    inter = torch.zeros((g.shape[0], p.shape[0]), dtype=torch.int64, device=g.device)
    for c0 in range(0, n, chunk):
        c1 = min(n, c0 + chunk)
        inter += (g[:, c0:c1].float() @ p[:, c0:c1].float().T).long()
    return inter, g[:, :n].sum(1, dtype=torch.int64), p[:, :n].sum(1, dtype=torch.int64)


def kernel_counts(g, p, n):
    from iggt_official_b200 import ops
    K, P = g.shape[0], p.shape[0]
    c = ops.mask_overlaps(g, p, n)
    return c[:K * P].view(K, P), c[K * P:K * P + K], c[K * P + K:]


def assert_counts(g, p, n):
    got, want = kernel_counts(g, p, n), brute(g, p, n)
    for a, b, what in zip(got, want, ("inter", "gsize", "psize")):
        assert torch.equal(a, b), (what, g.shape[0], p.shape[0], n, (a != b).sum().item())


SIZES = (1, 7, 64, 65, 200, 300)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 15, 16, 127, 129])
def test_mask_overlaps_small_n(n):
    for K in SIZES:
        for P in SIZES:
            assert_counts(rand_stack(K, n, K * 1000 + P), rand_stack(P, n, P * 1000 + K + 1, zero_row=False), n)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [508032, 2264192, 17172736])
def test_mask_overlaps_large_n(n):
    for K, P in ((1, 7), (64, 65), (65, 64), (200, 300), (300, 7)):
        assert_counts(rand_stack(K, n, 3 * K + P), rand_stack(P, n, 5 * P + K), n)
        torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("K,P", [(300, 300), (65, 7), (1, 1)])
def test_mask_overlaps_all_ones(K, P):
    """Every count at its largest: n = 16 x 1036^2 > 2^24 in every total, the largest slice in every CTA."""
    n = 17172736
    g = torch.ones((K, n), dtype=torch.uint8, device="cuda")
    p = torch.ones((P, n), dtype=torch.uint8, device="cuda")
    inter, gs, ps = kernel_counts(g, p, n)
    assert bool((inter == n).all()) and bool((gs == n).all()) and bool((ps == n).all())
    del g, p
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_mask_overlaps_repeats_bit_identical():
    n = 2264192
    g, p = rand_stack(128, n, 1), rand_stack(128, n, 2)
    first = [c.clone() for c in kernel_counts(g, p, n)]
    for _ in range(3):
        for a, b in zip(kernel_counts(g, p, n), first):
            assert torch.equal(a, b)


@pytest.mark.gpu
def test_mask_overlaps_launcher_rejects_unaligned_pitch():
    from iggt_official_b200 import _lib
    g = torch.zeros((4, 64), dtype=torch.uint8, device="cuda")
    out = torch.empty(4 * 4 + 8, dtype=torch.int64, device="cuda")
    lib = _lib.load()
    st = torch.cuda.current_stream().cuda_stream
    args = (out.data_ptr(), out.data_ptr() + 128, out.data_ptr() + 160, st)
    assert lib.iggt_mask_overlaps(g.data_ptr(), 4, 40, g.data_ptr(), 4, 64, 40, *args) < 0       # pitch 40
    assert lib.iggt_mask_overlaps(g.data_ptr() + 1, 4, 64, g.data_ptr(), 4, 64, 40, *args) < 0   # base + 1
    assert lib.iggt_mask_overlaps(g.data_ptr(), 4, 16, g.data_ptr(), 4, 64, 40, *args) < 0       # pitch < n
    torch.cuda.synchronize()


def blob_stack(K, shape, seed, device="cuda"):
    """[K, *shape] bool CUDA masks from a seeded nearest-centre label map (pixels past every centre's radius unset)."""
    gen = torch.Generator(device=device).manual_seed(seed)
    S, H, W = shape
    c = torch.rand((S, K, 2), generator=gen, device=device) * torch.tensor([H, W], device=device)
    yy, xx = torch.meshgrid(torch.arange(H, device=device), torch.arange(W, device=device), indexing="ij")
    lab = torch.empty((S, H, W), dtype=torch.int64, device=device)
    for s in range(S):
        best = torch.full((H, W), float("inf"), device=device)
        lab[s] = -1
        for k in range(K):
            d = (yy - c[s, k, 0]) ** 2 + (xx - c[s, k, 1]) ** 2
            upd = (d < best) & (d < (0.25 * min(H, W)) ** 2)
            best = torch.where(upd, d, best)
            lab[s][upd] = k
    return lab[None] == torch.arange(K, device=device)[:, None, None, None]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 37, 41), (2, 16, 32)])
def test_input_forms_agree(shape):
    from iggt_official_b200 import metrics
    g, p = blob_stack(9, shape, 1), blob_stack(12, shape, 2)
    gh, ph = g.cpu().numpy(), p.cpu().numpy()
    want = ref_instances.counts(gh, ph)
    n = int(np.prod(shape))
    if n % 16 == 0:                                     # a contiguous, aligned CUDA stack is read in place
        assert metrics._mask_stack(g, 9, n, g.device).data_ptr() == g.data_ptr()
    forms = {
        "cuda_stack": (g, p),
        "non_contiguous": (g.transpose(2, 3).contiguous().transpose(2, 3), torch.stack([p, p], 1).flatten(0, 1)[::2]),
        "cuda_list": (list(g), list(p)),
        "ndarray_stack": (gh, ph),
        "ndarray_list": (list(gh), list(ph)),
        "cpu_tensor_stack": (g.cpu(), p.cpu()),
        "mixed": (gh, p),
    }
    for form, (a, b) in forms.items():
        got = metrics._mask_counts(a, b)
        for x, y in zip(got, want):
            assert x.dtype == np.int64 and np.array_equal(x, y), form
    if torch.cuda.device_count() > 1:
        g1, p1 = g.to("cuda:1"), p.to("cuda:1")
        got = metrics._mask_counts(g1, p1)
        assert torch.cuda.current_device() == 0
        for x, y in zip(got, want):
            assert np.array_equal(x, y), "cuda:1"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(G.CASES))
def test_public_matches_fixture(name):
    from iggt_official_b200 import metrics
    g, p = G.case_masks(name)
    thr = G.CASES[name][2]
    assert tagged(metrics.evaluate_matched_instances(g, p, thr)) == golden(f"{name}_result")
    if len(g) and len(p):
        gt, pt = torch.from_numpy(np.stack(g)).cuda(), torch.from_numpy(np.stack(p)).cuda()
        assert tagged(metrics.evaluate_matched_instances(gt, pt, thr)) == golden(f"{name}_result")


@pytest.mark.gpu
def test_calculate_iou_matches_fixture():
    from iggt_official_b200 import metrics
    got = []
    for name, i, j in G.IOU_PAIRS:
        g, p = G.case_masks(name)
        got.append(metrics.calculate_iou(g[i], p[j]))
        assert tagged(metrics.calculate_iou(torch.from_numpy(g[i]).cuda(), torch.from_numpy(p[j]).cuda())) == \
            tagged(got[-1])
    assert tagged(got) == golden("iou_pairs")


@pytest.mark.gpu
@pytest.mark.parametrize("shape,K,P", [((3, 336, 504), 32, 40), ((8, 532, 532), 128, 128), ((8, 532, 532), 150, 90)])
def test_public_matches_oracle_large(shape, K, P):
    """Perturbed blob masks at the demo and part-head shapes: the public call equals the oracle's host arithmetic on
    brute-force counts, for every threshold."""
    from iggt_official_b200 import metrics
    g, p = blob_stack(K, shape, 11), blob_stack(P, shape, 11)
    n = int(np.prod(shape))
    p[: min(K, P) // 2] = g[: min(K, P) // 2].roll(3, dims=-1)     # overlapping pairs, shifted by 3 pixels
    inter, gs, ps = (x.cpu().numpy() for x in brute(g.view(K, n).view(torch.uint8), p.view(P, n).view(torch.uint8), n))
    for thr in (0.0, 0.5, 1.0):
        want = ref_instances.matched_from_counts(inter, gs, ps, thr)
        assert tagged(metrics.evaluate_matched_instances(g, p, thr)) == tagged(want), thr


@pytest.mark.gpu
def test_end_to_end_on_clustered_masks():
    """The instance masks of cluster_features_to_masks_mv on the seeded demo features (as scripts/bench_cluster.py makes
    them) scored against a seeded perturbation of themselves, at the demo shape: equal to the oracle."""
    from iggt_official_b200 import metrics
    from iggt_official_b200.utils import misc
    from oracle.make_golden_cluster import DEMO_KWARGS, KNN_K, demo_inputs
    pts, feats = demo_inputs(shape=(3, 336, 504))
    labels = misc.cluster_features_to_masks_mv(misc.knn_avg_features_pyg(pts, feats, k=KNN_K), **DEMO_KWARGS)
    rng = np.random.default_rng(5)
    gt = np.roll(labels, 4, axis=2)                               # shifted, relabelled, noisy ground truth
    ids = np.unique(gt)
    gt = rng.permutation(ids.max() + 1)[gt]
    noise = rng.random(gt.shape) < 0.03
    gt[noise] = rng.integers(0, ids.max() + 1, int(noise.sum()))
    pred_ids, gt_ids = np.unique(labels), np.unique(gt)
    pred_masks = torch.from_numpy(labels).cuda()[None] == torch.from_numpy(pred_ids).cuda()[:, None, None, None]
    gt_masks = [gt == k for k in gt_ids]
    assert len(pred_ids) > 1
    for thr in (0.0, 0.5):
        want = ref_instances.evaluate_matched_instances(gt_masks, pred_masks.cpu().numpy(), thr)
        assert tagged(metrics.evaluate_matched_instances(gt_masks, pred_masks, thr)) == tagged(want)
