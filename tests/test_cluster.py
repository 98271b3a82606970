"""HDBSCAN of the instance features (cluster_features_to_masks_mv, csrc/cluster.cu).

CPU: the host condensation (iggt_hdbscan_labels) against scikit-learn's make_single_linkage + tree_to_labels on the
same sorted MST, and the oracle's semantics worked out by hand.  GPU: core distances against a float64 KD-tree, the MST
weights against scipy's MST of the dense mutual-reachability matrix, labels against the oracle (scikit-learn)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_cluster as R                                         # noqa: E402

DEMO = {"eps": 0.06, "min_samples": 100, "min_cluster_size": 500}


def blobs(n, seed, k=6, spread=0.05, dim=8, noise_frac=0.05):
    """Seeded clustered 8-d data: k Gaussian blobs of unequal size and spread plus uniform background noise."""
    g = np.random.default_rng(seed)
    centres = g.uniform(-1, 1, (k, dim))
    w = g.uniform(0.5, 2.0, k)
    sizes = np.floor((n - int(n * noise_frac)) * w / w.sum()).astype(int)
    parts = [centres[i] + spread * g.uniform(0.5, 1.5) * g.standard_normal((s, dim)) for i, s in enumerate(sizes)]
    parts.append(g.uniform(-1.2, 1.2, (n - sizes.sum(), dim)))
    x = np.concatenate(parts).astype(np.float32)
    return x[g.permutation(n)]


def mutual_reachability(x, min_samples):
    """Dense float64 mutual-reachability matrix with the contrib min_samples (k-th nearest OTHER point)."""
    x = x.astype(np.float64)
    d = np.sqrt(((x[:, None] - x[None]) ** 2).sum(-1))
    core = np.sort(d, axis=1)[:, min_samples]                 # column 0 is the point itself
    return np.maximum(d, np.maximum(core[:, None], core[None])), core


def mst_from_dense(m):
    """scipy MST of a dense matrix -> [n-1, 3] rows (a, b, w) sorted by weight (stable)."""
    from scipy.sparse.csgraph import minimum_spanning_tree
    t = minimum_spanning_tree(m).tocoo()
    e = np.stack([t.row.astype(np.float64), t.col.astype(np.float64), t.data], 1)
    return e[np.argsort(e[:, 2], kind="mergesort")]


def sklearn_labels(mst, min_cluster_size, eps):
    from sklearn.cluster._hdbscan._linkage import MST_edge_dtype, make_single_linkage
    from sklearn.cluster._hdbscan._tree import tree_to_labels
    rec = np.empty(mst.shape[0], dtype=MST_edge_dtype)
    rec["current_node"] = mst[:, 0].astype(np.int64)
    rec["next_node"] = mst[:, 1].astype(np.int64)
    rec["distance"] = mst[:, 2]
    labels, _ = tree_to_labels(make_single_linkage(rec), min_cluster_size, "eom", False, eps, None)
    return labels.astype(np.int64)


def host_labels(mst, n, min_cluster_size, eps):
    from iggt_official_b200 import ops
    return ops.hdbscan_labels(mst, n, min_cluster_size, eps)


@pytest.mark.parametrize("n,seed,min_samples", [(3000, 0, 10), (1500, 1, 5), (800, 2, 20)])
def test_host_condensation_matches_sklearn(n, seed, min_samples):
    x = blobs(n, seed)
    mst = mst_from_dense(mutual_reachability(x, min_samples)[0])
    assert mst.shape == (n - 1, 3)
    seen_clusters = set()
    for mcs, eps in [(5, 0.0), (15, 0.0), (40, 0.0), (15, 0.05), (15, 0.2), (40, 0.3), (5, 10.0), (2, 0.0)]:
        want = sklearn_labels(mst, mcs, eps)
        got = host_labels(mst, n, mcs, eps)
        assert np.array_equal(got, want), (mcs, eps)
        seen_clusters.add(int(want.max()) + 1)
    # several clusters, and eps = 10 merges everything up to the root's children (a single cluster is not allowed)
    assert max(seen_clusters) >= 3 and min(seen_clusters) <= 2


def test_host_condensation_all_noise():
    x = blobs(400, 3, k=1, noise_frac=0.0)
    mst = mst_from_dense(mutual_reachability(x, 5)[0])
    for mcs, eps in [(300, 0.0), (250, 0.1)]:                       # no split leaves two parts of min_cluster_size
        want = sklearn_labels(mst, mcs, eps)
        assert (want == -1).all()
        assert np.array_equal(host_labels(mst, 400, mcs, eps), want)


def test_host_condensation_duplicates_and_ties():
    """Zero-weight edges (lambda = inf, which sklearn carries into inf / nan stabilities) and tied weights."""
    g = np.random.default_rng(4)
    base = blobs(600, 5, k=3)
    x = np.concatenate([base, base[:150], base[:150], np.repeat(base[200:201], 40, 0)])
    x = x[g.permutation(len(x))]
    n = len(x)
    m, _ = mutual_reachability(x, 3)
    # scipy reads a dense 0 as "no edge": keep the exact zeros explicitly in a sparse matrix
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import minimum_spanning_tree
    iu = np.triu_indices(n, 1)
    zero = m[iu] == 0
    assert zero.any()
    t = minimum_spanning_tree(csr_matrix((np.where(zero, 1e-300, m[iu]), iu), shape=(n, n))).tocoo()
    w = np.where(t.data == 1e-300, 0.0, t.data)
    mst = np.stack([t.row.astype(np.float64), t.col.astype(np.float64), w], 1)
    mst = mst[np.argsort(mst[:, 2], kind="mergesort")]
    assert (mst[:, 2] == 0).sum() >= 40                             # the 41 copies of one point
    # tied weights: round to a coarse grid so that many edges share a weight (any order of equal weights is an MST
    # order; both sides see the same one)
    tied = mst.copy()
    tied[:, 2] = np.round(tied[:, 2], 2)
    tied = tied[np.argsort(tied[:, 2], kind="mergesort")]
    for edges in (mst, tied):
        for mcs, eps in [(5, 0.0), (20, 0.0), (20, 0.05), (60, 0.0), (5, 0.3)]:
            want = sklearn_labels(edges, mcs, eps)
            assert np.array_equal(host_labels(edges, n, mcs, eps), want), (mcs, eps)


def test_oriented_mst_numbers_clusters_like_sklearn():
    """Any MST, oriented from the side of point 0 (the orientation of scikit-learn's Prim MST), gives exactly the labels
    of scikit-learn's own HDBSCAN, numbering included, on well-separated clusters.  (With background points between
    the clusters, the edges that join clusters can tie - two edges of one point weigh its core distance - and the
    numbering then follows scikit-learn's unstable sort of the Prim edges.)"""
    from iggt_official_b200 import ops
    g = np.random.default_rng(8)
    centres = 3.0 * np.eye(8)[:5]
    x = np.concatenate([c + 0.1 * g.standard_normal((150 + 40 * i, 8)) for i, c in enumerate(centres)]).astype(np.float32)
    x = x[g.permutation(len(x))]
    mst = mst_from_dense(mutual_reachability(x, 10)[0])
    flip = g.random(len(mst)) < 0.5                                  # scramble the orientation first
    mst[flip, 0], mst[flip, 1] = mst[flip, 1].copy(), mst[flip, 0].copy()
    got = ops.hdbscan_labels(ops.mst_orient(mst), len(x), 50, 0.0)
    want = R.hdbscan_labels(x, 0.0, 10, 50)
    assert want.max() == 4 and np.array_equal(got, want)


def test_host_condensation_rejects_a_non_tree():
    from iggt_official_b200 import ops
    bad = np.array([[0, 1, 0.5], [1, 0, 0.6]], np.float64)        # a cycle: point 2 is never joined
    with pytest.raises(RuntimeError, match="iggt_hdbscan_labels"):
        ops.hdbscan_labels(bad, 3, 2, 0.0)


def test_oracle_min_samples_offset():
    """Five points on a line: with the contrib min_samples = 2, the core distance is the distance to the 2nd nearest
    OTHER point; sklearn's min_samples = 3 counts the point itself and gives the same value."""
    from sklearn.neighbors import NearestNeighbors
    x = np.array([[0.0], [1.0], [3.0], [7.0], [15.0]])
    d, _ = NearestNeighbors(n_neighbors=3).fit(x).kneighbors(x)
    assert np.allclose(d[:, -1], [3.0, 2.0, 3.0, 6.0, 12.0])          # by hand: 2nd nearest other point
    _, core = mutual_reachability(x.astype(np.float32), 2)
    assert np.allclose(core, [3.0, 2.0, 3.0, 6.0, 12.0])


def test_oracle_jet_endpoints_and_all_noise_colour():
    assert np.allclose(R.jet(0.0), (0.0, 0.0, 0.5)) and np.allclose(R.jet(1.0), (0.5, 0.0, 0.0))
    from iggt_official_b200.utils.misc import jet_lut
    assert np.array_equal(jet_lut(), R.jet_lut())                   # the product restates the same table
    # every pixel noise -> every label 0 -> the single colour jet(0.5)
    x = np.zeros((1, 2, 3, 8), np.float32)
    labels = R.fill_noise(x.reshape(-1, 8), -np.ones(6, np.int64)).reshape(1, 2, 3)
    assert (labels == 0).all()
    col = R.colorize(labels)
    assert (col == (R.jet(0.5) * 255).astype(np.uint8)).all()


def test_palette_matches_the_oracle_colouring():
    from iggt_official_b200.utils.misc import label_palette
    for labels in (np.array([0]), np.arange(7), np.array([0, 1, 2, 5])):
        pal = label_palette(labels)
        masks = labels.reshape(1, 1, -1)
        assert np.array_equal(pal[labels].reshape(1, 1, -1, 3), R.colorize(masks))


def test_api_rejects_bad_input():
    from iggt_official_b200.utils.misc import cluster_features_to_masks_mv as f
    with pytest.raises(ValueError):
        f(np.zeros((4, 8), np.float32), eps=0.1, min_samples=2, min_cluster_size=5)
    with pytest.raises(ValueError):
        f(np.zeros((1, 4, 4, 8), np.float32), eps=0.1, min_samples=2)
    with pytest.raises(ValueError):
        f(np.zeros((1, 4, 4, 9), np.float32), eps=0.1, min_samples=2, min_cluster_size=5)
    with pytest.raises(ValueError):
        f(torch.zeros(1, 2, 2, 8), eps=0.1, min_samples=4, min_cluster_size=5)      # 4 points < min_samples + 1


# ------------------------------------------------------------------------------------------------ GPU

def _prep(x):
    from iggt_official_b200 import ops
    return ops.cluster_prepare(torch.from_numpy(np.pad(x, ((0, 0), (0, 8 - x.shape[1])))).cuda())


@pytest.mark.gpu
@pytest.mark.parametrize("kind,n,k", [("random", 5000, 1), ("random", 5000, 100), ("clustered", 20000, 100),
                                      ("clustered", 6000, 256), ("duplicates", 3000, 100), ("duplicates", 3000, 1),
                                      ("random", 700, 256), ("random", 300, 7), ("random", 1500, 512),
                                      ("clustered", 4097, 511)])
def test_device_core_distances(kind, n, k):
    from scipy.spatial import cKDTree
    from iggt_official_b200 import ops
    g = np.random.default_rng(n + k)
    if kind == "random":
        x = g.standard_normal((n, 8)).astype(np.float32)
    elif kind == "clustered":
        x = blobs(n, k)
    else:
        x = blobs(n // 2, k, k=3)
        x = np.concatenate([x, x[: n - len(x)]])                    # every point has an exact twin
    sorted8, orig, box = _prep(x)
    core2 = ops.cluster_core(sorted8, box, k)
    torch.cuda.synchronize()
    mine = np.empty(n)
    mine[orig.cpu().numpy()] = np.sqrt(core2.cpu().numpy().astype(np.float64))
    d, _ = cKDTree(x.astype(np.float64)).query(x.astype(np.float64), k=k + 1)
    want = d[:, -1] if k > 0 else d
    assert np.allclose(mine, want, rtol=2e-5, atol=1e-6)


@pytest.mark.gpu
@pytest.mark.parametrize("n,seed,min_samples", [(4000, 0, 10), (2500, 1, 100), (1000, 2, 3), (300, 3, 1)])
def test_device_mst(n, seed, min_samples):
    from scipy.sparse.csgraph import connected_components, minimum_spanning_tree
    from scipy.sparse import coo_matrix
    from iggt_official_b200 import ops
    x = blobs(n, seed)
    if seed == 1:
        x[: n // 10] = x[n // 10: 2 * (n // 10)]                   # duplicates: zero distances
    sorted8, orig, box = _prep(x)
    core2 = ops.cluster_core(sorted8, box, min_samples)
    a, b, w2, rounds = ops.cluster_mst(sorted8, box, orig, core2)
    torch.cuda.synchronize()
    a, b = a.cpu().numpy(), b.cpu().numpy()
    w = np.sqrt(w2.cpu().numpy().astype(np.float64))
    assert len(a) == n - 1 and rounds <= 40
    assert connected_components(coo_matrix((np.ones(n - 1), (a, b)), shape=(n, n)), directed=False)[0] == 1
    m, _ = mutual_reachability(x, min_samples)
    t = minimum_spanning_tree(np.where(m == 0, 1e-300, m)).tocoo()   # scipy drops dense zeros: keep them as tiny
    want = np.sort(np.where(t.data == 1e-300, 0.0, t.data))
    assert np.allclose(np.sort(w), want, rtol=1e-6, atol=1e-7)
    assert np.allclose(w, m[a, b], rtol=1e-6, atol=1e-7)          # each edge carries its own mutual reachability


def _ari(a, b):
    from sklearn.metrics import adjusted_rand_score
    return adjusted_rand_score(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("n,seed", [(20000, 10), (60000, 11)])
def test_device_labels_against_oracle(n, seed):
    from iggt_official_b200.utils.misc import cluster_features_to_masks_mv, hdbscan_device
    x = blobs(n, seed, k=8, spread=0.04)
    want_raw = R.hdbscan_labels(x, **DEMO)
    raw, _ = hdbscan_device(torch.from_numpy(x).cuda(), DEMO["eps"], DEMO["min_samples"], DEMO["min_cluster_size"])
    assert raw.max() == want_raw.max() and want_raw.max() >= 3
    assert _ari(raw, want_raw) >= 0.999
    assert ((raw == -1) != (want_raw == -1)).mean() <= 1e-3
    masks = cluster_features_to_masks_mv(x.reshape(1, 1, n, 8), **DEMO)
    assert masks.dtype == np.int64 and masks.shape == (1, 1, n) and (masks >= 0).all()
    # the fill itself, from the same labelled points: nearest labelled point up to fp32 near-ties
    assert (masks.reshape(-1) == R.fill_noise(x, raw)).mean() >= 0.999
    # against the oracle end to end: the background noise (5 %) is far from every cluster, so the few periphery
    # points labelled differently above are the nearest labelled points of many of them
    assert _ari(masks.reshape(-1), R.fill_noise(x, want_raw)) >= 0.99


@pytest.mark.gpu
def test_device_labels_exact_on_separated_blobs():
    """Well separated blobs (no background between them, see test_oriented_mst_numbers_clusters_like_sklearn): the
    labels (numbering included) and the colours equal the oracle's exactly, for C < 8 (zero-padded) and from a CUDA
    tensor."""
    from iggt_official_b200.utils.misc import cluster_features_to_masks_mv
    g = np.random.default_rng(21)
    centres = np.array([[0, 0, 0, 0, 0], [3, 0, 0, 0, 0], [0, 3, 0, 0, 0], [0, 0, 3, 0, 0], [0, 0, 0, 3, 3]], np.float64)
    x = np.concatenate([c + 0.1 * g.standard_normal((1200 + 300 * i, 5)) for i, c in enumerate(centres)]).astype(np.float32)
    x = x[g.permutation(len(x))].reshape(2, 1, -1, 5)
    kw = {"eps": 0.0, "min_samples": 10, "min_cluster_size": 200, "method": "dbscan"}
    want_m, want_c = R.cluster_features_to_masks_mv(x, apply_colormap=True, **kw)
    for inp in (x, torch.from_numpy(x).cuda()):
        m, c = cluster_features_to_masks_mv(inp, apply_colormap=True, **kw)
        assert m.dtype == np.int64 and c.dtype == np.uint8 and c.shape == x.shape[:3] + (3,)
        assert want_m.max() == 4 and np.array_equal(m, want_m)
        assert np.array_equal(c, want_c)


@pytest.mark.gpu
def test_device_all_noise_gives_label_zero():
    from iggt_official_b200.utils.misc import cluster_features_to_masks_mv
    x = np.random.default_rng(5).uniform(-1, 1, (1, 10, 30, 8)).astype(np.float32)
    m, c = cluster_features_to_masks_mv(x, True, eps=0.0, min_samples=5, min_cluster_size=200)
    assert (m == 0).all() and (c == (R.jet(0.5) * 255).astype(np.uint8)).all()
    with pytest.raises(ValueError, match="non-finite"):
        cluster_features_to_masks_mv(np.full((1, 10, 30, 8), np.nan, np.float32), eps=0.1, min_samples=5,
                                     min_cluster_size=20)


@pytest.mark.gpu
def test_device_demo_shape_against_golden():
    """The demo's call on demo-shaped features (3 x 336 x 504) smoothed by knn_avg_features_pyg, against the
    oracle's labels stored by oracle/make_golden_cluster.py."""
    from oracle.make_golden_cluster import KNN_K, OUT, demo_inputs
    from iggt_official_b200.utils.misc import cluster_features_to_masks_mv, knn_avg_features_pyg
    gold = np.load(OUT)
    pts, feats = demo_inputs()
    sm = knn_avg_features_pyg(pts, feats, k=KNN_K)                  # demo_inputs' features are already unit length
    m1, c1 = cluster_features_to_masks_mv(sm, method="dbscan", apply_colormap=True, **DEMO)
    m2, c2 = cluster_features_to_masks_mv(sm, method="dbscan", apply_colormap=True, **DEMO)
    assert np.array_equal(m1, m2) and np.array_equal(c1, c2)
    assert m1.shape == (3, 336, 504) and (m1 >= 0).all()
    assert _ari(m1.reshape(-1), gold["labels"].astype(np.int64)) >= 0.999
    # one colour per label
    pairs = np.unique(np.concatenate([m1.reshape(-1, 1), c1.reshape(-1, 3)], 1), axis=0)
    assert len(pairs) == len(np.unique(m1))
