"""Exact tests of the two point-search kernels behind the instance masks, csrc/cluster.cu (HDBSCAN core distances,
Borůvka MST, noise fill) and csrc/knn.cu (k-NN feature smoothing), against brute-force host references.

What the kernels promise.  Every search is exact for any point order: the Morton order only tightens the tile boxes,
and box and point distances use the same fp32 operations, so rounding never lets a pruned box hide a candidate.  The
MST is defined by the strict total order (weight, smaller original index, larger original index) on edges, so the tree
is unique.  The noise fill gives an unlabelled point the label of its nearest labelled point, ties to the lowest
original index.  Core distances are the k-th smallest squared distance to another point, 1 <= k <= 512.

Exact data.  On dyadic lattice points (small integers times 2^-s, `as_lattice` checks the range) every fp32
difference, square and fma of a squared distance is exact, so the kernels' distances equal the float64 ones bit for
bit whatever their operation order, and exact ties are plentiful.  The host references are then unique and bit-exact:
  core2[i]   the k-th smallest d2(i, j) over j != i, counted with multiplicity;
  MST        Prim's algorithm under the total order above (the unique tree, so also Kruskal's: the CPU tests check
             both on tie-heavy data, and the total weight against scipy);
  fill       the label of argmin_j (d2(i, j), j) over the labelled j;
  k-NN       the k smallest d2(i, .) without i, inf past n - 1; the features are small integers, so the fp32 sum is
             exact in any order and the mean is float32(sum) / float32(count).

Any data, any order (the `_any_order` tests).  On float data every search runs twice, in the library's Morton order
and in a random permutation, where every tile box spans nearly everything and nothing is pruned.  Mapped back to the
original indices the results agree bit for bit; k-NN index sets agree wherever the k-th and (k+1)-th distances differ,
and the means, summed in a different order, within k 2^-24 sum|f|.

The GPU tests reach an order other than Morton's by calling the reorder launchers through `ops._call`.

Negative controls, one-line changes to cluster.cu, each run against this file on an H100:
* fill tie rule `oj >= bo` -> `oj <= bo` (the highest index wins a tie): test_fill_exact[last_tile, empty_tiles,
  sparse_ids, ties] fail;
* Borůvka without the index comparison at `w2 == bw2`: test_mst_exact (8 of 11 cases, either another tree or a
  launcher error) and test_cluster_any_order fail;
* cl_reorder_kernel leaving the last warp's points out of the box: test_reorder_and_boxes, test_core_distances_exact
  [4097-1..3], test_mst_exact[blobs, far] and test_cluster_any_order[blobs] fail;
* CorePolicy::want `<` -> `<=` (also searches tiles that only tie the bound, still exact): every case passes.

Measured on an H100 80GB HBM3 (1980 MHz maximum SM clock), once at a 400 W and once at a 700 W power limit: the whole
file (135 cases; the second-device case needs two GPUs) in about 18 s of test time, 20 s with start-up.
"""
import functools
import math

import numpy as np
import pytest
import torch

TILE = 256                      # points per tile and per bounding box in both kernels


# ------------------------------------------------------------------------------------------------ data

def as_lattice(ints, shift):
    """integer coordinates -> float32 points ints * 2^-shift on which squared distances are exact in fp32"""
    ints = np.asarray(ints, np.int64)
    span = int(ints.max() - ints.min()) if ints.size else 0
    assert ints.shape[1] * span * span < 2 ** 24      # every partial sum of a squared distance fits in 24 bits
    return (ints * 2.0 ** -shift).astype(np.float32)


def lattice(n, dim, levels, shift, seed):
    """n points with coordinates drawn from {0 .. levels - 1} * 2^-shift"""
    return as_lattice(np.random.default_rng(seed).integers(0, levels, (n, dim)), shift)


def lattice_blobs(n, seed, centres, size=6, background=0.05, shift=6):
    """lattice blobs: a centre (integer vector) plus offsets in {0 .. size - 1}, and a share of background points
    anywhere in the centres' span"""
    g = np.random.default_rng(seed)
    centres = np.asarray(centres, np.int64)
    nb = int(n * background)
    pts = centres[g.integers(0, len(centres), n - nb)] + g.integers(0, size, (n - nb, centres.shape[1]))
    bg = g.integers(centres.min(), centres.max() + size, (nb, centres.shape[1]))
    return as_lattice(np.concatenate([pts, bg])[g.permutation(n)], shift)


def float_blobs(n, seed, k=6, dim=8, spread=0.05, background=0.05):
    """clustered float data: k Gaussian blobs of unequal size and spread plus uniform background points"""
    g = np.random.default_rng(seed)
    centres = g.uniform(-1, 1, (k, dim))
    w = g.uniform(0.5, 2.0, k)
    sizes = np.floor((n - int(n * background)) * w / w.sum()).astype(int)
    parts = [centres[i] + spread * g.uniform(0.5, 1.5) * g.standard_normal((s, dim)) for i, s in enumerate(sizes)]
    parts.append(g.uniform(-1.2, 1.2, (n - sizes.sum(), dim)))
    return np.concatenate(parts).astype(np.float32)[g.permutation(n)]


def scene(views, h, w, seed, outliers=0.01):
    """demo-like 3-D point maps: rippled surfaces from shifted cameras (1/z^2 density) with far outliers"""
    g = np.random.default_rng(seed)
    v, u = np.mgrid[0:h, 0:w].astype(np.float32)
    pts = []
    for s in range(views):
        z = 2.0 + 0.8 * np.sin(u / 17 + s) + 0.5 * np.cos(v / 11) + 0.02 * g.standard_normal((h, w))
        z = np.where(g.random((h, w)) < outliers, z * g.uniform(20, 200, (h, w)), z)
        pts.append(np.stack([(u - w / 2) / w * z + 0.3 * s, (v - h / 2) / w * z, z], -1))
    return np.stack(pts).reshape(-1, 3).astype(np.float32)


def small_int_feats(n, F, seed):
    return np.random.default_rng(seed).integers(-8, 9, (n, F)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ host references

def d2_block(x, rows, cols=None):
    """float64 squared distances from the points x[rows] to x[cols] (all points by default)"""
    x = x.astype(np.float64)
    y = x if cols is None else x[cols]
    return ((x[rows, None, :] - y[None, :, :]) ** 2).sum(-1)


def ref_nearest_d2(x, m, chunk=128):
    """[n, m]: every point's ascending squared distances to the other points (with multiplicity), inf past n - 1"""
    n = len(x)
    mm = min(m, n - 1)
    out = np.full((n, m), np.inf)
    for r0 in range(0, n, chunk):
        rows = np.arange(r0, min(n, r0 + chunk))
        d = d2_block(x, rows)
        d[np.arange(len(rows)), rows] = np.inf
        if 0 < mm < n - 1:
            d = np.partition(d, mm - 1, axis=1)[:, :mm]
        out[rows, :mm] = np.sort(d, axis=1)[:, :mm]
    return out


def ref_core2(x, k):
    return ref_nearest_d2(x, k)[:, k - 1]


def ref_mst(x, core2):
    """The minimum spanning tree of the mutual-reachability graph w2(i, j) = max(core2[i], core2[j], d2(i, j)) under
    the total order (w2, smaller index, larger index), by Prim's algorithm: every step adds the least edge out of the
    tree, which is in the unique tree.  -> (pairs [n-1, 2] with a < b, in lexicographic order; their w2)"""
    n = len(x)
    xd, c = x.astype(np.float64), core2.astype(np.float64)
    ids = np.arange(n)
    tree = np.zeros(n, bool)
    bw, blo, bhi = np.full(n, np.inf), np.full(n, n), np.full(n, n)    # each outside vertex's least edge to the tree
    pairs, ws = [], []
    v = 0
    for _ in range(n - 1):
        tree[v] = True
        w = np.maximum(np.maximum(c[v], c), ((xd - xd[v]) ** 2).sum(1))
        lo, hi = np.minimum(ids, v), np.maximum(ids, v)
        better = ~tree & ((w < bw) | ((w == bw) & ((lo < blo) | ((lo == blo) & (hi < bhi)))))
        bw[better], blo[better], bhi[better] = w[better], lo[better], hi[better]
        s = ~tree & (bw == np.where(tree, np.inf, bw).min())            # lexicographic minimum over the outside
        s &= blo == np.where(s, blo, n).min()
        v = int(np.argmin(np.where(s, bhi, n)))
        pairs.append((blo[v], bhi[v]))
        ws.append(bw[v])
    pairs = np.array(pairs, np.int64).reshape(-1, 2)
    o = np.lexsort((pairs[:, 1], pairs[:, 0]))
    return pairs[o], np.array(ws)[o]


def kruskal(x, core2):
    """Kruskal's algorithm over all pairs sorted by (w2, smaller index, larger index): the CPU cross-check of ref_mst"""
    n = len(x)
    i, j = np.triu_indices(n, 1)
    w = np.maximum(np.maximum(core2[i], core2[j]).astype(np.float64), ((x[i].astype(np.float64) - x[j]) ** 2).sum(1))
    parent = list(range(n))

    def find(a):
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a

    pairs, ws = [], []
    for e in np.lexsort((j, i, w)):
        ra, rb = find(i[e]), find(j[e])
        if ra != rb:
            parent[ra] = rb
            pairs.append((i[e], j[e]))
            ws.append(w[e])
    pairs = np.array(pairs, np.int64).reshape(-1, 2)
    o = np.lexsort((pairs[:, 1], pairs[:, 0]))
    return pairs[o], np.array(ws)[o]


def ref_fill(x, labels, chunk=256):
    """-> (labels after the fill, number of unlabelled points whose nearest labelled points carry different labels)"""
    lab = np.flatnonzero(labels >= 0)
    q = np.flatnonzero(labels < 0)
    out = labels.astype(np.int64)
    ties = 0
    for r0 in range(0, len(q), chunk):
        rows = q[r0:r0 + chunk]
        d = d2_block(x, rows, lab)
        out[rows] = labels[lab[np.argmin(d, axis=1)]]                    # the first minimum: the lowest index
        nearest = d == d.min(1, keepdims=True)
        lmax = np.where(nearest, labels[lab], -1).max(1)
        lmin = np.where(nearest, labels[lab], 1 << 30).min(1)
        ties += int((lmax != lmin).sum())
    return out, ties


def exact_mean(feats, idx):
    """mean of the feature rows idx >= 0 of every row: float32(exact sum of small integers) / float32(count)"""
    valid = idx >= 0
    s = (feats.astype(np.float64)[np.where(valid, idx, 0)] * valid[..., None]).sum(1)
    return s.astype(np.float32) / np.maximum(valid.sum(1), 1).astype(np.float32)[:, None]


def tile_boxes(xs):
    """[ceil(n / 256), 2 dim]: per-axis minimum, then maximum, of every tile of 256 consecutive points"""
    return np.stack([np.concatenate([xs[c:c + TILE].min(0), xs[c:c + TILE].max(0)]) for c in range(0, len(xs), TILE)])


def assert_bits(got, want, what=""):
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == np.float32 and want.dtype == np.float32 and got.shape == want.shape, (what, got.dtype, want.dtype)
    bad = got.view(np.uint32) != want.view(np.uint32)
    if bad.any():
        at = tuple(np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} differ, first at {at}: {got[at]!r} != {want[at]!r}")


def exact32(v):
    """float64 -> float32, asserting that the value is representable (the lattice references are exact)"""
    f = np.asarray(v).astype(np.float32)
    assert np.array_equal(f.astype(np.float64), np.asarray(v, np.float64))
    return f


# ------------------------------------------------------------------------------------------------ CPU: the references

def test_lattice_distances_are_exact_in_fp32():
    """The premise of the exact tests: on lattice points an fp32 squared distance does not depend on the operation
    order.  Summing the 8 squares in fp32 forwards and backwards both give the float64 value."""
    for x in (lattice(300, 8, 6, 6, 1), lattice_blobs(300, 2, [[0] * 8, [200] * 8], background=0.0),
              lattice(300, 3, 16, 4, 3)):
        d = x[:, None, :] - x[None, :, :]                                # fp32, exact
        fwd = np.zeros(d.shape[:2], np.float32)
        bwd = np.zeros(d.shape[:2], np.float32)
        for a in range(x.shape[1]):
            fwd = fwd + d[..., a] * d[..., a]
            bwd = bwd + d[..., -1 - a] * d[..., -1 - a]
        want = d2_block(x, np.arange(len(x)))
        assert np.array_equal(fwd, want) and np.array_equal(bwd, want)


def test_reference_distances_match_kdtree():
    from scipy.spatial import cKDTree
    g = np.random.default_rng(0)
    for n, dim, k in [(500, 8, 1), (500, 8, 17), (400, 3, 32), (300, 8, 299)]:
        x = g.standard_normal((n, dim))
        near = ref_nearest_d2(x, k)
        d, _ = cKDTree(x).query(x, k=k + 1)
        assert np.allclose(near, d[:, 1:] ** 2, rtol=1e-12, atol=0)
        assert np.allclose(ref_core2(x, k), d[:, k] ** 2, rtol=1e-12, atol=0)
    # fewer other points than k: inf-padded
    near = ref_nearest_d2(np.array([[0.0, 0, 0], [1, 0, 0], [3, 0, 0]]), 4)
    assert np.array_equal(near, [[1, 9, np.inf, np.inf], [1, 4, np.inf, np.inf], [4, 9, np.inf, np.inf]])
    assert np.array_equal(ref_nearest_d2(np.zeros((1, 3)), 2), [[np.inf, np.inf]])


def test_reference_mst_is_kruskal_and_minimal():
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import minimum_spanning_tree
    g = np.random.default_rng(1)
    for x, k in [(lattice(90, 8, 3, 2, 3), 3), (lattice(120, 8, 2, 1, 4), 5), (g.standard_normal((150, 8)), 4)]:
        n = len(x)
        core = ref_core2(x, k)
        pairs, w = ref_mst(x, core)
        kp, kw = kruskal(x, core)
        assert np.array_equal(pairs, kp) and np.array_equal(w, kw)      # ties included: the tree is unique
        i, j = np.triu_indices(n, 1)
        m = np.maximum(np.maximum(core[i], core[j]), ((x[i].astype(np.float64) - x[j]) ** 2).sum(1))
        t = minimum_spanning_tree(csr_matrix((np.where(m == 0, 1e-300, m), (i, j)), shape=(n, n)))  # keep zeros
        assert t.nnz == n - 1 and np.isclose(np.where(t.data == 1e-300, 0, t.data).sum(), w.sum(), rtol=1e-12)


def test_reference_mst_hand_cases():
    # all points identical: every weight is 0, and the order makes the tree the star around point 0
    pairs, w = ref_mst(np.zeros((6, 8), np.float32), np.zeros(6))
    assert np.array_equal(pairs, [[0, j] for j in range(1, 6)]) and (w == 0).all()
    # two points: one edge of weight max(core, d2) = d2
    pairs, w = ref_mst(np.array([[0.0] * 8, [0.5] + [0.0] * 7]), np.array([0.25, 0.25]))
    assert np.array_equal(pairs, [[0, 1]]) and np.array_equal(w, [0.25])
    # unit square, k = 1: core2 = 1, the four sides weigh 1 and the diagonals 2; the order keeps the sides
    # (0,1), (0,2), (1,3) and drops (2,3)
    sq = np.array([[0, 0], [1, 0], [0, 1], [1, 1]], np.float32)
    core = ref_core2(sq, 1)
    assert np.array_equal(core, [1, 1, 1, 1])
    pairs, w = ref_mst(sq, core)
    assert np.array_equal(pairs, [[0, 1], [0, 2], [1, 3]]) and np.array_equal(w, [1, 1, 1])


def test_reference_fill_hand_cases():
    x = np.array([[0], [4], [2], [1], [3]], np.float32)
    out, ties = ref_fill(x, np.array([5, 3, -1, -1, -1]))
    assert np.array_equal(out, [5, 3, 5, 5, 3]) and ties == 1               # x = 2 ties: index 0 wins
    out, ties = ref_fill(x, np.array([3, 5, -1, -1, -1]))
    assert np.array_equal(out, [3, 5, 3, 3, 5]) and ties == 1
    out, ties = ref_fill(np.array([[0], [2], [1], [1]], np.float32), np.array([-1, 7, -1, 0]))   # a twin at d = 0
    assert np.array_equal(out, [0, 7, 0, 0]) and ties == 0


def test_reference_mean_hand_case():
    f = np.array([[1.0], [2.0], [4.0], [8.0]], np.float32)
    out = exact_mean(f, np.array([[1, 2], [0, -1], [-1, -1], [3, 0]]))
    assert np.array_equal(out, np.array([[3.0], [1.0], [0.0], [4.5]], np.float32))


# ------------------------------------------------------------------------------------------------ GPU helpers

def _ops():
    from iggt_official_b200 import ops
    return ops


def cl_prepare(x, order=None):
    """points [n, <=8] -> (sorted8, orig, box) on the GPU: Morton order (ops.cluster_prepare) or the given order"""
    ops = _ops()
    x8 = torch.from_numpy(np.ascontiguousarray(np.pad(x, ((0, 0), (0, 8 - x.shape[1]))))).cuda()
    if order is None:
        return ops.cluster_prepare(x8)
    n = x8.shape[0]
    order = torch.from_numpy(np.ascontiguousarray(order, np.int64)).cuda()
    sorted8 = torch.full_like(x8, float("nan"))
    orig = torch.full((n,), -1, dtype=torch.int32, device=x8.device)
    box = torch.full(((n + TILE - 1) // TILE, 16), float("nan"), device=x8.device)
    ops._call(x8, "iggt_cluster_reorder", 0, 0, x8.data_ptr(), order.data_ptr(), n, sorted8.data_ptr(), orig.data_ptr(),
              box.data_ptr(), ops._STREAM)
    return sorted8, orig, box


def knn_reorder(p, order):
    ops = _ops()
    n = p.shape[0]
    order = torch.from_numpy(np.ascontiguousarray(order, np.int64)).cuda()
    sorted4 = torch.full((n, 4), float("nan"), device=p.device)
    aabb = torch.full(((n + TILE - 1) // TILE, 6), float("nan"), device=p.device)
    ops._call(p, "iggt_knn_reorder", 0, 0, p.data_ptr(), order.data_ptr(), n, sorted4.data_ptr(), aabb.data_ptr(),
              ops._STREAM)
    return sorted4, aabb


def knn_run(x, feats, k, order=None, stats=None):
    """-> (mean [n, F] or None, idx [n, k], d2 [n, k]) as numpy, at the original indices"""
    ops = _ops()
    p = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    f = None if feats is None else torch.from_numpy(feats).cuda()
    if order is None:
        out, idx, d2 = ops.knn_mean_features(p, f, k, return_graph=True, stats=stats)
    else:
        n = p.shape[0]
        sorted4, aabb = knn_reorder(p, order)
        out = None if f is None else torch.empty_like(f)
        idx = torch.empty((n, k), dtype=torch.int32, device=p.device)
        d2 = torch.empty((n, k), dtype=torch.float32, device=p.device)
        ops._call(p, "iggt_knn_mean_features", 0, 0, sorted4.data_ptr(), aabb.data_ptr(), n, k, ops._ptr(f),
                  0 if f is None else f.shape[1], ops._ptr(out), idx.data_ptr(), d2.data_ptr(), ops._ptr(stats),
                  ops._STREAM)
    return tuple(None if t is None else t.cpu().numpy() for t in (out, idx, d2))


def at_orig(v_sorted, orig):
    """a per-sorted-position result -> the same at the original indices"""
    v, o = v_sorted.cpu().numpy(), orig.cpu().numpy().astype(np.int64)
    assert np.array_equal(np.sort(o), np.arange(len(o)))
    out = np.empty_like(v)
    out[o] = v
    return out


def edge_set(a, b, w2):
    """device MST edges -> (pairs [n-1, 2] with a < b, in lexicographic order; their w2)"""
    a, b, w2 = (t.cpu().numpy() for t in (a, b, w2))
    pairs = np.stack([np.minimum(a, b), np.maximum(a, b)], 1).astype(np.int64)
    o = np.lexsort((pairs[:, 1], pairs[:, 0]))
    return pairs[o], w2[o]


def check_knn(x, feats, k, near, out, idx, d2):
    """device k-NN of lattice points against the reference rows `near` (width >= k)"""
    n = len(x)
    valid = idx >= 0
    assert (valid.sum(1) == min(k, n - 1)).all()
    assert (idx < n).all() and not (idx == np.arange(n)[:, None]).any()
    srt = np.sort(idx, 1)
    assert not ((srt[:, 1:] == srt[:, :-1]) & (srt[:, 1:] >= 0)).any(), "a neighbour appears twice"
    xd = x.astype(np.float64)
    slot = ((xd[np.where(valid, idx, 0)] - xd[:, None]) ** 2).sum(-1)
    assert_bits(np.where(valid, d2, 0), exact32(np.where(valid, slot, 0)), "d2 of each returned neighbour")
    assert np.isposinf(d2[~valid]).all()
    assert_bits(np.sort(d2, 1), exact32(near[:, :k]), "sorted neighbour distances")
    if feats is not None:
        assert_bits(out, exact_mean(feats, idx), "neighbour mean")


# ------------------------------------------------------------------------------------------------ 1. reorder and boxes

@pytest.mark.gpu
@pytest.mark.parametrize("order_kind", ["random", "morton"])
@pytest.mark.parametrize("n", [1, 255, 257, 513, 1000, 4097])
def test_reorder_and_boxes(n, order_kind):
    """sorted == x[order] bit for bit, orig == order, and every box the exact per-axis min / max of its tile, the
    ragged last tile included (the ±inf of the padding lanes must not leak into it)"""
    g = np.random.default_rng(n)
    x = g.standard_normal((n, 8)).astype(np.float32)
    order = g.permutation(n) if order_kind == "random" else None
    sorted8, orig, box = cl_prepare(x, order)
    o = orig.cpu().numpy().astype(np.int64)
    if order is None:
        assert np.array_equal(np.sort(o), np.arange(n))
        order = o
    assert np.array_equal(o, order)
    assert_bits(sorted8.cpu().numpy(), x[order], "sorted8")
    assert_bits(box.cpu().numpy(), tile_boxes(x[order]), "cluster boxes")
    p = np.ascontiguousarray(x[:, :3])
    sorted4, aabb = knn_reorder(torch.from_numpy(p).cuda(), order)
    s = sorted4.cpu().numpy()
    assert_bits(np.ascontiguousarray(s[:, :3]), p[order], "sorted4 xyz")
    assert np.array_equal(s.view(np.int32)[:, 3], order)
    assert_bits(aabb.cpu().numpy(), tile_boxes(p[order]), "k-NN boxes")


# ------------------------------------------------------------------------------------------------ 2. core distances

CORE_N = [2, 3, 31, 33, 63, 65, 255, 256, 257, 513, 4097]
CORE_K = [1, 2, 3, 192, 193, 256, 511, 512]
CORE_CASES = sorted({(n, k) for n in CORE_N for k in CORE_K + [n - 1] if 1 <= k < n and k <= 512})


@functools.lru_cache(maxsize=None)
def core_data(n):
    """8-d lattice points, a twentieth of them exact copies of others, and every point's sorted distances"""
    x = lattice(n, 8, 6, 6, seed=n)
    x[n - n // 20:] = x[:n // 20]
    return x, ref_nearest_d2(x, min(512, n - 1))


@pytest.mark.gpu
@pytest.mark.parametrize("n,k", CORE_CASES)
def test_core_distances_exact(n, k):
    x, near = core_data(n)
    sorted8, orig, box = cl_prepare(x)
    core2 = _ops().cluster_core(sorted8, box, k)
    assert_bits(at_orig(core2, orig), exact32(near[:, k - 1]), f"core2 n={n} k={k}")


# ------------------------------------------------------------------------------------------------ 3. MST

def mst_data(kind, n):
    if kind == "lattice":
        return lattice(n, 8, 6, 6, seed=n + 1)
    if kind == "blobs":                                  # lattice blobs with 5 % background
        return lattice_blobs(n, n, np.random.default_rng(n).integers(0, 4, (5, 8)) * 12)
    if kind == "identical":
        return np.full((n, 8), 0.375, np.float32)
    if kind == "far":                                    # two blobs far apart: whole tiles become one component
        return lattice_blobs(n, n, [[0] * 8, [200] * 8], background=0.0)
    raise ValueError(kind)


MST_CASES = [("lattice", 2, 1), ("lattice", 3, 1), ("lattice", 33, 2), ("lattice", 257, 3), ("lattice", 513, 16),
             ("lattice", 4097, 100), ("blobs", 4097, 10), ("blobs", 3001, 1), ("identical", 300, 5),
             ("identical", 2, 1), ("far", 3000, 10)]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,n,k", MST_CASES)
def test_mst_exact(kind, n, k):
    """The n - 1 device edges are the unique tree, each w2 is its pair's mutual reachability bit for bit, the
    launcher returns 0 (ops raises otherwise), and every Borůvka round at least halves the number of components."""
    ops = _ops()
    x = mst_data(kind, n)
    sorted8, orig, box = cl_prepare(x)
    core2 = ops.cluster_core(sorted8, box, k)
    a, b, w2, rounds = ops.cluster_mst(sorted8, box, orig, core2)
    core = at_orig(core2, orig)
    assert_bits(core, exact32(ref_core2(x, k)), "core2")
    pairs, w = edge_set(a, b, w2)
    own = np.maximum(np.maximum(core[pairs[:, 0]], core[pairs[:, 1]]).astype(np.float64),
                     ((x[pairs[:, 0]].astype(np.float64) - x[pairs[:, 1]]) ** 2).sum(1))
    assert_bits(w, exact32(own), "w2 of each device edge")
    want_pairs, want_w = ref_mst(x, core)
    assert np.array_equal(pairs, want_pairs), f"{int((pairs != want_pairs).any(1).sum())} edges differ"
    assert_bits(w, exact32(want_w), "w2")
    assert rounds <= math.ceil(math.log2(n)), rounds
    if kind == "identical":
        assert np.array_equal(pairs, [[0, j] for j in range(1, n)]) and (w == 0).all()


# ------------------------------------------------------------------------------------------------ 4. noise fill

FILL_CASES = ["one", "last_tile", "empty_tiles", "all", "sparse_ids", "ties"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", FILL_CASES)
def test_fill_exact(case):
    """labels at the original index equal the reference (labelled points keep their own), rgb == palette[label]"""
    ops = _ops()
    seed = FILL_CASES.index(case)
    g = np.random.default_rng(100 + seed)
    n = {"last_tile": 1000, "all": 777, "ties": 3000}.get(case, 2000)
    x = lattice(n, 8, 3, 2, seed) if case == "ties" else lattice(n, 8, 6, 6, seed)
    sorted8, orig, box = cl_prepare(x)
    lab_sorted = np.full(n, -1, np.int32)                # chosen by sorted position, where the tiles are
    pos = np.arange(n)
    if case == "one":
        lab_sorted[g.integers(n)] = 2
    elif case == "last_tile":                            # only in the last, ragged tile (232 points)
        sel = (pos >= n // TILE * TILE) & (g.random(n) < 0.3)
        lab_sorted[sel] = g.integers(0, 3, int(sel.sum()))
    elif case == "empty_tiles":                          # only in tiles 1 and 6 of 8: the rest have tcount == 0
        sel = np.isin(pos // TILE, [1, 6]) & (g.random(n) < 0.2)
        lab_sorted[sel] = g.integers(0, 4, int(sel.sum()))
    elif case == "all":
        lab_sorted[:] = g.integers(0, 5, n)
    elif case == "sparse_ids":                           # non-contiguous labels, 8-row palette
        sel = g.random(n) < 0.1
        lab_sorted[sel] = np.where(g.random(int(sel.sum())) < 0.5, 0, 7)
    else:                                                # a coarse lattice: exact ties between different labels
        sel = g.random(n) < 0.1
        lab_sorted[sel] = g.integers(0, 4, int(sel.sum()))
    labels = np.empty(n, np.int32)
    labels[orig.cpu().numpy().astype(np.int64)] = lab_sorted
    palette = g.integers(0, 256, (8, 3), dtype=np.uint8)
    want, ties = ref_fill(x, labels)
    if case == "ties":
        assert ties >= 100, ties
    out, rgb = ops.cluster_fill(sorted8, box, orig, torch.from_numpy(lab_sorted).cuda(), torch.from_numpy(palette).cuda())
    out, rgb = out.cpu().numpy(), rgb.cpu().numpy()
    assert np.array_equal(out, want), f"{int((out != want).sum())} labels differ"
    assert np.array_equal(rgb, palette[want])


# ------------------------------------------------------------------------------------------------ 5. k-NN

@functools.lru_cache(maxsize=None)
def knn_data(n):
    """3-d lattice points on 16^3 sites (duplicates and ties everywhere) and every point's 32 nearest distances"""
    x = lattice(n, 3, 16, 4, seed=n)
    return x, ref_nearest_d2(x, 32)


@pytest.mark.gpu
@pytest.mark.parametrize("F", [1, 3, 4, 8])
@pytest.mark.parametrize("k", [1, 8, 9, 16, 17, 24, 25, 32])
def test_knn_exact(k, F):
    """both sides of every KMAX template, scalar (F = 1, 3) and float4 (F = 4, 8) feature tails"""
    x, near = knn_data(3000)
    feats = small_int_feats(len(x), F, seed=10 * k + F)
    check_knn(x, feats, k, near, *knn_run(x, feats, k))


@pytest.mark.gpu
@pytest.mark.parametrize("n,k", [(1, 8), (2, 8), (17, 32), (33, 32), (9, 8)])
def test_knn_exact_few_points(n, k):
    """fewer other points than k (the slots past n - 1 stay empty) and single partial tiles"""
    x, near = knn_data(n)
    feats = small_int_feats(n, 3, seed=n)
    check_knn(x, feats, k, near, *knn_run(x, feats, k))


@pytest.mark.gpu
@pytest.mark.parametrize("k", [8, 32])
def test_knn_reverse_collinear(k):
    """Collinear points gathered in reverse order: candidates arrive in decreasing distance, so every one of them beats
    the current k-th and the per-thread queues fill up inside a tile (more drains than searched tiles)."""
    n = 1500
    x = as_lattice(np.stack([np.arange(n), np.zeros(n, np.int64), np.zeros(n, np.int64)], 1), 4)
    feats = small_int_feats(n, 4, seed=k)
    stats = torch.zeros(3, dtype=torch.int64, device="cuda")
    out, idx, d2 = knn_run(x, feats, k, order=np.arange(n)[::-1], stats=stats)
    check_knn(x, feats, k, ref_nearest_d2(x, k), out, idx, d2)
    _, computed, drains = stats.tolist()
    assert drains > computed, (computed, drains)


# ------------------------------------------------------------------------------------------------ 6. any order

def cluster_all(x, order, labels, k):
    """core2, MST and fill in one order -> results at the original indices"""
    ops = _ops()
    sorted8, orig, box = cl_prepare(x, order)
    core2 = ops.cluster_core(sorted8, box, k)
    a, b, w2, rounds = ops.cluster_mst(sorted8, box, orig, core2)
    lab_sorted = torch.from_numpy(labels[orig.cpu().numpy().astype(np.int64)]).cuda()
    fill, _ = ops.cluster_fill(sorted8, box, orig, lab_sorted)
    return (at_orig(core2, orig),) + edge_set(a, b, w2) + (fill.cpu().numpy(), rounds)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["blobs", "random"])
def test_cluster_any_order(kind):
    g = np.random.default_rng(7)
    x = float_blobs(3 * 112 * 168, 31) if kind == "blobs" else g.standard_normal((100000, 8)).astype(np.float32)
    n = len(x)
    labels = np.full(n, -1, np.int32)
    sel = g.random(n) < 0.1
    labels[sel] = g.integers(0, 6, int(sel.sum()))
    core_m, pairs_m, w_m, fill_m, rounds_m = cluster_all(x, None, labels, 100)
    core_r, pairs_r, w_r, fill_r, rounds_r = cluster_all(x, g.permutation(n), labels, 100)
    assert_bits(core_r, core_m, "core2")
    assert np.array_equal(pairs_r, pairs_m), f"{int((pairs_r != pairs_m).any(1).sum())} edges differ"
    assert_bits(w_r, w_m, "w2")
    assert np.array_equal(fill_r, fill_m), f"{int((fill_r != fill_m).sum())} labels differ"
    assert max(rounds_m, rounds_r) <= math.ceil(math.log2(n)), (rounds_m, rounds_r)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 20, 32])
@pytest.mark.parametrize("kind", ["scene", "random"])
def test_knn_any_order(kind, k):
    g = np.random.default_rng(8)
    x = scene(3, 112, 168, 9) if kind == "scene" else g.standard_normal((100000, 3)).astype(np.float32)
    n = len(x)
    feats = g.standard_normal((n, 8)).astype(np.float32)
    out_m, idx_m, d2_m = knn_run(x, feats, k)
    out_r, idx_r, d2_r = knn_run(x, feats, k, order=g.permutation(n))
    assert_bits(np.sort(d2_r, 1), np.sort(d2_m, 1), "sorted neighbour distances")
    same = (np.sort(idx_r, 1) == np.sort(idx_m, 1)).all(1)
    if k < 32:                                           # the k-th and (k+1)-th distance differ: one neighbour set
        d2_next = np.sort(knn_run(x, None, k + 1)[2], 1)
        apart = d2_next[:, k] != d2_next[:, k - 1]
        assert apart.mean() > 0.9 and same[apart].all(), (apart.mean(), int((apart & ~same).sum()))
    assert same.mean() > 0.9, same.mean()
    bound = k * 2.0 ** -24 * np.abs(feats.astype(np.float64)[idx_m.astype(np.int64)]).sum(1)
    err = np.abs(out_r.astype(np.float64) - out_m)
    assert (err[same] <= bound[same]).all(), float((err[same] / np.maximum(bound[same], 1e-300)).max())


# ------------------------------------------------------------------------------------------------ 7. second device

@pytest.mark.gpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_core_distances_on_a_second_device():
    """k = 256 needs the opt-in to more than 48 KB of dynamic shared memory, which holds per device: the same call on
    cuda:1 after one on cuda:0 (no set_device) gives the same bits."""
    ops = _ops()
    x, near = core_data(4097)
    got = []
    for dev in ("cuda:0", "cuda:1"):
        sorted8, orig, box = ops.cluster_prepare(torch.from_numpy(x).to(dev))
        got.append(at_orig(ops.cluster_core(sorted8, box, 256), orig))
    assert_bits(got[1], got[0], "core2 on cuda:1")
    assert_bits(got[0], exact32(near[:, 255]), "core2")
