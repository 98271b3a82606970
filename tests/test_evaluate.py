"""Scene evaluation (metrics.SceneEvaluator, csrc/evaluate.cu, the selection in csrc/pca.cu) and the ground-truth depth
helpers of postprocess.

CPU: the numpy oracle (oracle/ref_eval.py) against the unmodified reference's results (tests/golden/eval_ref.npz), the
host entry points against numpy / scipy bit for bit (rank and interpolation rules, nearest index map) and against
scipy (pose errors), argument errors and import hygiene.  GPU: the masked selection against numpy bit for bit, every
kernel against its host entry point or the oracle, and the public calls end to end against the fixture and the
oracle at the demo's shapes."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden_eval as G                                    # noqa: E402
from oracle import ref_eval                                                 # noqa: E402

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "eval_ref.npz"))
ULP32 = 2.0 ** -23


def sum_bound(n):
    """Relative error of the reference's pairwise float32 sum of n non-negative terms (numpy sums blocks of 128
    sequentially, then pairwise), plus the rounding of the mean and of the percentage."""
    return (19 + max(0.0, math.log2(max(n, 1) / 128))) * 2.0 ** -24 + 4 * 2.0 ** -24


def golden(name):
    return json.loads(str(GOLDEN[f"{name}_result"]))


def close(got, want, rel):
    if want is None or (isinstance(want, float) and math.isnan(want)):
        return got is None or (isinstance(got, float) and math.isnan(got))
    return abs(float(got) - float(want)) <= rel * abs(float(want))


def check_frame(got, want, n, lsq=False):
    bound = sum_bound(n)
    for key, w in want.items():
        g = float(got[key]) if not isinstance(got[key], (int, np.integer)) else int(got[key])
        if key in ("absrel", "mae", "rmse"):
            assert close(g, w, 2 * bound), (key, g, w)
        elif key == "inliers103" or (key == "scaling_factor" and lsq) or (lsq and key.startswith("delta")):
            assert close(g, w, (bound if lsq else 0) + 2 * ULP32), (key, g, w)
        else:
            assert (math.isnan(g) and math.isnan(w)) if isinstance(w, float) and math.isnan(w) else g == w, (key, g, w)


def check_pose(got, want):
    for key, w in want.items():
        g = got[key]
        if key in ("translation_errors", "rotation_errors"):
            g, w = np.asarray(g, float), np.asarray(w, float)
            tol = 1e-10 if key.startswith("rotation") else 1e-12 * np.abs(w).max()
            assert np.abs(g - w).max() <= tol, (key, g, w)
        elif key == "num_poses":
            assert g == w
        elif key.startswith("rotation"):
            assert abs(g - w) <= 1e-10, (key, g, w)
        else:
            assert abs(g - w) <= 1e-12 * abs(w) + 1e-15, (key, g, w)


def check_results(got, want, n, lsq=False):
    """got: a SceneEvaluator result (dicts of numpy scalars), want: the JSON of one; n pixels per frame."""
    got = json.loads(json.dumps(G.plain(got)))
    assert got.keys() == want.keys()
    dg, dw = got["depth_metrics"], want["depth_metrics"]
    assert dg.keys() == dw.keys()
    assert len(dg["per_frame"]) == len(dw["per_frame"])
    for fg, fw in zip(dg["per_frame"], dw["per_frame"]):
        assert fg.keys() == fw.keys()
        check_frame(fg, fw, n, lsq)
    bound = 2 * sum_bound(n) + 4 * ULP32
    for key, w in dw.items():
        if key == "per_frame":
            continue
        g = dg[key]
        if key.endswith("_std"):
            base = max(abs(dw[key.replace("_std", "_max")]), abs(dw[key.replace("_std", "_min")]))
            assert abs(g - w) <= 4 * bound * base, (key, g, w)
        elif isinstance(w, int):
            assert g == w, key
        else:
            assert close(g, w, bound), (key, g, w)
    check_pose(got["pose_metrics"], want["pose_metrics"])
    assert got["summary"].keys() == want["summary"].keys()


def case_inputs(name):
    sargs, eargs = G.CASES[name]
    gt, pred, gp, pp = G.scene(**sargs)
    return gt, pred, gp, pp, eargs


# ------------------------------------------------------------------------------------------------ CPU

@pytest.mark.parametrize("name", [n for n in G.CASES if n != "sparse"])
def test_oracle_matches_reference(name):
    gt, pred, gp, pp, e = case_inputs(name)
    got = ref_eval.evaluate_scene({"gt_depth": gt, "gt_extrinsic": gp}, {"depth": pred, "extrinsic": pp},
                                  e["alignment"], e["clip"])
    check_results(got, golden(name), gt[0].size, lsq=e["alignment"] == "least_squares")


def test_oracle_sparse_matches_reference():
    from iggt_official_b200 import metrics
    gt, pred, _, _, e = case_inputs("sparse")
    rec, _ = ref_eval.depth_records(gt, pred, e["alignment"], e["clip"], sparse=True)
    for i, want in enumerate(golden("sparse")):
        got = json.loads(json.dumps(G.plain(metrics._frame_metrics(rec[i], gt[0].size, e["alignment"]))))
        check_frame(got, want, gt[0].size)


def value_patterns(rng, n):
    kind = rng.integers(0, 6)
    if kind == 0:
        return rng.standard_normal(n).astype(np.float32)
    if kind == 1:
        return rng.integers(0, 4, n).astype(np.float32)                      # duplicates and zeros
    if kind == 2:
        return (rng.standard_normal(n) * 1e-39).astype(np.float32)           # subnormals
    if kind == 3:
        return -np.abs(rng.standard_normal(n) * 10 ** rng.uniform(-3, 3)).astype(np.float32)
    if kind == 4:
        x = rng.standard_normal(n).astype(np.float32)
        x[rng.random(n) < 0.2] = np.nan
        return x
    x = rng.standard_normal(n).astype(np.float32)
    x[rng.random(n) < 0.05] = np.inf
    return x


def test_quantile_rule_matches_numpy():
    from iggt_official_b200 import ops
    rng = np.random.default_rng(0)
    cases = 0
    for it in range(3000):
        n = int(rng.choice([1, 2, 3, 4, 5, rng.integers(1, 64), rng.integers(1, 5000)]))
        x = value_patterns(rng, n)
        x[x == 0] = 0.0                                     # numpy may return either sign of a zero
        s = np.sort(x)
        p = float(rng.choice([rng.uniform(0, 100), 0, 1, 2, 50, 98, 99, 100, 33.3, 66.7]))
        with np.errstate(all="ignore"), __import__("warnings").catch_warnings():
            __import__("warnings").simplefilter("ignore")
            want = {ops.QRULE_NUMPY: np.percentile(x, p), ops.QRULE_NUMPY_NAN: np.nanpercentile(x, p),
                    ops.QRULE_MEDIAN: np.median(x)}
        for rule, w in want.items():
            got = ops.quantile_rule(s, rule, p)
            assert np.float32(w).tobytes() == got.tobytes() or (np.isnan(w) and np.isnan(got)), (n, p, rule, w, got)
            cases += 1
    assert cases == 9000


@pytest.mark.parametrize("n", [(1 << 24) + 3, (1 << 24) + 1001])
def test_quantile_rule_past_2_24(n):
    from iggt_official_b200 import ops
    x = np.random.default_rng(n).standard_normal(n).astype(np.float32)
    s = np.sort(x)
    for p in (1.0, 37.5, 99.0):
        assert ops.quantile_rule(s, ops.QRULE_NUMPY, p).tobytes() == np.float32(np.percentile(x, p)).tobytes()
    assert ops.quantile_rule(s, ops.QRULE_MEDIAN).tobytes() == np.float32(np.median(x)).tobytes()


def test_zoom_index_matches_scipy():
    from scipy import ndimage
    from iggt_official_b200 import ops
    pairs = [(a, b) for a in range(1, 80, 3) for b in range(1, 80, 2)]
    pairs += [(336, 480), (504, 640), (518, 1168), (518, 1752), (40, 48), (56, 64), (1752, 518), (2, 1), (3, 2)]
    for a, b in pairs:
        x = np.arange(a, dtype=np.float64)[:, None]
        z = ndimage.zoom(x, [1 / (a / b), 1.0], order=0, mode="mirror", grid_mode=True)[:, 0].astype(np.int32)
        assert z.shape == (b,) and np.array_equal(ops.zoom_nearest_index(a, b), z), (a, b)


def pose_sets():
    rng = np.random.default_rng(5)
    R = G.rotation(rng, 40)
    ax = rng.standard_normal((40, 3))
    ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    ang = np.concatenate([rng.uniform(0, np.pi, 20), [0, 1e-9, 1e-6, 1e-3, np.pi, np.pi - 1e-9, np.pi - 1e-6,
                                                     np.pi - 1e-3], rng.uniform(0, np.pi, 12)])
    K = np.zeros((40, 3, 3))
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 2] = -ax[:, 2], ax[:, 1], -ax[:, 0]
    K = K - K.transpose(0, 2, 1)
    D = np.eye(3) + np.sin(ang)[:, None, None] * K + (1 - np.cos(ang))[:, None, None] * K @ K
    gt = np.concatenate([R, rng.standard_normal((40, 3, 1))], 2)
    pred = np.concatenate([R @ D, rng.standard_normal((40, 3, 1))], 2)
    return gt, pred


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_pose_errors_host_matches_scipy(dtype):
    from iggt_official_b200 import ops
    gt, pred = (a.astype(dtype).astype(np.float64) for a in pose_sets())
    t, r = ops.pose_errors_host(gt, pred)
    wt, wr = ref_eval.pose_errors(gt, pred)
    assert np.abs(r - wr).max() <= 1e-10
    assert np.all(np.abs(t - wt) <= 1e-12 * wt)


def test_pose_errors_host_left_handed_is_nan():
    from iggt_official_b200 import ops
    gt = np.concatenate([np.eye(3), np.zeros((3, 1))], 1)[None]
    pred = gt.copy()
    pred[0, 2, 2] = -1
    assert np.isnan(ops.pose_errors_host(gt, pred)[1][0])


def test_closed_form_inverse_se3():
    from iggt_official_b200 import postprocess
    _, ext, _ = G.camera_inputs()
    got = postprocess.closed_form_inverse_se3(ext)
    assert got.dtype == np.float64 and np.array_equal(got, GOLDEN["se3_inv"])
    t = postprocess.closed_form_inverse_se3(torch.from_numpy(ext))
    assert t.dtype == torch.float32                        # torch.bmm's fp32 dot products may round differently
    assert np.allclose(t.numpy(), GOLDEN["se3_inv"], rtol=0, atol=4 * ULP32 * np.abs(ext).max() ** 2 * 3)


def test_argument_errors():
    from iggt_official_b200 import metrics, ops, postprocess
    with pytest.raises(RuntimeError):
        ops.quantile_rule(np.zeros(3, np.float32), 7, 50)
    with pytest.raises(RuntimeError):
        ops.quantile_rule(np.zeros(3, np.float32), ops.QRULE_NUMPY, 101)
    with pytest.raises(ValueError):
        postprocess.threshold_depth_map(np.ones((4, 4), np.float32), max_percentile=101)
    with pytest.raises(ValueError):
        postprocess.closed_form_inverse_se3(np.zeros((2, 3, 3)))
    with pytest.raises(ValueError):
        metrics.PoseEvaluator().evaluate_poses(np.zeros((2, 3, 3)), np.zeros((2, 3, 3)))
    empty = metrics.PoseEvaluator().evaluate_poses(np.zeros((2, 3, 4)), np.zeros((3, 3, 4)))
    assert empty["num_poses"] == 0 and np.isnan(empty["rotation_error_mean"])


def test_import_hygiene():
    # torch itself may load some of these (e.g. tqdm): only what the new modules add counts
    code = ("import sys, numpy, torch; names = ('skimage', 'pandas', 'tqdm', 'scipy', 'cv2'); "
            "before = {m for m in names if m in sys.modules}; "
            "import iggt_official_b200.metrics, iggt_official_b200.postprocess; "
            "bad = [m for m in names if m in sys.modules and m not in before]; assert not bad, bad")
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, check=True)


# ------------------------------------------------------------------------------------------------ GPU

def numpy_row(x, m, rule, q):
    import warnings
    v = x[m]
    with warnings.catch_warnings(), np.errstate(all="ignore"):
        warnings.simplefilter("ignore")
        if v.size == 0:
            return np.float32(np.nan)
        if rule == 1:
            return np.float32(np.percentile(v, q))
        if rule == 2:
            return np.float32(np.nanpercentile(v, q))
        return np.float32(np.median(v))


def same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.array_equal(a.view(np.int32), b.view(np.int32)) or np.array_equal(a, b, equal_nan=True)


@pytest.mark.gpu
def test_select_matches_numpy():
    from iggt_official_b200 import ops
    rng = np.random.default_rng(1)
    rows, n = 12, 3001
    x = rng.standard_normal((rows, n)).astype(np.float32)
    x[3] = rng.integers(0, 5, n)                            # duplicates
    x[4, ::7] = np.nan                                      # NaN row
    x[5] = np.nan                                           # all NaN
    m = rng.random((rows, n)) < 0.6
    m[6] = False                                            # all masked
    m[7] = False
    m[7, 11] = True                                         # one value
    m[8] = False
    m[8, :2] = True                                         # even count 2
    m[9] = True                                             # odd count n
    m[10] = True
    m[10, 0] = False                                        # even count n - 1
    xt, mt = torch.from_numpy(x).cuda(), torch.from_numpy(m).cuda()
    for rule, qs in ((ops.QRULE_MEDIAN, [None]), (ops.QRULE_NUMPY, [1, 50, 99, 37.25]),
                     (ops.QRULE_NUMPY_NAN, [0, 1, 99, 100])):
        for mask in (None, mt):
            got, cnt = ops.select(xt, rule, [] if qs == [None] else qs, mask=mask, return_count=True)
            got = got.cpu().numpy()
            for r in range(rows):
                mm = np.ones(n, bool) if mask is None else m[r]
                want_cnt = mm.sum() - (np.isnan(x[r][mm]).sum() if rule == ops.QRULE_NUMPY_NAN else 0)
                assert cnt[r].item() == want_cnt
                for j, q in enumerate(qs):
                    assert same_bits(got[r, j], numpy_row(x[r], mm, rule, q)), (rule, r, q)


@pytest.mark.gpu
def test_select_past_2_24():
    from iggt_official_b200 import ops
    n = (1 << 24) + 4099
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn((1, n), device="cuda", generator=g)
    m = torch.rand((1, n), device="cuda", generator=g) < 0.999
    xn, mn = x.cpu().numpy()[0], m.cpu().numpy()[0]
    assert same_bits(ops.select(x, ops.QRULE_MEDIAN, mask=m).item(), np.median(xn[mn]))
    got = ops.select(x, ops.QRULE_NUMPY, [1.0, 99.0]).cpu().numpy()[0]
    assert same_bits(got, np.percentile(xn, [np.float32(1.0), np.float32(99.0)]).astype(np.float32))


@pytest.mark.gpu
def test_quantile_unchanged_by_rules():
    from iggt_official_b200 import ops
    y = torch.randn(3, 10007, device="cuda")
    q = (0.0, 0.02, 0.5, 0.98, 1.0)
    assert torch.equal(ops.quantile(y, q), ops.select(y, ops.QRULE_TORCH, q))
    assert torch.equal(ops.quantile(y, q), torch.quantile(y, torch.tensor(q, device="cuda"), dim=1).t())


@pytest.mark.gpu
def test_kernels_match_host_and_oracle():
    from iggt_official_b200 import ops
    gt, pred, gp, pp, _ = case_inputs("resize")
    S, H, W = gt.shape
    p = torch.from_numpy(pred[..., 0]).cuda()
    r = ops.resize_nearest(p, H, W).cpu().numpy()
    assert np.array_equal(r, pred[..., 0][:, ops.zoom_nearest_index(40, H)][:, :, ops.zoom_nearest_index(56, W)])
    g2, r2 = torch.from_numpy(gt).cuda().view(S, -1), torch.from_numpy(r).cuda().view(S, -1)
    for sparse in (False, True):
        mask = ops.depth_valid_mask(g2, r2, sparse)
        want_mask = (gt > 0) & ((r != 0) if sparse else True)
        assert np.array_equal(mask.cpu().numpy().reshape(gt.shape).astype(bool), want_mask)
        for align, clip in (("median", (0.1, 100.0)), ("least_squares", (0.1, 100.0)), (None, (0.1, 100.0)),
                            ("median", None)):
            mode = {"median": ops.ALIGN_MEDIAN, "least_squares": ops.ALIGN_LSQ, None: ops.ALIGN_NONE}[align]
            med = None
            if mode == ops.ALIGN_MEDIAN:
                med = torch.cat([ops.select(g2, ops.QRULE_MEDIAN, mask=mask),
                                 ops.select(r2, ops.QRULE_MEDIAN, mask=mask)], 1).t()
            rec, al = ops.depth_metrics(g2, r2, mask, mode, med, clip, sparse, want_aligned=True)
            rec = rec.cpu().numpy()
            want, want_al = ref_eval.depth_records(gt, r, align, clip, sparse)
            counts = [0, 1, 3, 6, 7, 8, 9, 11]
            assert np.array_equal(rec[:, counts], want[:, counts]), (align, clip, sparse)
            assert np.array_equal(rec[:, 10], want[:, 10])
            assert np.array_equal(al.cpu().numpy().reshape(gt.shape), want_al, equal_nan=True)
            has = rec[:, 0] > 0                             # a frame without valid pixels has no medians
            for f in (2, 4, 5, 12, 13):
                assert np.allclose(rec[has, f], want[has, f], rtol=1e-12, atol=0), (f, rec[:, f], want[:, f])
    t, rr = ops.pose_errors(torch.from_numpy(gp).cuda().double(), torch.from_numpy(pp).cuda().double())
    ht, hr = ops.pose_errors_host(gp, pp)
    assert np.allclose(t.cpu().numpy(), ht, rtol=1e-15, atol=0) and np.allclose(rr.cpu().numpy(), hr, rtol=1e-13,
                                                                                   atol=1e-13)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(G.CASES))
def test_evaluator_matches_reference(name):
    from iggt_official_b200 import metrics
    gt, pred, gp, pp, e = case_inputs(name)
    lsq = e["alignment"] == "least_squares"
    if e.get("sparse"):
        ev = metrics.DepthEvaluator(e["alignment"], e["clip"], sparse_pred=True)
        for i, want in enumerate(golden(name)):
            got = json.loads(json.dumps(G.plain(ev.evaluate_depth(gt[i], pred[i]))))
            check_frame(got, want, gt[0].size)
        return
    ev = metrics.SceneEvaluator(e["alignment"], e["clip"])
    res = ev.evaluate_scene({"gt_depth": gt, "gt_extrinsic": gp}, {"depth": pred, "extrinsic": pp})
    check_results(res, golden(name), gt[0].size, lsq)
    # CUDA tensors in place give the same result as ndarrays, and a second call the same bits
    res_t = ev.evaluate_scene({"gt_depth": torch.from_numpy(gt).cuda(), "gt_extrinsic": torch.from_numpy(gp).cuda()},
                              {"depth": torch.from_numpy(pred).cuda(), "extrinsic": torch.from_numpy(pp).cuda()})
    assert json.dumps(G.plain(res_t)) == json.dumps(G.plain(res))


@pytest.mark.gpu
@pytest.mark.parametrize("S,gt_hw,pred_hw", [(3, (480, 640), (336, 504)), (8, (1168, 1752), (518, 518))])
def test_evaluator_matches_oracle_at_demo_shapes(S, gt_hw, pred_hw):
    from iggt_official_b200 import metrics
    gt, pred, gp, pp = G.scene(seed=40 + S, S=S, gt_hw=gt_hw, pred_hw=pred_hw)
    ev = metrics.SceneEvaluator()
    res = ev.evaluate_scene({"gt_depth": gt, "gt_extrinsic": gp}, {"depth": pred, "extrinsic": pp})
    want = ref_eval.evaluate_scene({"gt_depth": gt, "gt_extrinsic": gp}, {"depth": pred, "extrinsic": pp})
    got_j, want_j = json.loads(json.dumps(G.plain(res))), json.loads(json.dumps(G.plain(want)))
    for fg, fw in zip(got_j["depth_metrics"]["per_frame"], want_j["depth_metrics"]["per_frame"]):
        for key, w in fw.items():                           # the oracle sums the same terms in fp64
            assert close(fg[key], w, 1e-12 if key in ("absrel", "mae", "rmse") else 0), (key, fg[key], w)
    check_pose(got_j["pose_metrics"], want_j["pose_metrics"])
    res2 = ev.evaluate_scene({"gt_depth": gt, "gt_extrinsic": gp}, {"depth": pred, "extrinsic": pp})
    assert json.dumps(G.plain(res2)) == json.dumps(G.plain(res))


@pytest.mark.gpu
def test_threshold_depth_map_matches_reference():
    from iggt_official_b200 import postprocess
    d = G.threshold_inputs()
    for key, args in (("thr_default", {}), ("thr_demo", dict(max_percentile=99, min_percentile=-1)),
                      ("thr_maxdepth", dict(max_percentile=95, min_percentile=5, max_depth=9.5))):
        for i in range(len(d)):                                          # one map, an ndarray, in place
            m = d[i].copy()
            assert postprocess.threshold_depth_map(m, **args) is m
            assert same_bits(m, GOLDEN[key][i]), (key, i)
        t = torch.from_numpy(d).cuda()                                   # the batch, a tensor, in place
        assert postprocess.threshold_depth_map(t, **args) is t
        assert same_bits(t.cpu().numpy(), GOLDEN[key]), key


@pytest.mark.gpu
def test_depth_to_world_coords_points_matches_reference():
    from iggt_official_b200 import postprocess
    depth, ext, K = G.camera_inputs()
    for i in range(2):
        w, c, m = postprocess.depth_to_world_coords_points(depth[i], ext[i], K[i])
        assert np.array_equal(c, GOLDEN["cam_cam"][i]) and np.array_equal(m, GOLDEN["cam_mask"][i])
        ref = GOLDEN["cam_world"][i]
        ulp = np.spacing(np.linalg.norm(ref, axis=-1).astype(np.float32)).astype(np.float64)
        assert np.all(np.abs(w - ref) <= 4 * ulp[..., None])
    w, c, m = postprocess.depth_to_world_coords_points(torch.from_numpy(depth).cuda(), torch.from_numpy(ext).cuda(),
                                                       torch.from_numpy(K).cuda())
    assert np.array_equal(c.cpu().numpy(), GOLDEN["cam_cam"]) and np.array_equal(m.cpu().numpy(), GOLDEN["cam_mask"])
