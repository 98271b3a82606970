"""numpy restatement of the scene evaluation (iggt/metrics.py:257-671) with fp64 sums, and of the ground-truth depth
helpers' arithmetic.  It runs wherever numpy and scipy do (no reference checkout), at any size: the GPU tests compare
against it at shapes where no fixture is stored, and scripts/bench_eval.py times it as the CPU baseline.

The per-pixel terms are the reference's fp32 ones in its operation order; where the reference sums float32 terms
pairwise in float32, this sums the same terms in float64 (np.sum over the terms cast to float64).  The nearest resize is
scipy.ndimage.zoom(order=0, grid_mode=True)'s index map, which skimage.transform.resize(order=0) calls.  Records use
the layout of iggt_depth_metrics (include/iggt_b200.h), so the per-frame dicts come from the same host code."""
import numpy as np
from scipy.spatial.transform import Rotation


def zoom_index(n_in, n_out):
    k = np.arange(n_out, dtype=np.float64)
    s = np.floor(((k + 0.5) * (n_in / n_out) - 0.5) + 0.5).astype(np.int64)
    return np.clip(s, 0, n_in - 1)


def resize_nearest(pred, H, W):
    """pred [S,h,w] float32 -> [S,H,W]."""
    return pred[:, zoom_index(pred.shape[1], H)][:, :, zoom_index(pred.shape[2], W)]


def frame_record(gt, pred, alignment="median", clip=(0.1, 100.0), sparse=False):
    """One frame (gt, pred float32 [H,W] at the GT resolution) -> (record [16] float64, aligned prediction)."""
    r = np.zeros(16)
    pm = pred != 0 if sparse else np.ones(pred.shape, bool)
    valid = (gt > 0) & pm
    r[0] = valid.sum()
    p = pred
    if alignment == "median" and valid.any():
        g_med, p_med = np.median(gt[valid]), np.median(pred[valid])
        r[12], r[13] = g_med, p_med
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = g_med / p_med
        if np.isfinite(ratio):
            p, r[10], r[11] = pred * ratio, ratio, 1
    elif alignment == "least_squares" and valid.any():
        gv, pv = gt[valid], pred[valid]
        r[12], r[13] = np.sum((gv * pv).astype(np.float64)), np.sum((pv * pv).astype(np.float64))
        with np.errstate(divide="ignore", invalid="ignore"):
            scale = np.float32(r[12] / r[13])
        if np.isfinite(scale) and scale > 0:
            p, r[10], r[11] = pred * scale, scale, 1
    if r[11] == 0:
        r[10] = 1.0
    if clip is not None:
        p = np.clip(p, clip[0], clip[1]) * pm
    ev = valid & (p != 0) if sparse else valid
    r[1] = ev.sum()
    g, q = gt[ev], p[ev]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        rel = np.nan_to_num(np.abs(q - g) / g, nan=0, posinf=0, neginf=0)
        r1 = np.nan_to_num(g / q, nan=2.03, posinf=2.03, neginf=2.03)
        r2 = np.nan_to_num(q / g, nan=0, posinf=0, neginf=0)
        mx = np.maximum(r1, r2)
        d = g - q
        ratio = np.maximum(g / q, q / g)
    r[2] = np.sum(rel.astype(np.float64))
    r[3] = np.count_nonzero((0 < mx) & (mx < 1.03))
    r[4] = np.sum(np.abs(d).astype(np.float64))
    r[5] = np.sum((d * d).astype(np.float64))
    ratio = ratio[np.isfinite(ratio)]
    r[6] = ratio.size
    for k, t in enumerate((1.25, 1.25 ** 2, 1.25 ** 3)):
        r[7 + k] = np.count_nonzero(ratio < t)
    return r, p


def depth_records(gt, pred, alignment="median", clip=(0.1, 100.0), sparse=False):
    """gt [S,H,W], pred [S,h,w] (or [...,1]) float32 -> (records [S,16], aligned [S,H,W])."""
    gt = np.asarray(gt, np.float32)
    pred = np.asarray(pred, np.float32)
    gt = gt[..., 0] if gt.ndim == 4 else gt
    pred = pred[..., 0] if pred.ndim == 4 else pred
    pred = pred[:gt.shape[0]]
    if pred.shape[1:] != gt.shape[1:]:
        pred = resize_nearest(pred, gt.shape[1], gt.shape[2])
    out = [frame_record(gt[i], pred[i], alignment, clip, sparse) for i in range(gt.shape[0])]
    return np.stack([o[0] for o in out]), np.stack([o[1] for o in out])


def evaluate_scene(gt_data, predictions, alignment="median", clip=(0.1, 100.0)):
    """The SceneEvaluator result dict, with the per-frame values formed from fp64 records."""
    from iggt_official_b200 import metrics
    ev = metrics.SceneEvaluator(alignment, clip)
    results = {"depth_metrics": {}, "pose_metrics": {}, "summary": {}}
    if "gt_depth" in gt_data and "depth" in predictions:
        rec, _ = depth_records(gt_data["gt_depth"], predictions["depth"], alignment, clip)
        total = int(np.prod(np.shape(gt_data["gt_depth"])[1:3]))
        frames = [dict(metrics._frame_metrics(rec[i], total, alignment), frame_id=i) for i in range(len(rec))]
        results["depth_metrics"] = ev._aggregate_depth_metrics(frames)
        results["depth_metrics"]["per_frame"] = frames
    if "gt_extrinsic" in gt_data and "extrinsic" in predictions:
        t, r = pose_errors(gt_data["gt_extrinsic"], predictions["extrinsic"])
        results["pose_metrics"] = {
            "translation_error_mean": np.mean(t), "translation_error_median": np.median(t),
            "translation_error_std": np.std(t), "translation_error_max": np.max(t), "translation_error_min": np.min(t),
            "rotation_error_mean": np.mean(r), "rotation_error_median": np.median(r),
            "rotation_error_std": np.std(r), "rotation_error_max": np.max(r), "rotation_error_min": np.min(r),
            "num_poses": len(t), "translation_errors": t, "rotation_errors": r}
    results["summary"] = ev._create_summary(results)
    return results


def pose_errors(gt, pred):
    """[N,3,4] or [N,4,4] -> (translation errors, rotation errors in degrees), float64, with scipy's Rotation."""
    gt = np.asarray(gt, np.float64)[:, :3, :4]
    pred = np.asarray(pred, np.float64)[:, :3, :4]
    t = np.linalg.norm(gt[:, :, 3] - pred[:, :, 3], axis=1)
    r = np.array([np.degrees(Rotation.from_matrix(g[:, :3].T @ p[:, :3]).magnitude()) for g, p in zip(gt, pred)])
    return t, r


def threshold_depth_map(depth, max_percentile=99, min_percentile=1, max_depth=-1):
    """One float32 map, in place, as the reference."""
    if max_depth > 0:
        depth[depth > max_depth] = 0.0
    hi = np.nanpercentile(depth, max_percentile) if max_percentile > 0 else None
    lo = np.nanpercentile(depth, min_percentile) if min_percentile > 0 else None
    if hi is not None and hi > 0:
        depth[depth > hi] = 0.0
    if lo is not None and lo > 0:
        depth[depth < lo] = 0.0
    return depth
