"""Scene evaluation on the GPU: DepthEvaluator, PoseEvaluator and SceneEvaluator with the reference's names, arguments
and result structure (iggt/metrics.py:257-727, which demo.py:99 and :145-163 run whenever a scene has ground truth).

The reference evaluates frame by frame in numpy on the host.  Here a scene's depth maps are evaluated in one batch of
launches (csrc/evaluate.cu, the selection in csrc/pca.cu): nearest resize of the predictions to the GT resolution,
the validity mask, the masked medians (np.median's rule), the aligned / clipped prediction and every per-pixel term in
the reference's fp32 operation order, with fp64 sums reduced in a fixed order.  One device-to-host copy brings back the
per-frame records; the per-frame values and the aggregation over the N frames are formed on the host in numpy, with
the reference's dtypes.  Pose errors are one launch in fp64 with scipy's rotation magnitude.

Inputs are the reference's ndarrays or CUDA tensors (used in place) in its shapes: depth (N,H,W) or (N,H,W,1), poses
(N,3,4) or (N,4,4).  Depth is evaluated in float32.  Two differences remain: the sums are fp64 where the reference
sums float32 terms pairwise in float32, and the resize follows scipy.ndimage.zoom(order=0, grid_mode=True), which is
what skimage.transform.resize(order=0) calls.  4x4 poses are widened to fp64 like 3x4 ones (the reference keeps a
float32 4x4 in float32).  No import of skimage, pandas, tqdm, scipy or cv2.

Instance masks (iggt/metrics.py:16-80): calculate_iou and evaluate_matched_instances with the reference's results and
result types.  The device does all the pixel-sized work in one launch (csrc/instances.cu: exact intersection counts and
mask sizes on the 8-bit tensor cores); the K x P rest (IoU, 1 - IoU, the assignment, the threshold and the means) is
formed on the host in numpy with the reference's dtypes, the assignment by scipy's algorithm restated in the library."""
import json
import logging
from typing import Any, Dict, Optional, Tuple

import numpy as np
import torch

from . import ops

logger = logging.getLogger(__name__)

_ALIGN = {"median": ops.ALIGN_MEDIAN, "least_squares": ops.ALIGN_LSQ}
_AGG_KEYS = ("absrel", "inliers103", "pred_depth_density", "mae", "rmse", "delta_1", "delta_2", "delta_3",
             "valid_ratio")


def _device_of(*xs):
    for x in xs:
        if isinstance(x, torch.Tensor) and x.is_cuda:
            return x.device
    if not torch.cuda.is_available():
        raise RuntimeError("scene evaluation runs on a CUDA device (there is no CPU fallback on this path)")
    return torch.device("cuda", torch.cuda.current_device())


def _depth_batch(x, device, name):
    """(N,H,W) or (N,H,W,1) ndarray / tensor -> contiguous fp32 CUDA tensor [N,H,W] (a CUDA fp32 input is used in place)."""
    t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
    if t.dim() == 4 and t.shape[-1] == 1:
        t = t[..., 0]
    if t.dim() != 3:
        raise ValueError(f"{name}: expected (N,H,W) or (N,H,W,1) depth maps, got {tuple(x.shape)}")
    return t.to(device=device, dtype=torch.float32).contiguous()


def _empty_depth_metrics():
    return {"absrel": np.nan, "inliers103": np.nan, "pred_depth_density": 0.0, "mae": np.nan, "rmse": np.nan,
            "delta_1": np.nan, "delta_2": np.nan, "delta_3": np.nan, "scaling_factor": np.nan, "valid_pixels": 0,
            "total_pixels": 0, "valid_ratio": 0.0}


def _frame_metrics(r, total, alignment):
    """One frame's result dict from its fp64 record, in the reference's dtypes: fp32 means of fp32 terms, fp64
    percentages of boolean means and of the density."""
    valid = int(r[0])
    if valid == 0:
        logger.warning("No valid pixels for depth evaluation")
        return _empty_depth_metrics()
    if alignment is None or alignment not in _ALIGN:
        scale = 1.0
    elif r[11] == 0.0:
        logger.warning("%s alignment failed, using original prediction",
                       "Median" if alignment == "median" else "Least squares")
        scale = 1.0
    else:
        scale = np.float32(r[10])
    n_eval = int(r[1])
    hundred = np.float32(100.0)
    nan = np.nan
    m = {"absrel": nan, "inliers103": nan, "pred_depth_density": np.float64(n_eval) / total * 100,
         "mae": nan, "rmse": nan, "delta_1": nan, "delta_2": nan, "delta_3": nan}
    if n_eval > 0:
        m["absrel"] = np.float32(r[2] / n_eval) * hundred
        m["inliers103"] = (np.float32(r[3]) / np.float32(n_eval)) * hundred
        m["mae"] = np.float32(r[4] / n_eval)
        m["rmse"] = np.sqrt(np.float32(r[5] / n_eval))
        finite = r[6]
        if finite > 0:
            for k in range(3):
                m[f"delta_{k + 1}"] = np.float64(r[7 + k]) / finite * 100
    m["scaling_factor"] = scale
    m["valid_pixels"] = np.int64(valid)
    m["total_pixels"] = total
    m["valid_ratio"] = np.int64(valid) / total
    return m


def _is_cuda(x):
    return isinstance(x, torch.Tensor) and x.is_cuda


def _is_bool(m):
    return m.dtype == torch.bool if isinstance(m, torch.Tensor) else m.dtype == np.bool_


def _mask_rows(masks, name):
    """masks: a stacked [K, ...] bool ndarray / tensor or a sequence of bool masks -> (list of per-mask arrays or the
    stack itself, K, mask shape).  Non-bool dtypes raise TypeError, masks of different shapes ValueError."""
    if isinstance(masks, (np.ndarray, torch.Tensor)):
        if not _is_bool(masks):
            raise TypeError(f"{name}: expected boolean masks, got {masks.dtype}")
        if masks.ndim < 1:
            raise ValueError(f"{name}: expected a stack [K, ...] of masks, got a scalar")
        return masks, masks.shape[0], tuple(masks.shape[1:])
    rows = [m if isinstance(m, (np.ndarray, torch.Tensor)) else np.asarray(m) for m in masks]
    shape = None
    for m in rows:
        if not _is_bool(m):
            raise TypeError(f"{name}: expected boolean masks, got {m.dtype}")
        if shape is None:
            shape = tuple(m.shape)
        elif tuple(m.shape) != shape:
            raise ValueError(f"{name}: masks of different shapes {shape} and {tuple(m.shape)}")
    return rows, len(rows), shape


def _mask_stack(masks, K, n, device):
    """-> uint8 CUDA [K, ld] 0/1 stack for iggt_mask_overlaps.  A contiguous CUDA bool stack whose rows are a multiple
    of 16 bytes is used in place; anything else is copied once into a zero-padded [K, round_up(n, 16)] buffer."""
    if isinstance(masks, torch.Tensor) and masks.is_cuda and masks.device == device and masks.is_contiguous() \
            and n % 16 == 0 and masks.data_ptr() % 16 == 0:
        return masks.view(K, n).view(torch.uint8)
    ld = (n + 15) // 16 * 16
    if isinstance(masks, torch.Tensor):
        buf = torch.zeros((K, ld), dtype=torch.uint8, device=device)
        buf[:, :n].copy_(masks.reshape(K, n).to(device=device))
        return buf
    if isinstance(masks, np.ndarray) or not any(_is_cuda(m) for m in masks):
        host = np.zeros((K, ld), dtype=np.uint8)
        if isinstance(masks, np.ndarray):
            host[:, :n] = masks.reshape(K, n)
        else:
            for i, m in enumerate(masks):
                host[i, :n] = m.reshape(-1).numpy() if isinstance(m, torch.Tensor) else np.asarray(m).reshape(-1)
        return torch.from_numpy(host).to(device)
    buf = torch.zeros((K, ld), dtype=torch.uint8, device=device)
    for i, m in enumerate(masks):
        src = m.reshape(-1) if isinstance(m, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(m).reshape(-1))
        buf[i, :n].copy_(src.to(device=device))
    return buf


def _mask_counts(gt_masks, pred_masks):
    """(inter [K,P], gsize [K], psize [P]) int64 ndarrays of two non-empty mask sets, from one device launch and one
    copy to the host."""
    g, K, gshape = _mask_rows(gt_masks, "gt_masks")
    p, P, pshape = _mask_rows(pred_masks, "pred_masks")
    if gshape != pshape:
        raise ValueError(f"gt masks {gshape} and predicted masks {pshape} differ in shape")
    n = int(np.prod(gshape, dtype=np.int64))
    def tensors(m):
        return [m] if isinstance(m, torch.Tensor) else [] if isinstance(m, np.ndarray) else m
    device = _device_of(*tensors(g), *tensors(p))
    if n == 0:
        z = np.zeros
        return z((K, P), np.int64), z(K, np.int64), z(P, np.int64)
    counts = ops.mask_overlaps(_mask_stack(g, K, n, device), _mask_stack(p, P, n, device), n).cpu().numpy()
    return counts[:K * P].reshape(K, P), counts[K * P:K * P + K], counts[K * P + K:]


def _matched_from_counts(inter, gsize, psize, iou_threshold=0.5):
    """evaluate_matched_instances' results from the exact counts (inter [K,P], gsize [K], psize [P] int64, K, P > 0),
    with the reference's dtypes: an fp64 IoU matrix of int64 / int64 quotients (0.0 where the union is empty), the
    assignment of 1 - IoU, then the threshold and the numpy means of the matched pairs."""
    inter = np.asarray(inter, np.int64)
    gsize, psize = np.asarray(gsize, np.int64), np.asarray(psize, np.int64)
    union = gsize[:, None] + psize[None, :] - inter
    iou_matrix = np.zeros(inter.shape)
    pos = union > 0
    iou_matrix[pos] = inter[pos] / union[pos]
    gt_indices, pred_indices = ops.linear_sum_assignment(1 - iou_matrix)
    matches, matched_ious, matched_accs = [], [], []
    for gt_idx, pred_idx in zip(gt_indices, pred_indices):
        if iou_matrix[gt_idx, pred_idx] >= iou_threshold:
            matches.append((gt_idx, pred_idx))
            matched_ious.append(iou_matrix[gt_idx, pred_idx])
            tp_pixels, gt_pixels = inter[gt_idx, pred_idx], gsize[gt_idx]
            matched_accs.append(tp_pixels / gt_pixels if gt_pixels > 0 else 0)
    if not matches:
        return {"matched_miou": 0, "matched_macc": 0, "num_matches": 0}, []
    return {"matched_miou": np.mean(matched_ious), "matched_macc": np.mean(matched_accs),
            "num_matches": len(matches)}, matches


def calculate_iou(mask1, mask2):
    """IoU of two boolean masks of one shape (ndarrays or tensors): np.float64, or 0.0 when both are empty."""
    mask1, mask2 = (m if isinstance(m, (np.ndarray, torch.Tensor)) else np.asarray(m) for m in (mask1, mask2))
    inter, gsize, psize = _mask_counts(mask1[None], mask2[None])
    intersection = inter[0, 0]
    union = gsize[0] + psize[0] - intersection
    return intersection / union if union > 0 else 0.0


def evaluate_matched_instances(gt_masks, pred_masks, iou_threshold=0.5):
    """Optimal one-to-one matching of gt and predicted instance masks by IoU (scipy's linear_sum_assignment on
    1 - IoU), then the mean IoU and mean pixel accuracy (|g & p| / |g|) of the pairs with IoU >= iou_threshold.
    Masks: a stacked [K, ...] bool ndarray / tensor or a sequence of bool masks, all of one shape.
    Returns ({"matched_miou", "matched_macc", "num_matches"}, [(gt_index, pred_index), ...])."""
    if len(gt_masks) == 0 or len(pred_masks) == 0:
        return {"matched_miou": 0, "matched_macc": 0, "num_matches": 0}, []
    return _matched_from_counts(*_mask_counts(gt_masks, pred_masks), iou_threshold)


class DepthEvaluator:
    """Depth metrics of predictions against ground truth (median / least-squares / no scale alignment)."""

    def __init__(self, alignment: str = "median", clip_pred_depth: Optional[Tuple[float, float]] = (0.1, 100.0),
                 sparse_pred: bool = False):
        self.alignment = alignment
        self.clip_pred_depth = clip_pred_depth
        self.sparse_pred = sparse_pred

    def evaluate_frames(self, gt_depths, pred_depths, return_aligned=False):
        """All frames of gt (N,H,W[,1]) against the first N of pred (M,h,w[,1]) in one batch: a list of per-frame
        result dicts (and the aligned, clipped predictions [N,H,W] on the device with return_aligned)."""
        device = _device_of(gt_depths, pred_depths)
        gt = _depth_batch(gt_depths, device, "gt_depth")
        pred = _depth_batch(pred_depths, device, "depth")
        S, H, W = gt.shape
        if pred.shape[0] < S:
            raise ValueError(f"{S} ground-truth frames but {pred.shape[0]} predicted ones")
        pred = pred[:S]
        if pred.shape[1:] != gt.shape[1:]:
            pred = ops.resize_nearest(pred, H, W)
        gt2, pred2 = gt.view(S, H * W), pred.reshape(S, H * W)
        mask = ops.depth_valid_mask(gt2, pred2, self.sparse_pred)
        mode = _ALIGN.get(self.alignment, ops.ALIGN_NONE) if self.alignment is not None else ops.ALIGN_NONE
        medians = None
        if mode == ops.ALIGN_MEDIAN:
            medians = torch.cat([ops.select(gt2, ops.QRULE_MEDIAN, mask=mask),
                                 ops.select(pred2, ops.QRULE_MEDIAN, mask=mask)], dim=1).t()
        rec, aligned = ops.depth_metrics(gt2, pred2, mask, mode, medians, self.clip_pred_depth, self.sparse_pred,
                                         want_aligned=return_aligned)
        records = rec.cpu().numpy()
        frames = [_frame_metrics(records[i], H * W, self.alignment) for i in range(S)]
        return (frames, aligned.view(S, H, W)) if return_aligned else frames

    def evaluate_depth(self, gt_depth, pred_depth) -> Dict[str, float]:
        """One frame: gt (H,W) or (H,W,1) against pred (h,w) or (h,w,1)."""
        return self.evaluate_frames(gt_depth[None], pred_depth[None])[0]

    def _get_empty_depth_metrics(self) -> Dict[str, float]:
        return _empty_depth_metrics()


class PoseEvaluator:
    """Camera pose errors: translation distance and relative rotation angle (degrees) per frame."""

    def evaluate_poses(self, gt_poses, pred_poses) -> Dict[str, Any]:
        if tuple(gt_poses.shape) != tuple(pred_poses.shape):
            logger.error(f"Pose shape mismatch: GT {tuple(gt_poses.shape)}, Pred {tuple(pred_poses.shape)}")
            return self._get_empty_pose_metrics()
        for poses in (gt_poses, pred_poses):
            if tuple(poses.shape[-2:]) not in ((4, 4), (3, 4)):
                raise ValueError(f"Unsupported pose shape: {tuple(poses.shape)}")
        device = _device_of(gt_poses, pred_poses)
        g, p = self._rows34(gt_poses, device), self._rows34(pred_poses, device)
        t, r = ops.pose_errors(g, p)
        errs = torch.stack([t, r]).cpu().numpy()
        t_err, r_err = errs[0].copy(), errs[1].copy()
        if np.isnan(r_err).any():
            logger.warning("Failed to compute rotation error: non-positive determinant")
        return {
            "translation_error_mean": np.mean(t_err), "translation_error_median": np.median(t_err),
            "translation_error_std": np.std(t_err), "translation_error_max": np.max(t_err),
            "translation_error_min": np.min(t_err),
            "rotation_error_mean": np.mean(r_err), "rotation_error_median": np.median(r_err),
            "rotation_error_std": np.std(r_err), "rotation_error_max": np.max(r_err),
            "rotation_error_min": np.min(r_err),
            "num_poses": len(t_err), "translation_errors": t_err, "rotation_errors": r_err,
        }

    @staticmethod
    def _rows34(poses, device):
        t = poses if isinstance(poses, torch.Tensor) else torch.from_numpy(np.asarray(poses))
        return t[:, :3, :4].to(device=device, dtype=torch.float64).contiguous()

    def _get_empty_pose_metrics(self) -> Dict[str, Any]:
        m = {f"{kind}_error_{stat}": np.nan for kind in ("translation", "rotation")
             for stat in ("mean", "median", "std", "max", "min")}
        m.update(num_poses=0, translation_errors=np.array([]), rotation_errors=np.array([]))
        return m


class SceneEvaluator:
    """Depth and pose evaluation of one scene, with the reference's report and summary."""

    def __init__(self, depth_alignment: str = "median",
                 depth_clip_range: Optional[Tuple[float, float]] = (0.1, 100.0)):
        self.depth_evaluator = DepthEvaluator(alignment=depth_alignment, clip_pred_depth=depth_clip_range)
        self.pose_evaluator = PoseEvaluator()

    def evaluate_scene(self, gt_data: Dict[str, Any], predictions: Dict[str, Any]) -> Dict[str, Any]:
        results = {"depth_metrics": {}, "pose_metrics": {}, "summary": {}}
        if "gt_depth" in gt_data and "depth" in predictions:
            logger.info("Evaluating depth predictions...")
            frames = self.depth_evaluator.evaluate_frames(gt_data["gt_depth"], predictions["depth"])
            for i, f in enumerate(frames):
                f["frame_id"] = i
            results["depth_metrics"] = self._aggregate_depth_metrics(frames)
            results["depth_metrics"]["per_frame"] = frames
        if "gt_extrinsic" in gt_data and "extrinsic" in predictions:
            logger.info("Evaluating pose predictions...")
            results["pose_metrics"] = self.pose_evaluator.evaluate_poses(gt_data["gt_extrinsic"],
                                                                         predictions["extrinsic"])
        results["summary"] = self._create_summary(results)
        return results

    @staticmethod
    def _aggregate_depth_metrics(frames: list) -> Dict[str, float]:
        """mean / median / std / min / max over the frames whose value is finite (N numbers, on the host)."""
        if not frames:
            return {}
        agg = {}
        for key in _AGG_KEYS:
            vals = [f[key] for f in frames if key in f and np.isfinite(f[key])]
            if vals:
                for stat, fn in (("mean", np.mean), ("median", np.median), ("std", np.std), ("min", np.min),
                                 ("max", np.max)):
                    agg[f"{key}_{stat}"] = fn(vals)
        valid = sum(f["valid_pixels"] for f in frames)
        total = sum(f["total_pixels"] for f in frames)
        agg["total_valid_pixels"] = valid
        agg["total_pixels"] = total
        agg["overall_valid_ratio"] = valid / total if total > 0 else 0
        return agg

    @staticmethod
    def _create_summary(results: Dict[str, Any]) -> Dict[str, Any]:
        summary = {}
        d = results.get("depth_metrics")
        if d:
            summary["depth"] = {k: d.get(f"{k}_mean", np.nan)
                                for k in ("absrel", "inliers103", "pred_depth_density", "mae", "rmse", "delta_1")}
            summary["depth"]["valid_ratio"] = d.get("overall_valid_ratio", 0)
        p = results.get("pose_metrics")
        if p:
            summary["pose"] = {"translation_error": p.get("translation_error_mean", np.nan),
                               "rotation_error": p.get("rotation_error_mean", np.nan),
                               "num_poses": p.get("num_poses", 0)}
        return summary

    def save_evaluation_report(self, results: Dict[str, Any], save_path: str):
        """The results as JSON (arrays as lists, numpy scalars as Python numbers)."""
        def plain(o):
            if isinstance(o, np.ndarray):
                return o.tolist()
            if isinstance(o, np.floating):
                return float(o)
            if isinstance(o, np.integer):
                return int(o)
            if isinstance(o, dict):
                return {k: plain(v) for k, v in o.items()}
            if isinstance(o, list):
                return [plain(v) for v in o]
            return o

        with open(save_path, "w") as f:
            json.dump(plain(results), f, indent=2)
        logger.info(f"Evaluation report saved to {save_path}")

    def print_summary(self, results: Dict[str, Any]):
        bar = "=" * 60
        print("\n" + bar)
        print("SCENE EVALUATION SUMMARY")
        print(bar)
        summary = results.get("summary", {})
        if "depth" in summary:
            d = summary["depth"]
            print("\nDEPTH METRICS:")
            print(f"  AbsRel:     {d['absrel']:.4f}%")
            print(f"  Inliers103: {d['inliers103']:.4f}%")
            print(f"  Pred Density: {d['pred_depth_density']:.4f}%")
            print(f"  MAE:        {d['mae']:.4f}")
            print(f"  RMSE:       {d['rmse']:.4f}")
            print(f"  δ < 1.25:   {d['delta_1']:.4f}%")
            print(f"  Valid ratio: {d['valid_ratio']:.4f}")
        if "pose" in summary:
            p = summary["pose"]
            print("\nPOSE METRICS:")
            print(f"  Translation error: {p['translation_error']:.4f} m")
            print(f"  Rotation error:    {p['rotation_error']:.4f} deg")
            print(f"  Number of poses:   {p['num_poses']}")
        print("\n" + bar)
