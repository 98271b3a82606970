"""numpy + scipy statement of iggt/metrics.py:16-80 (calculate_iou, evaluate_matched_instances) from integer counts.

The counts are a float64 matrix product of the 0/1 masks (exact: every partial sum is an integer below 2^53), taken in
pixel chunks so large stacks fit in memory; the rest is the reference's arithmetic with its dtypes and scipy's
linear_sum_assignment.  Pinned to the unmodified reference by tests/golden/instances_ref.npz; the GPU tests compare
the port against it at shapes the fixture does not hold."""
import numpy as np
from scipy.optimize import linear_sum_assignment

CHUNK = 1 << 20


def stack(masks):
    """A sequence of bool masks of one shape, or a stacked [K, ...] bool array -> [K, n] bool."""
    a = masks if isinstance(masks, np.ndarray) else np.stack([np.asarray(m) for m in masks])
    return a.reshape(a.shape[0], -1)


def counts(gt_masks, pred_masks):
    """(inter [K,P], gsize [K], psize [P]) int64."""
    g, p = stack(gt_masks), stack(pred_masks)
    inter = np.zeros((g.shape[0], p.shape[0]), np.int64)
    for c0 in range(0, g.shape[1], CHUNK):
        gc, pc = g[:, c0:c0 + CHUNK].astype(np.float64), p[:, c0:c0 + CHUNK].astype(np.float64)
        inter += (gc @ pc.T).astype(np.int64)
    return inter, g.sum(1, dtype=np.int64), p.sum(1, dtype=np.int64)


def matched_from_counts(inter, gsize, psize, iou_threshold=0.5):
    K, P = inter.shape
    iou_matrix = np.zeros((K, P))
    for i in range(K):
        for j in range(P):
            union = gsize[i] + psize[j] - inter[i, j]
            iou_matrix[i, j] = inter[i, j] / union if union > 0 else 0.0
    gt_indices, pred_indices = linear_sum_assignment(1 - iou_matrix)
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


def evaluate_matched_instances(gt_masks, pred_masks, iou_threshold=0.5):
    if len(gt_masks) == 0 or len(pred_masks) == 0:
        return {"matched_miou": 0, "matched_macc": 0, "num_matches": 0}, []
    return matched_from_counts(*counts(gt_masks, pred_masks), iou_threshold)


def calculate_iou(mask1, mask2):
    inter, g, p = counts(np.asarray(mask1)[None], np.asarray(mask2)[None])
    union = g[0] + p[0] - inter[0, 0]
    return inter[0, 0] / union if union > 0 else 0.0
