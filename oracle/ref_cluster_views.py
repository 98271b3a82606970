"""CPU restatement of the reference's per-view clustering (iggt/utils/misc.py:174-269, cluster_features_to_masks).

Whatever `method` says, the reference runs HDBSCAN on each view on its own, fills that view's noise from its nearest
labelled pixel and colours it by its own labels.  This is a loop over oracle/ref_cluster.py's hdbscan_labels,
fill_noise and colorize (same contrib semantics, same `jet` table)."""
import numpy as np

from oracle.ref_cluster import colorize, fill_noise, hdbscan_labels


def cluster_features_to_masks(feature_map, method="kmeans", apply_colormap=False, **kwargs):
    """feature_map [N, H, W, C] -> masks [N, H, W] int32 (and colours [N, H, W, 3] uint8)."""
    feature_map = np.asarray(feature_map)
    if feature_map.ndim != 4:
        raise ValueError("feature_map must be [N, H, W, C]")
    n, h, w, c = feature_map.shape
    masks = np.zeros((n, h, w), np.int32)
    colours = np.zeros((n, h, w, 3), np.uint8)
    for i in range(n):
        pts = feature_map[i].reshape(-1, c)
        raw = hdbscan_labels(pts, kwargs.get("eps"), kwargs.get("min_samples"), kwargs.get("min_cluster_size"))
        masks[i] = fill_noise(pts, raw).reshape(h, w)
        colours[i] = colorize(masks[i:i + 1])[0]
    return (masks, colours) if apply_colormap else masks
