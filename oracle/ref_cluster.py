"""CPU restatement of the reference's multi-view clustering (iggt/utils/misc.py:81-170, called from demo.py:389-397).

The reference imports cuML's HDBSCAN or the scikit-learn-contrib `hdbscan` package; neither is installable here, so
the oracle runs scikit-learn's HDBSCAN with the contrib package's semantics.  The one difference between the two is
documented in the scikit-learn HDBSCAN class notes: scikit-learn's `min_samples` counts the point itself, the contrib
package's does not, so the contrib call `HDBSCAN(min_samples=m)` is `sklearn.cluster.HDBSCAN(min_samples=m + 1)`.

matplotlib is not installed either: `jet_lut()` restates its 256-entry `jet` table from matplotlib's public segment
data.  It has not been checked against a matplotlib install."""
import numpy as np

# matplotlib's `jet` segment data: per channel, (x, y0, y1) rows (y0 = value left of x, y1 = value right of x)
JET_SEGMENTS = {
    "red": ((0.0, 0.0, 0.0), (0.35, 0.0, 0.0), (0.66, 1.0, 1.0), (0.89, 1.0, 1.0), (1.0, 0.5, 0.5)),
    "green": ((0.0, 0.0, 0.0), (0.125, 0.0, 0.0), (0.375, 1.0, 1.0), (0.64, 1.0, 1.0), (0.91, 0.0, 0.0),
              (1.0, 0.0, 0.0)),
    "blue": ((0.0, 0.5, 0.5), (0.11, 1.0, 1.0), (0.34, 1.0, 1.0), (0.65, 0.0, 0.0), (1.0, 0.0, 0.0)),
}


def _channel_lut(seg, n):
    """matplotlib's piecewise-linear lookup table of one channel, sampled at n evenly spaced points of [0, 1]."""
    a = np.asarray(seg, np.float64)
    x, y0, y1 = a[:, 0] * (n - 1), a[:, 1], a[:, 2]
    xs = (n - 1) * np.linspace(0.0, 1.0, n)
    ind = np.searchsorted(x, xs)[1:-1]
    frac = (xs[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
    return np.clip(np.concatenate([[y1[0]], frac * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]]), 0.0, 1.0)


def jet_lut(n=256):
    """[n, 3] float64 RGB table of `jet`."""
    return np.stack([_channel_lut(JET_SEGMENTS[c], n) for c in ("red", "green", "blue")], 1)


def jet(x):
    """RGB of matplotlib's `jet(x)` for a scalar x in [0, 1]: the table entry min(int(x * 256), 255)."""
    return jet_lut()[min(int(x * 256), 255)]


def hdbscan_labels(points, eps, min_samples, min_cluster_size):
    """Raw HDBSCAN labels (-1 = noise) of points [n, C] with the contrib package's min_samples."""
    from sklearn.cluster import HDBSCAN
    return HDBSCAN(min_samples=min_samples + 1, min_cluster_size=min_cluster_size, cluster_selection_epsilon=eps,
                   allow_single_cluster=False, copy=True).fit(np.asarray(points, np.float64)).labels_.astype(np.int64)


def fill_noise(points, labels):
    """The reference's noise fill: every noise pixel takes the label of its nearest labelled pixel; all noise -> 0."""
    from sklearn.neighbors import NearestNeighbors
    labels = labels.copy()
    noise = labels == -1
    if noise.all():
        return np.zeros_like(labels)
    if noise.any():
        nbrs = NearestNeighbors(n_neighbors=1, algorithm="auto").fit(points[~noise])
        _, idx = nbrs.kneighbors(points[noise])
        labels[noise] = labels[~noise][idx[:, 0]]
    return labels


def colorize(masks):
    """The reference's colouring loop: sorted label j -> jet(j / (n - 1)) (jet(0.5) for one label), noise black."""
    n, h, w = masks.shape
    uniq = np.unique(masks)
    uniq = uniq[uniq != -1]
    k = len(uniq)
    color_map = {lab: list(jet(j / (k - 1)) if k > 1 else jet(0.5)) for j, lab in enumerate(uniq)}
    color_map[-1] = [0, 0, 0]
    out = np.zeros((n, h, w, 3), np.uint8)
    for i in range(n):
        px = np.array([color_map[lab] for lab in masks[i].reshape(-1)])
        out[i] = (px * 255).astype(np.uint8).reshape(h, w, 3)
    return out


def cluster_features_to_masks_mv(feature_map, apply_colormap=False, **kwargs):
    """feature_map [N, H, W, C] -> masks [N, H, W] int64 (and colours [N, H, W, 3] uint8)."""
    feature_map = np.asarray(feature_map)
    if feature_map.ndim != 4:
        raise ValueError("feature_map must be [N, H, W, C]")
    n, h, w, c = feature_map.shape
    pts = feature_map.reshape(-1, c)
    raw = hdbscan_labels(pts, kwargs.get("eps"), kwargs.get("min_samples"), kwargs.get("min_cluster_size"))
    masks = fill_noise(pts, raw).reshape(n, h, w)
    return (masks, colorize(masks)) if apply_colormap else masks
