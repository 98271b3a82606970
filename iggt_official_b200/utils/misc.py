"""Device-side instance clustering (SURVEY.md section 8f, row 2): the last step of the demo (demo.py:365-401).

`knn_avg_features_pyg` keeps the name and arguments of the reference helper (iggt/utils/misc.py:24-78), which builds
a k-NN graph over the un-projected points of ALL views with torch_geometric and averages the neighbours' features with
torch_scatter on the CPU; here it is one exact block-pruned search on the GPU (csrc/knn.cu).

`cluster_features_to_masks_mv` keeps the name, arguments and return values of the reference helper
(iggt/utils/misc.py:81-170), which runs cuML's or the contrib `hdbscan` package's HDBSCAN over all pixels on the host.
Here the core distances, the minimum spanning tree of the mutual-reachability graph and the noise fill run on the GPU
(csrc/cluster.cu); only the tree condensation and cluster selection, O(n) work over the MST edges, run on the host
inside the same library.  `cluster_features_to_masks` is the reference's per-view variant (iggt/utils/misc.py:174-269)
over the same pieces.

`apply_pca_colormap` keeps the name, argument and return type of the reference helper (iggt/utils/misc.py:272-332),
which runs torch.pca_lowrank and torch.quantile; here every stage is a kernel of csrc/pca.cu.

This module imports none of torch_geometric, torch_scatter, hdbscan, cuML, scikit-learn, matplotlib, cv2 or evo, so
the demo's import block can point here as a whole."""
import numpy as np
import torch

from .. import ops


def knn_avg_features_pyg(points_batch, features_batch, k, device="cuda"):
    """points_batch [N,H,W,3], features_batch [N,H,W,F] (tensor or ndarray) -> smoothed features [N,H,W,F] on `device`."""
    if isinstance(points_batch, np.ndarray):
        points_batch = torch.from_numpy(points_batch).float()
    if isinstance(features_batch, np.ndarray):
        features_batch = torch.from_numpy(features_batch).float()
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("iggt_official_b200 has no CPU path: knn_avg_features_pyg needs a CUDA device")
    points_batch = points_batch.to(device=device, dtype=torch.float32)
    features_batch = features_batch.to(device=device, dtype=torch.float32)
    N, H, W, F = features_batch.shape
    out = ops.knn_mean_features(points_batch.reshape(-1, 3), features_batch.reshape(-1, F), int(k))
    return out.view(N, H, W, F)


# matplotlib's `jet` segment data, per channel (x, y0, y1).  The table below restates matplotlib's lookup-table
# construction from this public data; matplotlib is not a dependency, and the table has not been checked against a
# matplotlib install.
_JET_SEGMENTS = (
    ((0.0, 0.0, 0.0), (0.35, 0.0, 0.0), (0.66, 1.0, 1.0), (0.89, 1.0, 1.0), (1.0, 0.5, 0.5)),
    ((0.0, 0.0, 0.0), (0.125, 0.0, 0.0), (0.375, 1.0, 1.0), (0.64, 1.0, 1.0), (0.91, 0.0, 0.0), (1.0, 0.0, 0.0)),
    ((0.0, 0.5, 0.5), (0.11, 1.0, 1.0), (0.34, 1.0, 1.0), (0.65, 0.0, 0.0), (1.0, 0.0, 0.0)),
)


def jet_lut(n=256):
    """[n, 3] float64: `jet` sampled at n evenly spaced points of [0, 1], piecewise linear between the segment rows."""
    out = []
    for seg in _JET_SEGMENTS:
        a = np.asarray(seg, np.float64)
        x, y0, y1 = a[:, 0] * (n - 1), a[:, 1], a[:, 2]
        xs = (n - 1) * np.linspace(0.0, 1.0, n)
        ind = np.searchsorted(x, xs)[1:-1]
        frac = (xs[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
        out.append(np.clip(np.concatenate([[y1[0]], frac * (y0[ind] - y1[ind - 1]) + y1[ind - 1], [y0[-1]]]), 0, 1))
    return np.stack(out, 1)


def label_palette(labels):
    """uint8 [max label + 1, 3]: the reference's colours, sorted label j -> jet(j / (k - 1)) (jet(0.5) if k == 1),
    truncated by (rgb * 255).astype(uint8).  `labels` holds the distinct non-negative labels."""
    uniq = np.unique(labels)
    lut = jet_lut()
    k = len(uniq)
    pal = np.zeros((int(uniq[-1]) + 1, 3), np.uint8)
    for j, lab in enumerate(uniq):
        x = j / (k - 1) if k > 1 else 0.5
        pal[lab] = (lut[min(int(x * 256), 255)] * 255).astype(np.uint8)
    return pal


def sorted_mst(a, b, w2):
    """Device MST edges -> [n-1, 3] float64 (a, b, weight) rows on the host, sorted by (weight, smaller index,
    larger index) so that equal weights keep a fixed order, each edge oriented from the side of point 0 as
    scikit-learn's Prim MST records it (which side is left in the single-linkage tree decides the cluster numbers)."""
    lo, hi = torch.minimum(a, b), torch.maximum(a, b)
    i = torch.argsort(hi, stable=True)
    i = i[torch.argsort(lo[i], stable=True)]
    i = i[torch.argsort(w2[i], stable=True)]
    mst = torch.stack([a[i].double(), b[i].double(), torch.sqrt(w2[i].double())], 1).cpu().numpy()
    return ops.mst_orient(np.ascontiguousarray(mst))


def hdbscan_device(x, eps, min_samples, min_cluster_size):
    """x [n, 8] fp32 CUDA -> (raw labels [n] int64 ndarray, -1 = noise; (sorted8, orig, box) of the tile search)."""
    sorted8, orig, box = ops.cluster_prepare(x)
    core2 = ops.cluster_core(sorted8, box, min_samples)
    a, b, w2, _ = ops.cluster_mst(sorted8, box, orig, core2)
    raw = ops.hdbscan_labels(sorted_mst(a, b, w2), x.shape[0], min_cluster_size, eps)
    return raw, (sorted8, orig, box)


def cluster_features_to_masks_mv(feature_map, apply_colormap=False, **kwargs):
    """HDBSCAN over the pixels of all views together, with the contrib `hdbscan` package's semantics (Euclidean,
    min_samples = neighbours besides the point itself, excess of mass, cluster_selection_epsilon = eps, no single
    cluster); noise pixels then take the label of their nearest labelled pixel in feature space (ties: lowest pixel
    index), and all labels become 0 if every pixel is noise.

    feature_map [N, H, W, C] (C <= 8; tensor or ndarray; CUDA tensors are used in place) and the keyword arguments
    eps, min_samples (<= 512) and min_cluster_size (>= 2); others (e.g. method="dbscan") are ignored.
    Returns masks [N, H, W] int64, and with apply_colormap also colours [N, H, W, 3] uint8, as ndarrays."""
    eps, min_samples, min_cluster_size = _cluster_args(feature_map, kwargs, "cluster_features_to_masks_mv")
    N, H, W, C = feature_map.shape
    n = N * H * W
    if n < min_samples + 1:
        raise ValueError(f"{n} points: HDBSCAN with min_samples={min_samples} needs at least {min_samples + 1}")
    x = _cuda_features(feature_map, "cluster_features_to_masks_mv")
    with torch.cuda.device(x.device):
        x = x.reshape(n, C).to(torch.float32)
        if not bool(torch.isfinite(x).all()):
            raise ValueError("feature_map has non-finite values")
        labels, rgb = _masks(x, eps, min_samples, min_cluster_size, apply_colormap)
        masks = labels.view(N, H, W).cpu().numpy()
        if not apply_colormap:
            return masks
        return masks, rgb.view(N, H, W, 3).cpu().numpy()


def _cluster_args(feature_map, kwargs, name):
    """Checks shared by both clustering entry points -> (eps, min_samples, min_cluster_size)."""
    if not (isinstance(feature_map, (torch.Tensor, np.ndarray)) and feature_map.ndim == 4):
        raise ValueError("feature_map must be a 4-D [N, H, W, C] tensor or ndarray")
    eps, min_samples, min_cluster_size = (kwargs.get(k) for k in ("eps", "min_samples", "min_cluster_size"))
    if eps is None or min_samples is None or min_cluster_size is None:
        raise ValueError(f"{name} needs eps, min_samples and min_cluster_size")
    eps, min_samples, min_cluster_size = float(eps), int(min_samples), int(min_cluster_size)
    if not (np.isfinite(eps) and eps >= 0 and 1 <= min_samples <= 512 and min_cluster_size >= 2):
        raise ValueError(f"unsupported eps={eps}, min_samples={min_samples}, min_cluster_size={min_cluster_size}")
    if not 1 <= feature_map.shape[3] <= 8:
        raise ValueError(f"feature_map has {feature_map.shape[3]} channels; 1 to 8 are supported")
    return eps, min_samples, min_cluster_size


def _cuda_features(feature_map, name):
    x = torch.as_tensor(feature_map)
    if not x.is_cuda:
        if not torch.cuda.is_available():
            raise RuntimeError(f"iggt_official_b200 has no CPU path: {name} needs a CUDA device")
        x = x.cuda()
    return x


def _masks(x, eps, min_samples, min_cluster_size, apply_colormap):
    """x [n, C] fp32 CUDA, finite -> (labels [n] int64, rgb [n, 3] uint8 or None) on the device: HDBSCAN, all-noise
    -> all 0, noise filled from the nearest labelled point, colours spread over `jet` by this call's labels."""
    x = torch.nn.functional.pad(x, (0, 8 - x.shape[1])).contiguous()   # zero channels leave the distances unchanged
    raw, (sorted8, orig, box) = hdbscan_device(x, eps, min_samples, min_cluster_size)
    if (raw < 0).all():
        raw = np.zeros_like(raw)
    label_sorted = torch.from_numpy(raw.astype(np.int32)).to(x.device)[orig.long()]
    palette = torch.from_numpy(label_palette(raw[raw >= 0])).to(x.device) if apply_colormap else None
    return ops.cluster_fill(sorted8, box, orig, label_sorted, palette)


def cluster_features_to_masks(feature_map, method="kmeans", apply_colormap=False, **kwargs):
    """The reference's per-view variant: HDBSCAN over the pixels of each view on its own, whatever `method` says,
    with the semantics of cluster_features_to_masks_mv; noise pixels take the label of the nearest labelled pixel of
    the same view, and a view whose pixels are all noise becomes all 0.  Colours are per view: view i's sorted labels
    are spread over `jet` by view i's own label count.

    feature_map [N, H, W, C] (C <= 8; tensor or ndarray) and eps, min_samples (<= 512), min_cluster_size (>= 2).
    Returns masks [N, H, W] int32, and with apply_colormap also colours [N, H, W, 3] uint8, as ndarrays."""
    eps, min_samples, min_cluster_size = _cluster_args(feature_map, kwargs, "cluster_features_to_masks")
    N, H, W, C = feature_map.shape
    if H * W < min_samples + 1:
        raise ValueError(f"{H * W} pixels per view: HDBSCAN with min_samples={min_samples} needs at least "
                         f"{min_samples + 1}")
    x = _cuda_features(feature_map, "cluster_features_to_masks")
    masks = np.zeros((N, H, W), np.int32)
    colours = np.zeros((N, H, W, 3), np.uint8)
    with torch.cuda.device(x.device):
        x = x.reshape(N, H * W, C).to(torch.float32)
        if not bool(torch.isfinite(x).all()):
            raise ValueError("feature_map has non-finite values")
        for i in range(N):
            labels, rgb = _masks(x[i], eps, min_samples, min_cluster_size, apply_colormap)
            masks[i] = labels.view(H, W).cpu().numpy()
            if apply_colormap:
                colours[i] = rgb.view(H, W, 3).cpu().numpy()
    return (masks, colours) if apply_colormap else masks


def apply_pca_colormap(image):
    """[N, H, W, C] float features (3 <= C <= 8) -> [N, H, W, 3] float32 colours in [0, 1] on the input's device (a CPU
    tensor is processed on the current CUDA device and returned on the CPU).

    One PCA over all N*H*W pixels together, so colours agree across views: the pixels are projected (uncentred, as the
    reference projects them) onto the first three principal axes of their sample covariance, and each channel is
    stretched from its 2 % to its 98 % quantile (torch.quantile's, bit for bit) and clamped to [0, 1]; a channel
    whose 98 % quantile is not above its 2 % quantile is 0.5.  Other float dtypes are computed in fp32.

    Against the reference: the PCA is exact (fp64 moments, Jacobi eigenvectors) where torch.pca_lowrank is
    randomised, and each axis has a fixed sign (largest-magnitude component positive), so the colours no longer
    change from run to run.  A flipped axis negates its channel before the stretch and swaps the two quantiles, so
    each output channel equals the reference's c or 1 - c up to fp32 rounding.  Only the axes' directions matter
    after the stretch.  torch.quantile's limit of 2^24 elements does not apply.
    Raises ValueError for a non-4-D input, C outside 3..8, a non-float dtype or non-finite values."""
    image = torch.as_tensor(image)
    if image.dim() != 4:
        raise ValueError("image must be a 4-D [N, H, W, C] tensor")
    N, H, W, C = image.shape
    if not 3 <= C <= 8:
        raise ValueError(f"image has {C} channels; 3 to 8 are supported")
    if not image.is_floating_point():
        raise ValueError(f"image must be a float tensor, got {image.dtype}")
    n = N * H * W
    if n == 0:
        raise ValueError("image has no pixels")
    on_cpu = not image.is_cuda
    if on_cpu and not torch.cuda.is_available():
        raise RuntimeError("iggt_official_b200 has no CPU path: apply_pca_colormap needs a CUDA device")
    x = image.cuda() if on_cpu else image
    with torch.cuda.device(x.device):
        x = x.reshape(n, C).to(torch.float32).contiguous()
        basis = ops.pca_basis(x)
        if int(basis.nonfinite.item()) != 0:                          # the call's one host synchronisation
            raise ValueError("image has non-finite values")
        y = ops.pca_project(x, basis.V)
        qv = ops.quantile(y, (0.02, 0.98))
        out = ops.pca_stretch(y, qv).view(N, H, W, 3)
    return out.cpu() if on_cpu else out
