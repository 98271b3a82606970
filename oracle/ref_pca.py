"""Float64 restatement of the reference's apply_pca_colormap (iggt/utils/misc.py:272-332, called from demo.py:372 and
demo.py:380) with an exact PCA.

The reference takes the principal axes from torch.pca_lowrank, which is randomised: each axis comes back with a sign
that depends on the global RNG state.  Here the axes are the eigenvectors of the sample covariance (numpy's eigh)
with the product's sign convention: the largest-magnitude component of each axis is positive (the first one on a
tie).  The projection is of the uncentred pixels, as in the reference, and the quantiles use torch.quantile's rank
rule: rank = float32(q) * float32(n - 1) in fp32, interpolated linearly between the floor and ceil order
statistics (here in float64).  Any size: no 2^24-element limit."""
import numpy as np

LOW_P, HIGH_P = 0.02, 0.98


def sign_convention(v):
    """Flip each column of v so that its largest-magnitude component (the first one on a tie) is positive."""
    v = np.array(v, np.float64)
    k = np.argmax(np.abs(v), axis=0)                  # argmax returns the first maximum
    return v * np.where(v[k, np.arange(v.shape[1])] < 0, -1.0, 1.0)


def pca_basis(x):
    """x [n, C] -> (evals [C] descending, evecs [C, C] float64, eigenvector j in column j, sign convention applied)."""
    xd = np.asarray(x, np.float64)
    cov = np.cov(xd, rowvar=False, ddof=1) if xd.shape[0] > 1 else np.zeros((xd.shape[1],) * 2)
    w, v = np.linalg.eigh(cov)
    order = np.argsort(-w, kind="stable")
    return w[order], sign_convention(v[:, order])


def quantile(row, q):
    """torch.quantile(row, q)'s rank rule with float64 interpolation."""
    row = np.asarray(row, np.float64)
    n = row.shape[0]
    r = np.float32(q) * np.float32(n - 1)
    lo = min(int(r), n - 1)
    hi = min(int(np.ceil(r)), n - 1)
    s = np.partition(row, (lo, hi))
    w = float(r - np.float32(int(r)))
    return s[lo] + w * (s[hi] - s[lo])


def apply_pca_colormap(image, return_parts=False):
    """image [N, H, W, C] -> [N, H, W, 3] float64 in [0, 1] (and, with return_parts, (y [n, 3], lo [3], hi [3]))."""
    image = np.asarray(image)
    n_, h, w_, c = image.shape
    flat = image.reshape(-1, c).astype(np.float64)
    _, v = pca_basis(flat)
    y = flat @ v[:, :3]
    out = np.empty_like(y)
    lo, hi = np.empty(3), np.empty(3)
    for j in range(3):
        lo[j], hi[j] = quantile(y[:, j], LOW_P), quantile(y[:, j], HIGH_P)
        out[:, j] = np.clip((y[:, j] - lo[j]) / (hi[j] - lo[j]), 0.0, 1.0) if hi[j] > lo[j] else 0.5
    out = out.reshape(n_, h, w_, 3)
    return (out, (y, lo, hi)) if return_parts else out


def align_flips(got, want):
    """Per channel, `want` or 1 - `want`, whichever is closer to `got` (an axis of opposite sign stretches to 1 - c)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    out = want.copy()
    for j in range(want.shape[-1]):
        if np.abs(got[..., j] - (1.0 - want[..., j])).max() < np.abs(got[..., j] - want[..., j]).max():
            out[..., j] = 1.0 - want[..., j]
    return out
