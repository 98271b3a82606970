"""tests/golden/eval_ref.npz: the UNMODIFIED reference SceneEvaluator / DepthEvaluator (iggt/metrics.py),
threshold_depth_map (iggt/datasets/utils/misc.py:488-541), depth_to_world_coords_points and closed_form_inverse_se3
(iggt/utils/geometry.py:183-320) on seeded synthetic scenes.

The reference modules import matplotlib, torch_geometric, torch_scatter, hdbscan / cuML, evo and cv2 at import time
without using them here; they are stubbed as oracle/make_golden_pca.py stubs them.  skimage is not installed, so
skimage.transform.resize is stood in by what skimage >= 0.19 runs for resize(order=0, anti_aliasing=False):
scipy.ndimage.zoom(image, 1 / (in / out) per axis, order=0, mode="mirror", grid_mode=True).  The scenes are regenerated from
their seeds by the tests (scene(), CASES); so are the threshold and camera inputs
(threshold_inputs(), camera_inputs()).  Under numpy 2, nan_to_num(scalar, copy=False) raises where numpy 1 copied (metrics.py:103, every
frame); the maker gives the reference module numpy 1's meaning of copy=False (copy when needed) and nothing else.
Run once:  python -m oracle.make_golden_eval"""
import importlib.util
import json
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "eval_ref.npz")


def _skimage_stub():
    from scipy import ndimage

    def resize(image, output_shape, order=None, anti_aliasing=None, **_):
        assert order == 0 and not anti_aliasing
        factors = np.divide(image.shape, output_shape)
        return ndimage.zoom(image, [1 / f for f in factors], order=0, mode="mirror", grid_mode=True)

    sk = types.ModuleType("skimage")
    sk.transform = types.ModuleType("skimage.transform")
    sk.transform.resize = resize
    sys.modules["skimage"], sys.modules["skimage.transform"] = sk, sk.transform


def reference_modules():
    from oracle.make_golden_pca import _Stub, install_stubs
    from oracle.shims import REFERENCE_ROOT
    install_stubs()
    sys.modules.setdefault("cv2", _Stub("cv2"))
    _skimage_stub()
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)

    def load(name, rel):
        spec = importlib.util.spec_from_file_location(name, os.path.join(REFERENCE_ROOT, rel))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod
    ref_metrics = load("ref_metrics", "iggt/metrics.py")
    compat = types.ModuleType("numpy")
    compat.__dict__.update(np.__dict__)
    compat.nan_to_num = lambda x, copy=True, **k: np.nan_to_num(x, copy=copy or not isinstance(x, np.ndarray), **k)
    ref_metrics.np = compat
    return (ref_metrics, load("ref_misc", "iggt/datasets/utils/misc.py"),
            load("ref_geometry", "iggt/utils/geometry.py"))


def rotation(rng, n):
    q = rng.standard_normal((n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    x, y, z, w = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(n, 3, 3)


def scene(seed, S, gt_hw, pred_hw, empty_frame=None, zero_median_frame=None):
    """Seeded GT depth [S,H,W] (about 10 % invalid zeros), prediction [S,h,w,1] (a scaled, noisy GT sampled at the
    prediction's resolution) and [S,3,4] float32 camera-from-world poses (predictions perturbed by small rotations,
    one exactly equal, one turned by nearly 180 degrees)."""
    rng = np.random.default_rng(seed)
    H, W = gt_hw
    h, w = pred_hw
    yy, xx = np.meshgrid(np.linspace(0, 1, H), np.linspace(0, 1, W), indexing="ij")
    gt = np.stack([2 + 3 * yy + np.sin(6 * xx + i) + 0.2 * rng.standard_normal((H, W)) for i in range(S)])
    gt = np.where(rng.random(gt.shape) < 0.1, 0, gt).astype(np.float32)
    iy = np.minimum((np.arange(h) * H) // h, H - 1)
    ix = np.minimum((np.arange(w) * W) // w, W - 1)
    pred = (gt[:, iy][:, :, ix] * 0.37 + 0.05 * rng.standard_normal((S, h, w))).astype(np.float32)
    pred = np.abs(pred) + 0.01
    if empty_frame is not None:
        gt[empty_frame] = 0
    if zero_median_frame is not None:
        pred[zero_median_frame, : (2 * h) // 3] = 0
    R = rotation(rng, S)
    t = rng.standard_normal((S, 3))
    small = rotation(np.random.default_rng(seed + 100), S)
    Rp = R @ (np.eye(3) + 0.02 * (small - small.transpose(0, 2, 1)))
    if S > 1:
        Rp[0] = R[0]
    if S > 2:
        Rp[2] = R[2] @ np.diag([-1.0, -1.0, 1.0])
    gt_pose = np.concatenate([R, t[:, :, None]], 2).astype(np.float32)
    pred_pose = np.concatenate([Rp, (t + 0.05 * rng.standard_normal((S, 3)))[:, :, None]], 2).astype(np.float32)
    return gt, pred[..., None], gt_pose, pred_pose


CASES = {   # name: (scene args, SceneEvaluator args or DepthEvaluator args with sparse)
    "same": (dict(seed=1, S=3, gt_hw=(48, 64), pred_hw=(48, 64)), dict(alignment="median", clip=(0.1, 100.0))),
    "resize": (dict(seed=2, S=5, gt_hw=(48, 64), pred_hw=(40, 56), empty_frame=1, zero_median_frame=3),
               dict(alignment="median", clip=(0.1, 100.0))),
    "lsq": (dict(seed=3, S=3, gt_hw=(48, 64), pred_hw=(40, 56)), dict(alignment="least_squares", clip=(0.1, 100.0))),
    "none": (dict(seed=4, S=3, gt_hw=(48, 64), pred_hw=(40, 56)), dict(alignment=None, clip=(0.1, 100.0))),
    "noclip": (dict(seed=5, S=3, gt_hw=(48, 64), pred_hw=(40, 56)), dict(alignment="median", clip=None)),
    "sparse": (dict(seed=6, S=3, gt_hw=(48, 64), pred_hw=(40, 56), zero_median_frame=2),
               dict(alignment="median", clip=(0.1, 100.0), sparse=True)),
    "one": (dict(seed=7, S=1, gt_hw=(48, 64), pred_hw=(40, 56)), dict(alignment="median", clip=(0.1, 100.0))),
}


def plain(o):
    if isinstance(o, np.ndarray):
        return o.tolist()
    if isinstance(o, (np.floating, np.integer)):
        return o.item()
    if isinstance(o, dict):
        return {k: plain(v) for k, v in o.items()}
    if isinstance(o, list):
        return [plain(v) for v in o]
    return o


def threshold_inputs():
    rng = np.random.default_rng(21)
    d = (rng.gamma(2.0, 2.0, (3, 48, 64))).astype(np.float32)
    d[0, :4] = np.nan
    d[1, rng.random((48, 64)) < 0.3] = 0
    d[2, 5, 5] = 50.0
    return d


def camera_inputs():
    rng = np.random.default_rng(31)
    depth = rng.uniform(0.5, 8.0, (2, 48, 64)).astype(np.float32)
    depth[0, 0, :5] = 0
    R = rotation(rng, 2)
    ext = np.concatenate([R, 0.3 * rng.standard_normal((2, 3, 1))], 2).astype(np.float32)
    K = np.array([[[60.0, 0, 31.5], [0, 58.0, 23.5], [0, 0, 1]]] * 2, np.float32)
    return depth, ext, K


if __name__ == "__main__":
    ref_metrics, ref_misc, ref_geometry = reference_modules()
    out = {}
    for name, (sargs, eargs) in CASES.items():
        gt, pred, gp, pp = scene(**sargs)
        if eargs.get("sparse"):
            ev = ref_metrics.DepthEvaluator(eargs["alignment"], eargs["clip"], sparse_pred=True)
            res = [ev.evaluate_depth(gt[i], pred[i]) for i in range(len(gt))]
        else:
            ev = ref_metrics.SceneEvaluator(eargs["alignment"], eargs["clip"])
            res = ev.evaluate_scene({"gt_depth": gt, "gt_extrinsic": gp}, {"depth": pred, "extrinsic": pp})
        out[f"{name}_result"] = np.array(json.dumps(plain(res)))
    d = threshold_inputs()
    out["thr_default"] = np.stack([ref_misc.threshold_depth_map(m.copy()) for m in d])
    out["thr_demo"] = np.stack([ref_misc.threshold_depth_map(m.copy(), 99, -1) for m in d])
    out["thr_maxdepth"] = np.stack([ref_misc.threshold_depth_map(m.copy(), 95, 5, max_depth=9.5) for m in d])
    depth, ext, K = camera_inputs()
    w, c, m = zip(*[ref_geometry.depth_to_world_coords_points(depth[i], ext[i], K[i]) for i in range(2)])
    out["cam_world"], out["cam_cam"], out["cam_mask"] = np.stack(w), np.stack(c), np.stack(m)
    out["se3_inv"] = ref_geometry.closed_form_inverse_se3(ext)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")
