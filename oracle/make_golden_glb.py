"""tests/golden/glb_ref.npz: the UNMODIFIED reference predictions_to_glb (visual_util.py:38-390) on seeded scenes.

trimesh, matplotlib and gradio are not installed.  trimesh is replaced by a recording stub: PointCloud keeps its
vertices and colours, Trimesh its vertices, faces and face colours (trimesh's default grey, RGBA), Scene its
add_geometry calls and the apply_transform matrix; creation.cone is oracle/ref_glb.cone.  matplotlib's colormap
registry returns oracle/ref_glb.gist_rainbow.  Both restatements are unverified (see oracle/ref_glb.py).  gradio is a
bare stub, and so are the modules oracle/make_golden_pca.py stubs for the reference's iggt.utils imports.  The module's
numpy is wrapped only to record np.percentile's first result (the confidence threshold) and np.linalg.norm's result
(the scene scale).  The inputs are regenerated from their seeds by the tests (case_inputs, CASES).
Run once:  python -m oracle.make_golden_glb"""
import importlib.util
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "glb_ref.npz")


def _rotations(rng, n):
    q = rng.standard_normal((n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    x, y, z, w = q.T
    return np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                     2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                     2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).reshape(n, 3, 3)


def scene(seed, S=3, H=28, W=42, conf="uniform", images="nchw", black=0.0, white=0.0):
    """Seeded predictions as the demo holds them after its squeeze: world points and points from depth [S,H,W,3],
    confidences [S,H,W] float32, images (NCHW float32 in [0, 1]), HDBSCAN-style uint8 colours [S,H,W,3], PCA
    colours as a [1,S,H,W,3] float32 torch tensor, extrinsics [S,3,4] float32.  `conf`: "uniform" (1 + gamma),
    "ties" (few distinct values, many at the threshold), "nan" (one NaN), "small" (a share at or below 1e-5).
    `black` / `white`: share of pixels set to black / white in the images, the palette and the PCA colours."""
    import torch
    rng = np.random.default_rng(seed)
    yy, xx = np.meshgrid(np.linspace(-1, 1, H), np.linspace(-1.5, 1.5, W), indexing="ij")
    depth = 2 + 0.5 * np.sin(3 * xx)[None] + 0.3 * rng.standard_normal((S, H, W))
    wp = np.stack([xx[None] * depth, yy[None] * depth, depth], -1) + 0.1 * rng.standard_normal((S, H, W, 3))
    wpd = wp + 0.05 * rng.standard_normal(wp.shape)
    if conf == "ties":
        c = 1 + rng.integers(0, 4, (S, H, W)).astype(np.float64)
    else:
        c = 1 + rng.gamma(2.0, 1.0, (S, H, W))
    c = c.astype(np.float32)
    if conf == "nan":
        c[1, 3, 5] = np.nan
    if conf == "small":
        c[rng.random(c.shape) < 0.2] = 0
        c[0, 0, :4] = np.float32(1e-5)
    dc = (1 + rng.gamma(2.0, 1.0, (S, H, W))).astype(np.float32)
    img = rng.random((S, H, W, 3)).astype(np.float32)
    pal = rng.integers(0, 256, (S, H, W, 3)).astype(np.uint8)
    pca = rng.random((S, H, W, 3)).astype(np.float32)
    for share, value in ((black, 0), (white, 1)):
        sel = rng.random((S, H, W)) < share
        img[sel], pca[sel], pal[sel] = value, value, 0 if value == 0 else 1     # palette: c -> (256 - c) % 256
    pal[0, 0, 0] = (17, 3, 251)
    R = _rotations(rng, S)
    ext = np.concatenate([R, rng.standard_normal((S, 3, 1))], 2).astype(np.float32)
    pred = {"world_points": wp.astype(np.float32), "world_points_conf": c,
            "world_points_from_depth": wpd.astype(np.float32), "depth_conf": dc,
            "images": img.transpose(0, 3, 1, 2).copy() if images == "nchw" else img,
            "features": pal, "pca_features": torch.from_numpy(pca)[None], "extrinsic": ext}
    return pred


CASES = {   # name: (scene args, predictions_to_glb keyword arguments)
    "rgb50": (dict(seed=1), dict(conf_thres=50.0)),
    "demo": (dict(seed=2), dict(conf_thres=0.3, filter_by_frames="All", prediction_mode="Pointmap Regression")),
    "zero": (dict(seed=3, conf="small"), dict(conf_thres=0.0)),
    "none_ties": (dict(seed=4, conf="ties"), dict(conf_thres=None)),
    "ties50": (dict(seed=5, conf="ties", S=2, H=12, W=16), dict(conf_thres=50.0)),
    "nan": (dict(seed=6, conf="nan", S=2, H=12, W=16), dict(conf_thres=50.0)),
    "empty_black": (dict(seed=7, black=1.0, S=2, H=12, W=16), dict(conf_thres=20.0, mask_black_bg=True)),
    "frame_bg": (dict(seed=8, black=0.1, white=0.1), dict(conf_thres=30.0, filter_by_frames="1: frame_001.png",
                                                           mask_black_bg=True, mask_white_bg=True)),
    "mask": (dict(seed=9, black=0.1, white=0.1), dict(conf_thres=0.3, vis_mode="mask", mask_black_bg=True,
                                                       mask_white_bg=True)),
    "pca_depth": (dict(seed=10, white=0.1), dict(conf_thres=25.0, vis_mode="pca", mask_white_bg=True,
                                                 prediction_mode="Predicted Depthmap")),
    "nowp": (dict(seed=11, S=2, H=12, W=16), dict(conf_thres=40.0, filter_by_frames="garbage", show_cam=False)),
    "nhwc_frame0": (dict(seed=12, images="nhwc", S=2, H=12, W=16), dict(conf_thres=60.0, filter_by_frames="0")),
}


def case_inputs(name):
    """(predictions, keyword arguments) of case `name`; the "nowp" case drops world_points and depth_conf."""
    sargs, kw = CASES[name]
    pred = scene(**sargs)
    if name == "nowp":
        del pred["world_points"], pred["depth_conf"]
    return pred, dict(kw)


class _Rec:
    def __init__(self):
        self.geometry, self.transform, self.percentiles, self.norms = [], None, [], []


REC = _Rec()


def _trimesh_stub():
    from oracle import ref_glb
    tm = types.ModuleType("trimesh")

    class Scene:
        def add_geometry(self, g):
            REC.geometry.append(g)

        def apply_transform(self, m):
            assert REC.transform is None
            REC.transform = np.array(m, copy=True)

    class PointCloud:
        def __init__(self, vertices, colors):
            self.vertices, self.colors = np.array(vertices, copy=True), np.array(colors, copy=True)

    class Trimesh:
        def __init__(self, vertices, faces):
            self.vertices, self.faces = np.array(vertices, copy=True), np.array(faces, copy=True)
            self.visual = types.SimpleNamespace(face_colors=np.tile(np.array([102, 102, 102, 255], np.uint8),
                                                                    (len(self.faces), 1)))

    def cone(radius, height, sections=None):
        v, f = ref_glb.cone(radius, height, sections)
        return types.SimpleNamespace(vertices=v, faces=f)

    tm.Scene, tm.PointCloud, tm.Trimesh = Scene, PointCloud, Trimesh
    tm.creation = types.SimpleNamespace(cone=cone)
    def get_cmap(name):
        assert name == "gist_rainbow"
        return ref_glb.gist_rainbow
    sys.modules["matplotlib"].colormaps = types.SimpleNamespace(get_cmap=get_cmap)   # install_stubs' placeholder
    sys.modules["trimesh"] = tm


def reference_predictions_to_glb():
    from oracle.make_golden_pca import _Stub, install_stubs
    from oracle.shims import REFERENCE_ROOT
    install_stubs()
    _trimesh_stub()
    for name in ("gradio", "cv2"):
        sys.modules.setdefault(name, _Stub(name))
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    spec = importlib.util.spec_from_file_location("ref_visual_util", os.path.join(REFERENCE_ROOT, "visual_util.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    rec_np = types.ModuleType("numpy")
    rec_np.__dict__.update(np.__dict__)

    def percentile(*a, **k):
        r = np.percentile(*a, **k)
        REC.percentiles.append(r)
        return r

    def norm(*a, **k):
        r = np.linalg.norm(*a, **k)
        REC.norms.append(r)
        return r
    rec_np.percentile = percentile
    rec_np.linalg = types.SimpleNamespace(norm=norm, inv=np.linalg.inv)
    mod.np = rec_np
    return mod.predictions_to_glb


def run(fn, pred, kw):
    """One reference call -> the records oracle/ref_glb.predictions_to_glb returns."""
    global REC
    REC = _Rec()
    fn(pred, **kw)
    cloud, meshes = REC.geometry[0], REC.geometry[1:]
    thr_q = 10.0 if kw.get("conf_thres", 50.0) is None else kw.get("conf_thres", 50.0)
    return dict(points=cloud.vertices, colors=cloud.colors,
                cameras=[(m.vertices, m.faces, tuple(int(c) for c in m.visual.face_colors[0, :3])) for m in meshes],
                transform=REC.transform, threshold=0.0 if thr_q == 0.0 else REC.percentiles[0],
                scene_scale=REC.norms[0] if REC.norms else 1)


def flatten(name, r):
    out = {f"{name}_points": r["points"], f"{name}_colors": r["colors"], f"{name}_transform": r["transform"],
           f"{name}_threshold": np.asarray(r["threshold"]), f"{name}_scene_scale": np.asarray(r["scene_scale"])}
    if r["cameras"]:
        out[f"{name}_cam_vertices"] = np.stack([c[0] for c in r["cameras"]])
        out[f"{name}_cam_faces"] = np.stack([c[1] for c in r["cameras"]])
        out[f"{name}_cam_colors"] = np.array([c[2] for c in r["cameras"]], np.uint8)
    return out


if __name__ == "__main__":
    fn = reference_predictions_to_glb()
    out = {}
    for name in CASES:
        pred, kw = case_inputs(name)
        out.update(flatten(name, run(fn, pred, kw)))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")
