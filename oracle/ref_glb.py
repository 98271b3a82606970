"""numpy restatement of the reference point-cloud export (visual_util.py:38-390, predictions_to_glb and its camera
helpers), returning what oracle/make_golden_glb.py records from the unmodified reference: the point cloud's vertices
and colours, each camera glyph's vertices, faces and colour, the scene transform, the confidence threshold and the
scene scale.  Host numpy (float32 data, float64 cameras), no GPU; the tests pin it to tests/golden/glb_ref.npz and then
use it at full size.

Two library pieces the reference calls are restated here from their public definitions, unverified (neither library
is installed): matplotlib's `gist_rainbow` colormap and trimesh's `creation.cone(r, h, sections=4)`."""
import numpy as np
from scipy.spatial.transform import Rotation

# matplotlib's gist_rainbow: a list colormap, (x, (r, g, b)) per control point (unverified restatement)
GIST_RAINBOW = ((0.000, (1.00, 0.00, 0.16)), (0.030, (1.00, 0.00, 0.00)), (0.215, (1.00, 1.00, 0.00)),
                (0.400, (0.00, 1.00, 0.00)), (0.586, (0.00, 1.00, 1.00)), (0.770, (0.00, 0.00, 1.00)),
                (0.954, (1.00, 0.00, 1.00)), (1.000, (1.00, 0.00, 0.75)))


def gist_rainbow_lut(n=256):
    """[n, 3] float64: the list colormap's table, piecewise linear between the control points sampled at n evenly
    spaced points (matplotlib's lookup-table construction, gamma 1)."""
    x = np.array([p[0] for p in GIST_RAINBOW]) * (n - 1)
    xs = (n - 1) * np.linspace(0.0, 1.0, n)
    ind = np.searchsorted(x, xs)[1:-1]
    frac = (xs[1:-1] - x[ind - 1]) / (x[ind] - x[ind - 1])
    cols = []
    for c in range(3):
        y = np.array([p[1][c] for p in GIST_RAINBOW], np.float64)
        cols.append(np.clip(np.concatenate([[y[0]], frac * (y[ind] - y[ind - 1]) + y[ind - 1], [y[-1]]]), 0, 1))
    return np.stack(cols, 1)


def gist_rainbow(x, n=256):
    """RGBA tuple of floats for a Python float x in [0, 1], as a matplotlib colormap samples a scalar: row
    int(x * n) of the table (x == 1 -> the last row), alpha 1."""
    r, g, b = gist_rainbow_lut(n)[min(int(x * n), n - 1)]
    return (float(r), float(g), float(b), 1.0)


def cone(radius, height, sections=4):
    """trimesh.creation.cone's mesh (unverified restatement): vertex 0 the base centre, a ring of `sections` vertices
    at z = 0 from angle 0 counter-clockwise, the apex (0, 0, height) last; base faces around vertex 0, then the sides.
    Returns (vertices [sections + 2, 3] float64, faces [2 * sections, 3] int64)."""
    theta = np.linspace(0.0, 2.0 * np.pi, sections + 1)[:-1]
    ring = np.stack([radius * np.cos(theta), radius * np.sin(theta), np.zeros(sections)], 1)
    vertices = np.concatenate([[[0.0, 0.0, 0.0]], ring, [[0.0, 0.0, height]]]).astype(np.float64)
    k = np.arange(sections)
    a, b = 1 + k, 1 + (k + 1) % sections
    faces = np.concatenate([np.stack([np.zeros(sections, np.int64), b, a], 1),
                            np.stack([a, b, np.full(sections, sections + 1)], 1)]).astype(np.int64)
    return vertices, faces


def camera_faces(faces, nv):
    """The glyph's triangles: for every cone face not touching vertex 0, six triangles joining it to the scaled copy
    (offset nv) and the turned copy (offset 2 nv); then all of them again with the winding reversed."""
    tris = []
    for f in faces:
        if 0 in f:
            continue
        v1, v2, v3 = (int(v) for v in f)
        tris += [(v1, v2, v2 + nv), (v1, v1 + nv, v3), (v3 + nv, v2, v3),
                 (v1, v2, v2 + 2 * nv), (v1, v1 + 2 * nv, v3), (v3 + 2 * nv, v2, v3)]
    tris += [(c, b, a) for a, b, c in tris]
    return np.array(tris)


def apply_affine(m, pts):
    """pts [k, 3] -> (pts, 1) m^T without the homogeneous divide."""
    mt = m.swapaxes(-1, -2)
    return (np.asarray(pts) @ mt[..., :-1, :] + mt[..., -1:, :])[..., :3]


def euler(axis, degrees):
    out = np.eye(4)
    out[:3, :3] = Rotation.from_euler(axis, degrees, degrees=True).as_matrix()
    return out


OPENGL = np.diag([1.0, -1.0, -1.0, 1.0])


def camera_glyph(cam_to_world, scene_scale):
    """(vertices [3 * nv, 3] float64, faces) of one camera: a four-sided cone of width scale / 20 and height
    scale / 10, plus a copy scaled by 0.95 and a copy turned by 2 degrees, apex at the camera centre."""
    width, height = scene_scale * 0.05, scene_scale * 0.1
    turn = euler("z", 45)
    turn[2, 3] = -height
    full = cam_to_world @ OPENGL @ turn
    v, f = cone(width, height)
    both = np.concatenate([v, 0.95 * v, apply_affine(euler("z", 2), v)])
    return apply_affine(full, both), camera_faces(f, len(v))


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def predictions_to_glb(predictions, conf_thres=50.0, filter_by_frames="all", mask_black_bg=False, mask_white_bg=False,
                       show_cam=True, prediction_mode="Predicted Pointmap", vis_mode="rgb"):
    """The records of one export (dict): points, colors, cameras [(vertices, faces, rgb)], transform, threshold,
    scene_scale."""
    thr_q = 10.0 if conf_thres is None else conf_thres
    frame = None
    if filter_by_frames not in ("all", "All"):
        try:
            frame = int(filter_by_frames.split(":")[0])
        except (ValueError, IndexError):
            frame = None
    if "Pointmap" in prediction_mode and "world_points" in predictions:
        pts, conf_key = predictions["world_points"], "world_points_conf"
    else:
        pts, conf_key = predictions["world_points_from_depth"], "depth_conf"
    pts = np.asarray(pts)
    conf = np.asarray(predictions[conf_key]) if conf_key in predictions else np.ones_like(pts[..., 0])
    src = {"rgb": "images", "mask": "features", "pca": "pca_features"}[vis_mode]
    img = _np(predictions[src])
    cams = np.asarray(predictions["extrinsic"])
    if frame is not None:
        pts, conf, img, cams = pts[frame][None], conf[frame][None], img[frame][None], cams[frame][None]
    if img.ndim == 4 and img.shape[1] == 3:
        img = img.transpose(0, 2, 3, 1)
    rgb = (img.reshape(-1, 3) * 255).astype(np.uint8)
    conf = conf.reshape(-1)
    threshold = 0.0 if thr_q == 0.0 else np.percentile(conf, thr_q)
    keep = (conf >= threshold) & (conf > 1e-5)
    if mask_black_bg:
        keep &= rgb.sum(axis=1) >= 16
    if mask_white_bg:
        keep &= ~np.all(rgb > 240, axis=1)
    points, colors = pts.reshape(-1, 3)[keep], rgb[keep]
    if points.size == 0:
        points, colors, scene_scale = np.array([[1, 0, 0]]), np.array([[255, 255, 255]]), 1
    else:
        lo, hi = np.percentile(points, 5, axis=0), np.percentile(points, 95, axis=0)
        scene_scale = np.linalg.norm(hi - lo)
    ext = np.zeros((len(cams), 4, 4))
    ext[:, :3, :4] = cams
    ext[:, 3, 3] = 1
    cameras = []
    if show_cam:
        for i in range(len(cams)):
            v, f = camera_glyph(np.linalg.inv(ext[i]), scene_scale)
            rgb_i = tuple(int(255 * c) for c in gist_rainbow(i / len(cams))[:3])
            cameras.append((v, f, rgb_i))
    transform = np.linalg.inv(ext[0]) @ OPENGL @ euler("y", 180)
    return dict(points=points, colors=colors, cameras=cameras, transform=transform, threshold=threshold,
                scene_scale=scene_scale)
