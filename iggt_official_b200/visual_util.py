"""Point-cloud export on the GPU: `predictions_to_glb` keeps the name, arguments and defaults of the reference helper
(visual_util.py:38-238), which the demo calls three times per scene (demo.py:642, vis_mode rgb / mask / pca).  The
reference masks, compacts and takes percentiles in numpy after copying every point to the host, then builds a
trimesh.Scene.  Here the per-point work runs in csrc/pointcloud.cu and the selection of csrc/pca.cu, and only the
kept points cross to the host, already packed as the GLB's point section.  The cameras are host float64 numpy code,
the reference's own arithmetic.

The result is a `GlbScene`, not a trimesh.Scene: its `export(file_obj)` writes glTF 2.0 binary (the only call the demo
makes on the result), and its attributes hold the points, colours, camera glyphs and scene transform.

Semantics kept from the reference, including two of its quirks:
  - a uint8 colour source (the demo's `mask` mode passes HDBSCAN's uint8 palette) is multiplied by 255 in uint8, which
    wraps: channel c is written as (256 - c) % 256.  The reference writes these colours; so does this function;
  - the scene alignment inv(E0) @ opengl @ rot_y(180) is not applied to the vertices; it is the root node's matrix,
    as trimesh's Scene.apply_transform moves the base frame rather than the geometry.
Differences: an unknown vis_mode raises ValueError (the reference fails later); mask_sky with a target_dir raises
NotImplementedError (the reference downloads an ONNX sky-segmentation model); point, confidence and colour counts
that differ raise ValueError.

Two library pieces are restated from their public definitions and have not been checked against the libraries,
which are not dependencies: matplotlib's `gist_rainbow` table (camera colours) and trimesh's
`creation.cone(r, h, sections=4)` (the camera glyph's vertex and face order).

This module imports none of trimesh, matplotlib, gradio, cv2, onnxruntime or scipy."""
import json
import os
import struct

import numpy as np
import torch

from . import ops
from .utils.misc import segment_lut

_COLOR_KEYS = {"rgb": "images", "mask": "features", "pca": "pca_features"}

# matplotlib's gist_rainbow: a list colormap, (x, (r, g, b)) per control point.  Restated from memory of its public
# definition; not verified against a matplotlib install.
_GIST_RAINBOW = ((0.000, (1.00, 0.00, 0.16)), (0.030, (1.00, 0.00, 0.00)), (0.215, (1.00, 1.00, 0.00)),
                 (0.400, (0.00, 1.00, 0.00)), (0.586, (0.00, 1.00, 1.00)), (0.770, (0.00, 0.00, 1.00)),
                 (0.954, (1.00, 0.00, 1.00)), (1.000, (1.00, 0.00, 0.75)))


def gist_rainbow_lut(n=256):
    """[n, 3] float64: the gist_rainbow table (a list colormap becomes segment data with y0 = y1 per point)."""
    return segment_lut([[(x, c[k], c[k]) for x, c in _GIST_RAINBOW] for k in range(3)], n)


def camera_color(i, num_cameras):
    """(r, g, b) ints of camera i: gist_rainbow(i / num_cameras) as a colormap samples a float (row int(x * 256)),
    each channel truncated by int(255 * x)."""
    x = i / num_cameras
    row = gist_rainbow_lut()[min(int(x * 256), 255)]
    return tuple(int(255 * float(v)) for v in row)


def rotation_matrix(axis, degrees):
    """[4, 4] float64 rotation about 'x', 'y' or 'z', computed as scipy's Rotation.from_euler(axis, degrees,
    degrees=True).as_matrix() computes it: the half-angle quaternion, then the quaternion-to-matrix products."""
    t = np.deg2rad(degrees)
    q = np.zeros(4)
    q[3] = np.cos(t / 2)
    q["xyz".index(axis)] = np.sin(t / 2)
    x, y, z, w = q
    x2, y2, z2, w2 = x * x, y * y, z * z, w * w
    xy, zw, xz, yw, yz, xw = x * y, z * w, x * z, y * w, y * z, x * w
    out = np.eye(4)
    out[:3, :3] = [[x2 - y2 - z2 + w2, 2 * (xy - zw), 2 * (xz + yw)],
                   [2 * (xy + zw), -x2 + y2 - z2 + w2, 2 * (yz - xw)],
                   [2 * (xz - yw), 2 * (yz + xw), -x2 - y2 + z2 + w2]]
    return out


OPENGL = np.diag([1.0, -1.0, -1.0, 1.0])       # flips y and z


def cone(radius, height, sections=4):
    """trimesh.creation.cone's mesh, restated (unverified vertex and face order): vertex 0 the base centre, a ring of
    `sections` vertices at z = 0 from angle 0 counter-clockwise, the apex (0, 0, height) last; the base triangles
    around vertex 0, then the sides.  (vertices float64, faces int64)."""
    theta = np.linspace(0.0, 2.0 * np.pi, sections + 1)[:-1]
    ring = np.stack([radius * np.cos(theta), radius * np.sin(theta), np.zeros(sections)], 1)
    vertices = np.concatenate([[[0.0, 0.0, 0.0]], ring, [[0.0, 0.0, height]]])
    k = np.arange(sections)
    a, b = 1 + k, 1 + (k + 1) % sections
    faces = np.concatenate([np.stack([np.zeros(sections, np.int64), b, a], 1),
                            np.stack([a, b, np.full(sections, sections + 1)], 1)])
    return vertices.astype(np.float64), faces.astype(np.int64)


def transform_points(m, pts):
    """pts [k, 3] through the affine [4, 4] m, as the reference's transform_points does it: pts @ m[:3, :3]^T +
    m[:3, 3], no homogeneous divide."""
    mt = m.swapaxes(-1, -2)
    return (np.asarray(pts) @ mt[..., :-1, :] + mt[..., -1:, :])[..., :3]


def camera_faces(faces, nv):
    """visual_util.py:357-390: six triangles per cone face not touching vertex 0, joining it to the scaled copy
    (offset nv) and the turned copy (offset 2 nv), then all of them with the winding reversed."""
    tris = []
    for f in faces:
        if 0 in f:
            continue
        v1, v2, v3 = (int(v) for v in f)
        tris += [(v1, v2, v2 + nv), (v1, v1 + nv, v3), (v3 + nv, v2, v3),
                 (v1, v2, v2 + 2 * nv), (v1, v1 + 2 * nv, v3), (v3 + 2 * nv, v2, v3)]
    tris += [(c, b, a) for a, b, c in tris]
    return np.array(tris, np.int64)


def camera_glyph(cam_to_world, scene_scale):
    """visual_util.py:241-288: (vertices float64 [3 nv, 3], faces int64) of one camera - a four-sided cone of width
    scale * 0.05 and height scale * 0.1 turned by 45 degrees, a copy scaled by 0.95 and a copy turned by 2 degrees,
    with the apex at the camera centre."""
    width, height = scene_scale * 0.05, scene_scale * 0.1
    turn = rotation_matrix("z", 45)
    turn[2, 3] = -height
    full = cam_to_world @ OPENGL @ turn
    v, f = cone(width, height, sections=4)
    both = np.concatenate([v, 0.95 * v, transform_points(rotation_matrix("z", 2), v)])
    return transform_points(full, both), camera_faces(f, len(v))


# ---------------------------------------------------------------------------------------------------- GLB writer
_GLB_MAGIC, _GLB_JSON, _GLB_BIN = 0x46546C67, 0x4E4F534A, 0x004E4942
_FLOAT, _UBYTE, _UINT = 5126, 5121, 5125
_ARRAY_BUFFER, _ELEMENT_ARRAY_BUFFER = 34962, 34963


def _pad4(n):
    return (n + 3) & ~3


class GlbScene:
    """A point cloud plus camera glyphs under one root transform.

    points [m, 3] float32 and colors [m, 4] uint8 RGBA (alpha 255, as trimesh stores point colours); cameras: a list of
    (vertices [k, 3] float64, faces [f, 3] int64, rgba tuple); transform [4, 4] float64, the root node's matrix.
    bounds: the per-axis (min, max) of the points (NaNs left out), computed from them when None.  threshold and
    scene_scale: the confidence threshold and the scale the glyphs were sized by.
    `export` writes glTF 2.0 binary."""

    def __init__(self, points, colors, cameras, transform, bounds=None, threshold=None, scene_scale=None,
                 point_section=None):
        self.points = np.ascontiguousarray(points, dtype=np.float32)
        self.colors = np.ascontiguousarray(colors, dtype=np.uint8)
        if self.points.ndim != 2 or self.points.shape[1] != 3 or self.colors.shape != (len(self.points), 4):
            raise ValueError("points must be [m, 3] and colors [m, 4] with the same m")
        self.cameras = list(cameras)
        self.transform = np.asarray(transform, dtype=np.float64)
        if bounds is None:
            with np.errstate(invalid="ignore"):
                bounds = (np.nanmin(self.points, 0), np.nanmax(self.points, 0)) if len(self.points) else None
        self.bounds = bounds
        self.threshold, self.scene_scale = threshold, scene_scale
        self._point_section = point_section            # the packed xyz + RGBA bytes, when they came so from the device

    def _parts(self):
        """The GLB file as a list of byte strings."""
        m = len(self.points)
        section = self._point_section
        if section is None:
            section = memoryview(self.points.tobytes() + self.colors.tobytes())
        views = [dict(buffer=0, byteOffset=0, byteLength=12 * m, target=_ARRAY_BUFFER),
                 dict(buffer=0, byteOffset=12 * m, byteLength=4 * m, target=_ARRAY_BUFFER)]
        lo, hi = self.bounds
        accessors = [dict(bufferView=0, componentType=_FLOAT, count=m, type="VEC3", min=[float(v) for v in lo],
                          max=[float(v) for v in hi]),
                     dict(bufferView=1, componentType=_UBYTE, normalized=True, count=m, type="VEC4")]
        meshes = [dict(primitives=[dict(attributes=dict(POSITION=0, COLOR_0=1), mode=0)])]
        materials, tail, offset = [], [], 16 * m
        for i, (verts, faces, rgba) in enumerate(self.cameras):
            v32 = np.ascontiguousarray(verts, dtype=np.float32)
            idx = np.ascontiguousarray(faces, dtype=np.uint32).reshape(-1)
            for arr, target in ((v32, _ARRAY_BUFFER), (idx, _ELEMENT_ARRAY_BUFFER)):
                views.append(dict(buffer=0, byteOffset=offset, byteLength=arr.nbytes, target=target))
                tail.append(arr.tobytes())
                offset += arr.nbytes                     # float32 and uint32 data: every offset stays 4-aligned
            accessors.append(dict(bufferView=len(views) - 2, componentType=_FLOAT, count=len(v32), type="VEC3",
                                  min=[float(v) for v in v32.min(0)], max=[float(v) for v in v32.max(0)]))
            accessors.append(dict(bufferView=len(views) - 1, componentType=_UINT, count=int(idx.size), type="SCALAR"))
            rgba = tuple(rgba) + (255,) * (4 - len(rgba))
            materials.append(dict(pbrMetallicRoughness=dict(baseColorFactor=[c / 255.0 for c in rgba],
                                                            metallicFactor=0.0, roughnessFactor=1.0),
                                  doubleSided=True))
            meshes.append(dict(primitives=[dict(attributes=dict(POSITION=len(accessors) - 2),
                                                indices=len(accessors) - 1, mode=4, material=i)]))
        nodes = [dict(matrix=[float(v) for v in self.transform.T.reshape(-1)],
                      children=list(range(1, len(meshes) + 1)))] + [dict(mesh=j) for j in range(len(meshes))]
        doc = dict(asset=dict(version="2.0", generator="iggt_official_b200"), scene=0, scenes=[dict(nodes=[0])],
                   nodes=nodes, meshes=meshes, accessors=accessors, bufferViews=views,
                   buffers=[dict(byteLength=offset)])
        if materials:
            doc["materials"] = materials
        js = json.dumps(doc, separators=(",", ":")).encode()
        js += b" " * (_pad4(len(js)) - len(js))
        bin_len = _pad4(offset)
        total = 12 + 8 + len(js) + 8 + bin_len
        return ([struct.pack("<III", _GLB_MAGIC, 2, total), struct.pack("<II", len(js), _GLB_JSON), js,
                 struct.pack("<II", bin_len, _GLB_BIN), section] + tail + [b"\0" * (bin_len - offset)])

    def export(self, file_obj=None, file_type="glb"):
        """Write the scene as glTF 2.0 binary to a path or a binary file object; with file_obj None, return the
        bytes."""
        if str(file_type).lower() != "glb":
            raise ValueError(f"only glb export is supported, got {file_type!r}")
        parts = self._parts()
        if file_obj is None:
            return b"".join(parts)
        if isinstance(file_obj, (str, os.PathLike)):
            with open(file_obj, "wb") as f:
                for p in parts:
                    f.write(p)
        else:
            for p in parts:
                file_obj.write(p)
        return None


# ---------------------------------------------------------------------------------------------------- device side
def _on_device(x, device):
    """An ndarray or CPU tensor copied once to `device`, or a CUDA tensor there as it is; contiguous."""
    if isinstance(x, torch.Tensor):
        return x.detach().to(device).contiguous()
    return torch.from_numpy(np.ascontiguousarray(np.asarray(x))).to(device)


def _host(x):
    return x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def predictions_to_glb(predictions, conf_thres=50.0, filter_by_frames="all", mask_black_bg=False, mask_white_bg=False,
                       show_cam=True, mask_sky=False, target_dir=None, prediction_mode="Predicted Pointmap",
                       vis_mode="rgb"):
    """visual_util.py:38-238 on the GPU -> GlbScene.

    predictions: a dict of ndarrays (copied to the current CUDA device once) or CUDA tensors (used in place), as the
    demo holds them: world_points / world_points_from_depth [S,H,W,3] float32, world_points_conf / depth_conf
    [S,H,W] float32 (ones when missing), images NCHW float32, features uint8 [S,H,W,3], pca_features e.g.
    [1,S,H,W,3] float32, extrinsic [S,3,4].  conf_thres: a percentile of the confidences (None -> 10, 0 -> keep every
    confidence > 1e-5).  filter_by_frames: "all" or "<index>: ..." (an unparsable value means all)."""
    if not isinstance(predictions, dict):
        raise ValueError("predictions must be a dictionary")
    if vis_mode not in _COLOR_KEYS:
        raise ValueError(f"vis_mode must be one of {sorted(_COLOR_KEYS)}, got {vis_mode!r}")
    if mask_sky and target_dir is not None:
        raise NotImplementedError("mask_sky needs the ONNX sky-segmentation model, which is not supported")
    if conf_thres is None:
        conf_thres = 10.0
    if conf_thres != 0.0 and not 0.0 <= conf_thres <= 100.0:
        raise ValueError("Percentiles must be in the range [0, 100]")
    frame = None
    if filter_by_frames != "all" and filter_by_frames != "All":
        try:
            frame = int(filter_by_frames.split(":")[0])
        except (ValueError, IndexError):
            pass
    if "Pointmap" in prediction_mode and "world_points" in predictions:
        pts, conf = predictions["world_points"], predictions.get("world_points_conf")
    else:
        pts, conf = predictions["world_points_from_depth"], predictions.get("depth_conf")
    images = predictions[_COLOR_KEYS[vis_mode]]
    cams = _host(predictions["extrinsic"])
    if frame is not None:
        pts, images, cams = pts[frame][None], images[frame][None], cams[frame][None]
        conf = None if conf is None else conf[frame][None]

    device = pts.device if isinstance(pts, torch.Tensor) and pts.is_cuda else torch.device("cuda",
                                                                                            torch.cuda.current_device())
    pts = _on_device(pts, device)
    if pts.dtype != torch.float32 or pts.dim() < 1 or pts.shape[-1] != 3:
        raise ValueError(f"points must be float32 [..., 3], got {pts.dtype} {tuple(pts.shape)}")
    n = pts.numel() // 3
    if n == 0:
        raise ValueError("no points")
    conf = torch.ones(n, dtype=torch.float32, device=device) if conf is None else _on_device(conf, device)
    if conf.dtype != torch.float32 or conf.numel() != n:
        raise ValueError(f"confidences must be float32 with one value per point ({n}), got {conf.dtype} "
                         f"{tuple(conf.shape)}")
    img = _on_device(images, device)
    if img.dtype not in (torch.float32, torch.uint8):
        raise ValueError(f"colours must be float32 or uint8, got {img.dtype}")
    if not (img.dim() == 4 and img.shape[1] == 3):          # NCHW stays as it is; anything else is channels-last
        if img.numel() % 3:
            raise ValueError(f"channels-last colours of shape {tuple(img.shape)} do not reshape to [-1, 3]")
        img = img.reshape(-1, 3)
    if (img.numel() // 3) != n:
        raise ValueError(f"{img.numel() // 3} colours for {n} points")

    with torch.cuda.device(device):
        stats = torch.empty(16, dtype=torch.int32, device=device)   # threshold, p5/p95 per axis, count, min, max
        f = stats.view(torch.float32)
        thr = None
        if conf_thres != 0.0:
            thr = f[0:1]
            ops.select(conf.view(1, n), ops.QRULE_NUMPY, [conf_thres], out=thr.view(1, 1))
        bg = (ops.PC_MASK_BLACK if mask_black_bg else 0) | (ops.PC_MASK_WHITE if mask_white_bg else 0)
        mask, planes, rgba, ws = ops.pointcloud_select(pts.view(n, 3), conf.view(n), thr, img, bg)
        ops.select(planes, ops.QRULE_NUMPY, [5.0, 95.0], mask=mask.view(1, n).expand(3, n), out=f[1:7].view(3, 2))
        packed = ops.pointcloud_compact(pts.view(n, 3), mask, rgba, ws, stats[7:8], f[8:14])
        st = stats.cpu().numpy()
        fs = st.view(np.float32)
        m = int(st[7]) & 0xffffffff
        section = None
        if m:
            host = torch.empty(16 * m, dtype=torch.uint8, pin_memory=True)
            host.copy_(packed[:16 * m])
            section = host.numpy()

    threshold = fs[0] if conf_thres != 0.0 else 0.0
    if m == 0:
        points, colors, scene_scale, bounds = (np.array([[1, 0, 0]], np.float32), np.full((1, 4), 255, np.uint8), 1,
                                               None)
    else:
        points = section[:12 * m].view(np.float32).reshape(m, 3)
        colors = section[12 * m:].reshape(m, 4)
        scene_scale = np.linalg.norm(fs[[2, 4, 6]] - fs[[1, 3, 5]])
        bounds = (fs[8:11].copy(), fs[11:14].copy())

    num_cameras = len(cams)
    ext = np.zeros((num_cameras, 4, 4))
    ext[:, :3, :4] = cams
    ext[:, 3, 3] = 1
    cameras = []
    if show_cam:
        for i in range(num_cameras):
            verts, faces = camera_glyph(np.linalg.inv(ext[i]), scene_scale)
            cameras.append((verts, faces, camera_color(i, num_cameras) + (255,)))
    transform = np.linalg.inv(ext[0]) @ OPENGL @ rotation_matrix("y", 180)
    return GlbScene(points, colors, cameras, transform, bounds, threshold, scene_scale,
                    None if section is None else memoryview(section))
