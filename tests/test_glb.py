"""Point-cloud export (visual_util.predictions_to_glb, csrc/pointcloud.cu, the selection in csrc/pca.cu) and the GLB
writer.

CPU: the numpy oracle (oracle/ref_glb.py) against the unmodified reference's records (tests/golden/glb_ref.npz) bit for
bit, the host camera code against the fixture, the rotations against scipy, the GLB writer through a small parser,
argument errors and import hygiene.  GPU: every fixture case through the public function from ndarrays and from CUDA
tensors, the kernels on their own against numpy (n = 1, n not a multiple of the tile, 16 x 1036^2 points), the
public function against the oracle at the demo's shapes, and repeated exports byte for byte."""
import io
import json
import os
import struct
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import make_golden_glb as G                                     # noqa: E402
from oracle import ref_glb                                                  # noqa: E402
from iggt_official_b200 import visual_util as V                             # noqa: E402

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "glb_ref.npz"))
FIELDS = ("points", "colors", "transform", "threshold", "scene_scale", "cam_vertices", "cam_faces", "cam_colors")


def golden(name):
    return {k[len(name) + 1:]: GOLDEN[k] for k in GOLDEN.files
            if k.startswith(name + "_") and k[len(name) + 1:] in FIELDS}


def same(a, b):
    """Equal values, dtypes and shapes, NaNs included (bit for bit for floats)."""
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def parse_glb(data):
    """(JSON document, BIN chunk bytes) of a GLB file, checking the container's layout."""
    magic, version, length = struct.unpack_from("<III", data, 0)
    assert magic == 0x46546C67 and version == 2 and length == len(data)
    jlen, jtype = struct.unpack_from("<II", data, 12)
    assert jtype == 0x4E4F534A and jlen % 4 == 0
    js = data[20:20 + jlen]
    assert js == js.rstrip(b" ") + b" " * (len(js) - len(js.rstrip(b" ")))     # padded with spaces
    blen, btype = struct.unpack_from("<II", data, 20 + jlen)
    assert btype == 0x004E4942 and blen % 4 == 0 and 28 + jlen + blen == len(data)
    return json.loads(js), data[28 + jlen:]


def accessor_array(doc, binary, index):
    acc = doc["accessors"][index]
    view = doc["bufferViews"][acc["bufferView"]]
    assert view["byteOffset"] % 4 == 0 and acc.get("byteOffset", 0) % 4 == 0
    dtype = {5126: np.float32, 5121: np.uint8, 5125: np.uint32}[acc["componentType"]]
    width = {"SCALAR": 1, "VEC3": 3, "VEC4": 4}[acc["type"]]
    assert view["byteLength"] == acc["count"] * width * np.dtype(dtype).itemsize
    raw = binary[view["byteOffset"]:view["byteOffset"] + view["byteLength"]]
    return np.frombuffer(raw, dtype).reshape(acc["count"], width), acc


def check_glb(scene, data):
    """The GLB holds the scene's arrays bit for bit, with the accessor metadata the spec requires."""
    doc, binary = parse_glb(data)
    assert doc["asset"]["version"] == "2.0" and len(binary) >= doc["buffers"][0]["byteLength"]
    root = doc["nodes"][doc["scenes"][doc["scene"]]["nodes"][0]]
    assert same(np.array(root["matrix"], np.float64).reshape(4, 4).T, scene.transform)
    meshes = [doc["meshes"][doc["nodes"][c]["mesh"]] for c in root["children"]]
    assert len(meshes) == 1 + len(scene.cameras)
    prim = meshes[0]["primitives"][0]
    assert prim["mode"] == 0
    pos, acc = accessor_array(doc, binary, prim["attributes"]["POSITION"])
    assert acc["type"] == "VEC3" and same(pos, scene.points)
    assert acc["min"] == [float(v) for v in np.nanmin(scene.points, 0)]
    assert acc["max"] == [float(v) for v in np.nanmax(scene.points, 0)]
    col, acc = accessor_array(doc, binary, prim["attributes"]["COLOR_0"])
    assert acc["type"] == "VEC4" and acc["normalized"] is True and same(col, scene.colors)
    for mesh, (verts, faces, rgba) in zip(meshes[1:], scene.cameras):
        prim = mesh["primitives"][0]
        assert prim["mode"] == 4
        v, acc = accessor_array(doc, binary, prim["attributes"]["POSITION"])
        assert same(v, verts.astype(np.float32))
        assert acc["min"] == [float(x) for x in v.min(0)] and acc["max"] == [float(x) for x in v.max(0)]
        idx, _ = accessor_array(doc, binary, prim["indices"])
        assert same(idx.reshape(-1, 3).astype(np.int64), faces)
        mat = doc["materials"][prim["material"]]["pbrMetallicRoughness"]["baseColorFactor"]
        assert mat == [c / 255.0 for c in rgba]


# ------------------------------------------------------------------------------------------------ CPU

@pytest.mark.parametrize("name", list(G.CASES))
def test_oracle_matches_reference(name):
    pred, kw = G.case_inputs(name)
    got = G.flatten(name, ref_glb.predictions_to_glb(pred, **kw))
    want = golden(name)
    assert sorted(k[len(name) + 1:] for k in got) == sorted(want)
    for k, w in want.items():
        assert same(got[f"{name}_{k}"], w), k


@pytest.mark.parametrize("name", list(G.CASES))
def test_cameras_match_reference(name):
    """The package's host camera code against the reference's records, from the fixture's scene scale."""
    pred, kw = G.case_inputs(name)
    want = golden(name)
    cams = pred["extrinsic"]
    frame = {"1: frame_001.png": 1, "0": 0}.get(kw.get("filter_by_frames"))
    if frame is not None:
        cams = cams[frame][None]
    ext = np.zeros((len(cams), 4, 4))
    ext[:, :3, :4] = cams
    ext[:, 3, 3] = 1
    assert same(np.linalg.inv(ext[0]) @ V.OPENGL @ V.rotation_matrix("y", 180), want["transform"])
    if not kw.get("show_cam", True):
        assert "cam_vertices" not in want
        return
    scale = want["scene_scale"][()]
    for i in range(len(cams)):
        verts, faces = V.camera_glyph(np.linalg.inv(ext[i]), scale)
        assert same(verts, want["cam_vertices"][i]) and same(faces, want["cam_faces"][i])
        assert V.camera_color(i, len(cams)) == tuple(int(c) for c in want["cam_colors"][i])
        assert faces.shape == (48, 3)
        centre = np.linalg.inv(ext[i])[:3, 3]
        assert np.abs(verts[5] - centre).max() <= 1e-12 * (1 + np.abs(centre).max())     # the cone's apex


def test_rotations_match_scipy():
    from scipy.spatial.transform import Rotation
    for axis in "xyz":
        for deg in (0, 2, 30, 45, 90, 135, 180, -45, 270, 1e-3):
            assert same(V.rotation_matrix(axis, deg)[:3, :3], Rotation.from_euler(axis, deg, degrees=True).as_matrix())


def test_restatements_agree():
    assert same(V.gist_rainbow_lut(), ref_glb.gist_rainbow_lut())
    for s in (1, 2, 3, 7, 8, 16, 100):
        for i in range(s):
            assert V.camera_color(i, s) == tuple(int(255 * c) for c in ref_glb.gist_rainbow(i / s)[:3])
    for a, b in zip(V.cone(0.3, 0.7), ref_glb.cone(0.3, 0.7)):
        assert same(a, b)


def random_scene(rng, m, cams):
    pts = rng.standard_normal((m, 3)).astype(np.float32)
    if m > 3:
        pts[1, 0], pts[2, 1] = np.nan, -0.0
    col = np.concatenate([rng.integers(0, 256, (m, 3)), np.full((m, 1), 255)], 1).astype(np.uint8)
    cameras = [(rng.standard_normal((18, 3)), rng.integers(0, 18, (48, 3)).astype(np.int64), (10 * i, 20, 30, 255))
               for i in range(cams)]
    q = np.linalg.qr(rng.standard_normal((3, 3)))[0]
    transform = np.eye(4)
    transform[:3, :3], transform[:3, 3] = q, rng.standard_normal(3)
    return V.GlbScene(pts, col, cameras, transform)


@pytest.mark.parametrize("m,cams", [(1, 0), (5, 1), (1001, 3), (4096, 8)])
def test_glb_writer_roundtrip(m, cams, tmp_path):
    scene = random_scene(np.random.default_rng(m + cams), m, cams)
    data = scene.export()
    check_glb(scene, data)
    path = tmp_path / "scene.glb"
    assert scene.export(file_obj=str(path)) is None and path.read_bytes() == data
    buf = io.BytesIO()
    scene.export(file_obj=buf, file_type="glb")
    assert buf.getvalue() == data


def test_glb_writer_errors():
    scene = random_scene(np.random.default_rng(0), 4, 1)
    with pytest.raises(ValueError):
        scene.export(file_type="ply")
    with pytest.raises(ValueError):
        V.GlbScene(np.zeros((3, 3), np.float32), np.zeros((2, 4), np.uint8), [], np.eye(4))


def test_argument_errors():
    pred, _ = G.case_inputs("rgb50")
    with pytest.raises(ValueError):
        V.predictions_to_glb([pred])
    with pytest.raises(ValueError):
        V.predictions_to_glb(pred, vis_mode="depth")
    with pytest.raises(NotImplementedError):
        V.predictions_to_glb(pred, mask_sky=True, target_dir="scene")
    with pytest.raises(ValueError):
        V.predictions_to_glb(pred, conf_thres=150.0)


def test_import_hygiene():
    names = ("trimesh", "matplotlib", "gradio", "cv2", "onnxruntime", "scipy")
    code = (f"import sys, numpy, torch; names = {names!r}; before = {{m for m in names if m in sys.modules}}; "
            "import iggt_official_b200.visual_util; "
            "bad = [m for m in names if m in sys.modules and m not in before]; assert not bad, bad")
    subprocess.run([sys.executable, "-c", code], cwd=ROOT, check=True)


# ------------------------------------------------------------------------------------------------ GPU

def to_cuda(pred):
    return {k: (torch.as_tensor(v) if not isinstance(v, torch.Tensor) else v).cuda() for k, v in pred.items()}


def check_against(scene, want):
    """scene (GlbScene) against records in the fixture's layout, bit for bit."""
    pts, cols = want["points"], want["colors"]
    if pts.dtype != np.float32:                                              # the reference's single-point fallback
        assert same(scene.points, pts.astype(np.float32)) and same(scene.colors[:, :3], cols.astype(np.uint8))
        assert scene.scene_scale == 1 and int(want["scene_scale"]) == 1
    else:
        assert same(scene.points, pts) and same(scene.colors[:, :3], cols)
        assert same(np.float32(scene.scene_scale), want["scene_scale"]) and isinstance(scene.scene_scale, np.float32)
    assert (scene.colors[:, 3] == 255).all()
    assert np.array_equal(np.asarray(scene.threshold, want["threshold"].dtype), want["threshold"], equal_nan=True)
    assert same(scene.transform, want["transform"])
    if "cam_vertices" not in want:
        assert scene.cameras == []
        return
    assert len(scene.cameras) == len(want["cam_vertices"])
    for (v, f, rgba), wv, wf, wc in zip(scene.cameras, want["cam_vertices"], want["cam_faces"], want["cam_colors"]):
        assert same(v, wv) and same(f, wf) and tuple(rgba) == tuple(int(c) for c in wc) + (255,)


def records(r):
    """oracle/ref_glb records -> the fixture's layout."""
    return {k[len("x_"):]: v for k, v in G.flatten("x", r).items()}


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["numpy", "cuda"])
@pytest.mark.parametrize("name", list(G.CASES))
def test_public_matches_fixture(name, source):
    pred, kw = G.case_inputs(name)
    if source == "cuda":
        pred = to_cuda(pred)
    before = {k: (v.clone() if isinstance(v, torch.Tensor) else v.copy()) for k, v in pred.items()}
    scene = V.predictions_to_glb(pred, **kw)
    check_against(scene, golden(name))
    check_glb(scene, scene.export())
    assert before.keys() == pred.keys()
    for k, v in before.items():                                              # predictions is not modified
        assert same(v.cpu().numpy() if isinstance(v, torch.Tensor) else v,
                    pred[k].cpu().numpy() if isinstance(pred[k], torch.Tensor) else pred[k]), k


@pytest.mark.gpu
def test_public_argument_errors():
    pred, _ = G.case_inputs("rgb50")
    bad = dict(pred, images=pred["images"].astype(np.float64))
    with pytest.raises(ValueError):
        V.predictions_to_glb(bad)
    with pytest.raises(ValueError):                                          # [1,S,H,W,3]: frame 0 is every frame
        V.predictions_to_glb(pred, vis_mode="pca", filter_by_frames="0")
    with pytest.raises(ValueError):
        V.predictions_to_glb(dict(pred, world_points_conf=pred["world_points_conf"][:, :-1]))
    with pytest.raises(ValueError):
        V.predictions_to_glb(dict(pred, world_points=pred["world_points"].astype(np.float64)))


def kernel_inputs(n, seed, kind):
    rng = np.random.default_rng(seed)
    pts = rng.standard_normal((n, 3)).astype(np.float32)
    conf = (1 + rng.gamma(2.0, 1.0, n)).astype(np.float32)
    conf[rng.random(n) < 0.05] = 0.0
    if n > 8:
        pts[3, 1], pts[5] = np.nan, (-0.0, 0.0, -0.0)
        conf[7] = np.nan
    col = (rng.integers(0, 256, (n, 3)).astype(np.uint8) if kind == "u8"
           else rng.random((n, 3)).astype(np.float32))
    if n > 64:
        col[rng.random(n) < 0.1] = 0 if kind == "u8" else 1.0
        col[rng.random(n) < 0.1] = 1 if kind == "u8" else 0.0
    return pts, conf, col


def numpy_select(pts, conf, col, thr, bg):
    rgb = (col * 255).astype(np.uint8)
    keep = (conf >= thr) & (conf > 1e-5)
    if bg & 1:
        keep &= rgb.sum(axis=1) >= 16
    if bg & 2:
        keep &= ~np.all(rgb > 240, axis=1)
    return keep, rgb


def run_kernels(pts, conf, col, thr, bg):
    from iggt_official_b200 import ops
    n = len(pts)
    P, C, K = (torch.from_numpy(a).cuda() for a in (pts, conf, col))
    stats = torch.zeros(16, dtype=torch.int32, device="cuda")
    f = stats.view(torch.float32)
    f[0] = float(thr)
    mask, planes, rgba, ws = ops.pointcloud_select(P, C, f[0:1], K, bg)
    q = ops.select(planes, ops.QRULE_NUMPY, [5.0, 95.0], mask=mask.view(1, n).expand(3, n))
    packed = ops.pointcloud_compact(P, mask, rgba, ws, stats[7:8], f[8:14])
    packed2 = ops.pointcloud_compact(P, mask, rgba, ws, stats[7:8], f[8:14])
    torch.cuda.synchronize()
    st = stats.cpu().numpy()
    m = int(st[7])
    return (mask.cpu().numpy(), rgba.cpu().numpy().view(np.uint8).reshape(n, 4), q.cpu().numpy(), m,
            st.view(np.float32)[8:14], packed[:16 * m].cpu().numpy(), packed2[:16 * m].cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("n,kind,bg", [(1, "f32", 0), (1000, "f32", 3), (1025, "u8", 1), (5000, "u8", 2),
                                       (3 * 1024, "f32", 0), (16 * 1036 * 1036, "u8", 3)])
def test_kernels_against_numpy(n, kind, bg):
    pts, conf, col = kernel_inputs(n, n, kind)
    thr = np.float32(np.percentile(conf, 30.0)) if n > 1 else np.float32(0.0)
    mask, rgba, q, m, mm, packed, packed2 = run_kernels(pts, conf, col, thr, bg)
    keep, rgb = numpy_select(pts, conf, col, thr, bg)
    assert same(mask.astype(bool), keep) and same(rgba[:, :3], rgb) and (rgba[:, 3] == 255).all()
    sel = pts[keep]
    assert m == len(sel)
    assert packed.tobytes() == packed2.tobytes()                            # deterministic
    assert same(packed[:12 * m].view(np.float32).reshape(m, 3), sel)       # pixel order
    assert same(packed[12 * m:].reshape(m, 4)[:, :3], rgb[keep])
    with np.errstate(invalid="ignore"):
        for j in range(3):
            fin = sel[:, j][~np.isnan(sel[:, j])]
            if len(fin):
                lo, hi = np.sort(fin)[[0, -1]]                               # -0 orders below +0
                assert same(mm[j], lo) and same(mm[3 + j], hi), j
            if len(sel):
                want = np.array([np.percentile(sel[:, j], 5.0), np.percentile(sel[:, j], 95.0)])  # scalar q: fp32
                assert want.dtype == np.float32 and np.array_equal(q[j], want, equal_nan=True), (j, q[j], want)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 336, 504), (8, 532, 532)])
@pytest.mark.parametrize("vis_mode,kw", [("rgb", dict(conf_thres=0.3, prediction_mode="Pointmap Regression")),
                                         ("mask", dict(conf_thres=50.0, mask_black_bg=True, mask_white_bg=True,
                                                       filter_by_frames="2: x")),
                                         ("pca", dict(conf_thres=20.0))])
def test_full_size_against_oracle(shape, vis_mode, kw):
    S, H, W = shape
    pred = G.scene(seed=40 + S, S=S, H=H, W=W, black=0.05, white=0.05)
    scene = V.predictions_to_glb(pred, vis_mode=vis_mode, **kw)
    check_against(scene, records(ref_glb.predictions_to_glb(pred, vis_mode=vis_mode, **kw)))


@pytest.mark.gpu
def test_export_is_deterministic():
    pred = to_cuda(G.scene(seed=77, S=3, H=336, W=504))
    a = V.predictions_to_glb(pred, conf_thres=0.3, vis_mode="pca").export()
    b = V.predictions_to_glb(pred, conf_thres=0.3, vis_mode="pca").export()
    assert a == b
