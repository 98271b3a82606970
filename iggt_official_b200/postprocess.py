"""Device-side post-processing of a prediction dict (SURVEY.md section 8f, row 1).

Same names and argument meaning as the reference helpers `iggt.utils.pose_enc.pose_encoding_to_extri_intri` and
`iggt.utils.geometry.unproject_depth_map_to_point_map`, but on CUDA tensors, so demo.py's
"predictions -> .cpu().numpy() -> per-frame numpy loop" (demo.py:340-355) becomes two kernel launches.

The ground-truth helpers the demo's loader uses (demo.py:38, 46: threshold_depth_map, closed_form_inverse_se3,
depth_to_world_coords_points) keep the reference names and argument meaning as well."""
import numpy as np
import torch

from . import ops


def pose_encoding_to_extri_intri(pose_encoding: torch.Tensor, image_size_hw=None, pose_encoding_type="absT_quaR_FoV",
                                 build_intrinsics=True):
    if pose_encoding_type != "absT_quaR_FoV":
        raise NotImplementedError
    H, W = image_size_hw if image_size_hw is not None else (0, 0)
    return ops.pose_to_cameras(pose_encoding.float(), int(H), int(W), build_intrinsics and image_size_hw is not None)


def unproject_depth_map_to_point_map(depth_map: torch.Tensor, extrinsics_cam: torch.Tensor, intrinsics_cam: torch.Tensor):
    """depth [S,H,W,1] or [S,H,W]; extrinsics [S,3,4]; intrinsics [S,3,3]  ->  world points [S,H,W,3] (CUDA)."""
    world, _ = ops.unproject_depth(depth_map.float(), extrinsics_cam.float(), intrinsics_cam.float())
    return world


def _cuda_f32(x, name):
    """ndarray -> fp32 CUDA copy; tensor -> itself (it must be a CUDA fp32 tensor)."""
    if isinstance(x, torch.Tensor):
        if not x.is_cuda or x.dtype != torch.float32:
            raise ValueError(f"{name}: expected a CUDA float32 tensor or an ndarray")
        return x
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).cuda()


def threshold_depth_map(depth_map, max_percentile=99, min_percentile=1, max_depth=-1):
    """iggt.datasets.utils.misc.threshold_depth_map on the GPU, for one map (H,W) or a batch (S,H,W) with one pair of
    percentiles per map.  In place, returning its argument: values > max_depth (if > 0) become 0, then values above the
    max_percentile-th / below the min_percentile-th np.nanpercentile (when that percentile is > 0 and the threshold is
    > 0) become 0.  An ndarray is processed in float32 on the current CUDA device and written back."""
    if depth_map is None:
        return None
    for p in (max_percentile, min_percentile):
        if p > 0 and not p <= 100:
            raise ValueError("Percentiles must be in the range [0, 100]")
    if depth_map.ndim not in (2, 3):
        raise ValueError(f"expected a (H,W) or (S,H,W) depth map, got {tuple(depth_map.shape)}")
    t = _cuda_f32(depth_map, "depth_map")
    d = t.contiguous()
    flat = d.view(1 if d.dim() == 2 else d.shape[0], -1)
    if max_depth > 0:
        ops.depth_zero_outside(flat, max_depth=float(max_depth))
    qs = [float(p) for p in (max_percentile, min_percentile) if p > 0]
    if qs:
        thr = torch.zeros((flat.shape[0], 2), dtype=torch.float32, device=flat.device)
        got = ops.select(flat, ops.QRULE_NUMPY_NAN, qs)
        cols = [c for c, p in enumerate((max_percentile, min_percentile)) if p > 0]
        thr[:, cols] = got
        ops.depth_zero_outside(flat, thr, use_hi=max_percentile > 0, use_lo=min_percentile > 0)
    if isinstance(depth_map, torch.Tensor):
        if d.data_ptr() != depth_map.data_ptr():
            depth_map.copy_(d)
    else:
        depth_map[...] = d.cpu().numpy()
    return depth_map


def closed_form_inverse_se3(se3):
    """Inverse of each (N,4,4) or (N,3,4) [R | t] as (N,4,4) [R^T | -R^T t]: an ndarray gives a float64 ndarray (R^T t
    in the input's dtype), a tensor a tensor of its dtype on its device."""
    if tuple(se3.shape[-2:]) not in ((4, 4), (3, 4)):
        raise ValueError(f"se3 must be of shape (N,4,4), got {tuple(se3.shape)}.")
    R, T = se3[:, :3, :3], se3[:, :3, 3:]
    if isinstance(se3, torch.Tensor):
        Rt = R.transpose(1, 2)
        out = torch.eye(4, dtype=R.dtype, device=R.device).repeat(len(R), 1, 1)
        out[:, :3, :3] = Rt
        out[:, :3, 3:] = -torch.bmm(Rt, T)
        return out
    Rt = np.transpose(R, (0, 2, 1))
    out = np.tile(np.eye(4), (len(R), 1, 1))
    out[:, :3, :3] = Rt
    out[:, :3, 3:] = -np.matmul(Rt, T)
    return out


def depth_to_world_coords_points(depth_map, extrinsic, intrinsic, z_far=100.0, eps=1e-8):
    """iggt.utils.geometry.depth_to_world_coords_points on the GPU: depth (H,W) with a (3,4)/(4,4) camera-from-world
    extrinsic and a (3,3) intrinsic, or a batch (S,H,W) with (S,3,4)/(S,4,4) and (S,3,3) -> (world (..,H,W,3),
    cam (..,H,W,3), mask (..,H,W) bool).  World points come from iggt_unproject_depth (R^T (X - t) in fp32); camera
    coordinates are computed in fp64 and rounded to fp32 as the reference's numpy does.  ndarray inputs give ndarrays,
    tensors give CUDA tensors."""
    if depth_map is None:
        return None, None, None
    as_numpy = not isinstance(depth_map, torch.Tensor)
    d = _cuda_f32(depth_map, "depth_map")
    single = d.dim() == 2
    d = d[None] if single else d
    S = d.shape[0]
    dev = d.device
    e = extrinsic if isinstance(extrinsic, torch.Tensor) else torch.from_numpy(np.asarray(extrinsic))
    k = intrinsic if isinstance(intrinsic, torch.Tensor) else torch.from_numpy(np.asarray(intrinsic))
    e = e.reshape(S, e.shape[-2], 4)
    k = k.reshape(S, 3, 3).to(device=dev, dtype=torch.float64)
    if tuple(e.shape[-2:]) not in ((3, 4), (4, 4)):
        raise ValueError(f"extrinsic must be (3,4) or (4,4), got {tuple(extrinsic.shape)}")
    if bool((k[:, 0, 1] != 0).any()) or bool((k[:, 1, 0] != 0).any()):
        raise ValueError("Intrinsic matrix must have zero skew")
    world, mask = ops.unproject_depth(d, e[:, :3, :4].to(device=dev, dtype=torch.float32), k.float(), eps=eps,
                                      z_far=z_far)
    cam = ops.depth_to_cam(d, k)
    if single:
        world, cam, mask = world[0], cam[0], mask[0]
    if as_numpy:
        return world.cpu().numpy(), cam.cpu().numpy(), mask.cpu().numpy()
    return world, cam, mask
