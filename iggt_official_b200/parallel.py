"""View sharding over the GPUs of one box (SURVEY.md section 8e; new design -- the reference is single-GPU).

Rank r holds views [r*S_loc, (r+1)*S_loc) of every scene.  DINOv2, frame blocks and every dense head are
per-view, so they need no communication; each of the 24 global blocks needs the K and V of all views:
one NCCL all-gather of the rank's K|V rows ([B*S_loc*T, 2048] 16-bit) per global block, after which the
local queries attend to the full key set with the same flash kernel (exact softmax).  The camera head needs
the S camera tokens of layer 23 (one tiny all-gather).
"""
from typing import Optional

import torch
import torch.distributed as dist

from . import ops


def _trace_begin():
    """bench.py's per-kernel trace (ops.TRACE) also gets a row for the exchange step: CUDA events on the current stream
    around the K|V staging copy + the collective (torch's NCCL work joins the current stream at both ends)."""
    if ops.TRACE is None:
        return None
    e0 = torch.cuda.Event(enable_timing=True)
    e0.record()
    return e0


def _trace_end(e0, name, nbytes):
    if e0 is None:
        return
    e1 = torch.cuda.Event(enable_timing=True)
    e1.record()
    ops.TRACE.append((name, 0.0, float(nbytes), e0, e1, ()))


def make_kv_gather(group, world: int, B: int, S_loc: int, T: int):
    """Returns f(qkv[M_loc, 3072]) -> (K view, V view, Lk) over all ranks' tokens, scene-major."""
    M_loc = B * S_loc * T

    def gather(qkv: torch.Tensor):
        dev, dt = qkv.device, qkv.dtype
        ev = _trace_begin()
        send = qkv[:, 1024:].contiguous()                                  # [M_loc, 2048]  (K | V)
        recv = torch.empty((world, M_loc, 2048), dtype=dt, device=dev)
        dist.all_gather_into_tensor(recv.view(world * M_loc, 2048), send, group=group)
        if B > 1:  # rows arrive (rank, scene, view, token); attention wants (scene, rank, view, token)
            recv = recv.view(world, B, S_loc * T, 2048).transpose(0, 1).contiguous()
        _trace_end(ev, "nccl_all_gather_kv", (world + 1) * M_loc * 2048 * 2.0)
        kv = recv.view(world * M_loc, 2048)
        return kv[:, :1024], kv[:, 1024:], world * S_loc * T

    return gather


class FusedKVGather:
    """The same gather WITHOUT a collective on the data path (default when torch symmetric memory is available;
    IGGT_FUSED_GATHER=0 selects the NCCL all-gather): every rank owns a symmetric buffer [2 parities, B, S*T, 2048]
    (the buffers of all ranks are mapped into every process over NVLink / NVSwitch), and the qkv GEMM of a global block
    stores the K | V chunks of each finished tile straight into ALL ranks' buffers through per-rank tensor maps
    (csrc/gemm.cuh, gather_maps; TMA stores to peer memory) - the transfer rides under the GEMM tile by tile instead of a
    staging copy + NCCL all-gather afterwards, and the rows land in (scene, rank, view, token) order, i.e. already in the
    layout the attention kernel reads.  What is left between GEMM and attention is a barrier on the symmetric-memory
    signal pads (capturable in the CUDA graph).  Two parities: block l+2 may only overwrite parity p once every rank has
    finished reading block l's keys, which the barrier of block l+1 guarantees."""

    def __init__(self, group, world: int, rank: int, B: int, S_loc: int, T: int, dtype, device):
        import torch.distributed._symmetric_memory as symm_mem
        self.group, self.world, self.B = group, world, B
        self.M_loc = S_loc * T                        # this rank's rows per scene
        self.Lk = world * self.M_loc                  # keys per scene
        shape = (2, B, self.Lk, 2048)
        self.buf = symm_mem.empty(shape, dtype=dtype, device=device)
        self.hdl = symm_mem.rendezvous(self.buf, group)
        self.maps = []
        for parity in range(2):
            windows = []
            for r in range(world):
                peer = self.hdl.get_buffer(r, shape, dtype)
                windows.append(peer[parity, 0, rank * self.M_loc:])          # first row of this rank's window
            self.maps.append(ops.kv_gather_maps(windows, self.M_loc, 2048, 2048, B, self.Lk * 2048, dtype, device))
        self.parity = 0

    def gemm_args(self):
        return {"gather_maps": self.maps[self.parity], "n_gather": self.world, "gather_rows": self.M_loc}

    def __call__(self, qkv: torch.Tensor):
        ev = _trace_begin()
        self.hdl.barrier(channel=self.parity)        # every rank's tiles have landed in every buffer
        _trace_end(ev, "symm_barrier_kv", 0.0)
        kv = self.buf[self.parity].view(self.B * self.Lk, 2048)
        self.parity ^= 1
        return kv[:, :1024], kv[:, 1024:], self.Lk


_FUSED = {}
_FUSED_FAILED = []


def make_fused_kv_gather(group, world: int, rank: int, B: int, S_loc: int, T: int, dtype, device):
    """FusedKVGather when it applies (symmetric memory available, not disabled with IGGT_FUSED_GATHER=0), else None -
    the caller then uses the NCCL all-gather."""
    import os
    import warnings
    if os.environ.get("IGGT_FUSED_GATHER", "1") == "0" or world < 2 or _FUSED_FAILED or not torch.cuda.is_available():
        return None
    key = (id(group), world, rank, B, S_loc, T, dtype, str(device))
    if key not in _FUSED:
        try:
            _FUSED[key] = FusedKVGather(group, world, rank, B, S_loc, T, dtype, device)
        except Exception as e:     # no symmetric memory on this system / build: keep the collective
            _FUSED_FAILED.append(repr(e))
            warnings.warn(f"fused K|V gather unavailable ({e!r}); using the NCCL all-gather")
            return None
    g = _FUSED[key]
    g.parity = 0
    return g


def gather_camera_tokens(tokens23: torch.Tensor, group, world: int) -> torch.Tensor:
    """tokens23 [B, S_loc, T, 2048] (local) -> camera tokens [B, S, 2048] of all views."""
    cam = tokens23[:, :, 0].contiguous()                                   # [B, S_loc, 2048]
    if world == 1:
        return cam
    B, S_loc, C = cam.shape
    ev = _trace_begin()
    recv = torch.empty((world, B, S_loc, C), dtype=cam.dtype, device=cam.device)
    dist.all_gather_into_tensor(recv.view(-1), cam.view(-1), group=group)
    _trace_end(ev, "nccl_all_gather_camera_tokens", (world + 1) * cam.numel() * 4.0)
    return recv.permute(1, 0, 2, 3).reshape(B, world * S_loc, C).contiguous()


def camera_poses(model, tokens, cam: torch.Tensor, rank: int, world: int, group, hd, iters: int = 4):
    """Camera head of the view-sharded forward.  `cam` [B, S, 2048]: the gathered camera tokens.  The head only couples the
    views of ONE scene (reference iggt/heads/camera_head.py:114-121: attention over S), so with B >= 2 scenes every rank
    refines ceil(B / world) of them and the poses (iters x B x S x 9 floats) are all-gathered - instead of every rank
    streaming the head's 216 M parameters once per group of scenes.  B = 1 (and IGGT_CAMERA_BY_SCENE=0): replicated."""
    import os
    B, S, _ = cam.shape
    if world == 1 or B < 2 or os.environ.get("IGGT_CAMERA_BY_SCENE", "1") == "0":
        return model.camera_head(tokens, num_iterations=iters, compute_dtype=hd, camera_tokens=cam)
    q = -(-B // world)                                                     # scenes per rank (the last ranks may own none)
    b0, b1 = min(rank * q, B), min((rank + 1) * q, B)
    mine = torch.zeros((iters, q, S, 9), dtype=torch.float32, device=cam.device)
    if b1 > b0:
        poses = model.camera_head(tokens, num_iterations=iters, compute_dtype=hd, camera_tokens=cam[b0:b1].contiguous())
        mine[:, :b1 - b0] = torch.stack(poses)
    ev = _trace_begin()
    allp = torch.empty((world,) + tuple(mine.shape), dtype=torch.float32, device=cam.device)
    dist.all_gather_into_tensor(allp.view(-1), mine.view(-1), group=group)
    _trace_end(ev, "nccl_all_gather_poses", (world + 1) * mine.numel() * 4.0)
    full = allp.permute(1, 0, 2, 3, 4).reshape(iters, world * q, S, 9)[:, :B]
    return [full[i].contiguous() for i in range(iters)]


def shard_views(model, group=None):
    """Configure `model` (IGGT / VGGT) for view-sharded execution over `group` (default: WORLD)."""
    if not dist.is_initialized():
        raise RuntimeError("torch.distributed is not initialised")
    group = group if group is not None else dist.group.WORLD
    model.aggregator.process_group = group
    model._shard_group = group
    return model


def _check_equal_shards(model, shape, group, world):
    """`all_gather_into_tensor` needs the same [B, S_loc, 3, H, W] on every rank; verify it once per shape (a host-side
    object all-gather, outside any CUDA-graph capture) and fail with a description instead of a hang / garbage."""
    seen = model.__dict__.setdefault("_shard_shapes_ok", set())
    if world <= 1 or shape in seen or (torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()):
        return
    shapes = [None] * world
    dist.all_gather_object(shapes, shape, group=group)
    if any(s != shape for s in shapes):
        raise ValueError(f"view sharding needs the same number of views and the same image size on every rank, got {shapes}")
    seen.add(shape)


@torch.no_grad()
def forward_sharded(model, images_local: torch.Tensor, rank: int, world: int, group=None):
    """images_local [B, S_loc, 3, H, W]: this rank's views.  Returns the prediction dict for the local
    views (pose_enc covers all S views, identical on every rank)."""
    group = group if group is not None else dist.group.WORLD
    model.aggregator.process_group = group if world > 1 else None
    if images_local.dim() == 4:
        images_local = images_local.unsqueeze(0)
    B, S_loc = images_local.shape[:2]
    _check_equal_shards(model, tuple(images_local.shape), group, world)
    dt, hd = model._dtype(), model._head_dtype()
    tokens, psi = model.aggregator(images_local, compute_dtype=dt, view_offset=rank * S_loc,
                                   total_views=world * S_loc)
    cam = gather_camera_tokens(tokens[23], group, world)
    pred = {"pose_enc": camera_poses(model, tokens, cam, rank, world, group, hd)}
    d, dc = model.depth_head(tokens, images=images_local, patch_start_idx=psi, compute_dtype=hd)
    out = model.point_head(tokens, images=images_local, patch_start_idx=psi, compute_dtype=hd)
    pred["depth"], pred["depth_conf"] = d, dc
    pred["world_points"], pred["world_points_conf"] = out[0], out[1]
    if getattr(model, "_with_part", False) and getattr(model, "part_enabled", True):
        maps = model.part_adaptor(tokens, images=images_local, patch_start_idx=psi, compute_dtype=hd)
        pred["part_feat"] = model.part_head(maps, point_feature=out[2], images=images_local, patch_start_idx=psi,
                                            compute_dtype=hd)
    pred["images"] = images_local
    return model._check(pred)
