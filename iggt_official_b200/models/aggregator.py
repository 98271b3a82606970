"""Hopper-native Aggregator: DINOv2 ViT-L/14-reg tokeniser + 24 x (frame, global) attention blocks.

Same interface as the reference `iggt.models.aggregator.Aggregator` (iggt/models/aggregator.py:186-275):
`forward(images[B,S,3,H,W]) -> (list of 24 [B,S,T,2C] fp32 tensors, patch_start_idx)`; only the layers the
heads read (4, 11, 17, 23) are materialised unless `keep_all_layers` is set (the others are None).

Every block is 7 launches of the C-ABI kernels (include/iggt_b200.h):
  LayerNorm -> qkv GEMM (+bias, q/k-LayerNorm(64), 2-D RoPE) -> flash attention -> proj GEMM (TMA reduce-add
  of gamma1 * (.) into the fp32 residual) -> LayerNorm -> fc1 GEMM (+bias, erf-GELU) -> fc2 GEMM (reduce-add).
The fp32 residual stream, fp32 LayerNorm statistics and 16-bit GEMM / attention operands are the reference's
own precision policy under `torch.amp.autocast` (demo.py:191-195).
"""
import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn.functional as F

from .. import ops
from ..layout import Node

KEEP_LAYERS = (4, 11, 17, 23)
PATCH = 14
NUM_REG = 4
NUM_SPECIAL = 1 + NUM_REG
HEADS = 16
KP = 640  # 3*14*14 = 588 im2col columns padded to a multiple of 64


class _BlockW:
    __slots__ = ("n1w", "n1b", "qkv_w", "qkv_b", "qn_w", "qn_b", "kn_w", "kn_b", "proj_w", "proj_b", "ls1",
                 "n2w", "n2b", "fc1_w", "fc1_b", "fc2_w", "fc2_b", "ls2")


def pack_block(blk, dtype, device, qk_norm) -> _BlockW:
    w = _BlockW()
    f32 = lambda p: p.detach().to(device=device, dtype=torch.float32).contiguous()
    h16 = lambda p: p.detach().to(device=device, dtype=dtype).contiguous()
    # autocast casts a Linear's bias to the 16-bit dtype like its other operands (pinned against real autocast by
    # tests/test_oracle_amp.py); the epilogues add it in fp32, so it is rounded once here
    b16 = lambda p: p.detach().to(device=device, dtype=dtype).to(torch.float32).contiguous()
    w.n1w, w.n1b = f32(blk.norm1.weight), f32(blk.norm1.bias)
    w.qkv_w, w.qkv_b = h16(blk.attn.qkv.weight), b16(blk.attn.qkv.bias)
    if qk_norm:
        w.qn_w, w.qn_b = f32(blk.attn.q_norm.weight), f32(blk.attn.q_norm.bias)
        w.kn_w, w.kn_b = f32(blk.attn.k_norm.weight), f32(blk.attn.k_norm.bias)
    else:
        w.qn_w = w.qn_b = w.kn_w = w.kn_b = None
    w.proj_w, w.proj_b = h16(blk.attn.proj.weight), b16(blk.attn.proj.bias)
    w.ls1 = f32(blk.ls1.gamma)
    w.n2w, w.n2b = f32(blk.norm2.weight), f32(blk.norm2.bias)
    w.fc1_w, w.fc1_b = h16(blk.mlp.fc1.weight), b16(blk.mlp.fc1.bias)
    w.fc2_w, w.fc2_b = h16(blk.mlp.fc2.weight), b16(blk.mlp.fc2.bias)
    w.ls2 = f32(blk.ls2.gamma)
    return w


def rope_tables(npos: int, device):
    """cos/sin [npos, 16] of the per-axis 32-wide RoPE, base 100 (iggt/layers/rope.py:103-112)."""
    exponents = torch.arange(0, 32, 2, device=device).float() / 32
    inv_freq = 1.0 / (100.0 ** exponents)
    ang = torch.einsum("i,j->ij", torch.arange(npos, device=device, dtype=torch.float32), inv_freq)
    return ang.cos().contiguous(), ang.sin().contiguous()


def token_positions(gh: int, gw: int, device) -> torch.Tensor:
    """(y, x) + 1 for patch tokens, (0, 0) for the 5 special tokens -> int32 [T, 2]
    (iggt/layers/rope.py:24-59, iggt/models/aggregator.py:236-245)."""
    yy, xx = torch.meshgrid(torch.arange(gh, device=device), torch.arange(gw, device=device), indexing="ij")
    p = torch.stack([yy.reshape(-1), xx.reshape(-1)], -1) + 1
    return torch.cat([torch.zeros(NUM_SPECIAL, 2, dtype=p.dtype, device=device), p], 0).int().contiguous()


def _require_cuda(images: torch.Tensor):
    """The product path has no CPU fallback.  (tests/test_model_wiring.py replaces this hook AND every launcher of
    `ops` with PyTorch statements to exercise the host-side graph on the CPU.)"""
    if not images.is_cuda:
        raise RuntimeError("iggt_official_b200 runs on CUDA (sm_90a) only; there is no CPU fallback")


class Aggregator(Node):
    def __init__(self):
        super().__init__()
        self.patch_start_idx = NUM_SPECIAL
        self.keep_all_layers = False
        self._pk = None
        self._pk_key = None
        self._pos_cache: Dict[Tuple, torch.Tensor] = {}
        # view sharding (set by parallel.shard_views): this rank owns views [view_offset, view_offset+S_loc)
        self.process_group = None

    # ------------------------------------------------------------------ packing
    def invalidate(self):
        self._pk = None
        self._pos_cache.clear()

    def _packed(self, dtype, device):
        key = (dtype, str(device))
        if self._pk is not None and self._pk_key == key:
            return self._pk
        pe = self.patch_embed
        pk = {}
        w = pe.patch_embed.proj.weight.detach().to(device).reshape(1024, 588)
        wp = torch.zeros(1024, KP, device=device, dtype=dtype)
        wp[:, :588] = w.to(dtype)
        pk["pe_w"] = wp
        pk["pe_b"] = pe.patch_embed.proj.bias.detach().to(device, dtype).to(torch.float32).contiguous()   # as above
        pk["cls"] = pe.cls_token.detach().to(device, torch.float32).reshape(-1).contiguous()
        pk["reg"] = pe.register_tokens.detach().to(device, torch.float32).reshape(NUM_REG, -1).contiguous()
        pk["dino_norm_w"] = pe.norm.weight.detach().to(device, torch.float32).contiguous()
        pk["dino_norm_b"] = pe.norm.bias.detach().to(device, torch.float32).contiguous()
        pk["dino"] = [pack_block(getattr(pe.blocks, str(i)), dtype, device, False) for i in range(24)]
        pk["frame"] = [pack_block(getattr(self.frame_blocks, str(i)), dtype, device, True) for i in range(24)]
        pk["global"] = [pack_block(getattr(self.global_blocks, str(i)), dtype, device, True) for i in range(24)]
        pk["cam"] = self.camera_token.detach().to(device, torch.float32).reshape(2, -1).contiguous()
        pk["regtok"] = self.register_token.detach().to(device, torch.float32).reshape(2, NUM_REG, -1).contiguous()
        self._pk, self._pk_key = pk, key
        return pk

    def _dino_pos(self, gh, gw, device):
        """DINOv2 learned pos-embed, bicubic(+antialias) resized when the grid is not the native square
        (iggt/layers/vision_transformer.py:183-215).  Cached per grid; not on the hot path."""
        key = (gh, gw, str(device))
        if key not in self._pos_cache:
            pe = self.patch_embed.pos_embed.detach().to(device, torch.float32)
            n = pe.shape[1] - 1
            m = int(math.sqrt(n))
            if not (gh * gw == n and gh == gw):
                patch = F.interpolate(pe[:, 1:].reshape(1, m, m, -1).permute(0, 3, 1, 2), size=(gh, gw),
                                      mode="bicubic", antialias=True)
                pe = torch.cat([pe[:, :1], patch.permute(0, 2, 3, 1).reshape(1, gh * gw, -1)], 1)
            self._pos_cache[key] = pe.reshape(1 + gh * gw, -1).contiguous()
        return self._pos_cache[key]

    # ------------------------------------------------------------------ one transformer block
    @staticmethod
    def _block(x, w: _BlockW, eps, num_seq, Lq, T, rope, kv_gather=None):
        M = x.shape[0]
        dt = w.qkv_w.dtype
        h = torch.empty((M, 1024), dtype=dt, device=x.device)
        ops.layernorm(x, w.n1w, w.n1b, eps, h)
        fused = kv_gather.gemm_args() if hasattr(kv_gather, "gemm_args") else {}   # K|V gather fused into this GEMM
        if rope is None:
            qkv = ops.gemm_qkv(h, w.qkv_w, w.qkv_b, 1024)
        else:
            qkv = ops.gemm_qkv(h, w.qkv_w, w.qkv_b, 1024, qk_norm=True, qn_w=w.qn_w, qn_b=w.qn_b, kn_w=w.kn_w,
                               kn_b=w.kn_b, rope_cos=rope[0], rope_sin=rope[1], pos_yx=rope[2], T=T, **fused)
        q = qkv[:, :1024]
        if kv_gather is None:
            k, v, Lk = qkv[:, 1024:2048], qkv[:, 2048:], Lq
        else:
            k, v, Lk = kv_gather(qkv)
        o = ops.attention(q, k, v, num_seq, Lq, Lk, HEADS)
        ops.gemm_resid32(o, w.proj_w, x, w.proj_b, w.ls1, round_out16=True)
        ops.layernorm(x, w.n2w, w.n2b, eps, h)
        f = ops.gemm_store16(h, w.fc1_w, w.fc1_b, act=1)
        ops.gemm_resid32(f, w.fc2_w, x, w.fc2_b, w.ls2, round_out16=True)

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, images: torch.Tensor, compute_dtype: Optional[torch.dtype] = None,
                view_offset: int = 0, total_views: Optional[int] = None):
        """images [B,S_loc,3,H,W] fp32 in [0,1] (CUDA).  With view sharding, S_loc views of every scene live
        on this rank, `view_offset` is the scene-index of the first one and `total_views` the scene size."""
        if images.dim() != 5:
            raise ValueError("expected images of shape [B, S, 3, H, W]")
        B, S, C_in, H, W = images.shape
        if C_in != 3:
            raise ValueError(f"Expected 3 input channels, got {C_in}")                 # aggregator.py:202-203
        assert H % PATCH == 0 and W % PATCH == 0, "Input image size must be a multiple of the patch size"
        _require_cuda(images)
        dt = compute_dtype or (torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else torch.float16)
        dev = images.device
        pk = self._packed(dt, dev)
        NI, gh, gw = B * S, H // PATCH, W // PATCH
        P = gh * gw
        T = NUM_SPECIAL + P
        M = NI * T
        img = images.reshape(NI, 3, H, W).float().contiguous()

        # --- DINOv2 tokeniser (vision_transformer.py:217-281)
        A = ops.patchify(img, KP, dt)
        pe16 = ops.gemm_store16(A, pk["pe_w"], pk["pe_b"])
        x = torch.empty((M, 1024), dtype=torch.float32, device=dev)
        ops.dino_assemble(pe16, pk["cls"], pk["reg"], self._dino_pos(gh, gw, dev), x, NI, P, NUM_REG, 1024)
        for i in range(24):
            self._block(x, pk["dino"][i], 1e-6, NI, T, T, None)
        y = torch.empty((M, 1024), dtype=torch.float32, device=dev)
        ops.layernorm(x, pk["dino_norm_w"], pk["dino_norm_b"], 1e-6, y, groups=NI, rows_out=P, rows_in=T,
                      in_off=NUM_SPECIAL, out_rows_per_group=T, out_off=NUM_SPECIAL)
        del x, A, pe16
        ops.special_tokens(pk["cam"], pk["regtok"], y, NI, T, NUM_REG, 1024, S, view_offset)

        # --- alternating attention (aggregator.py:254-270)
        cos, sin = rope_tables(max(gh, gw) + 1, dev)
        rope = (cos, sin, token_positions(gh, gw, dev))
        keep = range(24) if self.keep_all_layers else KEEP_LAYERS
        out: List[Optional[torch.Tensor]] = [None] * 24
        group = self.process_group
        world = dist.get_world_size(group) if group is not None else 1
        S_tot = total_views if total_views is not None else S * world
        gather = None
        if world > 1:
            from ..parallel import make_fused_kv_gather, make_kv_gather
            gather = make_fused_kv_gather(group, world, view_offset // S, B, S, T, dt, dev) or \
                make_kv_gather(group, world, B, S, T)
        for i in range(24):
            self._block(y, pk["frame"][i], 1e-5, NI, T, T, rope)
            if i in keep:
                out[i] = torch.empty((B, S, T, 2048), dtype=torch.float32, device=dev)
                out[i].view(M, 2048)[:, :1024].copy_(y)
            self._block(y, pk["global"][i], 1e-5, B, S * T, T, rope, kv_gather=gather)
            if i in keep:
                out[i].view(M, 2048)[:, 1024:].copy_(y)
        return out, self.patch_start_idx
