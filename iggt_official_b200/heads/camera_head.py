"""Hopper-native camera head: iterative pose refinement on the S camera tokens
(reference: iggt/heads/camera_head.py:83-154, iggt/heads/head_act.py:12-35).

M = B*S rows of width 2048 against 216 M parameters: every Linear is a weight stream (fp32 activations, 16-bit
weights, fp32 accumulate).  For B*S <= 16 the whole head - 4 iterations x (embed, AdaLN, 4 blocks, pose branch) - is ONE
persistent launch (`iggt_camera_head`, csrc/camera.cu: the producer warp streams weights across phase boundaries, a
device-wide barrier separates the ~27 phases of an iteration).  Scenes of more than 16 views and devices with fewer
than 128 SMs (an H100 PCIe, a MIG slice) run layer by layer: `iggt_skinny_gemm`, `iggt_small_attention`,
`iggt_layernorm`, with the AdaLN modulate in torch arithmetic.  Scenes with more views than `iggt_small_attention` holds
in shared memory (197 and up at head dim 128) take `iggt_token_attention`, which streams the keys, so the view count
is bounded by device memory only.
"""
import ctypes
from typing import List

import torch

from .. import _lib, ops
from ..layout import Node

DIM = 2048
HEADS = 16
FUSED_MIN_SMS = 128            # the one-launch kernel's grid holds every phase in <= 4 tiles per CTA only from 128 SMs

_sm_counts = {}


def _sm_count(device) -> int:
    """Multiprocessor count of `device` (iggt_device_info), read once per device."""
    idx = torch.device(device).index
    idx = torch.cuda.current_device() if idx is None else idx
    if idx not in _sm_counts:
        n = ctypes.c_int(0)
        with torch.cuda.device(idx):
            _lib.check(_lib.load().iggt_device_info(None, ctypes.byref(n)), "iggt_device_info")
        _sm_counts[idx] = n.value
    return _sm_counts[idx]


def _f32(p, device):
    return p.detach().to(device, torch.float32).contiguous()


class CameraHead(Node):
    def __init__(self):
        super().__init__()
        self._pk = None
        self._pk_key = None

    def invalidate(self):
        self._pk = None

    def _packed(self, dtype, device):
        key = (dtype, str(device))
        if self._pk is not None and self._pk_key == key:
            return self._pk
        h16 = lambda p: p.detach().to(device=device, dtype=dtype).contiguous()
        pk = {}
        for i in range(4):
            b = self.trunk._modules[str(i)]
            pk[f"t{i}"] = dict(
                n1w=_f32(b.norm1.weight, device), n1b=_f32(b.norm1.bias, device),
                qkv_w=h16(b.attn.qkv.weight), qkv_b=_f32(b.attn.qkv.bias, device),
                proj_w=h16(b.attn.proj.weight), proj_b=_f32(b.attn.proj.bias, device), ls1=_f32(b.ls1.gamma, device),
                n2w=_f32(b.norm2.weight, device), n2b=_f32(b.norm2.bias, device),
                fc1_w=h16(b.mlp.fc1.weight), fc1_b=_f32(b.mlp.fc1.bias, device),
                fc2_w=h16(b.mlp.fc2.weight), fc2_b=_f32(b.mlp.fc2.bias, device), ls2=_f32(b.ls2.gamma, device))
        pk["tok_w"], pk["tok_b"] = _f32(self.token_norm.weight, device), _f32(self.token_norm.bias, device)
        pk["trk_w"], pk["trk_b"] = _f32(self.trunk_norm.weight, device), _f32(self.trunk_norm.bias, device)
        ew = torch.zeros(DIM, 16, device=device, dtype=dtype)       # K = 9 padded to 16 for 16-byte rows
        ew[:, :9] = self.embed_pose.weight.detach().to(device, dtype)
        pk["emb_w"], pk["emb_b"] = ew, _f32(self.embed_pose.bias, device)
        mod = self.poseLN_modulation._modules["1"]
        pk["mod_w"], pk["mod_b"] = h16(mod.weight), _f32(mod.bias, device)
        pk["pb1_w"], pk["pb1_b"] = h16(self.pose_branch.fc1.weight), _f32(self.pose_branch.fc1.bias, device)
        pk["pb2_w"], pk["pb2_b"] = h16(self.pose_branch.fc2.weight), _f32(self.pose_branch.fc2.bias, device)
        pk["empty"] = _f32(self.empty_pose_tokens, device).reshape(1, 9)
        e16 = torch.zeros(16, dtype=torch.float32, device=device)
        e16[:9] = pk["empty"].view(-1)
        pk["empty16"] = e16
        pk["cstruct"] = self._cstruct(pk)
        self._pk, self._pk_key = pk, key
        return pk

    @staticmethod
    def _cstruct(pk):
        """iggt_camera_weights for the one-launch kernel: raw pointers into the packed tensors (kept alive by `pk`)."""
        w = _lib.CameraWeights()
        P = lambda t: ctypes.c_void_p(t.data_ptr())
        w.emb_w, w.emb_b, w.mod_w, w.mod_b = P(pk["emb_w"]), P(pk["emb_b"]), P(pk["mod_w"]), P(pk["mod_b"])
        for i in range(4):
            t = pk[f"t{i}"]
            for name in ("n1w", "n1b", "qkv_w", "qkv_b", "proj_w", "proj_b", "ls1", "n2w", "n2b", "fc1_w", "fc1_b", "fc2_w",
                         "fc2_b", "ls2"):
                setattr(w.blk[i], name, P(t[name]))
        w.tok_w, w.tok_b, w.trk_w, w.trk_b = P(pk["tok_w"]), P(pk["tok_b"]), P(pk["trk_w"]), P(pk["trk_b"])
        w.pb1_w, w.pb1_b, w.pb2_w, w.pb2_b = P(pk["pb1_w"]), P(pk["pb1_b"]), P(pk["pb2_w"]), P(pk["pb2_b"])
        w.empty = P(pk["empty16"])
        return w

    @staticmethod
    def _rows(fn, x, *a, **k):
        """skinny GEMM handles <= 32 rows per launch; larger B*S go in row chunks."""
        if x.shape[0] <= 32:
            return fn(x, *a, **k)
        outs = []
        for r in range(0, x.shape[0], 32):
            kk = dict(k)
            if kk.get("resid") is not None:
                kk["resid"] = kk["resid"][r:r + 32]
            outs.append(fn(x[r:r + 32], *a, **kk))
        return torch.cat(outs, 0)

    def _block(self, x, w, B, S):
        M = x.shape[0]
        h = torch.empty_like(x)
        ops.layernorm(x, w["n1w"], w["n1b"], 1e-5, h)
        qkv = self._rows(ops.skinny_gemm, h, w["qkv_w"], w["qkv_b"])
        # scenes with more views than small_attention holds in shared memory stream their keys (token_attention)
        attend = ops.small_attention if ops._small_attention_fits(S, DIM // HEADS) else ops.token_attention
        o = attend(qkv, B, S, HEADS, DIM // HEADS)
        x = self._rows(ops.skinny_gemm, o, w["proj_w"], w["proj_b"], gamma=w["ls1"], resid=x)
        ops.layernorm(x, w["n2w"], w["n2b"], 1e-5, h)
        f = self._rows(ops.skinny_gemm, h, w["fc1_w"], w["fc1_b"], act=1)
        return self._rows(ops.skinny_gemm, f, w["fc2_w"], w["fc2_b"], gamma=w["ls2"], resid=x)

    @torch.no_grad()
    def forward(self, aggregated_tokens_list: List[torch.Tensor], num_iterations: int = 4, compute_dtype=None,
                camera_tokens: torch.Tensor = None) -> List[torch.Tensor]:
        """`camera_tokens` [B,S,2048] (already gathered over ranks) overrides tokens_list[-1][:, :, 0]."""
        if camera_tokens is None:
            tok = aggregated_tokens_list[-1]
            camera_tokens = tok[:, :, 0]
        B, S, C = camera_tokens.shape
        dev = camera_tokens.device
        dt = compute_dtype or (torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else torch.float16)
        pk = self._packed(dt, dev)
        M = B * S
        if S <= 16 and camera_tokens.is_cuda and _sm_count(dev) >= FUSED_MIN_SMS:
            rows = camera_tokens.reshape(M, C)                    # a strided view of tokens[:, :, 0]: no copy
            if rows.dtype != torch.float32 or rows.stride(1) != 1:
                rows = rows.float().contiguous()
            if M <= 16:
                poses = ops.camera_head(pk["cstruct"], pk, rows, B, S, num_iterations, dt)
            else:
                # scenes only meet in nothing here (the token attention is per scene): one launch per group of scenes
                # that fits the kernel's 16 rows - the weights are re-streamed per group (1.4 ms each), still well under
                # the ~180 launches of the layer-by-layer path
                per = max(1, 16 // S)
                poses = torch.cat([ops.camera_head(pk["cstruct"], pk, rows[b0 * S:(b0 + per) * S], min(per, B - b0), S,
                                                   num_iterations, dt) for b0 in range(0, B, per)], 1)
            return [poses[i].view(B, S, 9) for i in range(num_iterations)]
        return self._layers(camera_tokens, pk, num_iterations)

    def _layers(self, camera_tokens, pk, num_iterations):
        """The head layer by layer on camera_tokens [B,S,2048] with the packed weights `pk` of `_packed`."""
        B, S, C = camera_tokens.shape
        M = B * S
        dev = camera_tokens.device
        raw = camera_tokens.reshape(M, C).float().contiguous()
        pt = torch.empty_like(raw)
        ops.layernorm(raw, pk["tok_w"], pk["tok_b"], 1e-5, pt)
        ptn = torch.empty_like(raw)
        ops.layernorm(pt, None, None, 1e-6, ptn)                      # adaln_norm (no affine, eps 1e-6)
        pred = None
        outs = []
        for _ in range(num_iterations):
            inp = torch.zeros((M, 16), dtype=torch.float32, device=dev)
            inp[:, :9] = pk["empty"] if pred is None else pred
            e = self._rows(ops.skinny_gemm, inp, pk["emb_w"], pk["emb_b"], act=4)          # SiLU(embed_pose(.))
            mod = self._rows(ops.skinny_gemm, e, pk["mod_w"], pk["mod_b"])
            shift, scale, gate = mod[:, :DIM], mod[:, DIM:2 * DIM], mod[:, 2 * DIM:]
            x = (gate * (ptn * (1 + scale) + shift) + pt).contiguous()
            for i in range(4):
                x = self._block(x, pk[f"t{i}"], B, S)
            xn = torch.empty_like(x)
            ops.layernorm(x, pk["trk_w"], pk["trk_b"], 1e-5, xn)
            hdn = self._rows(ops.skinny_gemm, xn, pk["pb1_w"], pk["pb1_b"], act=1)
            d = self._rows(ops.skinny_gemm, hdn, pk["pb2_w"], pk["pb2_b"])
            pred = d if pred is None else pred + d
            outs.append(torch.cat([pred[:, :7], torch.relu(pred[:, 7:])], -1).view(B, S, 9))
        return outs
