"""Hopper-native track head (SURVEY.md 8f row 4): the `query_points` branch of `IGGT.forward` / `VGGT.forward`.

Interface of the reference `iggt.heads.track_head.TrackHead.forward(aggregated_tokens_list, images, patch_start_idx,
query_points, iters)` (iggt/heads/track_head.py:73-109) -> (list of per-iteration tracks [B,S,N,2] in image pixels,
visibility [B,S,N], confidence [B,S,N]).

* Feature extractor = the DPT pyramid / fusion kernels of `dpt_head.py` in the tracker configuration (128 features, no
  positional embedding, output at half resolution; reference dpt_head.py:192-262 with for_tracker=True, down_ratio=2).
* Tracker = BaseTrackerPredictor (track_modules/base_track_predictor.py:85-209).  Rows of every per-track tensor are
  ordered (scene, track, frame), which is the layout the update transformer's time attention wants.  The correlation
  lookup never builds the correlation volume (`ops.corr_sample`); the update transformer (blocks.py:19-144) runs on the
  wgmma GEMM / attention kernels with its 48-wide heads zero-padded to 64 (padded q/k columns add nothing to the
  scores, padded v columns are dropped by the padded out_proj) and a fp32 token stream like the trunk.
The reference evaluates this head in fp32 / TF32; GEMM operands here are 16-bit with fp32 accumulation.
"""
import math
from typing import Dict, List

import torch

from .. import ops
from ..layout import Node
from .dpt_head import DPTHead, PATCH

STRIDE = 2                    # track_head.py:25 (and down_ratio of the feature extractor, :57)
C = 128                       # latent_dim
HID, HEADS, HD, HDP = 384, 8, 48, 64
VIRT = 64
TDIM = 3 * C + 4              # 388
KCORR, KIN, NFLOW = 576, 392, 136     # 567 / 388 / 130 padded to TMA-legal widths


def _f32(p, device):
    return p.detach().to(device, torch.float32).contiguous()


def _padk(w, k, dtype, device):
    """[N, K0] -> [N, k] 16-bit, zero padded along K."""
    out = torch.zeros((w.shape[0], k), dtype=dtype, device=device)
    out[:, :w.shape[1]] = w.detach().to(device)
    return out


def _pad_heads_rows(w, b, parts, dtype, device):
    """in_proj rows [parts*384, 384] (+ bias) -> [parts*512, 384]: every 48-wide head padded to 64 zero rows."""
    w = w.detach().to(device, torch.float32).view(parts, HEADS, HD, HID)
    wp = torch.zeros((parts, HEADS, HDP, HID), dtype=torch.float32, device=device)
    wp[:, :, :HD] = w
    bp = torch.zeros((parts, HEADS, HDP), dtype=torch.float32, device=device)
    bp[:, :, :HD] = b.detach().to(device, torch.float32).view(parts, HEADS, HD)
    return wp.view(parts * HEADS * HDP, HID).to(dtype).contiguous(), bp.view(-1).contiguous()


def _pad_heads_cols(w, dtype, device):
    """out_proj [384, 384] -> [384, 512]: columns of the padded head dims are zero."""
    w = w.detach().to(device, torch.float32).view(HID, HEADS, HD)
    wp = torch.zeros((HID, HEADS, HDP), dtype=torch.float32, device=device)
    wp[:, :, :HD] = w
    return wp.view(HID, HEADS * HDP).to(dtype).contiguous()


class TrackFeatureExtractor(DPTHead):
    """DPTHead(features=128, pos_embed=False, for_tracker=True, down_ratio=2): tokens -> NHWC [B*S, H/2, W/2, 128]."""
    pos_embed_enabled = False

    def __init__(self):
        super().__init__(output_dim=0, activation="none")

    @torch.no_grad()
    def forward(self, aggregated_tokens_list, images, patch_start_idx, frames_chunk_size=8, compute_dtype=None):
        B, S, _, H, W = images.shape
        dev = images.device
        dt = compute_dtype or (torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else torch.float16)
        pk = self._packed(dt, dev)
        gh, gw = H // PATCH, W // PATCH
        T = patch_start_idx + gh * gw
        NI = B * S
        hf, wf = int(gh * PATCH / STRIDE), int(gw * PATCH / STRIDE)
        out = torch.empty((NI, hf, wf, C), dtype=dt, device=dev)
        chunk = frames_chunk_size or NI
        for n0 in range(0, NI, chunk):
            n1 = min(n0 + chunk, NI)
            feats = self._pyramid(pk, aggregated_tokens_list, NI, n0, n1, gh, gw, T, W / H, dt, dev)
            o, _ = self._scratch(pk, feats)
            out[n0:n1].copy_(ops.upsample_bilinear(o, hf, wf))
        return out


class TrackHead(Node):
    def __init__(self, iters: int = 4):
        super().__init__()
        self.feature_extractor = TrackFeatureExtractor()
        self.tracker = Node()
        self.iters = iters
        self._pk = None
        self._pk_key = None
        self._tab: Dict = {}

    def invalidate(self):
        self._pk = None
        self._tab.clear()

    # ------------------------------------------------------------------ packing
    def _pack_block(self, pk, name, blk, dtype, device, cross):
        attn = blk.cross_attn if cross else blk.attn
        pk[name + "n1"] = (_f32(blk.norm1.weight, device), _f32(blk.norm1.bias, device))
        pk[name + "n2"] = (_f32(blk.norm2.weight, device), _f32(blk.norm2.bias, device))
        if cross:
            pk[name + "nc"] = (_f32(blk.norm_context.weight, device), _f32(blk.norm_context.bias, device))
            pk[name + "q"] = _pad_heads_rows(attn.in_proj_weight[:HID], attn.in_proj_bias[:HID], 1, dtype, device)
            pk[name + "kv"] = _pad_heads_rows(attn.in_proj_weight[HID:], attn.in_proj_bias[HID:], 2, dtype, device)
        else:
            pk[name + "qkv"] = _pad_heads_rows(attn.in_proj_weight, attn.in_proj_bias, 3, dtype, device)
        pk[name + "o"] = (_pad_heads_cols(attn.out_proj.weight, dtype, device), _f32(attn.out_proj.bias, device))
        pk[name + "fc1"] = (blk.mlp.fc1.weight.detach().to(device, dtype).contiguous(), _f32(blk.mlp.fc1.bias, device))
        pk[name + "fc2"] = (blk.mlp.fc2.weight.detach().to(device, dtype).contiguous(), _f32(blk.mlp.fc2.bias, device))

    def _packed(self, dtype, device):
        key = (dtype, str(device))
        if self._pk is not None and self._pk_key == key:
            return self._pk
        t = self.tracker
        pk = {}
        pk["fmap_norm"] = (_f32(t.fmap_norm.weight, device), _f32(t.fmap_norm.bias, device))
        pk["corr1"] = (_padk(t.corr_mlp.fc1.weight, KCORR, dtype, device), _f32(t.corr_mlp.fc1.bias, device))
        pk["corr2"] = (t.corr_mlp.fc2.weight.detach().to(device, dtype).contiguous(), _f32(t.corr_mlp.fc2.bias, device))
        pk["ref_tok"] = _f32(t.query_ref_token, device).view(2, TDIM).contiguous()
        u = t.updateformer
        pk["in_norm"] = (_f32(u.input_norm.weight, device), _f32(u.input_norm.bias, device))
        pk["in_proj"] = (_padk(u.input_transform.weight, KIN, dtype, device), _f32(u.input_transform.bias, device))
        pk["virt"] = _f32(u.virual_tracks, device).view(VIRT, HID).contiguous()
        pk["out_norm"] = (_f32(u.output_norm.weight, device), _f32(u.output_norm.bias, device))
        wf = torch.zeros((NFLOW, HID), dtype=dtype, device=device)
        wf[:C + 2] = u.flow_head.weight.detach().to(device)
        bf = torch.zeros(NFLOW, dtype=torch.float32, device=device)
        bf[:C + 2] = u.flow_head.bias.detach().to(device)
        pk["flow"] = (wf, bf)
        for i in range(6):
            self._pack_block(pk, f"t{i}.", u.time_blocks._modules[str(i)], dtype, device, False)
            self._pack_block(pk, f"sv{i}.", u.space_virtual_blocks._modules[str(i)], dtype, device, False)
            self._pack_block(pk, f"p2v{i}.", u.space_point2virtual_blocks._modules[str(i)], dtype, device, True)
            self._pack_block(pk, f"v2p{i}.", u.space_virtual2point_blocks._modules[str(i)], dtype, device, True)
        pk["ffeat_norm"] = (_f32(t.ffeat_norm.weight, device), _f32(t.ffeat_norm.bias, device))
        pk["ffeat"] = (t.ffeat_updater._modules["0"].weight.detach().to(device, dtype).contiguous(),
                       _f32(t.ffeat_updater._modules["0"].bias, device))
        wv = torch.zeros((8, C), dtype=dtype, device=device)
        wv[0] = t.vis_predictor._modules["0"].weight.detach().to(device)[0]
        wv[1] = t.conf_predictor._modules["0"].weight.detach().to(device)[0]
        bv = torch.zeros(8, dtype=torch.float32, device=device)
        bv[0] = t.vis_predictor._modules["0"].bias.detach().to(device)[0]
        bv[1] = t.conf_predictor._modules["0"].bias.detach().to(device)[0]
        pk["scores"] = (wv, bv)
        self._pk, self._pk_key = pk, key
        return pk

    def _sincos(self, n, device):
        """get_1d_sincos_pos_embed_from_grid(194, arange(n)) (track_modules/utils.py:66-88): [n, 194] fp32."""
        key = (n, str(device))
        if key not in self._tab:
            omega = torch.arange(TDIM // 4, dtype=torch.double, device=device) / (TDIM / 4.0)
            out = torch.arange(n, dtype=torch.double, device=device)[:, None] * (1.0 / 10000 ** omega)[None, :]
            self._tab[key] = torch.cat([torch.sin(out), torch.cos(out)], 1).float().contiguous()
        return self._tab[key]

    def _pos_embed(self, qp, HH, WW):
        """Bilinear sample (border padding) of the separable 2-D sin/cos table at the query points: the x half only
        depends on x, the y half only on y, so it is two 1-D interpolations.  qp [B,N,2] -> [B*N, 388]."""
        def lerp(tab, v, n):
            v = v.clamp(0, n - 1)
            i0 = v.floor()
            f = (v - i0)[..., None]
            i0 = i0.long()
            i1 = (i0 + 1).clamp(max=n - 1)
            return tab[i0] * (1 - f) + tab[i1] * f
        px = lerp(self._sincos(WW, qp.device), qp[..., 0], WW)
        py = lerp(self._sincos(HH, qp.device), qp[..., 1], HH)
        return torch.cat([px, py], -1).reshape(-1, TDIM).contiguous()

    # ------------------------------------------------------------------ update transformer
    @staticmethod
    def _mlp_tail(pk, name, xn32, dt):
        h16 = torch.empty(xn32.shape, dtype=dt, device=xn32.device)
        ops.layernorm_rows(xn32, *pk[name + "n2"], out16=h16)
        m = ops.gemm_store16(h16, *pk[name + "fc1"], act=1)
        ops.gemm_resid32(m, pk[name + "fc2"][0], xn32, bias=pk[name + "fc2"][1])
        return xn32

    def _attn_block(self, pk, name, x32, num_seq, L, dt):
        """AttnBlock (modules.py:136-178); its `x = self.norm1(x)` rebinding makes the NORMALISED input the residual."""
        xn32 = torch.empty_like(x32)
        xn16 = torch.empty(x32.shape, dtype=dt, device=x32.device)
        ops.layernorm_rows(x32, *pk[name + "n1"], out32=xn32, out16=xn16)
        qkv = ops.gemm_store16(xn16, *pk[name + "qkv"])
        W = HEADS * HDP
        a = ops.attention(qkv[:, :W], qkv[:, W:2 * W], qkv[:, 2 * W:], num_seq, L, L, HEADS, scale=1.0 / math.sqrt(HD))
        ops.gemm_resid32(a, pk[name + "o"][0], xn32, bias=pk[name + "o"][1])
        return self._mlp_tail(pk, name, xn32, dt)

    def _cross_block(self, pk, name, x32, ctx32, num_seq, Lq, Lk, dt):
        """CrossAttnBlock (modules.py:181-218), same residual convention."""
        xn32 = torch.empty_like(x32)
        xn16 = torch.empty(x32.shape, dtype=dt, device=x32.device)
        c16 = torch.empty(ctx32.shape, dtype=dt, device=x32.device)
        ops.layernorm_rows(x32, *pk[name + "n1"], out32=xn32, out16=xn16)
        ops.layernorm_rows(ctx32, *pk[name + "nc"], out16=c16)
        q = ops.gemm_store16(xn16, *pk[name + "q"])
        kv = ops.gemm_store16(c16, *pk[name + "kv"])
        W = HEADS * HDP
        a = ops.attention(q, kv[:, :W], kv[:, W:], num_seq, Lq, Lk, HEADS, scale=1.0 / math.sqrt(HD))
        ops.gemm_resid32(a, pk[name + "o"][0], xn32, bias=pk[name + "o"][1])
        return self._mlp_tail(pk, name, xn32, dt)

    def _update_former(self, pk, xin16, B, N, S, dt):
        """EfficientUpdateFormer.forward (blocks.py:101-144) on the already input-normalised rows [B*N*S, 392]."""
        tok = ops.gemm_store32(xin16, *pk["in_proj"])                                    # [B*N*S, 384], rows (b, n, s)
        NV = N + VIRT
        full = torch.cat([tok.view(B, N, S, HID), pk["virt"].view(1, VIRT, 1, HID).expand(B, VIRT, S, HID)], 1).contiguous()
        for i in range(6):
            full = self._attn_block(pk, f"t{i}.", full.view(B * NV * S, HID), B * NV, S, dt)
            sp = full.view(B, NV, S, HID).permute(0, 2, 1, 3)                              # (b, s, n')
            pt = sp[:, :, :N].reshape(B * S * N, HID)
            vt = sp[:, :, N:].reshape(B * S * VIRT, HID)
            vt = self._cross_block(pk, f"v2p{i}.", vt, pt, B * S, VIRT, N, dt)
            vt = self._attn_block(pk, f"sv{i}.", vt, B * S, VIRT, dt)
            pt = self._cross_block(pk, f"p2v{i}.", pt, vt, B * S, N, VIRT, dt)
            sp = torch.cat([pt.view(B, S, N, HID), vt.view(B, S, VIRT, HID)], 2)
            full = sp.permute(0, 2, 1, 3).contiguous()
        out = full.view(B, NV, S, HID)[:, :N].reshape(B * N * S, HID) + tok
        o16 = torch.empty(out.shape, dtype=dt, device=out.device)
        ops.layernorm_rows(out, *pk["out_norm"], out16=o16)
        return ops.gemm_store32(o16, *pk["flow"])                                        # [rows, 136] (130 valid)

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, aggregated_tokens_list: List[torch.Tensor], images: torch.Tensor, patch_start_idx: int,
                query_points: torch.Tensor = None, iters: int = None, compute_dtype=None, trace: list = None,
                teacher: list = None):
        B, S, _, H, W = images.shape
        dev = images.device
        dt = compute_dtype or (torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else torch.float16)
        iters = self.iters if iters is None else iters
        fmaps = self.feature_extractor(aggregated_tokens_list, images, patch_start_idx, compute_dtype=dt)
        return self.track(fmaps, query_points, B, S, iters, dt, trace, teacher)

    @torch.no_grad()
    def track(self, fmaps, query_points, B, S, iters, dt, trace=None, teacher=None):
        """fmaps NHWC [B*S, HH, WW, 128] 16-bit (un-normalised), query_points [B,N,2] image pixels.
        Test hooks (the refinement loop is numerically chaotic on synthetic weights, so parity is checked iteration by
        iteration): `trace` collects every iteration's transformer input / output, `teacher[i] = (coords [B,S,N,2] in
        feature pixels, track feats [B,S,N,128])` replaces the state at the start of iteration i."""
        pk = self._packed(dt, fmaps.device)
        HH, WW = fmaps.shape[1], fmaps.shape[2]
        if min(HH, WW) < 64:
            raise RuntimeError("the 7-level correlation pyramid needs feature maps of at least 64 x 64 "
                               "(the reference's avg_pool2d fails the same way, blocks.py:173)")
        N = query_points.shape[1]
        rows = B * N * S
        levels = [ops.layernorm16(fmaps, *pk["fmap_norm"], eps=1e-5)]
        for _ in range(6):
            levels.append(ops.avgpool2_nhwc(levels[-1]))
        qp = (query_points.to(fmaps.device, torch.float32) / float(STRIDE)).contiguous()
        coords0 = qp[:, :, None, :].expand(B, N, S, 2).contiguous()
        frame0 = levels[0].view(B, S, HH, WW, C)[:, 0].contiguous()
        tf = ops.sample_bilinear_nhwc(frame0, qp)[:, :, None, :].expand(B, N, S, C).reshape(rows, C).contiguous()
        pos = self._pos_embed(qp, HH, WW)
        coords = coords0.view(rows, 2).clone()
        preds = []
        for it in range(iters):
            if teacher is not None and teacher[it] is not None:
                coords = teacher[it][0].to(fmaps.device, torch.float32).permute(0, 2, 1, 3).reshape(rows, 2).contiguous()
                tf = teacher[it][1].to(fmaps.device, torch.float32).permute(0, 2, 1, 3).reshape(rows, C).contiguous()
            A = ops.corr_sample(levels, tf, coords, B, N, S, KCORR)
            h = ops.gemm_store16(A, *pk["corr1"], act=1)
            fcorr = ops.gemm_store32(h, *pk["corr2"])
            if trace is not None:
                xin, raw = ops.track_input(coords, fcorr, tf, pos, pk["ref_tok"], *pk["in_norm"], S, dt, KIN, want_raw=True)
            else:
                xin = ops.track_input(coords, fcorr, tf, pos, pk["ref_tok"], *pk["in_norm"], S, dt, KIN)
            delta = self._update_former(pk, xin, B, N, S, dt)
            if trace is not None:
                trace.append({"x_in": raw.view(B, N, S, TDIM).clone(), "delta": delta[:, :C + 2].reshape(B, N, S, C + 2).clone()})
            d16 = torch.empty((rows, C), dtype=dt, device=fmaps.device)
            ops.layernorm_rows(delta[:, 2:C + 2], *pk["ffeat_norm"], out16=d16)           # GroupNorm(1, C) on [rows, C]
            tf = tf + ops.gemm_store32(d16, *pk["ffeat"], act=1)
            coords = (coords + delta[:, :2]).view(B, N, S, 2)
            coords[:, :, 0] = coords0[:, :, 0]
            coords = coords.view(rows, 2).contiguous()
            preds.append((coords * float(STRIDE)).view(B, N, S, 2).permute(0, 2, 1, 3).contiguous())
        sc = torch.sigmoid(ops.gemm_store32(tf.to(dt), *pk["scores"])[:, :2]).view(B, N, S, 2).permute(3, 0, 2, 1)
        return preds, sc[0].contiguous(), sc[1].contiguous()
