"""Hopper-native DPT dense head (depth / 3-D points, and the feature pyramid the part head consumes).

Interface of the reference `iggt.heads.dpt_head.DPTHead.forward(aggregated_tokens_list, images,
patch_start_idx, frames_chunk_size)` (iggt/heads/dpt_head.py:130-190); returns (preds, conf) or, with
`use_point_feat`, (preds, conf, (out2, out3, out4)) where the feature maps are NHWC 16-bit tensors.

All activations are NHWC 16-bit; every convolution runs on the wgmma implicit-GEMM kernel
(`iggt_conv_nhwc` / `iggt_gemm_store16`) with fp32 accumulation.  Fusions relative to the reference graph:
  * ResidualConvUnit's in-place ReLU (SURVEY F10): producers emit relu(x) directly (act / act_post flags),
    the skip-adds ride in the conv epilogue (resid, resid2);
  * FeatureFusionBlock's 1x1 `out_conv` commutes with the bilinear upsample (bilinear weights sum to 1), so
    it runs at the low resolution (4x fewer pixels); rounding differs at the 1e-7 level (SURVEY E-19);
  * ConvTranspose(k == stride) = GEMM + pixel shuffle; the stride-2 conv = im2col + GEMM;
  * final upsample + pos-embed in one pass; 1x1 (32 -> out) + exp / inverse-log / 1+exp in one pass.
The reference runs these heads in fp32 / TF32 (iggt/models/vggt.py:189); 16-bit operands with fp32 accumulate
have the same 10-bit mantissa as TF32 when the compute dtype is fp16.
"""
import os
from typing import Dict, List, Tuple

import torch

from .. import ops
from ..layout import Node

PATCH = 14
LAYERS = (4, 11, 17, 23)
FUSED_TAIL = os.environ.get("IGGT_FUSED_TAIL", "1") != "0"


def uv_pos_tables(gh: int, gw: int, ch: int, aspect: float, device) -> Tuple[torch.Tensor, torch.Tensor]:
    """Split form of `_apply_pos_embed` (iggt/heads/dpt_head.py:274-284, iggt/heads/utils.py:11-108):
    embedding[y, x] = 0.1 * [sin(u w) | cos(u w) | sin(v w) | cos(v w)], each ch/4 wide, w_k = 100^(-k/(ch/4))
    evaluated in float64 -> tabx [gw, ch/2] (depends on x only), taby [gh, ch/2]."""
    dg = (aspect ** 2 + 1.0) ** 0.5
    sx, sy = aspect / dg, 1.0 / dg
    xs = torch.linspace(-sx * (gw - 1) / gw, sx * (gw - 1) / gw, gw, dtype=torch.float32, device=device)
    ys = torch.linspace(-sy * (gh - 1) / gh, sy * (gh - 1) / gh, gh, dtype=torch.float32, device=device)
    q = ch // 4
    omega = torch.arange(q, dtype=torch.double, device=device) / q
    omega = 1.0 / 100 ** omega

    def emb(p):
        o = p.double()[:, None] * omega[None, :]
        return (torch.cat([torch.sin(o), torch.cos(o)], 1).float() * 0.1).contiguous()

    return emb(xs), emb(ys)


def pack_conv3x3(w, dtype, device):
    """[Cout, Cin, 3, 3] -> [Cout, 9*Cin] tap-major (k = (ky*3+kx)*Cin + ci)."""
    return w.detach().to(device).permute(0, 2, 3, 1).reshape(w.shape[0], -1).to(dtype).contiguous()


def pack_deconv(w, b, dtype, device):
    """ConvTranspose2d weight [Cin, Cout, k, k] -> GEMM B [(dy*k+dx)*Cout + co, Cin]; bias tiled k*k times."""
    k = w.shape[2]
    wp = w.detach().to(device).permute(2, 3, 1, 0).reshape(k * k * w.shape[1], w.shape[0]).to(dtype).contiguous()
    return wp, b.detach().to(device, torch.float32).repeat(k * k).contiguous()


def dense_tail(up, pk, mode):
    """`output_conv2` + head activation on the full-resolution 128-channel map: one launch of the tall-box kernel
    (csrc/tailconv.cu; the 32-channel map stays in fp32 registers).  IGGT_FUSED_TAIL=0 selects the two-launch form
    (generic implicit-GEMM conv -> 16-bit map -> per-pixel tail) for A/B checks."""
    if FUSED_TAIL and up.shape[3] == 128 and pk["oc2a.w"].shape[0] == 32:
        return ops.dpt_tail_fused(up, pk["oc2a.w"], pk["oc2a.b"], pk["oc2b.w"], pk["oc2b.b"], mode)
    z = ops.conv_nhwc(up, pk["oc2a.w"], pk["oc2a.b"], act=2)
    return ops.dpt_tail(z, pk["oc2b.w"], pk["oc2b.b"], mode)


def _f32(p, device):
    return p.detach().to(device, torch.float32).contiguous()


class DPTHead(Node):
    def __init__(self, output_dim: int, activation: str, use_point_feat: bool = False):
        super().__init__()
        self.output_dim = output_dim
        self.activation = activation
        self.use_point_feat = use_point_feat
        self._pk = None
        self._pk_key = None
        self._pe_cache: Dict = {}

    def invalidate(self):
        self._pk = None
        self._pe_cache.clear()

    # ------------------------------------------------------------------ packing
    def _pack_scratch(self, pk, dtype, device):
        s = self.scratch
        for i in range(1, 5):
            pk[f"rn{i}"] = pack_conv3x3(getattr(s, f"layer{i}_rn").weight, dtype, device)
            rn = getattr(s, f"refinenet{i}")
            for u in ("resConfUnit1", "resConfUnit2"):
                if u in rn._modules:
                    unit = rn._modules[u]
                    for c in ("conv1", "conv2"):
                        pk[f"r{i}.{u}.{c}.w"] = pack_conv3x3(unit._modules[c].weight, dtype, device)
                        pk[f"r{i}.{u}.{c}.b"] = _f32(unit._modules[c].bias, device)
            pk[f"r{i}.out.w"] = rn.out_conv.weight.detach().to(device).reshape(rn.out_conv.weight.shape[0], -1).to(dtype).contiguous()
            pk[f"r{i}.out.b"] = _f32(rn.out_conv.bias, device)
        pk["oc1.w"] = pack_conv3x3(s.output_conv1.weight, dtype, device)
        pk["oc1.b"] = _f32(s.output_conv1.bias, device)
        if "output_conv2" not in s._modules:          # tracker feature extractor (for_tracker=True): features only
            return
        oc2 = s.output_conv2
        pk["oc2a.w"] = pack_conv3x3(oc2._modules["0"].weight, dtype, device)
        pk["oc2a.b"] = _f32(oc2._modules["0"].bias, device)
        pk["oc2b.w"] = _f32(oc2._modules["2"].weight, device).reshape(oc2._modules["2"].weight.shape[0], -1).contiguous()
        pk["oc2b.b"] = _f32(oc2._modules["2"].bias, device)

    def _packed(self, dtype, device):
        key = (dtype, str(device))
        if self._pk is not None and self._pk_key == key:
            return self._pk
        pk = {"norm_w": _f32(self.norm.weight, device), "norm_b": _f32(self.norm.bias, device)}
        for i in range(4):
            pr = self.projects._modules[str(i)]
            pk[f"proj{i}.w"] = pr.weight.detach().to(device).reshape(pr.weight.shape[0], -1).to(dtype).contiguous()
            pk[f"proj{i}.b"] = _f32(pr.bias, device)
        r = self.resize_layers._modules
        pk["rs0.w"], pk["rs0.b"] = pack_deconv(r["0"].weight, r["0"].bias, dtype, device)
        pk["rs1.w"], pk["rs1.b"] = pack_deconv(r["1"].weight, r["1"].bias, dtype, device)
        pk["rs3.w"] = pack_conv3x3(r["3"].weight, dtype, device)
        pk["rs3.b"] = _f32(r["3"].bias, device)
        self._pack_scratch(pk, dtype, device)
        self._pk, self._pk_key = pk, key
        return pk

    def _pe(self, gh, gw, ch, aspect, device, dtype, full: bool):
        """full=True: [gh*gw, ch] 16-bit addend for the GEMM epilogue; else the split fp32 tables."""
        key = (gh, gw, ch, aspect, str(device), dtype, full)
        if key not in self._pe_cache:
            tx, ty = uv_pos_tables(gh, gw, ch, aspect, device)
            if full:
                e = torch.cat([tx[None].expand(gh, gw, ch // 2), ty[:, None].expand(gh, gw, ch // 2)], -1)
                self._pe_cache[key] = e.reshape(gh * gw, ch).to(dtype).contiguous()
            else:
                self._pe_cache[key] = (tx, ty)
        return self._pe_cache[key]

    # ------------------------------------------------------------------ building blocks
    @staticmethod
    def _rcu_tail(pk, i, s):
        """RCU2 + out_conv of FeatureFusionBlock i on the (already relu'd) sum s -> low-res projected map."""
        t = ops.conv_nhwc(s, pk[f"r{i}.resConfUnit2.conv1.w"], pk[f"r{i}.resConfUnit2.conv1.b"], act=2)
        o = ops.conv_nhwc(t, pk[f"r{i}.resConfUnit2.conv2.w"], pk[f"r{i}.resConfUnit2.conv2.b"], resid=s)
        NB, h, w, C = o.shape
        p = ops.gemm_store16(o.view(NB * h * w, C), pk[f"r{i}.out.w"], pk[f"r{i}.out.b"])
        return p.view(NB, h, w, -1)

    @staticmethod
    def _fuse(pk, i, x0, a):
        """relu(x0 + RCU1(a)) with a = relu(layer_rn output): both skip-adds and the ReLU in one epilogue."""
        t = ops.conv_nhwc(a, pk[f"r{i}.resConfUnit1.conv1.w"], pk[f"r{i}.resConfUnit1.conv1.b"], act=2)
        return ops.conv_nhwc(t, pk[f"r{i}.resConfUnit1.conv2.w"], pk[f"r{i}.resConfUnit1.conv2.b"], resid=a,
                             resid2=x0, act_post=2)

    def _pyramid(self, pk, tokens_list, NI, n0, n1, gh, gw, T, aspect, dt, dev):
        """LN -> 1x1 proj (+pos-embed) -> resize, for views [n0, n1): four NHWC maps at 4g, 2g, g, ceil(g/2)."""
        nb = n1 - n0
        P = gh * gw
        feats = []
        for li, layer in enumerate(LAYERS):
            tok = tokens_list[layer]
            if tok is None:
                raise RuntimeError(f"aggregated_tokens_list[{layer}] was not materialised")
            tok2 = tok.reshape(-1, tok.shape[-1])[n0 * T:n1 * T]
            xn = torch.empty((nb * P, tok.shape[-1]), dtype=dt, device=dev)
            ops.layernorm(tok2, pk["norm_w"], pk["norm_b"], 1e-5, xn, groups=nb, rows_out=P, rows_in=T,
                          in_off=T - P, out_rows_per_group=P, out_off=0)
            oc = pk[f"proj{li}.w"].shape[0]
            add = self._pe(gh, gw, oc, aspect, dev, dt, True) if self.pos_embed_enabled else None
            x = ops.gemm_store16(xn, pk[f"proj{li}.w"], pk[f"proj{li}.b"], addend=add, add_rows=P)
            if li == 0:
                y = ops.gemm_store16(x, pk["rs0.w"], pk["rs0.b"])
                x = ops.deconv_shuffle(y, nb, gh, gw, oc, 4)
            elif li == 1:
                y = ops.gemm_store16(x, pk["rs1.w"], pk["rs1.b"])
                x = ops.deconv_shuffle(y, nb, gh, gw, oc, 2)
            elif li == 2:
                x = x.view(nb, gh, gw, oc)
            else:
                A, ho, wo = ops.im2col3x3_s2(x.view(nb, gh, gw, oc))
                x = ops.gemm_store16(A, pk["rs3.w"], pk["rs3.b"]).view(nb, ho, wo, -1)
            feats.append(x)
        return feats

    pos_embed_enabled = True

    def _scratch(self, pk, feats):
        """scratch_forward (iggt/heads/dpt_head.py:286-316) -> (out1 at 8g after output_conv1, (out2,out3,out4))."""
        l = [ops.conv_nhwc(f, pk[f"rn{i + 1}"], None, act=2) for i, f in enumerate(feats)]  # relu(layer_rn(.))
        p4 = self._rcu_tail(pk, 4, l[3])
        out4 = ops.upsample_bilinear(p4, l[2].shape[1], l[2].shape[2])
        p3 = self._rcu_tail(pk, 3, self._fuse(pk, 3, out4, l[2]))
        out3 = ops.upsample_bilinear(p3, l[1].shape[1], l[1].shape[2])
        p2 = self._rcu_tail(pk, 2, self._fuse(pk, 2, out3, l[1]))
        out2 = ops.upsample_bilinear(p2, l[0].shape[1], l[0].shape[2])
        p1 = self._rcu_tail(pk, 1, self._fuse(pk, 1, out2, l[0]))
        out1 = ops.upsample_bilinear(p1, 2 * p1.shape[1], 2 * p1.shape[2])
        o = ops.conv_nhwc(out1, pk["oc1.w"], pk["oc1.b"])
        return o, (out2, out3, out4)

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, aggregated_tokens_list: List[torch.Tensor], images: torch.Tensor, patch_start_idx: int,
                frames_chunk_size: int = 8, compute_dtype=None):
        B, S, _, H, W = images.shape
        dev = images.device
        dt = compute_dtype or (torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else torch.float16)
        pk = self._packed(dt, dev)
        gh, gw = H // PATCH, W // PATCH
        T = patch_start_idx + gh * gw
        NI = B * S
        aspect = W / H
        oc = self.output_dim
        mode = 0 if self.activation == "exp" else 1
        preds = torch.empty((NI, H, W, oc - 1), dtype=torch.float32, device=dev)
        conf = torch.empty((NI, H, W), dtype=torch.float32, device=dev)
        f2, f3, f4 = [], [], []
        chunk = frames_chunk_size or NI
        tx, ty = self._pe(gh * PATCH, gw * PATCH, 128, aspect, dev, dt, False)
        for n0 in range(0, NI, chunk):
            n1 = min(n0 + chunk, NI)
            feats = self._pyramid(pk, aggregated_tokens_list, NI, n0, n1, gh, gw, T, aspect, dt, dev)
            o, (o2, o3, o4) = self._scratch(pk, feats)
            up = ops.upsample_bilinear(o, gh * PATCH, gw * PATCH, tx, ty)
            m, c = dense_tail(up, pk, mode)
            preds[n0:n1].copy_(m)
            conf[n0:n1].copy_(c)
            if self.use_point_feat:
                f2.append(o2); f3.append(o3); f4.append(o4)
        preds = preds.view(B, S, H, W, oc - 1)
        conf = conf.view(B, S, H, W)
        if self.use_point_feat:
            return preds, conf, (torch.cat(f2), torch.cat(f3), torch.cat(f4))
        return preds, conf
