"""Hopper-native part (instance-feature) path.

`PartAdaptor`  = reference `SamProjector` (iggt/heads/adaptor.py:140-226): LN -> 1x1 proj -> per-level resize
                 stacks (ConvTranspose k4/s2/p1, k2/s2, Conv3x3/s2, `Projects` with eval-mode BatchNorm folded
                 into the convolutions).  The PositionEmbeddingSine the reference also computes is discarded by
                 IGGT.forward (iggt/models/vggt.py:208) and is not computed here.
`PartHead`     = reference `PartHead` (iggt/heads/part_head.py:14-243): RefineNet fusion of the adaptor maps with
                 point-head features injected by cross_attention_2 (g^2 tokens, 8 heads x 32) and the
                 overlapping-window cross attention SwinCA/OCAB at (4g)^2, then SwinSA/HAB at (8g)^2, bilinear
                 to HxW, 3x3 -> ReLU -> 1x1 -> 8 raw channels [B,S,8,H,W].
                 `cross_attention_1` never reaches the output (SURVEY F4) and is not evaluated.
All convolutions / Linear layers run on the wgmma GEMM / implicit-GEMM kernels; window attentions, small-C
LayerNorms and the channel-attention run on the kernels in csrc/part.cu.
"""
from typing import List

import torch

from .. import ops
from ..layout import Node
from .dpt_head import DPTHead, LAYERS, PATCH, _f32, dense_tail, pack_conv3x3, pack_deconv


def _h16(p, dtype, device):
    return p.detach().to(device=device, dtype=dtype).contiguous()


def fold_bn(conv_w, bn, device):
    """conv (no bias) followed by eval-mode BatchNorm2d -> (w', b') in fp32 (adaptor.py:12-24)."""
    scale = (bn.weight.detach().to(device).float() / torch.sqrt(bn.running_var.detach().to(device).float() + 1e-5))
    w = conv_w.detach().to(device).float() * scale.view(-1, 1, 1, 1)
    b = bn.bias.detach().to(device).float() - bn.running_mean.detach().to(device).float() * scale
    return w, b.contiguous()


def pad_rows(w, rows):
    out = torch.zeros((rows,) + tuple(w.shape[1:]), dtype=w.dtype, device=w.device)
    out[:w.shape[0]] = w
    return out


class PartAdaptor(Node):
    def __init__(self):
        super().__init__()
        self._pk = None
        self._pk_key = None

    def invalidate(self):
        self._pk = None

    def _pack_projects(self, pk, name, mod, dtype, device):
        w, b = fold_bn(mod.input_proj._modules["0"].weight, mod.input_proj._modules["1"], device)
        pk[name + ".in.w"], pk[name + ".in.b"] = w.reshape(w.shape[0], -1).to(dtype).contiguous(), b
        w, b = fold_bn(mod.residual_conv._modules["0"].weight, mod.residual_conv._modules["1"], device)
        pk[name + ".r1.w"], pk[name + ".r1.b"] = pack_conv3x3(w, dtype, device), b
        w, b = fold_bn(mod.residual_conv._modules["3"].weight, mod.residual_conv._modules["4"], device)
        pk[name + ".r2.w"], pk[name + ".r2.b"] = pack_conv3x3(w, dtype, device), b
        ow = mod.output_proj.weight
        pk[name + ".out.w"] = ow.detach().to(device).reshape(ow.shape[0], -1).to(dtype).contiguous()
        pk[name + ".out.b"] = _f32(mod.output_proj.bias, device)

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
        l0 = r["0"]._modules
        for j in ("0", "2"):                                    # ConvTranspose2d k4 s2 p1: [Cin, Cout, 4, 4]
            w = l0[j].weight.detach().to(device)
            pk[f"l0.ct{j}.w"] = w.permute(2, 3, 1, 0).reshape(16 * w.shape[1], w.shape[0]).to(dtype).contiguous()
            pk[f"l0.ct{j}.b"] = _f32(l0[j].bias, device)
        self._pack_projects(pk, "l0.p1", l0["1"], dtype, device)
        self._pack_projects(pk, "l0.p3", l0["3"], dtype, device)
        l1 = r["1"]._modules
        pk["l1.ct.w"], pk["l1.ct.b"] = pack_deconv(l1["0"].weight, l1["0"].bias, dtype, device)
        self._pack_projects(pk, "l1.p", l1["1"], dtype, device)
        self._pack_projects(pk, "l2.p", r["2"]._modules["1"], dtype, device)
        l3 = r["3"]._modules
        pk["l3.c.w"], pk["l3.c.b"] = pack_conv3x3(l3["0"].weight, dtype, device), _f32(l3["0"].bias, device)
        self._pack_projects(pk, "l3.p", l3["1"], dtype, device)
        self._pk, self._pk_key = pk, key
        return pk

    @staticmethod
    def _projects(pk, name, x):
        """`Projects.forward` (adaptor.py:28-35) with BatchNorm folded: relu(1x1) -> relu(3x3) -> 3x3 + skip -> 1x1."""
        NB, h, w, C = x.shape
        a = ops.gemm_store16(x.view(-1, C), pk[name + ".in.w"], pk[name + ".in.b"], act=2).view(NB, h, w, -1)
        t = ops.conv_nhwc(a, pk[name + ".r1.w"], pk[name + ".r1.b"], act=2)
        s = ops.conv_nhwc(t, pk[name + ".r2.w"], pk[name + ".r2.b"], resid=a)
        o = ops.gemm_store16(s.view(-1, s.shape[-1]), pk[name + ".out.w"], pk[name + ".out.b"])
        return o.view(NB, h, w, -1)

    @staticmethod
    def _deconv_k4s2p1(pk, name, x):
        NB, h, w, C = x.shape
        y = ops.gemm_store16(x.view(-1, C), pk[name + ".w"], None)
        return ops.col2im_k4s2p1(y, pk[name + ".b"], NB, h, w, pk[name + ".w"].shape[0] // 16)

    @torch.no_grad()
    def forward(self, aggregated_tokens_list, images, patch_start_idx, compute_dtype=None, frames=None):
        """-> [res1, res2, res3, res4] NHWC 16-bit maps at 4g, 2g, g, ceil(g/2) for views `frames` (n0, n1)."""
        B, S, _, H, W = images.shape
        dev = images.device
        dt = compute_dtype or (torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else torch.float16)
        pk = self._packed(dt, dev)
        gh, gw = H // PATCH, W // PATCH
        P = gh * gw
        T = patch_start_idx + P
        n0, n1 = frames if frames is not None else (0, B * S)
        nb = n1 - n0
        outs = []
        for li, layer in enumerate(LAYERS):
            tok = aggregated_tokens_list[layer]
            tok2 = tok.reshape(-1, tok.shape[-1])[n0 * T:n1 * T]
            xn = torch.empty((nb * P, tok.shape[-1]), dtype=dt, device=dev)
            ops.layernorm(tok2, pk["norm_w"], pk["norm_b"], 1e-5, xn, groups=nb, rows_out=P, rows_in=T,
                          in_off=T - P, out_rows_per_group=P, out_off=0)
            x = ops.gemm_store16(xn, pk[f"proj{li}.w"], pk[f"proj{li}.b"]).view(nb, gh, gw, -1)
            if li == 0:
                x = self._projects(pk, "l0.p1", self._deconv_k4s2p1(pk, "l0.ct0", x))
                x = self._projects(pk, "l0.p3", self._deconv_k4s2p1(pk, "l0.ct2", x))
            elif li == 1:
                y = ops.gemm_store16(x.view(-1, x.shape[-1]), pk["l1.ct.w"], pk["l1.ct.b"])
                x = self._projects(pk, "l1.p", ops.deconv_shuffle(y, nb, gh, gw, x.shape[-1], 2))
            elif li == 2:
                x = self._projects(pk, "l2.p", x)
            else:
                A, ho, wo = ops.im2col3x3_s2(x)
                x = self._projects(pk, "l3.p", ops.gemm_store16(A, pk["l3.c.w"], pk["l3.c.b"]).view(nb, ho, wo, -1))
            outs.append(x)
        return outs


class PartHead(DPTHead):
    """Inherits the RefineNet building blocks (`_rcu_tail`, `_fuse`, `_pack_scratch`) from DPTHead."""

    def __init__(self):
        super().__init__(output_dim=8, activation="norm", use_point_feat=False)

    # ------------------------------------------------------------------ packing
    def _pack_swin_common(self, pk, name, m, dtype, device, C):
        pk[name + ".pe_w"], pk[name + ".pe_b"] = _f32(m.patch_embed.norm.weight, device), _f32(m.patch_embed.norm.bias, device)
        pk[name + ".norm_w"], pk[name + ".norm_b"] = _f32(m.norm.weight, device), _f32(m.norm.bias, device)
        pk[name + ".cab.w"], pk[name + ".cab.b"] = pack_conv3x3(m.conv_after_body.weight, dtype, device), _f32(m.conv_after_body.bias, device)
        cbu = m.conv_before_upsample._modules["0"]
        pk[name + ".cbu.w"], pk[name + ".cbu.b"] = pack_conv3x3(cbu.weight, dtype, device), _f32(cbu.bias, device)
        pk[name + ".last.w"], pk[name + ".last.b"] = pack_conv3x3(m.conv_last.weight, dtype, device), _f32(m.conv_last.bias, device)
        ab = m.atten_block
        for n in ("norm1", "norm2"):
            pk[f"{name}.{n}_w"], pk[f"{name}.{n}_b"] = _f32(ab._modules[n].weight, device), _f32(ab._modules[n].bias, device)
        pk[name + ".fc1.w"], pk[name + ".fc1.b"] = _h16(ab.mlp.fc1.weight, dtype, device), _f32(ab.mlp.fc1.bias, device)
        pk[name + ".fc2.w"], pk[name + ".fc2.b"] = _h16(ab.mlp.fc2.weight, dtype, device), _f32(ab.mlp.fc2.bias, device)

    def _packed(self, dtype, device):
        key = (dtype, str(device))
        if self._pk is not None and self._pk_key == key:
            return self._pk
        pk = {}
        self._pack_scratch(pk, dtype, device)
        # cross_attention_2: 8 heads x 32, zero-padded to 8 x 64 so the d=64 flash kernel applies unchanged
        ca = self.cross_attention_2

        def pad_heads_out(w, b):                     # Linear [256 -> 8x32]  ->  [8x64, 256]
            w4 = torch.zeros(8, 64, w.shape[1], device=device)
            w4[:, :32] = w.detach().to(device).float().view(8, 32, -1)
            b4 = torch.zeros(8, 64, device=device)
            b4[:, :32] = b.detach().to(device).float().view(8, 32)
            return w4.view(512, -1).to(dtype).contiguous(), b4.view(512).contiguous()

        pk["ca.q.w"], pk["ca.q.b"] = pad_heads_out(ca.projq.weight, ca.projq.bias)
        kw, kb = pad_heads_out(ca.projk.weight, ca.projk.bias)
        vw, vb = pad_heads_out(ca.projv.weight, ca.projv.bias)
        pk["ca.kv.w"], pk["ca.kv.b"] = torch.cat([kw, vw], 0).contiguous(), torch.cat([kb, vb], 0).contiguous()
        pw = torch.zeros(256, 8, 64, device=device)
        pw[:, :, :32] = ca.proj.weight.detach().to(device).float().view(256, 8, 32)
        pk["ca.o.w"], pk["ca.o.b"] = pw.view(256, 512).to(dtype).contiguous(), _f32(ca.proj.bias, device)
        # SwinCA / OCAB
        wc = self.window_cross_attention
        self._pack_swin_common(pk, "wc", wc, dtype, device, 256)
        ab = wc.atten_block
        pk["wc.q.w"], pk["wc.q.b"] = _h16(ab.q.weight, dtype, device), _f32(ab.q.bias, device)
        pk["wc.kv.w"] = torch.cat([ab.k.weight.detach(), ab.v.weight.detach()], 0).to(device, dtype).contiguous()
        pk["wc.kv.b"] = torch.cat([ab.k.bias.detach(), ab.v.bias.detach()], 0).to(device, torch.float32).contiguous()
        pk["wc.proj.w"], pk["wc.proj.b"] = _h16(ab.proj.weight, dtype, device), _f32(ab.proj.bias, device)
        pk["wc.table"] = _f32(ab.relative_position_bias_table, device)
        n_tab = pk["wc.table"].shape[0]
        pk["wc.rpi"] = (wc.relative_position_index_OCA.detach().to(device) % n_tab).int().contiguous()   # python-style wrap
        # SwinSA / HAB
        ws = self.window_self_atten
        self._pack_swin_common(pk, "ws", ws, dtype, device, 128)
        hb = ws.atten_block
        pk["ws.qkv.w"], pk["ws.qkv.b"] = _h16(hb.attn.qkv.weight, dtype, device), _f32(hb.attn.qkv.bias, device)
        pk["ws.proj.w"], pk["ws.proj.b"] = _h16(hb.attn.proj.weight, dtype, device), _f32(hb.attn.proj.bias, device)
        cab = hb.conv_block.cab._modules
        w0 = pad_rows(cab["0"].weight.detach().to(device).float(), 64)                       # 128 -> 42, padded to 64 out
        pk["ws.cab0.w"] = pack_conv3x3(w0, dtype, device)
        pk["ws.cab0.b"] = pad_rows(cab["0"].bias.detach().to(device).float(), 64).contiguous()
        w2 = cab["2"].weight.detach().to(device).float()                                      # 42 -> 128, padded to 64 in
        w2p = torch.zeros(w2.shape[0], 64, 3, 3, device=device)
        w2p[:, :w2.shape[1]] = w2
        pk["ws.cab2.w"], pk["ws.cab2.b"] = pack_conv3x3(w2p, dtype, device), _f32(cab["2"].bias, device)
        att = cab["3"].attention._modules
        pk["ws.se.w1"] = _f32(att["1"].weight, device).reshape(att["1"].weight.shape[0], -1).contiguous()
        pk["ws.se.b1"] = _f32(att["1"].bias, device)
        pk["ws.se.w2"] = _f32(att["3"].weight, device).reshape(att["3"].weight.shape[0], -1).contiguous()
        pk["ws.se.b2"] = _f32(att["3"].bias, device)
        self._pk, self._pk_key = pk, key
        return pk

    # ------------------------------------------------------------------ blocks
    @staticmethod
    def _swin_tail(pk, name, y, x_in):
        """norm -> conv_after_body + x -> conv 3x3 + LeakyReLU -> conv_last (window_sa.py:428-435,536-545)."""
        z = ops.layernorm16(y, pk[name + ".norm_w"], pk[name + ".norm_b"])
        z = ops.conv_nhwc(z, pk[name + ".cab.w"], pk[name + ".cab.b"], resid=x_in)
        z = ops.conv_nhwc(z, pk[name + ".cbu.w"], pk[name + ".cbu.b"], act=3)
        return ops.conv_nhwc(z, pk[name + ".last.w"], pk[name + ".last.b"])

    @staticmethod
    def _mlp_res(pk, name, x):
        """x + fc2(gelu(fc1(LN2(x))))"""
        C = x.shape[-1]
        y = ops.layernorm16(x, pk[name + ".norm2_w"], pk[name + ".norm2_b"])
        hdn = ops.gemm_store16(y.view(-1, C), pk[name + ".fc1.w"], pk[name + ".fc1.b"], act=1)
        x2 = x.view(-1, C)
        return ops.gemm_store16(hdn, pk[name + ".fc2.w"], pk[name + ".fc2.b"], addend=x2, add_rows=x2.shape[0]).view(x.shape)

    def _swin_ca(self, pk, x, kv):
        """SwinCA.forward on NHWC x (part features) and kv (point-head out2), both [nb, 4g, 4g, 256]."""
        nb, h, w, C = x.shape
        xt = ops.layernorm16(x, pk["wc.pe_w"], pk["wc.pe_b"])
        kt = ops.layernorm16(kv, pk["wc.pe_w"], pk["wc.pe_b"])
        xs = ops.layernorm16(xt, pk["wc.norm1_w"], pk["wc.norm1_b"])
        ks = ops.layernorm16(kt, pk["wc.norm1_w"], pk["wc.norm1_b"])
        q = ops.gemm_store16(xs.view(-1, C), pk["wc.q.w"], pk["wc.q.b"]).view(nb, h, w, C)
        kvp = ops.gemm_store16(ks.view(-1, C), pk["wc.kv.w"], pk["wc.kv.b"])
        k = kvp[:, :C].contiguous().view(nb, h, w, C)
        v = kvp[:, C:].contiguous().view(nb, h, w, C)
        o = ops.ocab_attention(q, k, v, pk["wc.table"], pk["wc.rpi"])
        xt2 = xt.view(-1, C)
        x1 = ops.gemm_store16(o.view(-1, C), pk["wc.proj.w"], pk["wc.proj.b"], addend=xt2, add_rows=xt2.shape[0]).view(nb, h, w, C)
        x2 = self._mlp_res(pk, "wc", x1)
        return self._swin_tail(pk, "wc", x2, x)

    def _swin_sa(self, pk, x):
        """SwinSA.forward on NHWC x [nb, 8g, 8g, 128]."""
        nb, h, w, C = x.shape
        xt = ops.layernorm16(x, pk["ws.pe_w"], pk["ws.pe_b"])
        xn = ops.layernorm16(xt, pk["ws.norm1_w"], pk["ws.norm1_b"])
        c1 = ops.conv_nhwc(xn, pk["ws.cab0.w"], pk["ws.cab0.b"], act=1)              # 128 -> 42(64), GELU
        c2 = ops.conv_nhwc(c1, pk["ws.cab2.w"], pk["ws.cab2.b"])                       # 42(64) -> 128
        mean = ops.channel_mean(c2)
        qkv = ops.gemm_store16(xn.view(-1, C), pk["ws.qkv.w"], pk["ws.qkv.b"]).view(nb, h, w, 3 * C)
        a = ops.window_attention(qkv)
        xt2 = xt.view(-1, C)
        y0 = ops.gemm_store16(a.view(-1, C), pk["ws.proj.w"], pk["ws.proj.b"], addend=xt2, add_rows=xt2.shape[0]).view(nb, h, w, C)
        y = ops.se_scale_add(y0, c2, mean, pk["ws.se.w1"], pk["ws.se.b1"], pk["ws.se.w2"], pk["ws.se.b2"], 0.01)
        y2 = self._mlp_res(pk, "ws", y)
        return self._swin_tail(pk, "ws", y2, x)

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, maps_fn, point_feature, images, patch_start_idx, compute_dtype=None, frames_chunk_size: int = 4):
        """`maps_fn(n0, n1)` -> adaptor maps for views [n0, n1) (or a list of 4 full maps); `point_feature` =
        (out2, out3, out4) NHWC maps from the point head.  Returns part_feat [B, S, 8, H, W] fp32."""
        B, S, _, H, W = images.shape
        gh, gw = H // PATCH, W // PATCH
        if gh % 2 or gw % 2:
            # reference: window_partition's view fails (iggt/heads/window_sa.py:71-75, SURVEY F2)
            raise RuntimeError(f"shape is invalid for input: the part head needs an even patch grid, got {gh}x{gw}")
        dev = images.device
        dt = compute_dtype or (torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else torch.float16)
        pk = self._packed(dt, dev)
        NI = B * S
        out = torch.empty((NI, 8, H, W), dtype=torch.float32, device=dev)
        pf2, pf3, pf4 = point_feature
        chunk = frames_chunk_size or NI
        for n0 in range(0, NI, chunk):
            n1 = min(n0 + chunk, NI)
            nb = n1 - n0
            maps = maps_fn(n0, n1) if callable(maps_fn) else [m[n0:n1] for m in maps_fn]
            l = [ops.conv_nhwc(f, pk[f"rn{i + 1}"], None, act=2) for i, f in enumerate(maps)]
            p4 = self._rcu_tail(pk, 4, l[3])
            o = ops.upsample_bilinear(p4, l[2].shape[1], l[2].shape[2])                      # [nb, g, g, 256]
            # cross_attention_2: q from the part map, k = v from point-head out4; output REPLACES the map
            g2 = o.shape[1] * o.shape[2]
            qp = ops.gemm_store16(o.view(-1, 256), pk["ca.q.w"], pk["ca.q.b"])
            kvp = ops.gemm_store16(pf4[n0:n1].reshape(-1, 256), pk["ca.kv.w"], pk["ca.kv.b"])
            att = ops.attention(qp, kvp[:, :512], kvp[:, 512:], nb, g2, g2, 8, scale=32 ** -0.5)
            o4 = ops.gemm_store16(att, pk["ca.o.w"], pk["ca.o.b"]).view(o.shape)
            p3 = self._rcu_tail(pk, 3, self._fuse(pk, 3, o4, l[2]))
            o3 = ops.upsample_bilinear(p3, l[1].shape[1], l[1].shape[2])
            p2 = self._rcu_tail(pk, 2, self._fuse(pk, 2, o3, l[1]))
            o2 = ops.upsample_bilinear(p2, l[0].shape[1], l[0].shape[2])
            o2 = self._swin_ca(pk, o2, pf2[n0:n1].contiguous())
            p1 = self._rcu_tail(pk, 1, self._fuse(pk, 1, o2, l[0]))
            o1 = ops.upsample_bilinear(p1, 2 * p1.shape[1], 2 * p1.shape[2])
            f = ops.conv_nhwc(o1, pk["oc1.w"], pk["oc1.b"])                                  # [nb, 8g, 8g, 128]
            f = self._swin_sa(pk, f)
            up = ops.upsample_bilinear(f, gh * PATCH, gw * PATCH)
            m, _ = dense_tail(up, pk, 2)
            out[n0:n1].copy_(m)
        return out.view(B, S, 8, H, W)
