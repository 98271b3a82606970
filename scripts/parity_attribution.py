"""CPU: where the end-to-end parity error of the native path comes from (no GPU needed; ~5 min on 16 threads).

The product's module graph is run with every C-ABI launcher replaced by its plain-PyTorch statement (tests/emu_ops.py,
the same statements the GPU kernel tests hold the CUDA kernels to), with fp16 operands, against oracle/ref_model.py on a
small stress-weight case.  Three measurements -> profiles/r02_parity_attribution.json:
 1. trunk noise floor: tokens of emulated trunk vs oracle(amp) layer by layer - two correct 16-bit realisations differ by
    ~1e-4 of a block's update per block (fp32 summation order flips 16-bit roundings), ~7e-4 after the 24 DINOv2 blocks;
 2. head policies on identical trunk tokens: exact fp32 heads / operands rounded to fp16 but fp32 storage (= TF32-like,
    what the reference's heads run on a GPU) / 16-bit storage as well (the product) - storage costs almost nothing,
    the 10-bit operand mantissa is the error;
 3. the point head layer by layer: rounding the operands of ONE layer at a time.
"""
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import emu_ops  # noqa: E402
from oracle import ref_model, weights  # noqa: E402
from iggt_official_b200 import ops  # noqa: E402
from iggt_official_b200.models import aggregator as agg_mod  # noqa: E402
from iggt_official_b200.models.vggt import VGGT  # noqa: E402
from test_model_wiring import EMU  # noqa: E402


def l2(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


def r16(t):
    return t.half().float()


def main():
    torch.set_num_threads(min(16, os.cpu_count() or 1))
    for n, f in EMU.items():
        setattr(ops, n, f)
    agg_mod._require_cuda = lambda images: None
    H, W, S = 42, 56, 2
    sd = weights.make_state_dict(1, "stress", prefixes=("aggregator.", "camera_head.", "depth_head.", "point_head."))
    m = VGGT()
    m.load_state_dict(sd, strict=False)
    m.eval()
    g = torch.Generator().manual_seed(5)
    images = torch.rand(1, S, 3, H, W, generator=g)
    amp = torch.float16
    report = {"case": f"vggt 1x{S}x{H}x{W} stress/1 fp16"}
    # ---- 1. trunk
    m.aggregator.keep_all_layers = True
    toks, psi = m.aggregator(images, compute_dtype=amp)
    ref = ref_model.aggregator(sd, images, amp, keep=tuple(range(24)))
    ref32 = ref_model.aggregator(sd, images, None, keep=tuple(range(24)))
    report["trunk_tokens"] = {str(i): {"emulated_vs_oracle_amp": l2(toks[i], ref[i]), "oracle_amp_vs_fp32": l2(ref[i], ref32[i])}
                              for i in (0, 4, 11, 17, 23)}
    refamp = ref_model.forward(sd, images, model="vggt", amp=amp, skip_part=True)
    ref_fp32 = ref_model.forward(sd, images, model="vggt", amp=None, skip_part=True)
    report["oracle_amp_vs_fp32"] = {k: l2(refamp[k], ref_fp32[k]) for k in ("depth", "depth_conf", "world_points", "world_points_conf")}
    # ---- 2./3. heads on the emulated trunk's tokens, operand rounding switched per layer
    state = {"i": 0, "round": set(), "names": [], "store16": False}

    def pick(tag, x):
        i = state["i"]
        state["i"] += 1
        if len(state["names"]) <= i:
            state["names"].append(f"{tag}{tuple(x.shape)}")
        return i in state["round"] or "all" in state["round"]

    def conv_nhwc(x, wp, bias=None, act=0, resid=None, taps=9, out=None, resid2=None, act_post=0):
        Cout, ks = wp.shape[0], (3 if taps == 9 else 1)
        rnd = pick("conv", x)
        xx, ww = (r16(x.float()), r16(wp.float())) if rnd else (x.float(), wp.float())
        v = F.conv2d(xx.permute(0, 3, 1, 2), ww.view(Cout, ks, ks, -1).permute(0, 3, 1, 2), bias, padding=ks // 2).permute(0, 2, 3, 1)
        v = emu_ops._act(v, act)
        if resid is not None:
            v = v + resid.float()
        if resid2 is not None:
            v = v + resid2.float()
        v = emu_ops._act(v, act_post).contiguous()
        return r16(v) if state["store16"] else v

    def gemm_store16(a, w, bias=None, act=0, addend=None, add_rows=0, out=None):
        rnd = pick("gemm", a)
        aa, ww = (r16(a.float()), r16(w.float())) if rnd else (a.float(), w.float())
        v = aa @ ww.t()
        if bias is not None:
            v = v + bias
        v = emu_ops._act(v, act)
        if addend is not None:
            v = v + addend.float().repeat(v.shape[0] // add_rows, 1)
        return r16(v) if state["store16"] else v

    def dpt_tail_fused(x, wp, bias, w2, b2, mode):
        rnd = pick("tailconv", x)
        xx, ww = (r16(x.float()), r16(wp.float())) if rnd else (x.float(), wp.float())
        z = F.relu(F.conv2d(xx.permute(0, 3, 1, 2), ww.view(32, 3, 3, 128).permute(0, 3, 1, 2), bias, padding=1)).permute(0, 2, 3, 1)
        return emu_ops.dpt_tail(z, w2, b2, mode)

    def upsample(x, Hh, Ww, tabx=None, taby=None, out=None):
        v = emu_ops.upsample_bilinear(x.float(), Hh, Ww, tabx, taby)
        return r16(v) if state["store16"] else v

    ops.conv_nhwc, ops.gemm_store16, ops.dpt_tail_fused, ops.upsample_bilinear = conv_nhwc, gemm_store16, dpt_tail_fused, upsample
    tokens = [t if t is not None else None for t in toks]

    def point_head(rset, store16=False):
        state["i"], state["round"], state["store16"] = 0, set(rset), store16
        m.point_head.invalidate()
        p, _ = m.point_head(tokens, images=images, patch_start_idx=psi, compute_dtype=torch.float32)
        return p

    exact = point_head(set())
    n = state["i"]
    tf32like = point_head({"all"})
    product = point_head({"all"}, store16=True)
    report["point_head_policies"] = {
        "exact_fp32_heads_vs_oracle_amp": l2(exact, refamp["world_points"]),
        "operands_fp16_storage_fp32_vs_oracle_amp": l2(tf32like, refamp["world_points"]),
        "product_16bit_storage_vs_oracle_amp": l2(product, refamp["world_points"]),
        "operands_fp16_vs_exact_heads_same_tokens": l2(tf32like, exact)}
    per_layer = []
    for i in range(n):
        per_layer.append({"layer": i, "op": state["names"][i], "world_points_err": l2(point_head({i}), exact)})
    report["point_head_per_layer_operand_rounding"] = per_layer
    report["point_head_rss_of_layers"] = sum(e["world_points_err"] ** 2 for e in per_layer) ** 0.5
    out = os.path.join(ROOT, "profiles", "r02_parity_attribution.json")
    json.dump(report, open(out, "w"), indent=1)
    print(json.dumps({k: v for k, v in report.items() if k != "point_head_per_layer_operand_rounding"}, indent=1))


if __name__ == "__main__":
    main()
