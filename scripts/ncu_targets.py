"""One launch of every CUDA kernel of the library at its C2 shape (8 views, 518 x 518; part path at 532 x 532), bracketed
by cudaProfilerStart/Stop so that ONE `ncu --set full --profile-from-start off` run captures them all:

  ncu --set full --clock-control none --import-source on --profile-from-start off -f -o gpurun_out/prof_<tag>_all \
      python scripts/ncu_targets.py

(`--only a,b` restricts to the named targets.)  Each target is launched once un-profiled first (kernel configuration,
allocator warm-up) and once inside the profiled range.  scripts/ncu_extract.py turns the report into the per-kernel CSV
rows kept under profiles/."""
import argparse
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from iggt_official_b200 import ops  # noqa: E402

DEV = "cuda"
DT = torch.float16


def rnd(*shape, dtype=DT, scale=1.0):
    return (torch.randn(*shape, device=DEV) * scale).to(dtype)


def targets():
    S, T, g = 8, 1374, 37
    M = S * T
    t = {}
    # ---- trunk
    x32 = rnd(M, 1024, dtype=torch.float32)
    w1, b1 = torch.rand(1024, device=DEV) + 0.5, rnd(1024, dtype=torch.float32)
    h16 = torch.empty(M, 1024, device=DEV, dtype=DT)
    t["layernorm"] = lambda: ops.layernorm(x32, w1, b1, 1e-5, h16)
    a = rnd(M, 1024)
    wqkv, bqkv = rnd(3072, 1024, scale=1 / 32), rnd(3072, dtype=torch.float32)
    from iggt_official_b200.models.aggregator import rope_tables, token_positions
    cos, sin = rope_tables(g + 1, DEV)
    pos = token_positions(g, g, DEV)
    nw = [torch.rand(64, device=DEV) + 0.5 for _ in range(4)]
    t["gemm_qkv"] = lambda: ops.gemm_qkv(a, wqkv, bqkv, 1024, qk_norm=True, qn_w=nw[0], qn_b=nw[1], kn_w=nw[2], kn_b=nw[3],
                                         rope_cos=cos, rope_sin=sin, pos_yx=pos, T=T)
    qkv = rnd(M, 3072)
    t["attention_frame"] = lambda: ops.attention(qkv[:, :1024], qkv[:, 1024:2048], qkv[:, 2048:], S, T, T, 16)
    t["attention_global"] = lambda: ops.attention(qkv[:, :1024], qkv[:, 1024:2048], qkv[:, 2048:], 1, M, M, 16)
    wp, bp, gam = rnd(1024, 1024, scale=1 / 32), rnd(1024, dtype=torch.float32), torch.rand(1024, device=DEV)
    t["gemm_resid32_proj"] = lambda: ops.gemm_resid32(a, wp, x32, bp, gam, round_out16=True)
    wf1, bf1 = rnd(4096, 1024, scale=1 / 32), rnd(4096, dtype=torch.float32)
    t["gemm_store16_fc1_gelu"] = lambda: ops.gemm_store16(a, wf1, bf1, act=1)
    a4 = rnd(M, 4096)
    wf2 = rnd(1024, 4096, scale=1 / 64)
    t["gemm_resid32_fc2"] = lambda: ops.gemm_resid32(a4, wf2, x32, bp, gam, round_out16=True)
    img = torch.rand(S, 3, 518, 518, device=DEV)
    t["patchify"] = lambda: ops.patchify(img, 640, DT)
    pe16 = rnd(S * g * g, 1024)
    cls, reg, dpos = rnd(1024, dtype=torch.float32), rnd(4, 1024, dtype=torch.float32), rnd(1 + g * g, 1024, dtype=torch.float32)
    t["dino_assemble"] = lambda: ops.dino_assemble(pe16, cls, reg, dpos, x32, S, g * g, 4, 1024)
    cam, regtok = rnd(2, 1024, dtype=torch.float32), rnd(2, 4, 1024, dtype=torch.float32)
    t["special_tokens"] = lambda: ops.special_tokens(cam, regtok, x32, S, T, 4, 1024, S, 0)
    # ---- camera head
    xs = rnd(8, 2048, dtype=torch.float32)
    wsk, bsk = rnd(6144, 2048, scale=1 / 45), rnd(6144, dtype=torch.float32)
    t["skinny_gemm_qkv"] = lambda: ops.skinny_gemm(xs, wsk, bsk)
    q8 = rnd(8, 6144, dtype=torch.float32)
    t["small_attention"] = lambda: ops.small_attention(q8, 1, 8, 16, 128)
    from iggt_official_b200.heads.camera_head import CameraHead
    from iggt_official_b200.layout import load_layout, populate
    torch.manual_seed(0)
    cam_mod = CameraHead()
    populate(cam_mod, load_layout(), "camera_head.")
    cam_mod = cam_mod.cuda()
    pk = cam_mod._packed(DT, torch.device("cuda"))
    cam_tok = rnd(8, 2048, dtype=torch.float32)
    t["camera_head_one_launch"] = lambda: ops.camera_head(pk["cstruct"], pk, cam_tok, 1, 8, 4, DT)
    cam_tok16 = rnd(16, 2048, dtype=torch.float32)
    t["camera_head_one_launch_16_rows"] = lambda: ops.camera_head(pk["cstruct"], pk, cam_tok16, 1, 16, 4, DT)
    t["attention_global_1of8_split3"] = lambda: ops.attention(qkv[:1374, :1024], qkv[:, 1024:2048], qkv[:, 2048:], 1, 1374, M, 16, splits=3)
    # ---- DPT heads
    f148 = rnd(S, 148, 148, 256)
    wc = rnd(256, 9 * 256, scale=1 / 48)
    bc = rnd(256, dtype=torch.float32)
    t["conv_nhwc_256_148"] = lambda: ops.conv_nhwc(f148, wc, bc, act=2)
    f296 = rnd(S, 296, 296, 256)
    woc1 = rnd(128, 9 * 256, scale=1 / 48)
    t["conv_nhwc_oc1_296"] = lambda: ops.conv_nhwc(f296, woc1, bc[:128].contiguous())
    f74 = rnd(S, 74, 74, 256)
    t["upsample_bilinear_74_148"] = lambda: ops.upsample_bilinear(f74, 148, 148)
    o296 = rnd(S, 296, 296, 128)
    from iggt_official_b200.heads.dpt_head import uv_pos_tables
    tx, ty = uv_pos_tables(518, 518, 128, 1.0, DEV)
    t["upsample_bilinear_pe_296_518"] = lambda: ops.upsample_bilinear(o296, 518, 518, tx, ty)
    up = rnd(S, 518, 518, 128)
    wt, bt = rnd(32, 9 * 128, scale=1 / 34), rnd(32, dtype=torch.float32)
    w2, b2 = rnd(4, 32, dtype=torch.float32, scale=0.2), rnd(4, dtype=torch.float32, scale=0.1)
    t["dpt_tail_fused"] = lambda: ops.dpt_tail_fused(up, wt, bt, w2, b2, 1)
    t["conv_nhwc_tail_generic"] = lambda: ops.conv_nhwc(up, wt, bt, act=2)
    y4 = rnd(S * g * g, 16 * 256)
    t["deconv_shuffle"] = lambda: ops.deconv_shuffle(y4, S, g, g, 256, 4)
    f37 = rnd(S, g, g, 1024)
    t["im2col3x3_s2"] = lambda: ops.im2col3x3_s2(f37)
    # ---- part path (532 x 532: g = 38)
    gp = 38
    q152 = rnd(4, 4 * gp, 4 * gp, 256)
    table, rpi = rnd(361, 4, dtype=torch.float32), torch.randint(0, 361, (64, 144), device=DEV, dtype=torch.int32)
    t["ocab_attention"] = lambda: ops.ocab_attention(q152, q152, q152, table, rpi)
    qkv304 = rnd(4, 8 * gp, 8 * gp, 384)
    t["window_attention"] = lambda: ops.window_attention(qkv304)
    l16w, l16b = torch.rand(256, device=DEV) + 0.5, rnd(256, dtype=torch.float32)
    t["layernorm16"] = lambda: ops.layernorm16(q152, l16w, l16b)
    ycol = rnd(4 * gp * gp, 16 * 256)
    t["col2im_k4s2p1"] = lambda: ops.col2im_k4s2p1(ycol, bc, 4, gp, gp, 256)
    c304 = rnd(4, 8 * gp, 8 * gp, 128)
    t["channel_mean"] = lambda: ops.channel_mean(c304)
    mean = rnd(4, 128, dtype=torch.float32)
    sw1, sb1, sw2, sb2 = rnd(4, 128, dtype=torch.float32), rnd(4, dtype=torch.float32), rnd(128, 4, dtype=torch.float32), rnd(128, dtype=torch.float32)
    t["se_scale_add"] = lambda: ops.se_scale_add(c304, c304, mean, sw1, sb1, sw2, sb2, 0.01)
    # ---- callers either side of the path (SURVEY 8f)
    pose = rnd(S, 9, dtype=torch.float32)
    t["pose_to_cameras"] = lambda: ops.pose_to_cameras(pose, 518, 518)
    depth = torch.rand(S, 518, 518, device=DEV) + 0.5
    extr, intr = ops.pose_to_cameras(pose, 518, 518)
    t["unproject_depth"] = lambda: ops.unproject_depth(depth, extr, intr)
    pts = torch.randn(2_000_000, 3, device=DEV)
    feats = torch.randn(2_000_000, 8, device=DEV)
    t["knn_mean_features"] = lambda: ops.knn_mean_features(pts, feats, 20)
    fm = rnd(S, 259, 259, 128)
    t["avgpool2_nhwc"] = lambda: ops.avgpool2_nhwc(fm)
    coords = torch.rand(S, 64, 2, device=DEV) * 250
    t["sample_bilinear_nhwc"] = lambda: ops.sample_bilinear_nhwc(fm, coords)
    lv = [fm]
    for _ in range(6):
        lv.append(ops.avgpool2_nhwc(lv[-1]))
    rows = 1 * 64 * S
    tg, cd = rnd(rows, 128, dtype=torch.float32), torch.rand(rows, 2, device=DEV) * 250
    t["corr_sample"] = lambda: ops.corr_sample(lv, tg, cd, 1, 64, S, 576)
    fc, ps_, rt = rnd(rows, 128, dtype=torch.float32), rnd(64, 388, dtype=torch.float32), rnd(2, 388, dtype=torch.float32)
    lw, lb = torch.rand(388, device=DEV) + 0.5, rnd(388, dtype=torch.float32)
    t["track_input"] = lambda: ops.track_input(cd, fc, tg, ps_, rt, lw, lb, S, DT, 392)
    xr = rnd(rows, 384, dtype=torch.float32)
    o16 = torch.empty(rows, 384, device=DEV, dtype=DT)
    lw2, lb2 = torch.rand(384, device=DEV) + 0.5, rnd(384, dtype=torch.float32)
    t["layernorm_rows"] = lambda: ops.layernorm_rows(xr, lw2, lb2, out16=o16)
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    t = targets()
    names = [n for n in t if not args.only or n in args.only.split(",")]
    for n in names:                       # un-profiled pass: configuration + allocator warm-up
        t[n]()
    torch.cuda.synchronize()
    torch.cuda.profiler.start()
    for n in names:
        t[n]()
        torch.cuda.synchronize()
    torch.cuda.profiler.stop()
    print("targets:", ",".join(names))


if __name__ == "__main__":
    main()
