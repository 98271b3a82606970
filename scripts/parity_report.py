"""GPU: end-to-end parity report of the native path against the oracle (fp32 and same-precision-policy).

usage: python scripts/parity_report.py [--case NAME ...]   (cases = tests/golden fixtures + larger shapes)
"""
import argparse
import glob
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_model, weights  # noqa: E402  (checker only)


def rel_l2(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


def rel_max(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-12)).item()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1x2x28x56,2x3x28x28,1x2x42x42,1x2x518x518")
    ap.add_argument("--kinds", default="stress,default")
    ap.add_argument("--dtype", default="float16")
    ap.add_argument("--model", default="vggt")
    args = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from iggt_official_b200.models.vggt import IGGT, VGGT
    dt = getattr(torch, args.dtype)
    model = (IGGT if args.model == "iggt" else VGGT)()
    report = []
    for kind in args.kinds.split(","):
        sd = weights.make_state_dict(1, kind)
        model.load_state_dict(sd, strict=False)
        model.eval().to("cuda")
        sd_gpu = {k: v.cuda() for k, v in sd.items() if not k.startswith("track_head.")}
        for shp in args.shapes.split(","):
            B, S, H, W = map(int, shp.split("x"))
            g = torch.Generator().manual_seed(B * 1000 + S * 100 + H)
            images = torch.rand(B, S, 3, H, W, generator=g).cuda()
            t0 = time.time()
            model.compute_dtype = dt
            out = model(images)
            torch.cuda.synchronize()
            t1 = time.time()
            ref32 = ref_model.forward(sd_gpu, images, model=args.model, amp=None, frames_chunk=2, skip_part=(args.model != "iggt"))
            refamp = ref_model.forward(sd_gpu, images, model=args.model, amp=dt, frames_chunk=2, skip_part=(args.model != "iggt"))
            row = {"kind": kind, "shape": shp, "dtype": args.dtype, "fwd_s": t1 - t0}
            for k in ("depth", "depth_conf", "world_points", "world_points_conf", "part_feat"):
                if k not in out or k not in ref32:
                    continue
                row[k] = {"vs_fp32_l2": rel_l2(out[k], ref32[k]), "vs_fp32_max": rel_max(out[k], ref32[k]),
                          "vs_amp_l2": rel_l2(out[k], refamp[k]), "vs_amp_max": rel_max(out[k], refamp[k]),
                          "amp_vs_fp32_l2": rel_l2(refamp[k], ref32[k]), "amp_vs_fp32_max": rel_max(refamp[k], ref32[k])}
            p, p32, pamp = (torch.stack(o["pose_enc"]) for o in (out, ref32, refamp))
            row["pose_enc"] = {"vs_fp32_l2": rel_l2(p, p32), "vs_fp32_max": rel_max(p, p32), "vs_amp_l2": rel_l2(p, pamp),
                               "vs_amp_max": rel_max(p, pamp), "amp_vs_fp32_l2": rel_l2(pamp, p32), "amp_vs_fp32_max": rel_max(pamp, p32)}
            print(json.dumps(row))
            report.append(row)
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(report, open(os.path.join(ROOT, "gpurun_out", f"parity_{args.model}_{args.dtype}.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
