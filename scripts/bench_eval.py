"""SceneEvaluator.evaluate_scene timed at the demo's shape (3 frames, GT 480 x 640 from predictions 336 x 504) and at
8 frames of GT 1168 x 1752 from 518 x 518 predictions, plus threshold_depth_map on each GT batch.

"ms_total_median": the median of 20 public calls on CUDA tensors, each ended by a device synchronise (evaluate_scene
ends in its device-to-host copy), after three warm-up calls.  "ms_by_stage_median": CUDA events around each stage of
the same pipeline (median of 20).  "oracle_cpu_s": the numpy oracle (oracle/ref_eval.py, the reference's per-frame
arithmetic with fp64 sums) on the host CPU for the same scene, for context.  The card's name, power limit and clocks
are read in the same run.  Prints one JSON line per shape."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler                                              # noqa: E402
from iggt_official_b200 import metrics, ops, postprocess                    # noqa: E402
from oracle import make_golden_eval, ref_eval                               # noqa: E402
from scripts.bench_pca import card                                          # noqa: E402

REPS = 20


def stages(gt, pred):
    """One evaluate_frames pipeline (median alignment, default clip) with CUDA events between the stages."""
    S, H, W = gt.shape
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
    ev[0].record()
    r = ops.resize_nearest(pred, H, W).view(S, -1)
    ev[1].record()
    g = gt.view(S, -1)
    mask = ops.depth_valid_mask(g, r, False)
    ev[2].record()
    med = torch.cat([ops.select(g, ops.QRULE_MEDIAN, mask=mask), ops.select(r, ops.QRULE_MEDIAN, mask=mask)], 1).t()
    ev[3].record()
    rec, _ = ops.depth_metrics(g, r, mask, ops.ALIGN_MEDIAN, med, (0.1, 100.0))
    ev[4].record()
    rec.cpu()
    ev[5].record()
    torch.cuda.synchronize()
    names = ("resize", "mask", "medians", "metrics", "records_d2h")
    return {k: ev[i].elapsed_time(ev[i + 1]) for i, k in enumerate(names)}


def timed(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    runs = []
    for _ in range(REPS):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        runs.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(runs)), float(min(runs))


def main():
    info = card()
    sampler = ClockSampler(0)
    sampler.start()
    shapes = {"demo_3x480x640_from_336x504": (3, (480, 640), (336, 504)),
              "8x1168x1752_from_518x518": (8, (1168, 1752), (518, 518))}
    lines = []
    for name, (S, gt_hw, pred_hw) in shapes.items():
        gt, pred, gp, pp = make_golden_eval.scene(seed=40 + S, S=S, gt_hw=gt_hw, pred_hw=pred_hw)
        gt_c, pred_c = torch.from_numpy(gt).cuda(), torch.from_numpy(pred).cuda()
        gd = {"gt_depth": gt_c, "gt_extrinsic": torch.from_numpy(gp).cuda()}
        pd = {"depth": pred_c, "extrinsic": torch.from_numpy(pp).cuda()}
        ev = metrics.SceneEvaluator()
        med, mn = timed(lambda: ev.evaluate_scene(gd, pd))
        per = [stages(gt_c, pred_c[..., 0]) for _ in range(REPS)]
        st = {k: float(np.median([p[k] for p in per])) for k in per[0]}
        work = gt_c.clone()
        thr_med, thr_min = timed(lambda: postprocess.threshold_depth_map(work.copy_(gt_c)))
        t0 = time.perf_counter()
        ref_eval.evaluate_scene({"gt_depth": gt, "gt_extrinsic": gp}, {"depth": pred, "extrinsic": pp})
        cpu_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        for m in gt.copy():
            ref_eval.threshold_depth_map(m)
        thr_cpu_s = time.perf_counter() - t0
        lines.append({"shape": name, "pixels": int(gt.size), "evaluate_scene_ms_median": med,
                      "evaluate_scene_ms_min": mn, "ms_by_stage_median": st,
                      "threshold_depth_map_ms_median": thr_med, "threshold_depth_map_ms_min": thr_min,
                      "oracle_cpu_s": cpu_s, "threshold_oracle_cpu_s": thr_cpu_s})
        del gt_c, pred_c, gd, pd, work
        torch.cuda.empty_cache()
    clocks = sampler.stop()
    for line in lines:
        line.update(card=info, clocks=clocks)
        print(json.dumps(line))


if __name__ == "__main__":
    main()
