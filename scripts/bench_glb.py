"""visual_util.predictions_to_glb plus export() to an in-memory buffer, timed at the demo's shape (3 x 336 x 504) and at
8 x 532 x 532, the rgb mode at the demo's conf_thres 0.3.

"ms_total_median": the median of 20 calls of predictions_to_glb(...).export(BytesIO) on CUDA tensors, after three
warm-up calls (the call ends in its device-to-host copies, so it needs no extra synchronise).  "ms_by_stage_median":
the same pipeline split into its stages (median of 20): the device stages between CUDA events, the copies and the
host stages (cameras, GLB writing) by the host clock after a synchronise.  "oracle_cpu_s": oracle/ref_glb.py (the
reference's numpy arithmetic, without trimesh's scene building or writing) on the host CPU, for context.  The card's
name, power limit and clocks are read in the same run.  Prints one JSON line per shape."""
import io
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler                                              # noqa: E402
from iggt_official_b200 import ops, visual_util                             # noqa: E402
from oracle import make_golden_glb, ref_glb                                 # noqa: E402
from scripts.bench_pca import card                                          # noqa: E402

REPS = 20
KW = dict(conf_thres=0.3, prediction_mode="Pointmap Regression", vis_mode="rgb")


def stages(pred):
    """One predictions_to_glb pipeline, stage by stage, as the public function runs it."""
    pts, conf, img = pred["world_points"], pred["world_points_conf"], pred["images"]
    n = pts.numel() // 3
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    stats = torch.empty(16, dtype=torch.int32, device=pts.device)
    f = stats.view(torch.float32)
    ev[0].record()
    ops.select(conf.view(1, n), ops.QRULE_NUMPY, [KW["conf_thres"]], out=f[0:1].view(1, 1))
    ev[1].record()
    mask, planes, rgba, ws = ops.pointcloud_select(pts.view(n, 3), conf.view(n), f[0:1], img, 0)
    ev[2].record()
    ops.select(planes, ops.QRULE_NUMPY, [5.0, 95.0], mask=mask.view(1, n).expand(3, n), out=f[1:7].view(3, 2))
    ev[3].record()
    packed = ops.pointcloud_compact(pts.view(n, 3), mask, rgba, ws, stats[7:8], f[8:14])
    ev[4].record()
    torch.cuda.synchronize()
    out = {k: ev[i].elapsed_time(ev[i + 1]) for i, k in enumerate(("threshold", "select", "percentiles", "compact"))}
    t0 = time.perf_counter()
    st = stats.cpu().numpy()
    t1 = time.perf_counter()
    m = int(st[7]) & 0xffffffff
    host = torch.empty(16 * m, dtype=torch.uint8, pin_memory=True)
    host.copy_(packed[:16 * m])
    t2 = time.perf_counter()
    out.update(stats_d2h=(t1 - t0) * 1e3, points_d2h=(t2 - t1) * 1e3, points=m, point_bytes=16 * m)
    return out


def host_stages(pred):
    """The host part of one call: the cameras (inside predictions_to_glb after the copies) and the GLB writing."""
    scene = visual_util.predictions_to_glb(pred, **KW)
    t0 = time.perf_counter()
    cams = pred["extrinsic"].cpu().numpy()
    ext = np.zeros((len(cams), 4, 4))
    ext[:, :3, :4] = cams
    ext[:, 3, 3] = 1
    for i in range(len(cams)):
        visual_util.camera_glyph(np.linalg.inv(ext[i]), scene.scene_scale)
    t1 = time.perf_counter()
    scene.export(io.BytesIO())
    t2 = time.perf_counter()
    return {"cameras": (t1 - t0) * 1e3, "export": (t2 - t1) * 1e3}


def main():
    info = card()
    sampler = ClockSampler(0)
    sampler.start()
    lines = []
    for S, H, W in ((3, 336, 504), (8, 532, 532)):
        host = make_golden_glb.scene(seed=40 + S, S=S, H=H, W=W)
        pred = {k: (v if isinstance(v, torch.Tensor) else torch.from_numpy(v)).cuda() for k, v in host.items()}

        def call():
            visual_util.predictions_to_glb(pred, **KW).export(io.BytesIO())
        for _ in range(3):
            call()
        torch.cuda.synchronize()
        runs = []
        for _ in range(REPS):
            t0 = time.perf_counter()
            call()
            runs.append((time.perf_counter() - t0) * 1e3)
        per = [dict(stages(pred), **host_stages(pred)) for _ in range(REPS)]
        st = {k: float(np.median([p[k] for p in per])) for k in per[0]}
        t0 = time.perf_counter()
        ref_glb.predictions_to_glb(host, **{k: v for k, v in KW.items()})
        cpu_s = time.perf_counter() - t0
        lines.append({"shape": f"{S}x{H}x{W}", "points_in": S * H * W, "ms_total_median": float(np.median(runs)),
                      "ms_total_min": float(min(runs)), "ms_by_stage_median": st, "oracle_cpu_s": cpu_s})
        del pred
        torch.cuda.empty_cache()
    clocks = sampler.stop()
    for line in lines:
        line.update(card=info, clocks=clocks)
        print(json.dumps(line))


if __name__ == "__main__":
    main()
