"""HDBSCAN instance clustering (cluster_features_to_masks_mv with the demo's parameters) timed stage by stage at the
demo shape (3 x 336 x 504) and at C2-with-part (8 x 532 x 532).

The features are oracle/make_golden_cluster.py's seeded demo features smoothed on the device by knn_avg_features_pyg.
Stages: Morton order + sort + reorder ("prepare"), core distances, Boruvka MST (its launcher synchronises once per
pointer-jumping pass), edge sort + copy to the host, host condensation, noise fill + colours + copy of the masks to
the host.  CUDA events around device stages, a host clock around the host stage; "total" is a host clock around the
whole public call.  The SM clock is sampled as bench.py samples it; the card's name and power limit are read once."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler                                              # noqa: E402
from iggt_official_b200 import ops                                          # noqa: E402
from iggt_official_b200.utils import misc                                   # noqa: E402
from oracle.make_golden_cluster import DEMO_KWARGS, KNN_K, demo_inputs      # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=20).stdout.strip().splitlines()[0]
        return dict(zip(("name", "power_limit", "sm_max_clock"), [f.strip() for f in out.split(",")]))
    except Exception:
        return {"name": torch.cuda.get_device_name(0)}


def stages(x, kw):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    ev[0].record()
    sorted8, orig, box = ops.cluster_prepare(x)
    ev[1].record()
    core2 = ops.cluster_core(sorted8, box, kw["min_samples"])
    ev[2].record()
    a, b, w2, rounds = ops.cluster_mst(sorted8, box, orig, core2)
    ev[3].record()
    mst = misc.sorted_mst(a, b, w2)
    ev[4].record()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    raw = ops.hdbscan_labels(mst, x.shape[0], kw["min_cluster_size"], kw["eps"])
    t_host = (time.perf_counter() - t0) * 1e3
    e5, e6 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e5.record()
    lab = torch.from_numpy(raw.astype(np.int32)).cuda()[orig.long()]
    pal = torch.from_numpy(misc.label_palette(raw[raw >= 0] if (raw >= 0).any() else np.zeros(1, np.int64))).cuda()
    labels, rgb = ops.cluster_fill(sorted8, box, orig, lab, pal)
    labels.cpu(), rgb.cpu()
    e6.record()
    torch.cuda.synchronize()
    names = ("prepare", "core_distances", "mst", "edge_sort_and_copy")
    out = {k: ev[i].elapsed_time(ev[i + 1]) for i, k in enumerate(names)}
    out.update(host_condense=t_host, fill_colour_and_copy=e5.elapsed_time(e6))
    return out, {"rounds": rounds, "clusters": int(raw.max()) + 1, "noise_fraction": float((raw < 0).mean())}


def main():
    res = {"card": card()}
    sampler = ClockSampler(0)
    sampler.start()
    for name, shape in {"C1_3x336x504": (3, 336, 504), "C2_8x532x532": (8, 532, 532)}.items():
        pts, feats = demo_inputs(shape=shape)
        sm = misc.knn_avg_features_pyg(pts, feats, k=KNN_K)
        x = sm.reshape(-1, 8).contiguous()
        misc.cluster_features_to_masks_mv(sm, apply_colormap=True, **DEMO_KWARGS)      # warm-up
        torch.cuda.synchronize()
        runs = []
        for _ in range(3):
            t0 = time.perf_counter()
            misc.cluster_features_to_masks_mv(sm, apply_colormap=True, **DEMO_KWARGS)
            runs.append((time.perf_counter() - t0) * 1e3)
        parts, info = stages(x, DEMO_KWARGS)
        res[name] = {"points": x.shape[0], "ms_total_median": sorted(runs)[1], "ms_total_runs": runs,
                     "ms_by_stage": parts, **info}
    res["clocks"] = sampler.stop()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
