"""apply_pca_colormap timed at the demo shape (3 x 336 x 504), at C2-with-part (8 x 532 x 532) and at 16 x 1036 x 1036
(17.2 M pixels, where the reference's torch.quantile raises), all with C = 8.

"total": the median of 25 calls of the public function on a CUDA tensor, each ended by a device synchronise, after
three warm-up calls.  "stages": CUDA events around each stage of the same pipeline (median of 25), with the bytes each
stage must move and the share of the H100 SXM data sheet's 3.35 TB/s that this is.  The card's name, power limit and
clocks are read in the same run; the SM clock is sampled during the run as bench.py samples it.  "ref_pca_cpu_s" is
the float64 oracle (oracle/ref_pca.py) on the host CPU, for context only.  The first two shapes use
oracle/make_golden_cluster.demo_inputs' unit features; the third uses seeded Gaussian features mixed by a random 8x8
matrix, generated on the device."""
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
from oracle import ref_pca                                                  # noqa: E402
from oracle.make_golden_cluster import demo_inputs                          # noqa: E402

PEAK_BW = 3.35e12
REPS = 25


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=20).stdout.strip().splitlines()[0]
    return dict(zip(("name", "power_limit", "sm_clock", "sm_max_clock"), [f.strip() for f in out.split(",")]))


def stage_bytes(n, C):
    """Bytes each stage must move: basis reads x once; project reads x and writes y [3, n]; the quantile reads y in
    three radix passes; the stretch reads y and writes out [n, 3]."""
    return {"basis": 4.0 * n * C, "project": 4.0 * n * C + 12.0 * n, "quantile": 3 * 12.0 * n, "stretch": 24.0 * n}


def stages(x):
    """One pipeline run with CUDA events: "basis" = moments pass + one-CTA reduction and Jacobi."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
    ev[0].record()
    b = ops.pca_basis(x)
    ev[1].record()
    b.nonfinite.item()
    ev[2].record()
    y = ops.pca_project(x, b.V)
    ev[3].record()
    qv = ops.quantile(y, (0.02, 0.98))
    ev[4].record()
    ops.pca_stretch(y, qv)
    ev[5].record()
    torch.cuda.synchronize()
    names = ("basis", "host_sync", "project", "quantile", "stretch")
    return {k: ev[i].elapsed_time(ev[i + 1]) for i, k in enumerate(names)}


def main():
    res = {"card": card()}
    sampler = ClockSampler(0)
    sampler.start()
    shapes = {"demo_3x336x504": (3, 336, 504), "C2_8x532x532": (8, 532, 532), "big_16x1036x1036": (16, 1036, 1036)}
    for name, shape in shapes.items():
        if name.startswith("big"):
            g = torch.Generator(device="cuda").manual_seed(16)
            mix = torch.randn(8, 8, device="cuda", generator=g)
            x = (torch.randn(int(np.prod(shape)), 8, device="cuda", generator=g) @ mix).view(*shape, 8)
        else:
            x = torch.from_numpy(demo_inputs(shape=shape)[1]).cuda()
        n = x.numel() // 8
        for _ in range(3):
            misc.apply_pca_colormap(x)
        torch.cuda.synchronize()
        runs = []
        for _ in range(REPS):
            t0 = time.perf_counter()
            misc.apply_pca_colormap(x)
            torch.cuda.synchronize()
            runs.append((time.perf_counter() - t0) * 1e3)
        flat = x.view(-1, 8)
        per = [stages(flat) for _ in range(REPS)]
        st = {k: float(np.median([p[k] for p in per])) for k in per[0]}
        nbytes = stage_bytes(n, 8)
        share = {k: (nbytes[k] / (st[k] * 1e-3)) / PEAK_BW for k in nbytes}
        entry = {"pixels": n, "ms_total_median": float(np.median(runs)), "ms_total_min": float(min(runs)),
                 "ms_by_stage_median": st, "bytes_by_stage": nbytes, "share_of_3.35TBps": share}
        if not name.startswith("big"):
            xc = x.cpu().numpy()
            t0 = time.perf_counter()
            ref_pca.apply_pca_colormap(xc)
            entry["ref_pca_cpu_s"] = time.perf_counter() - t0
        res[name] = entry
        del x, flat
        torch.cuda.empty_cache()
    res["clocks"] = sampler.stop()
    res["card_after"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
