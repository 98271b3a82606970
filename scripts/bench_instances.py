"""Instance-mask evaluation (evaluate_matched_instances) timed at the demo shape (3 x 336 x 504) and at C2-with-part
(8 x 532 x 532), with K = P in {32, 128} seeded random masks.

  public_cuda_ms:    the public call from CUDA bool stacks [K, S, H, W] (used in place), host clock around synchronised
                     calls, median of 20 after warm-up;
  public_ndarray_ms: the same from lists of host bool ndarrays (one padded host stack, one copy to the device);
  kernel_ms:         iggt_mask_overlaps alone (CUDA events, median of 20), and its bytes/s against the (K + P) N bytes
                     of the stacks and the 3.35 TB/s of the H100 SXM data sheet;
  assignment_ms:     the host assignment of the K x P cost matrix;
  oracle_numpy_ms:   the numpy oracle (float64 matmul counts + scipy) on the host, at the demo shape only.
The card's name, power limit and the SM clock are read in the same run (bench.py's sampler)."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler                                              # noqa: E402
from iggt_official_b200 import metrics, ops                                 # noqa: E402
from oracle import ref_instances                                            # noqa: E402
from scripts.bench_cluster import card                                      # noqa: E402

REPS = 20
PEAK_BYTES_PER_S = 3.35e12


def host_ms(fn, reps=REPS):
    fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def event_ms(fn, reps=REPS):
    fn()
    t = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        t.append(e0.elapsed_time(e1))
    return float(np.median(t))


def masks(K, shape, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    dens = torch.rand((K, 1, 1, 1), generator=gen, device="cuda") * 0.3
    return torch.rand((K, *shape), generator=gen, device="cuda") < dens


def main():
    res = {"card": card()}
    sampler = ClockSampler(0)
    sampler.start()
    for name, shape in {"C1_3x336x504": (3, 336, 504), "C2_8x532x532": (8, 532, 532)}.items():
        n = int(np.prod(shape))
        for K in (32, 128):
            g, p = masks(K, shape, 1), masks(K, shape, 2)
            gl, pl = list(g.cpu().numpy()), list(p.cpu().numpy())
            g8, p8 = g.view(K, n).view(torch.uint8), p.view(K, n).view(torch.uint8)
            r = {"pixels": n, "K": K, "P": K}
            r["public_cuda_ms"] = host_ms(lambda: metrics.evaluate_matched_instances(g, p))
            r["public_ndarray_ms"] = host_ms(lambda: metrics.evaluate_matched_instances(gl, pl))
            r["kernel_ms"] = event_ms(lambda: ops.mask_overlaps(g8, p8, n))
            r["kernel_bytes_per_s"] = 2 * K * n / (r["kernel_ms"] * 1e-3)
            r["kernel_fraction_of_3.35TBps"] = r["kernel_bytes_per_s"] / PEAK_BYTES_PER_S
            inter, gs, ps = metrics._mask_counts(g, p)
            union = gs[:, None] + ps[None, :] - inter
            cost = 1 - np.where(union > 0, inter / np.maximum(union, 1), 0.0)
            r["assignment_ms"] = host_ms(lambda: ops.linear_sum_assignment(cost))
            if name.startswith("C1"):
                t0 = time.perf_counter()
                ref_instances.evaluate_matched_instances(gl, pl)
                r["oracle_numpy_ms"] = (time.perf_counter() - t0) * 1e3
            res[f"{name}_K{K}"] = r
            del g, p, gl, pl, g8, p8
            torch.cuda.empty_cache()
    res["clocks"] = sampler.stop()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
