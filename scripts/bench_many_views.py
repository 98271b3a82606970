"""Forwards of many views per scene: VGGT at 518 x 518 (fp16 trunk, one scene) for S in {8, 64, 196, 197, 256}, and IGGT
with the part path at 532 x 532 for S in {64, 197}.  196 is the last view count whose camera head runs small_attention;
from 197 on it runs the key-streaming token_attention.  One JSON line per size:

* "ms": host clock around one forward ended by a device synchronise, after one warm-up forward at the same shape
  (median of --steps forwards);
* "views_per_s": S / ms;
* "peak_gb": torch.cuda.max_memory_allocated over the timed forwards, after reset_peak_memory_stats;
* "camera_head_ms": CUDA events around the model's camera_head inside the timed forwards (median);
* "outputs_ok": every output of the last forward has the shape of S views and is finite;
* the card's name, power limit and clocks, read in the same run, and the SM clock sampled during it.

A last line times ops.token_attention against ops.small_attention at the camera head's shapes (H = 16, d = 128) for
N in {64, 196}: CUDA events around 200 launches, median of 5 rounds.

The GPUs may be shared: before each size the free device memory is compared with an estimate from shapes, and the size
is reported as skipped instead of run when it does not fit.

  python scripts/bench_many_views.py [--steps 1] [--sizes 8,64,196,197,256] [--part-sizes 64,197]"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench import ClockSampler                                              # noqa: E402
from bench_pca import card                                                  # noqa: E402
from iggt_official_b200 import ops                                          # noqa: E402
from iggt_official_b200.models.vggt import IGGT, VGGT                       # noqa: E402


def estimate_bytes(S, size, part):
    """device memory a forward needs, from shapes: 16-bit and fp32 weights (7.8 GB), the four fp32 token layers the
    heads read (4 x 2048 x 4 B per token), the trunk's working buffers (about 20 KB per token), the fp32 outputs, and
    2 GB for the heads' per-chunk buffers; the part path adds a third"""
    T = (size // 14) ** 2 + 5
    tokens = S * T
    b = 7.8e9 + tokens * (4 * 2048 * 4 + 20e3) + S * size * size * 4 * (6 + (8 if part else 0)) + 2e9
    return b * (1.3 if part else 1.0)


def time_forward(model, S, size, steps):
    g = torch.Generator().manual_seed(0)
    images = torch.rand(1, S, 3, size, size, generator=g).cuda()
    cam_ms = []
    head = model.camera_head
    orig = head.forward

    def timed_head(*a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = orig(*a, **k)
        e1.record()
        cam_ms.append((e0, e1))
        return out

    with torch.no_grad():
        model(images)                                           # warm-up at this shape
        torch.cuda.synchronize()
        head.forward = timed_head
        torch.cuda.reset_peak_memory_stats()
        ms = []
        try:
            for _ in range(steps):
                t0 = time.perf_counter()
                out = model(images)
                torch.cuda.synchronize()
                ms.append(1e3 * (time.perf_counter() - t0))
        finally:
            head.forward = orig
    cam = sorted(e0.elapsed_time(e1) for e0, e1 in cam_ms)
    ms.sort()
    shapes = {"depth": (1, S, size, size, 1), "depth_conf": (1, S, size, size), "world_points": (1, S, size, size, 3),
              "world_points_conf": (1, S, size, size)}
    ok = all(tuple(out[k].shape) == v and bool(torch.isfinite(out[k]).all()) for k, v in shapes.items())
    ok = ok and len(out["pose_enc"]) == 4 and all(tuple(p.shape) == (1, S, 9) and bool(torch.isfinite(p).all())
                                                  for p in out["pose_enc"])
    if "part_feat" in out:
        ok = ok and out["part_feat"].shape[:2] == (1, S) and bool(torch.isfinite(out["part_feat"]).all())
    return ms[len(ms) // 2], cam[len(cam) // 2], torch.cuda.max_memory_allocated() / 1e9, ok


def attention_ab(N, launches=200, rounds=5):
    """median ms per launch of token_attention and small_attention on the same qkv [N, 3 * 2048]"""
    qkv = torch.randn(N, 3 * 2048, device="cuda", generator=torch.Generator(device="cuda").manual_seed(N))
    res = {}
    for name in ("small_attention", "token_attention"):
        fn = getattr(ops, name)
        for _ in range(10):
            fn(qkv, 1, N, 16, 128)
        per = []
        for _ in range(rounds):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(launches):
                fn(qkv, 1, N, 16, 128)
            e1.record()
            e1.synchronize()
            per.append(e0.elapsed_time(e1) / launches)
        per.sort()
        res[name] = round(per[len(per) // 2], 4)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--sizes", default="8,64,196,197,256")
    ap.add_argument("--part-sizes", default="64,197")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    info = card()
    runs = [(False, int(s), 518) for s in args.sizes.split(",") if s] + \
           [(True, int(s), 532) for s in args.part_sizes.split(",") if s]
    models = {}
    for part, S, size in runs:
        line = {"model": "IGGT+part" if part else "VGGT", "views": S, "image": size, "dtype": "fp16",
                "camera_attention": "small_attention" if ops._small_attention_fits(S, 128) else "token_attention",
                "card": info}
        if part not in models:
            models.clear()
            torch.cuda.empty_cache()
            torch.manual_seed(0)
            m = (IGGT if part else VGGT)().eval().cuda()
            m.compute_dtype = torch.float16
            models[part] = m
        free, _ = torch.cuda.mem_get_info()
        need = estimate_bytes(S, size, part)
        line["free_gb"], line["estimate_gb"] = round(free / 1e9, 1), round(need / 1e9, 1)
        if need > free + torch.cuda.memory_reserved() - torch.cuda.memory_allocated():
            line["skipped"] = "not enough free memory"
            print(json.dumps(line), flush=True)
            continue
        clk = ClockSampler()
        clk.start()
        ms, cam, peak, ok = time_forward(models[part], S, size, args.steps)
        line.update({"outputs_ok": ok, "ms": round(ms, 1), "views_per_s": round(S / ms * 1e3, 2), "camera_head_ms": round(cam, 2),
                     "camera_head_share": round(cam / ms, 4), "peak_gb": round(peak, 2), "steps": args.steps,
                     "clocks": clk.stop()})
        print(json.dumps(line), flush=True)
        torch.cuda.empty_cache()
    models.clear()
    torch.cuda.empty_cache()
    print(json.dumps({"attention_ms_per_launch": {N: attention_ab(N) for N in (64, 196)}, "card": info}), flush=True)


if __name__ == "__main__":
    main()
