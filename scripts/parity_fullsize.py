"""GPU: full-size parity report (BASELINE configs) of the native path against the oracle evaluated on the same GPU.
Writes gpurun_out/parity_fullsize.json (copied to profiles/ when judged).   python scripts/parity_fullsize.py [--quick]"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import parity_lib  # noqa: E402

CASES = [
    # model, B, S, H, W, trunk dtype, weights
    ("vggt", 1, 8, 518, 518, "float16", "stress"),      # C2
    ("vggt", 1, 8, 518, 518, "float16", "default"),
    ("vggt", 1, 8, 518, 518, "bfloat16", "stress"),
    ("iggt", 1, 8, 532, 532, "float16", "stress"),      # C2 with the part path (even patch grid)
    ("iggt", 1, 3, 336, 504, "float16", "stress"),      # C1 shape
    ("iggt", 1, 3, 336, 504, "bfloat16", "stress"),
    ("vggt", 2, 4, 518, 518, "bfloat16", "default"),    # C5-shaped (scenes x views), bf16
]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "parity_fullsize.json"))
    args = ap.parse_args()
    rows, models = [], {}
    for kind, B, S, H, W, dt, wk in (CASES[:1] + CASES[4:5] if args.quick else CASES):
        t0 = time.time()
        row = parity_lib.measure(kind, B, S, H, W, getattr(torch, dt), wkind=wk, models=models)
        row["seconds"] = time.time() - t0
        print(json.dumps(row), flush=True)
        rows.append(row)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    json.dump(rows, open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
