"""tests/golden/instances_ref.npz: the UNMODIFIED reference calculate_iou / evaluate_matched_instances
(iggt/metrics.py:16-80) on seeded instance masks.

The reference module is loaded as oracle/make_golden_eval.py loads it (reference_modules()).  The masks are
regenerated from their seeds by the tests (case_masks(), CASES, IOU_PAIRS); the results are stored as JSON with a type
tag on every value (tagged()), so the tests check the result types too.
Run once:  python -m oracle.make_golden_instances"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden", "instances_ref.npz")

SHAPE = (2, 23, 31)          # [S, H, W]: N = 1426 pixels, not a multiple of 16


def blob_labels(rng, centers, shape=SHAPE, radius=7.0):
    """Label map [S,H,W] int64: each pixel takes the index of its nearest centre (centres [S, c, 2] per view, in
    (y, x)), -1 where that centre is farther than `radius`."""
    S, H, W = shape
    yy, xx = np.mgrid[:H, :W]
    d2 = (yy[None, None] - centers[:, :, 0, None, None]) ** 2 + (xx[None, None] - centers[:, :, 1, None, None]) ** 2
    lab = d2.argmin(1)
    lab[d2.min(1) > radius ** 2] = -1
    return lab


def blob_masks(seed, K, P, shape=SHAPE):
    """K gt masks from a seeded blob label map and P predicted ones from a perturbed copy of it (the first min(K, P)
    centres moved by about a pixel, the rest new); a label no pixel takes gives an all-False mask."""
    rng = np.random.default_rng(seed)
    S, H, W = shape
    gc = rng.uniform((0, 0), (H, W), (S, K, 2))
    pc = rng.uniform((0, 0), (H, W), (S, P, 2))
    m = min(K, P)
    pc[:, :m] = gc[:, :m] + rng.normal(0, 1.2, (S, m, 2))
    g, p = blob_labels(rng, gc, shape), blob_labels(rng, pc, shape, radius=7.5)
    return [g == k for k in range(K)], [p == k for k in range(P)]


def case_masks(name):
    kind, args, _ = CASES[name]
    if kind == "blobs":
        return blob_masks(*args)
    if kind == "empty":
        g, p = blob_masks(11, 4, 5)
        return ([], p) if args == "gt" else (g, [])
    if kind == "dups":                    # duplicated masks, exact gt copies among the predictions, all-False ones
        g, p = blob_masks(12, 6, 6)
        z = np.zeros(SHAPE, bool)
        return [g[0], g[1], g[1], g[2], z, g[3]], [g[1], p[1], g[0], z, p[2], g[1], p[0], p[4]]
    if kind == "disjoint":                # gt only in view 0, pred only in view 1: every IoU is 0 (cost 1 everywhere)
        K, P = args
        g, _ = blob_masks(13, K, 1)
        _, p = blob_masks(14, 1, P)
        for m in g:
            m[1] = False
        for m in p:
            m[0] = False
        return g, p
    raise KeyError(name)


CASES = {   # name: (kind, args, iou_threshold)
    "k_lt_p": ("blobs", (1, 6, 9), 0.5),
    "k_gt_p": ("blobs", (2, 11, 5), 0.5),
    "k_eq_p": ("blobs", (3, 8, 8), 0.5),
    "k_lt_p_thr0": ("blobs", (4, 7, 10), 0.0),
    "k_gt_p_thr0": ("blobs", (5, 10, 7), 0.0),
    "k_eq_p_thr1": ("blobs", (6, 9, 9), 1.0),
    "empty_gt": ("empty", "gt", 0.5),
    "empty_pred": ("empty", "pred", 0.5),
    "dups": ("dups", None, 0.5),
    "dups_thr0": ("dups", None, 0.0),
    "dups_thr1": ("dups", None, 1.0),
    "disjoint_wide": ("disjoint", (3, 6), 0.0),
    "disjoint_tall": ("disjoint", (6, 3), 0.0),
    "disjoint_half": ("disjoint", (5, 5), 0.5),
}

IOU_PAIRS = [("k_eq_p", 0, 0), ("k_eq_p", 1, 3), ("dups", 1, 0), ("dups", 4, 3), ("dups", 0, 2), ("disjoint_wide", 0, 0)]


def tagged(o):
    """A result as JSON-able data with the type of every value: ["f64", x] for np.float64, ["float", x], ["i64", i],
    ["int", i], ["tuple", [...]], lists and dicts as they are."""
    if isinstance(o, np.float64):
        return ["f64", float(o)]
    if isinstance(o, np.int64):
        return ["i64", int(o)]
    if isinstance(o, bool):
        return ["bool", o]
    if isinstance(o, float):
        return ["float", o]
    if isinstance(o, int):
        return ["int", o]
    if isinstance(o, tuple):
        return ["tuple", [tagged(v) for v in o]]
    if isinstance(o, list):
        return [tagged(v) for v in o]
    if isinstance(o, dict):
        return {k: tagged(v) for k, v in o.items()}
    raise TypeError(type(o))


if __name__ == "__main__":
    from oracle.make_golden_eval import reference_modules
    ref_metrics = reference_modules()[0]
    out = {}
    for name, (_, _, thr) in CASES.items():
        g, p = case_masks(name)
        out[f"{name}_result"] = np.array(json.dumps(tagged(ref_metrics.evaluate_matched_instances(g, p, thr))))
    ious = []
    for name, i, j in IOU_PAIRS:
        g, p = case_masks(name)
        ious.append(tagged(ref_metrics.calculate_iou(g[i], p[j])))
    out["iou_pairs"] = np.array(json.dumps(ious))
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")
