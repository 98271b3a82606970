"""tests/golden/cluster_demo.npz: the oracle's HDBSCAN labels for a seeded, demo-shaped feature map (3 x 336 x 504).

`demo_inputs` builds un-projected-depth-like points and unit 8-d part features whose instances are 3-D regions seen
by every view; the features are smoothed over the k = 20 nearest 3-D points (oracle/ref_knn.py) and clustered with
the demo's parameters (demo.py:78-83).  Only labels are stored: the GPU test regenerates the features from the seed.
scikit-learn's HDBSCAN takes tens of minutes on this many points; run once:  python -m oracle.make_golden_cluster"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DEMO_KWARGS = {"eps": 0.06, "min_samples": 100, "min_cluster_size": 500}
SEED, SHAPE, KNN_K = 11, (3, 336, 504), 20
OUT = os.path.join(ROOT, "tests", "golden", "cluster_demo.npz")


def demo_inputs(seed=SEED, shape=SHAPE, n_objects=10, noise=0.08, outliers=0.01):
    """points [S,H,W,3] and unit features [S,H,W,8] (float32).  Instances are the 3-D Voronoi cells of n_objects sites;
    each instance has a random unit feature centre, and far outliers carry random unit features."""
    g = np.random.default_rng(seed)
    s_, h, w = shape
    v, u = np.mgrid[0:h, 0:w].astype(np.float32)
    pts = []
    for s in range(s_):
        z = 2.0 + 0.8 * np.sin(u / 17 + s) + 0.5 * np.cos(v / 11) + 0.02 * g.standard_normal((h, w))
        far = g.random((h, w)) < outliers
        z = np.where(far, z * g.uniform(20, 200, (h, w)), z).astype(np.float32)
        pts.append(np.stack([(u - w / 2) / w * z + 0.3 * s, (v - h / 2) / w * z, z], -1))
    pts = np.stack(pts).astype(np.float32)
    sites = np.stack([g.uniform(-1.0, 1.6, n_objects), g.uniform(-0.6, 0.6, n_objects), g.uniform(1.0, 3.5, n_objects)], 1)
    d2 = ((pts.reshape(-1, 1, 3) - sites[None].astype(np.float32)) ** 2).sum(-1)
    obj = d2.argmin(1)
    centres = g.standard_normal((n_objects, 8))
    centres /= np.linalg.norm(centres, axis=1, keepdims=True)
    feats = centres[obj] + noise * g.standard_normal((obj.size, 8))
    far = pts.reshape(-1, 3)[:, 2] > 8.0
    feats[far] = g.standard_normal((int(far.sum()), 8))
    feats /= np.linalg.norm(feats, axis=1, keepdims=True)
    return pts, feats.astype(np.float32).reshape(*shape, 8)


if __name__ == "__main__":
    from oracle import ref_cluster, ref_knn
    pts, feats = demo_inputs()
    t0 = time.time()
    sm = ref_knn.knn_avg_features(pts, feats, KNN_K)
    t1 = time.time()
    x = sm.reshape(-1, 8)
    raw = ref_cluster.hdbscan_labels(x, **DEMO_KWARGS)
    t2 = time.time()
    filled = ref_cluster.fill_noise(x, raw)
    print(f"knn {t1 - t0:.1f} s, hdbscan {t2 - t1:.1f} s on {x.shape[0]} points: {raw.max() + 1} clusters, "
          f"{(raw == -1).mean():.4f} noise")
    np.savez_compressed(OUT, labels_raw=raw.astype(np.int16), labels=filled.astype(np.int16),
                        seed=SEED, shape=np.array(SHAPE), knn_k=KNN_K)
    print("wrote", OUT)
