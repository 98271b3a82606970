"""tests/golden/pca_ref.npz: the UNMODIFIED reference apply_pca_colormap (iggt/utils/misc.py:272-332) on seeded
features.

The reference module imports matplotlib, torch_geometric, torch_scatter, hdbscan / cuML and, through
iggt/utils/vo_eval.py, evo at import time; apply_pca_colormap uses none of them.  They are stubbed here as far as the
import needs (in the style of oracle/shims.py), and the function runs under torch.manual_seed(0) on the CPU, as the
unmodified demo runs it.  Stored: the full output at 2 x 48 x 64 and a seeded sample of 4096 pixels at the demo shape
(3 x 336 x 504), both from oracle/make_golden_cluster.demo_inputs' unit 8-d features; the tests regenerate the inputs
from the seeds.  Run once:  python -m oracle.make_golden_pca"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, "tests", "golden", "pca_ref.npz")
SMALL_SEED, SMALL_SHAPE = 3, (2, 48, 64)
DEMO_SEED, DEMO_SHAPE = 11, (3, 336, 504)
SAMPLE_SEED, SAMPLE = 7, 4096

_STUBS = ("matplotlib", "matplotlib.cm", "matplotlib.pyplot", "torch_geometric", "torch_geometric.nn",
          "torch_scatter", "hdbscan", "evo", "evo.main_ape", "evo.main_rpe", "evo.core", "evo.core.sync",
          "evo.core.metrics", "evo.core.trajectory", "evo.tools", "evo.tools.file_interface", "evo.tools.plot")


class _Stub(types.ModuleType):
    """A module whose every attribute is a placeholder: enough for `from m import name` at import time."""

    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return lambda *a, **k: None


def install_stubs():
    for name in _STUBS:
        if name not in sys.modules:
            sys.modules[name] = _Stub(name)
    for name in _STUBS:                                   # parents expose their stubbed children as attributes
        parent, _, child = name.rpartition(".")
        if parent:
            setattr(sys.modules[parent], child, sys.modules[name])


def reference_apply_pca_colormap():
    from oracle.shims import REFERENCE_ROOT
    install_stubs()
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    from iggt.utils.misc import apply_pca_colormap
    return apply_pca_colormap


def features(seed, shape):
    from oracle.make_golden_cluster import demo_inputs
    return demo_inputs(seed=seed, shape=shape)[1]


def sample_index(n):
    return np.sort(np.random.default_rng(SAMPLE_SEED).choice(n, SAMPLE, replace=False))


if __name__ == "__main__":
    import torch
    f = reference_apply_pca_colormap()
    small = features(SMALL_SEED, SMALL_SHAPE)
    torch.manual_seed(0)
    out_small = f(torch.from_numpy(small)).numpy()
    demo = features(DEMO_SEED, DEMO_SHAPE)
    torch.manual_seed(0)
    out_demo = f(torch.from_numpy(demo)).numpy().reshape(-1, 3)
    idx = sample_index(out_demo.shape[0])
    np.savez_compressed(OUT, small=out_small.astype(np.float32), small_seed=SMALL_SEED, small_shape=np.array(SMALL_SHAPE),
                        demo_idx=idx.astype(np.int32), demo_sample=out_demo[idx].astype(np.float32), demo_seed=DEMO_SEED,
                        demo_shape=np.array(DEMO_SHAPE))
    print("wrote", OUT, os.path.getsize(OUT), "bytes")
