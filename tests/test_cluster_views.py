"""Per-view HDBSCAN clustering (utils.misc.cluster_features_to_masks, the reference's iggt/utils/misc.py:174-269):
every view is clustered, noise-filled and coloured on its own, against oracle/ref_cluster_views.py."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_cluster as R                                         # noqa: E402
from oracle import ref_cluster_views as RV                                  # noqa: E402

KW = {"eps": 0.0, "min_samples": 10, "min_cluster_size": 250, "method": "dbscan"}


def separated_view(sizes, seed, dim=5):
    """Well-separated Gaussian blobs (3 apart, spread 0.1) of the given sizes, shuffled: [sum(sizes), dim] fp32."""
    g = np.random.default_rng(seed)
    centres = 3.0 * np.eye(dim)[: len(sizes)]
    x = np.concatenate([c + 0.1 * g.standard_normal((s, dim)) for c, s in zip(centres, sizes)]).astype(np.float32)
    return x[g.permutation(len(x))]


def noise_view(n, seed, dim=5):
    return np.random.default_rng(seed).uniform(-1, 1, (n, dim)).astype(np.float32)


def test_too_small_view_raises_before_any_launch():
    from iggt_official_b200.utils.misc import cluster_features_to_masks as f
    with pytest.raises(ValueError):
        f(np.zeros((3, 2, 2, 8), np.float32), eps=0.1, min_samples=4, min_cluster_size=5)    # 4 pixels per view
    with pytest.raises(ValueError):
        f(np.zeros((4, 8), np.float32), eps=0.1, min_samples=2, min_cluster_size=5)
    with pytest.raises(ValueError):
        f(np.zeros((1, 4, 4, 9), np.float32), eps=0.1, min_samples=2, min_cluster_size=5)
    with pytest.raises(ValueError):
        f(np.zeros((1, 4, 4, 8), np.float32), eps=0.1, min_samples=2)


def test_oracle_colours_each_view_by_its_own_labels():
    masks = np.array([[[0, 1, 1]], [[2, 2, 2]]], np.int64)
    cols = np.stack([R.colorize(masks[i:i + 1])[0] for i in range(2)])
    assert np.array_equal(cols[0, 0, 0], (R.jet(0.0) * 255).astype(np.uint8))
    assert np.array_equal(cols[0, 0, 1], (R.jet(1.0) * 255).astype(np.uint8))
    assert (cols[1] == (R.jet(0.5) * 255).astype(np.uint8)).all()        # a view with one label: jet(0.5)


# ------------------------------------------------------------------------------------------------ GPU

@pytest.mark.gpu
def test_per_view_masks_and_colours_equal_the_oracle():
    """Three views with 2, 5 and 3 clusters: labels (numbering included) and colours exactly as the oracle's, from an
    ndarray and from a CUDA tensor."""
    from iggt_official_b200.utils.misc import cluster_features_to_masks
    views = [separated_view([700, 800], 1), separated_view([300, 280, 320, 290, 310], 2),
             separated_view([500, 450, 550], 3)]
    x = np.stack(views).reshape(3, 30, 50, 5)
    want_m, want_c = RV.cluster_features_to_masks(x, apply_colormap=True, **KW)
    assert [int(want_m[i].max()) + 1 for i in range(3)] == [2, 5, 3]
    for inp in (x, torch.from_numpy(x).cuda()):
        m, c = cluster_features_to_masks(inp, apply_colormap=True, **KW)
        assert m.dtype == np.int32 and m.shape == (3, 30, 50) and c.dtype == np.uint8 and c.shape == (3, 30, 50, 3)
        assert np.array_equal(m, want_m)
        assert np.array_equal(c, want_c)
    m_only = cluster_features_to_masks(x, **KW)
    assert np.array_equal(m_only, want_m)


@pytest.mark.gpu
def test_all_noise_view_becomes_zero_while_others_keep_their_labels():
    from iggt_official_b200.utils.misc import cluster_features_to_masks
    x = np.stack([separated_view([700, 800], 4), noise_view(1500, 5), separated_view([400, 500, 600], 6)])
    assert (R.hdbscan_labels(x[1], KW["eps"], KW["min_samples"], KW["min_cluster_size"]) == -1).all()
    x = x.reshape(3, 1, 1500, 5)
    want_m, want_c = RV.cluster_features_to_masks(x, apply_colormap=True, **KW)
    m, c = cluster_features_to_masks(x, apply_colormap=True, **KW)
    assert (m[1] == 0).all() and (c[1] == (R.jet(0.5) * 255).astype(np.uint8)).all()
    assert m[0].max() == 1 and m[2].max() == 2
    assert np.array_equal(m, want_m) and np.array_equal(c, want_c)


@pytest.mark.gpu
def test_one_view_equals_the_multi_view_call():
    from iggt_official_b200.utils.misc import cluster_features_to_masks, cluster_features_to_masks_mv
    g = np.random.default_rng(9)
    x = np.concatenate([separated_view([600, 700, 800], 7), g.uniform(-0.5, 3.5, (100, 5)).astype(np.float32)])
    x = x[g.permutation(len(x))].reshape(1, 40, 55, 5)
    m1, c1 = cluster_features_to_masks(x, apply_colormap=True, **KW)
    m2, c2 = cluster_features_to_masks_mv(x, apply_colormap=True, **KW)
    assert m1.dtype == np.int32 and m2.dtype == np.int64
    assert np.array_equal(m1, m2) and np.array_equal(c1, c2)
