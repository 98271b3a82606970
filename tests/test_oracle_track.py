"""The track-head oracle (SURVEY.md 8f row 4) against the fixture produced by the unmodified reference
(`VGGT.forward(images, query_points)`, oracle/make_golden_track.py).  CPU only: this pins the restatement that the native
track head (heads/track_head.py) is tested against in tests/test_track_wiring.py (CPU) and tests/test_track_gpu.py."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_model, ref_track, weights                           # noqa: E402

FIX = os.path.join(ROOT, "tests", "golden", "track_vggt_s3_140x154.pt")


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-12)).item()


def test_track_oracle_matches_reference_fixture():
    """Teacher-forced: the refinement loop is chaotic on synthetic weights (fp32 re-association grows ~100x per
    iteration), so every iteration starts from the REFERENCE's recorded state and must reproduce the reference's
    transformer input, transformer output, new coordinates and final scores."""
    rec = torch.load(FIX)
    c = rec["case"]
    sd = weights.make_state_dict(c["wseed"], c["kind"], prefixes=("aggregator.", "track_head."))
    g = torch.Generator().manual_seed(c["iseed"])
    images = torch.rand(c["S"], 3, c["H"], c["W"], generator=g)[None]
    with torch.no_grad():
        tokens = ref_model.aggregator(sd, images)
        fmaps = ref_track.track_features(sd, tokens, c["H"], c["W"])
        assert _rel(fmaps.mean((3, 4)), rec["fmaps_mean"]) < 2e-5
        assert _rel(fmaps[..., :4, :4], rec["fmaps_corner"]) < 2e-5
        st = ref_track.TrackerState(sd, rec["query_points"][None].float(), fmaps)
        B, N, S, C = st.B, st.N, st.S, st.C
        iters = rec["x_in"].shape[0]
        assert rec["x_in"].shape == (iters, B, N, S, 388) and rec["delta"].shape == (iters, B, N, S, 130)
        tail = (st.pos + st.ref_tok).view(B, N, S, -1)[..., -C:]
        coords = st.coords0.clone()
        for i in range(iters):
            # the reference's own track features of this iteration, recovered from its transformer input
            tf = (rec["x_in"][i][..., -C:] - tail).permute(0, 2, 1, 3)
            if i == 0:
                assert _rel(tf, st.track_feats0) < 1e-5
            x = st.transformer_input(coords, tf)                          # correlation pyramid, corr MLP, embeddings
            assert _rel(x, rec["x_in"][i]) < 1e-4, (i, _rel(x, rec["x_in"][i]))
            delta = ref_track.update_former(sd, "track_head.tracker.updateformer.", rec["x_in"][i])
            assert _rel(delta, rec["delta"][i]) < 1e-4, (i, _rel(delta, rec["delta"][i]))
            new_coords, new_tf = st.apply_delta(coords, tf, rec["delta"][i])
            assert (new_coords * ref_track.STRIDE - rec["track_all_iters"][i]).abs().max().item() < 1e-3   # pixels
            coords = rec["track_all_iters"][i] / ref_track.STRIDE
        vis, conf = st.scores(new_tf)
        assert (vis - rec["vis"]).abs().max().item() < 1e-4 and (conf - rec["conf"]).abs().max().item() < 1e-4
        assert torch.equal(rec["track"], rec["track_all_iters"][-1])
        # free-running: identical in the first iteration, then allowed to drift (chaos), frame 0 stays pinned
        preds, _, _ = ref_track.track_head(sd, tokens, c["H"], c["W"], rec["query_points"])
        assert (preds[0] - rec["track_all_iters"][0]).abs().max().item() < 1e-3
        assert torch.equal(preds[-1][:, 0], rec["query_points"][None])


def test_embedding_layouts():
    """utils.py:18-127: the first half of the 2-D sin/cos channels encodes x (constant along y), the second half y;
    the flow embedding interleaves sin / cos per coordinate."""
    pe = ref_track.sincos_2d(388, 5, 7)
    assert pe.shape == (1, 388, 5, 7) and torch.isfinite(pe).all()
    assert torch.equal(pe[0, :194, 0], pe[0, :194, 4]) and not torch.equal(pe[0, :194, :, 0], pe[0, :194, :, 6])
    assert torch.equal(pe[0, 194:, :, 0], pe[0, 194:, :, 6]) and not torch.equal(pe[0, 194:, 0], pe[0, 194:, 4])
    e = ref_track.embedding_2d(torch.tensor([[[0.0, 0.0], [1.0, -2.0]]]), 64)
    assert e.shape == (1, 2, 128)
    assert torch.equal(e[0, 0, 0::2], torch.zeros(64)) and torch.equal(e[0, 0, 1::2], torch.ones(64))
