"""GPU: the track head (SURVEY.md 8f row 4) end to end: the whole `VGGT.forward(images, query_points)` branch
teacher-forced against the fixture of the unmodified reference (the refinement loop is chaotic on synthetic weights, see
tests/test_oracle_track.py), and one free-running iteration.  Each kernel of csrc/track.cu, and the flash-attention
kernel at the update transformer's shapes, is tested element by element in tests/test_track_bounds_gpu.py."""
import os
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

FIX = os.path.join(ROOT, "tests", "golden", "track_vggt_s3_140x154.pt")


def _rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).abs().max() / b.float().abs().max().clamp_min(1e-12)).item()


def test_forward_with_query_points_teacher_forced():
    from oracle import ref_model, ref_track, weights
    from iggt_official_b200.models.vggt import VGGT
    rec = torch.load(FIX)
    c = rec["case"]
    sd = weights.make_state_dict(c["wseed"], c["kind"])
    m = VGGT()
    m.load_state_dict(sd, strict=False)
    m.eval().to("cuda")
    m.compute_dtype = torch.float16
    g = torch.Generator().manual_seed(c["iseed"])
    images = torch.rand(c["S"], 3, c["H"], c["W"], generator=g)
    qp = rec["query_points"]
    # 1. the public call: keys, shapes, frame 0 pinned to the query points
    out = m(images.cuda(), query_points=qp.cuda())
    assert out["track"].shape == (1, c["S"], c["N"], 2) and out["vis"].shape == (1, c["S"], c["N"]) == out["conf"].shape
    assert torch.equal(out["track"][:, 0].cpu(), qp[None]) and torch.isfinite(out["track"]).all()
    # 2. feature extractor against the reference's maps
    tokens, psi = m.aggregator(images.cuda()[None], compute_dtype=torch.float16)
    fm = m.track_head.feature_extractor(tokens, images.cuda()[None], psi, compute_dtype=torch.float16)   # NHWC
    fm_nchw = fm.float().permute(0, 3, 1, 2).view(1, c["S"], 128, *fm.shape[1:3])
    assert _rel(fm_nchw.mean((3, 4)), rec["fmaps_mean"]) < 2e-2
    assert _rel(fm_nchw[..., :4, :4], rec["fmaps_corner"]) < 2e-2
    # 3. every refinement iteration from the reference's own state
    sdt = {k: v for k, v in sd.items() if k.startswith("track_head.")}
    ref_fm = torch.zeros(1)                                                             # only shapes / pos / ref token needed
    st = ref_track.TrackerState(sdt, qp[None].float(), fm_nchw.cpu())
    B, N, S, C = st.B, st.N, st.S, st.C
    tail = (st.pos + st.ref_tok).view(B, N, S, -1)[..., -C:]
    iters = rec["x_in"].shape[0]
    teacher = []
    for i in range(iters):
        coords = st.coords0 if i == 0 else rec["track_all_iters"][i - 1] / ref_track.STRIDE
        teacher.append((coords, (rec["x_in"][i][..., -C:] - tail).permute(0, 2, 1, 3)))
    trace = []
    preds, vis, conf = m.track_head(tokens, images.cuda()[None], psi, query_points=qp[None].cuda(),
                                    compute_dtype=torch.float16, trace=trace, teacher=teacher)
    for i in range(iters):
        assert _rel(trace[i]["x_in"], rec["x_in"][i]) < 3e-2, (i, _rel(trace[i]["x_in"], rec["x_in"][i]))
        assert _rel(trace[i]["delta"], rec["delta"][i]) < 6e-2, (i, _rel(trace[i]["delta"], rec["delta"][i]))
        assert (preds[i].cpu() - rec["track_all_iters"][i]).abs().max().item() < 0.5   # pixels
    assert (vis.cpu() - rec["vis"]).abs().max().item() < 5e-2 and (conf.cpu() - rec["conf"]).abs().max().item() < 5e-2


def test_free_running_first_iteration_and_13_views():
    """(a) One free-running refinement iteration (no teacher forcing: the module's own feature maps, correlation lookup
    and state) against the oracle's tracker run on the SAME 16-bit feature maps - the first iteration is before the
    loop turns chaotic, so it is compared directly.  (b) S = 13 views with query points: the reference's frame-chunk
    path raises for S > 12 (SURVEY F3); here it must simply work, and frame 0 stays pinned to the query points."""
    from oracle import ref_track, weights
    from iggt_official_b200.models.vggt import VGGT
    rec = torch.load(FIX)
    c = rec["case"]
    sd = weights.make_state_dict(c["wseed"], c["kind"])
    m = VGGT()
    m.load_state_dict(sd, strict=False)
    m.eval().to("cuda")
    m.compute_dtype = torch.float16
    g = torch.Generator().manual_seed(c["iseed"])
    images = torch.rand(c["S"], 3, c["H"], c["W"], generator=g).cuda()
    qp = rec["query_points"]
    tokens, psi = m.aggregator(images[None], compute_dtype=torch.float16)
    fm = m.track_head.feature_extractor(tokens, images[None], psi, compute_dtype=torch.float16)
    preds, vis, conf = m.track_head.track(fm, qp[None].cuda(), 1, c["S"], 1, torch.float16)
    sdt = {k: v for k, v in sd.items() if k.startswith("track_head.")}
    fm_nchw = fm.float().permute(0, 3, 1, 2).view(1, c["S"], 128, *fm.shape[1:3]).cpu()
    want, wvis, wconf = ref_track.tracker(sdt, qp[None].float(), fm_nchw, iters=1)
    assert (preds[0].cpu() - want[0]).abs().max().item() < 0.5                     # pixels, after one update
    assert (vis.cpu() - wvis).abs().max().item() < 5e-2 and (conf.cpu() - wconf).abs().max().item() < 5e-2
    g13 = torch.Generator().manual_seed(3)
    imgs13 = torch.rand(13, 3, 140, 154, generator=g13).cuda()
    out = m(imgs13, query_points=qp.cuda())
    assert out["track"].shape == (1, 13, c["N"], 2) and out["vis"].shape == (1, 13, c["N"]) == out["conf"].shape
    assert torch.equal(out["track"][:, 0].cpu(), qp[None]) and torch.isfinite(out["track"]).all()
    assert torch.isfinite(out["vis"]).all() and torch.isfinite(out["conf"]).all()
