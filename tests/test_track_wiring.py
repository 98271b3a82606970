"""Host-side wiring of the native track head (heads/track_head.py) WITHOUT a GPU: the C-ABI launchers are replaced by
their plain-PyTorch statements (tests/emu_ops.py) and the module is driven teacher-forced against the fixture of the
unmodified reference.  This pins row orders, the 48->64 head padding, the K / N zero padding, the separable positional
embedding and the update-transformer plumbing; the CUDA kernels themselves are compared with the same statements in
the GPU tests."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import emu_ops                                                              # noqa: E402
from oracle import ref_model, ref_track, weights                           # noqa: E402

FIX = os.path.join(ROOT, "tests", "golden", "track_vggt_s3_140x154.pt")


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-12)).item()


def test_track_module_wiring_teacher_forced(monkeypatch):
    from iggt_official_b200.heads import track_head as TH
    from iggt_official_b200.layout import load_layout, populate
    rec = torch.load(FIX)
    c = rec["case"]
    sd = weights.make_state_dict(c["wseed"], c["kind"], prefixes=("aggregator.", "track_head."))
    head = TH.TrackHead()
    populate(head, load_layout(), "track_head.")
    missing, unexpected = head.load_state_dict({k[len("track_head."):]: v for k, v in sd.items() if k.startswith("track_head.")})
    assert not missing and not unexpected
    for name in ("gemm_store16", "gemm_store32", "gemm_resid32", "attention", "layernorm16", "layernorm_rows",
                 "avgpool2_nhwc", "sample_bilinear_nhwc", "corr_sample", "track_input"):
        monkeypatch.setattr(TH.ops, name, getattr(emu_ops, name))
    g = torch.Generator().manual_seed(c["iseed"])
    images = torch.rand(c["S"], 3, c["H"], c["W"], generator=g)[None]
    with torch.no_grad():
        tokens = ref_model.aggregator(sd, images)
        fmaps = ref_track.track_features(sd, tokens, c["H"], c["W"])                    # [B,S,128,HH,WW] fp32
        st = ref_track.TrackerState(sd, rec["query_points"][None].float(), fmaps)
        B, N, S, C = st.B, st.N, st.S, st.C
        tail = (st.pos + st.ref_tok).view(B, N, S, -1)[..., -C:]
        iters = rec["x_in"].shape[0]
        teacher = []
        for i in range(iters):                                                           # the reference's own states
            coords = st.coords0 if i == 0 else rec["track_all_iters"][i - 1] / ref_track.STRIDE
            tf = (rec["x_in"][i][..., -C:] - tail).permute(0, 2, 1, 3)
            teacher.append((coords, tf))
        trace = []
        nhwc = fmaps.view(B * S, C, *fmaps.shape[-2:]).permute(0, 2, 3, 1).contiguous()  # "16-bit" maps kept in fp32
        preds, vis, conf = head.track(nhwc, rec["query_points"][None], B, S, iters, torch.float32, trace, teacher)
    for i in range(iters):
        assert _rel(trace[i]["x_in"], rec["x_in"][i]) < 1e-4, (i, _rel(trace[i]["x_in"], rec["x_in"][i]))
        assert _rel(trace[i]["delta"], rec["delta"][i]) < 2e-4, (i, _rel(trace[i]["delta"], rec["delta"][i]))
        assert (preds[i] - rec["track_all_iters"][i]).abs().max().item() < 2e-3        # pixels
    assert preds[-1].shape == rec["track"].shape and torch.equal(preds[-1][:, 0], rec["query_points"][None])
    assert (vis - rec["vis"]).abs().max().item() < 1e-4 and (conf - rec["conf"]).abs().max().item() < 1e-4


def test_query_points_run_by_default():
    """The track branch is on by default (reference: iggt/models/vggt.py:220-226): with CPU tensors the call reaches
    the CUDA-only guard of the hot path instead of a NotImplementedError / an opt-in switch."""
    import pytest
    from iggt_official_b200.models.vggt import VGGT
    with pytest.raises(RuntimeError, match="CUDA"):
        VGGT()(torch.zeros(2, 3, 28, 28), query_points=torch.zeros(3, 2))


def test_corr_lookup_without_the_volume_equals_volume_sampling():
    """The kernel's formulation (dot products on the integer pixels under the window, interpolated afterwards) against
    the reference's (sample the full correlation volume), down to 1 x 1, 1 x 2 and 2 x 1 pyramid levels."""
    g = torch.Generator().manual_seed(2)
    B, N, S = 1, 4, 2
    rows = B * N * S
    for h, w in ((70, 77), (64, 130), (130, 64)):
        lv = [torch.randn(B * S, h, w, 128, generator=g)]
        for _ in range(6):
            lv.append(emu_ops.avgpool2_nhwc(lv[-1]))
        targets = torch.randn(rows, 128, generator=g)
        coords = torch.rand(rows, 2, generator=g) * torch.tensor([w + 3.0, h + 4.0]) - 2.0   # windows hang over every border
        coords[0] = torch.tensor([0.0, 0.0])
        coords[1] = torch.tensor([w - 1.0, h - 1.0])
        a = emu_ops.corr_sample(lv, targets, coords, B, N, S)
        b = emu_ops.corr_sample_direct(lv, targets, coords, B, N, S)
        for lvl in range(7):
            blk = slice(lvl * 81, (lvl + 1) * 81)
            assert (a[:, blk] - b[:, blk]).abs().max().item() < 1e-4 * max(a[:, blk].abs().max().item(), 1e-3), (h, w, lvl)
