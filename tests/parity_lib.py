"""TEST INFRASTRUCTURE (GPU): full-size parity of the native forward against oracle/ref_model.py evaluated on the same
device.  For one configuration `measure()` returns, per output key, the relative L2 / max distances

  vs_amp   product  vs  oracle(amp = trunk dtype, heads fp32)        <- the parity number
  vs_fp32  product  vs  oracle(fp32 everywhere)
  gap_amp  oracle(amp) vs oracle(fp32)      the reference's own autocast-vs-fp32 gap on these inputs
  gap_tf32 oracle(amp, cuDNN TF32 convolutions = PyTorch's default on GPU, which is what the reference's heads run
           under iggt/models/vggt.py:189) vs oracle(amp, exact-fp32 convolutions)

so that a tolerance can be stated in units of the noise two independent 16-bit realisations of the same network have
between them.  Used by tests/test_fullsize_parity_gpu.py (asserts) and scripts/parity_fullsize.py (report)."""
import torch

from oracle import ref_model, weights

KEYS = ("depth", "depth_conf", "world_points", "world_points_conf", "part_feat")


def rel_l2(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


def rel_max(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-12)).item()


def _oracle(sd, images, kind, amp, tf32):
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return ref_model.forward(sd, images, model=kind, amp=amp, frames_chunk=2, skip_part=(kind != "iggt"))
    finally:
        torch.backends.cudnn.allow_tf32 = False


def measure(kind, B, S, H, W, dtype, wkind="stress", wseed=1, models=None, with_tf32_gap=True):
    from iggt_official_b200.models.vggt import IGGT, VGGT
    dev = torch.device("cuda")
    prefixes = ("aggregator.", "camera_head.", "depth_head.", "point_head.") + (("part_adaptor.", "part_head.") if kind == "iggt" else ())
    sd = weights.make_state_dict(wseed, wkind, prefixes=prefixes)
    if models is not None and kind in models:
        model = models[kind]
    else:
        model = (IGGT if kind == "iggt" else VGGT)()
        if models is not None:
            models[kind] = model
    model.load_state_dict(sd, strict=False)
    model.eval().to(dev)
    model.compute_dtype = dtype
    g = torch.Generator().manual_seed(B * 1000 + S * 100 + H)
    images = torch.rand(B, S, 3, H, W, generator=g).to(dev)
    out = model(images)
    torch.cuda.synchronize()
    out = {k: (torch.stack(v) if isinstance(v, list) else v).float().cpu() for k, v in out.items() if k != "images"}
    sdg = {k: v.to(dev) for k, v in sd.items()}
    refs = {}
    for name, amp, tf32 in (("fp32", None, False), ("amp", dtype, False)) + ((("amp_tf32", dtype, True),) if with_tf32_gap else ()):
        r = _oracle(sdg, images, kind, amp, tf32)
        refs[name] = {k: (torch.stack(v) if isinstance(v, list) else v).float().cpu() for k, v in r.items() if k != "images"}
        del r
        torch.cuda.empty_cache()
    row = {"model": kind, "shape": [B, S, H, W], "dtype": str(dtype).replace("torch.", ""), "weights": f"{wkind}/{wseed}"}
    for k in KEYS + ("pose_enc",):
        if k not in out or k not in refs["amp"]:
            continue
        e = {"vs_amp_l2": rel_l2(out[k], refs["amp"][k]), "vs_amp_max": rel_max(out[k], refs["amp"][k]),
             "vs_fp32_l2": rel_l2(out[k], refs["fp32"][k]), "gap_amp_l2": rel_l2(refs["amp"][k], refs["fp32"][k]),
             "gap_amp_max": rel_max(refs["amp"][k], refs["fp32"][k])}
        if with_tf32_gap:
            e["gap_tf32_l2"] = rel_l2(refs["amp_tf32"][k], refs["amp"][k])
        row[k] = e
    return row
