"""Drop-in model classes: `IGGT` and `VGGT` with the reference constructor, `forward(images,
query_points=None)` signature, output dictionary and `state_dict` layout (iggt/models/vggt.py:14-230),
running on the sm_90a kernels of this package.

    from iggt_official_b200.models.vggt import IGGT      # instead of iggt.models.vggt
    model = IGGT(); model.load_state_dict(ckpt, strict=False); model.eval().to("cuda")
    with torch.no_grad(), torch.amp.autocast("cuda", dtype=torch.float16):
        predictions = model(images)                       # [S,3,H,W] or [B,S,3,H,W] in [0,1]

Differences from the reference that a caller can observe:
  * CUDA only (no CPU fallback); the trunk's 16-bit compute dtype follows the enclosing autocast (fp16 when there
    is none -- the reference would run fp32).
  * The heads do NOT follow autocast, like the reference's (iggt/models/vggt.py:189 disables it and runs them in
    fp32 with TF32 convolutions): their GEMM / conv operands are fp16 (the same 10-bit mantissa as TF32) with fp32
    accumulation whatever the trunk dtype is.  `model.head_dtype = torch.bfloat16` trades 3 mantissa bits for fp32's
    exponent range; `model.check_finite = True` makes forward raise FloatingPointError when an output is not
    finite (e.g. a checkpoint whose head activations exceed fp16's 65504) instead of returning inf / nan.
  * S > 12 views works (the reference's frame-chunk path raises TypeError, SURVEY F3), and any number of views per
    scene is accepted: the camera head's token attention streams its keys above 196 views, so the view count is
    bounded by device memory only.
  * `query_points` runs the native track head (heads/track_head.py, reference iggt/models/vggt.py:220-226) and adds
    `track`, `vis`, `conf` to the dictionary exactly like the reference; S > 12 works there too.
"""
from typing import Optional

import torch
import torch.nn as nn

from ..heads.camera_head import CameraHead
from ..heads.dpt_head import DPTHead
from ..layout import Node, load_layout, populate
from .aggregator import Aggregator

try:  # the reference mixes this in for from_pretrained / save_pretrained (vggt.py:4,132)
    from huggingface_hub import PyTorchModelHubMixin
except Exception:  # pragma: no cover
    class PyTorchModelHubMixin:  # type: ignore
        pass


class _Base(nn.Module, PyTorchModelHubMixin):
    _with_part = False

    def __init__(self, img_size=518, patch_size=14, embed_dim=1024, only_train_adaptor=False):
        super().__init__()
        entries = load_layout(img_size, patch_size, embed_dim)
        self.aggregator = Aggregator()
        self.camera_head = CameraHead()
        self.point_head = DPTHead(output_dim=4, activation="inv_log", use_point_feat=self._with_part)
        self.depth_head = DPTHead(output_dim=2, activation="exp", use_point_feat=False)
        from ..heads.track_head import TrackHead
        self.track_head = TrackHead()
        if self._with_part:
            from ..heads.part_head import PartAdaptor, PartHead
            self.part_adaptor = PartAdaptor()
            self.part_head = PartHead()
        for name, mod in self.named_children():
            populate(mod, entries, name + ".")
        self.compute_dtype: Optional[torch.dtype] = None     # trunk: None = follow autocast, else fp16
        self.head_dtype: Optional[torch.dtype] = None        # heads: None = fp16 (TF32's mantissa), or torch.bfloat16
        self.check_finite = False                            # raise if an output is inf / nan (costs a sync)
        self.register_load_state_dict_post_hook(lambda module, incompatible: module.invalidate_packed())

    _pack_generation = 0

    def invalidate_packed(self):
        self._pack_generation += 1             # graphs.GraphedForward keys its captured graphs on this
        for m in self.modules():
            if m is not self and hasattr(m, "invalidate"):
                m.invalidate()

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self.invalidate_packed()
        return out

    def _dtype(self):
        if self.compute_dtype is not None:
            return self.compute_dtype
        return torch.get_autocast_dtype("cuda") if torch.is_autocast_enabled("cuda") else torch.float16

    def _head_dtype(self):
        return self.head_dtype if self.head_dtype is not None else torch.float16

    def _check(self, predictions):
        if not self.check_finite:
            return predictions
        for k, v in predictions.items():
            for t in (v if isinstance(v, (list, tuple)) else [v]):
                if torch.is_tensor(t) and t.is_floating_point() and k != "images" and not torch.isfinite(t).all():
                    raise FloatingPointError(
                        f"prediction '{k}' is not finite: head activations left the range of {self._head_dtype()}; "
                        "set model.head_dtype = torch.bfloat16 (fp32's exponent range) for this checkpoint")
        return predictions

    @torch.no_grad()
    def forward(self, images: torch.Tensor, query_points: torch.Tensor = None):
        if len(images.shape) == 4:
            images = images.unsqueeze(0)
        if query_points is not None:
            if len(query_points.shape) == 2:
                query_points = query_points.unsqueeze(0)       # vggt.py:179-180
        dt, hd = self._dtype(), self._head_dtype()
        tokens, psi = self.aggregator(images, compute_dtype=dt)
        predictions = {}
        predictions["pose_enc"] = self.camera_head(tokens, compute_dtype=hd)
        depth, depth_conf = self.depth_head(tokens, images=images, patch_start_idx=psi, compute_dtype=hd)
        predictions["depth"] = depth
        predictions["depth_conf"] = depth_conf
        if self._with_part:
            pts, pconf, point_feat = self.point_head(tokens, images=images, patch_start_idx=psi, compute_dtype=hd)
        else:
            pts, pconf = self.point_head(tokens, images=images, patch_start_idx=psi, compute_dtype=hd)
        predictions["world_points"] = pts
        predictions["world_points_conf"] = pconf
        if self._with_part:
            maps = self.part_adaptor(tokens, images=images, patch_start_idx=psi, compute_dtype=hd)
            predictions["part_feat"] = self.part_head(maps, point_feature=point_feat, images=images,
                                                      patch_start_idx=psi, compute_dtype=hd)
        if query_points is not None:                             # vggt.py:220-226
            track_list, vis, conf = self.track_head(tokens, images=images, patch_start_idx=psi,
                                                    query_points=query_points, compute_dtype=hd)
            predictions["track"] = track_list[-1]
            predictions["vis"] = vis
            predictions["conf"] = conf
        predictions["images"] = images
        return self._check(predictions)


class VGGT(_Base):
    """Reference `VGGT` (iggt/models/vggt.py:14-95): IGGT minus the part path. Its state_dict is the IGGT
    layout without `part_adaptor.*` / `part_head.*`."""
    _with_part = False


class IGGT(_Base):
    """Reference `IGGT` (iggt/models/vggt.py:132-230)."""
    _with_part = True
