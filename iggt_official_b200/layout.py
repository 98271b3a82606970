"""Checkpoint (`state_dict`) layout of the reference `IGGT` module tree and a builder that materialises
it as nested nn.Modules, so `load_state_dict` / `utils/model.py:align_and_update_state_dicts` /
`PyTorchModelHubMixin` keep working against the native implementation (SURVEY.md section 8b, Appendix C).

`state_layout.json` lists the 2053 (name, shape, dtype) entries of `IGGT().state_dict()` for the default
constructor arguments (img_size 518, patch 14, embed_dim 1024); tests/test_layout.py checks it against the
manifest extracted from the unmodified reference.
"""
import json
import math
import os

import torch
import torch.nn as nn

_HERE = os.path.dirname(os.path.abspath(__file__))
_BUFFER_LEAVES = ("running_mean", "running_var", "num_batches_tracked", "relative_position_index_SA",
                  "relative_position_index_OCA")


def load_layout(img_size=518, patch_size=14, embed_dim=1024):
    if patch_size != 14 or embed_dim != 1024:
        raise NotImplementedError("the native kernels are specialised for patch_size=14, embed_dim=1024 "
                                  "(the only configuration the reference checkpoint uses)")
    with open(os.path.join(_HERE, "state_layout.json")) as f:
        entries = [(k, tuple(s), getattr(torch, d)) for k, s, d in json.load(f)]
    n_pos = 1 + (img_size // patch_size) ** 2
    return [(k, (1, n_pos, embed_dim) if k == "aggregator.patch_embed.pos_embed" else s, d) for k, s, d in entries]


def calculate_rpi_sa(ws=8):
    """Relative-position index of an 8x8 window (reference buffer `relative_position_index_SA`,
    iggt/heads/window_sa.py:379-391)."""
    c = torch.stack(torch.meshgrid(torch.arange(ws), torch.arange(ws), indexing="ij")).flatten(1)
    rel = (c[:, :, None] - c[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += ws - 1
    rel[:, :, 1] += ws - 1
    rel[:, :, 0] *= 2 * ws - 1
    return rel.sum(-1)


def calculate_rpi_oca(ws=8, overlap_ratio=0.5):
    """Index of the 8x8 query window against its 12x12 overlapping key window (reference buffer
    `relative_position_index_OCA`, iggt/heads/window_sa.py:497-523; contains negative entries that wrap)."""
    wse = ws + int(overlap_ratio * ws)
    co = torch.stack(torch.meshgrid(torch.arange(ws), torch.arange(ws), indexing="ij")).flatten(1)
    ce = torch.stack(torch.meshgrid(torch.arange(wse), torch.arange(wse), indexing="ij")).flatten(1)
    rel = (ce[:, None, :] - co[:, :, None]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += ws - wse + 1
    rel[:, :, 1] += ws - wse + 1
    rel[:, :, 0] *= ws + wse - 1
    return rel.sum(-1)


class Node(nn.Module):
    """Plain container; children / parameters are attached by `populate`."""


def _init_tensor(name, shape, dtype):
    leaf = name.rsplit(".", 1)[-1]
    if dtype == torch.int64:
        if leaf == "relative_position_index_SA":
            return calculate_rpi_sa(8)
        if leaf == "relative_position_index_OCA":
            return calculate_rpi_oca(8)
        return torch.zeros(shape, dtype=dtype)
    if leaf == "gamma":
        return torch.full(shape, 1.0 if name.startswith("aggregator.patch_embed.") else 0.01)
    if leaf == "running_var" or (len(shape) == 1 and leaf == "weight"):
        return torch.ones(shape)
    if leaf in ("bias", "running_mean", "empty_pose_tokens", "mask_token"):
        return torch.zeros(shape)
    if leaf in ("camera_token", "register_token", "cls_token", "register_tokens"):
        return torch.randn(shape) * 1e-6
    if len(shape) >= 2:
        fan_in = 1
        for s in shape[1:]:
            fan_in *= s
        return torch.randn(shape) / math.sqrt(max(fan_in, 1)) if leaf != "pos_embed" else torch.randn(shape) * 0.02
    return torch.zeros(shape)


def populate(root: nn.Module, entries, prefix: str):
    """Attach every layout entry under `prefix` to `root` (creating intermediate Node containers)."""
    for name, shape, dtype in entries:
        if not name.startswith(prefix):
            continue
        parts = name[len(prefix):].split(".")
        mod = root
        for p in parts[:-1]:
            if p not in mod._modules:
                mod.add_module(p, Node())
            mod = mod._modules[p]
        t = _init_tensor(name, shape, dtype)
        if parts[-1] in _BUFFER_LEAVES:
            mod.register_buffer(parts[-1], t)
        else:
            mod.register_parameter(parts[-1], nn.Parameter(t, requires_grad=False))
