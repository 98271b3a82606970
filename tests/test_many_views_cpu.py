"""Scenes of more views than the camera head's small_attention holds (197 and up), without a GPU:

* the tile walk of `token_attention_kernel` in fp32 torch (tests/token_attention_ref.py) stays inside the per-element
  bound tests/test_many_views_gpu.py holds the kernel to, at every shape that test runs, and the bound rejects the same
  walk with one rescale left out (so it is not vacuous);
* `ops.token_attention` refuses the arguments its launcher refuses with a ValueError, before any device work;
* the model graph with emulated launchers reaches `token_attention` at 197 views and equals the same graph with an
  unbounded small_attention forced in; the view-sharded forward (gloo, 2 ranks x 100 views) equals the unsharded one.
"""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import token_attention_ref as ta                                            # noqa: E402

KERNEL_N = [1, 2, 33, 63, 64, 65, 196, 197, 256, 257, 500, 1000, 2049]       # tests/test_many_views_gpu.py
ADVERSARIAL_N = [197, 257, 1000]
H, D = 16, 128


def token_attention_emu(qkv, B, N, H, d):
    """the launcher replaced by the fp32 statement of its tile walk"""
    return ta.tile_walk(qkv, B, N, H, d)


# ------------------------------------------------------------------------------------- tile walk against the bound
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("N", KERNEL_N)
def test_tile_walk_is_inside_the_bound(N, B):
    qkv = ta.random_qkv(B, N, H, D, seed=37 + N)
    o64, bound = ta.reference_and_bound(qkv, B, N, H, D)
    r = ta.worst_ratio(ta.tile_walk(qkv, B, N, H, D), o64, bound)
    print(f"[bound] tile walk N={N} B={B}: {r:.3g}")
    assert r <= 1.0


@pytest.mark.parametrize("N", ADVERSARIAL_N)
@pytest.mark.parametrize("kind", ta.ADVERSARIAL)
def test_tile_walk_is_inside_the_bound_at_adversarial_logits(kind, N):
    qkv = ta.logits_qkv(1, N, H, D, ta.adversarial_logits(kind, N, seed=N), seed=N)
    o64, bound = ta.reference_and_bound(qkv, 1, N, H, D)
    out = ta.tile_walk(qkv, 1, N, H, D)
    assert torch.isfinite(out).all()
    r = ta.worst_ratio(out, o64, bound)
    print(f"[bound] tile walk {kind} N={N}: {r:.3g}")
    assert r <= 1.0


@pytest.mark.parametrize("N", [257, 1000])
def test_bound_rejects_a_walk_with_one_rescale_skipped(N):
    """increasing logits: every tile raises the max, so leaving out the last tile's rescale keeps the earlier keys at
    their old weight; the bound must see that"""
    qkv = ta.logits_qkv(1, N, H, D, ta.adversarial_logits("increasing", N, seed=N), seed=N)
    o64, bound = ta.reference_and_bound(qkv, 1, N, H, D)
    last = -(-N // ta.KT) - 1
    good = ta.worst_ratio(ta.tile_walk(qkv, 1, N, H, D), o64, bound)
    bad = ta.worst_ratio(ta.tile_walk(qkv, 1, N, H, D, skip_rescale_at=last), o64, bound)
    print(f"[bound] increasing N={N}: walk {good:.3g}, walk without the last rescale {bad:.3g}")
    assert good <= 1.0 < bad


# ------------------------------------------------------------------------------------------------- argument checks
@pytest.mark.parametrize("B,N,Hh,d,why", [(0, 197, 16, 128, ">= 1"), (1, 0, 16, 128, ">= 1"), (1, 197, 0, 16, ">= 1"),
                                          (1, 197, 16, 0, "head dim"), (1, 197, 16, 100, "head dim"),
                                          (1, 197, 16, 160, "head dim"), (1, 197, 16, -32, "head dim"),
                                          (1, 65535 * 16 + 1, 16, 128, "views per scene"),
                                          (2 ** 31 - 1, 10 ** 6, 2 ** 31 - 1, 128, "64-bit"),
                                          (2 ** 20, 197, 2 ** 12, 128, "scene-heads"),
                                          (1, 197, 16, 128, "fp32 qkv of shape")])
def test_token_attention_refuses_bad_arguments_before_device_work(B, N, Hh, d, why):
    """each argument the launcher would refuse (and an operand of the wrong shape) raises a ValueError naming the
    problem, on a CPU tensor, so before any device work"""
    from iggt_official_b200 import ops
    with pytest.raises(ValueError, match="token_attention: .*" + why.replace("^", "\\^")):
        ops.token_attention(torch.zeros(1, 3 * 2048), B, N, Hh, d)


def test_small_attention_fits_is_the_shared_memory_cap():
    from iggt_official_b200 import ops
    assert ops._small_attention_fits(196, 128) and not ops._small_attention_fits(197, 128)
    assert ops._small_attention_fits(256, 64) and not ops._small_attention_fits(257, 32)


# ------------------------------------------------------------------------------------ the model graph, emulated
def _emulated(monkeypatch, calls):
    from test_model_wiring import EMU
    from iggt_official_b200 import ops
    from iggt_official_b200.models import aggregator as agg_mod
    for name, fn in EMU.items():
        monkeypatch.setattr(ops, name, fn)

    def count(name, fn):
        def wrapped(*a, **k):
            calls[name] = calls.get(name, 0) + 1
            return fn(*a, **k)
        return wrapped
    monkeypatch.setattr(ops, "small_attention", count("small_attention", EMU["small_attention"]))
    monkeypatch.setattr(ops, "token_attention", count("token_attention", token_attention_emu))
    monkeypatch.setattr(agg_mod, "_require_cuda", lambda images: None)
    return ops


def test_model_graph_reaches_token_attention_above_the_cap(monkeypatch):
    """197 views of 28 x 28 (9 tokens each): the camera head's 16 block passes run token_attention, and the forward
    equals the same graph with an unbounded small_attention emulation forced in (fp32: only the summation order of the
    attention differs)."""
    from oracle import weights
    from iggt_official_b200.models.vggt import VGGT
    torch.set_num_threads(8)
    calls = {}
    ops = _emulated(monkeypatch, calls)
    m = VGGT()
    m.load_state_dict(weights.make_state_dict(4, "default"), strict=False)
    m.eval()
    m.compute_dtype = m.head_dtype = torch.float32
    S = 197
    images = torch.rand(1, S, 3, 28, 28, generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        out = m(images)
    assert calls == {"token_attention": 16}, calls
    monkeypatch.setattr(ops, "_small_attention_fits", lambda N, d: True)
    with torch.no_grad():
        ref = m(images)
    assert calls == {"token_attention": 16, "small_attention": 16}, calls
    pe, rp = torch.stack(out["pose_enc"]), torch.stack(ref["pose_enc"])
    assert pe.shape == (4, 1, S, 9) and torch.isfinite(pe).all()
    assert ((pe - rp).abs().max() / rp.abs().max()).item() < 1e-5
    for k in ("depth", "depth_conf", "world_points", "world_points_conf"):
        assert torch.equal(out[k], ref[k]), k                               # the camera head feeds no other output


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _sharded_worker(rank, world, port, S, ret):
    """The view-sharded forward with the launchers replaced by their PyTorch statements; every rank also runs the
    unsharded forward and compares its own views."""
    sys.path.insert(0, HERE)
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(4)
    from test_model_wiring import EMU
    from iggt_official_b200 import ops
    from iggt_official_b200.models import aggregator as agg_mod
    from iggt_official_b200.models.vggt import VGGT
    from iggt_official_b200.parallel import forward_sharded
    for name, fn in EMU.items():
        setattr(ops, name, fn)
    calls = []
    ops.token_attention = lambda *a: calls.append(a[2]) or token_attention_emu(*a)
    agg_mod._require_cuda = lambda images: None
    torch.manual_seed(0)                                   # identical random-init weights on every rank
    m = VGGT().eval()
    m.compute_dtype = m.head_dtype = torch.float32
    images = torch.rand(1, S, 3, 28, 28, generator=torch.Generator().manual_seed(3))
    S_loc = S // world
    mine = images[:, rank * S_loc:(rank + 1) * S_loc].contiguous()
    with torch.no_grad():
        out = forward_sharded(m, mine, rank, world)
        m.aggregator.process_group = None
        ref = m(images)
    ok = calls == [S] * 32                                 # 16 block passes in each forward, over all S views
    for k in ("depth", "depth_conf", "world_points", "world_points_conf"):
        a, b = out[k], ref[k][:, rank * S_loc:(rank + 1) * S_loc]
        ok = ok and a.shape == b.shape and ((a - b).abs().max() / b.abs().max()).item() < 1e-5
    rp = torch.stack(ref["pose_enc"])
    pe = ((torch.stack(out["pose_enc"]) - rp).abs().max() / rp.abs().max()).item()       # fp32 summation order only
    ret[rank] = bool(ok and pe < 1e-5)
    dist.destroy_process_group()


def test_view_sharded_forward_of_200_views_equals_unsharded_forward():
    world = 2
    ret = mp.Manager().dict()
    mp.spawn(_sharded_worker, args=(world, _free_port(), 200, ret), nprocs=world, join=True)
    assert ret[0] and ret[1]
