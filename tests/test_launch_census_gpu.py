"""A census of the real forward's GEMM, convolution, attention and DPT-tail launches, each checked element by element
at the model's own shapes, and the launch sequence checked bit for bit (GPU, except the coverage guard).

1. Census.  Seeded stress weights (oracle.weights), real forwards of four configurations:
     c2_fp16   VGGT 1 x 8 x 518^2, fp16 trunk                (the benchmark's C2 workload)
     c2_bf16   the same with a bf16 trunk
     iggt_532  IGGT 1 x 8 x 532^2, fp16                      (even 38 x 38 grid: the part path)
     demo      IGGT 1 x 3 x 336 x 504 (24 x 36 grid), bf16 heads, 64 query points (the track head)
   The `ops` launchers below are wrapped (the model calls them as module attributes).  Every call is keyed by its
   signature: the launcher, every shape and stride, the dtype, the epilogue flags and the schedule (iggt_gemm_plan's
   bn / stream_k / grid, attention_plan's kv splits, the conv's spatial tile grid).  The first and the last call of
   each signature keep their inputs and output (the in-place gemm_resid32 its x from before the launch): the trunk's
   late blocks carry larger activations than its first ones.  Each kept launch is then held to the float64 statement
   of the synthetic tests (tests/launch_refs.py, tests/ulp_bounds.py), built per image, per head or per block of rows:
     gemm_store16 / conv_nhwc  RN16 of the ACC interval through the activation, + resid, + resid2, act_post; 1 ulp
     gemm_store32              ACC of the magnitude sum (GELU: its interval and error)
     gemm_resid32              x + gamma RN16(acc + b) on whole tiles (round_out16), else x + gamma (acc + b)
     gemm_qkv                  test_qkv_bounds_gpu.py's Gaussian statement (ambiguous LayerNorm inputs widened)
     attention                 bound 1 (check_attn_bound1)
     dpt_tail_fused            test_heads_bounds_gpu.py's tail statement, 2^-18 of A
   Exact operands: for every gemm_store16 and conv_nhwc signature one more launch with integer A and W = integers x
   2^-e (every partial sum a multiple of 2^-e below 2^(24-e): fp32 accumulation is exact in any order) must equal
   bit for bit the fp32 epilogue restated in torch (acc + b, activation, + addend / resid / resid2, act_post, one
   RN16), or for act = 1 be within GELU_ERR of gelu64(RN16(acc + b)).  That pins the tap and channel-block order and the
   image / tile mapping at the heads' ragged grids independently of the data.
   Negative controls at one real signature each: bias dropped, resid2 dropped, the conv statement of the neighbouring
   16-pixel tile column, the global attention with the keys of another view.  Each must fail.

   The share of 16-bit outputs off RN16 of the float64 value grows with K and with real activations (FRAC was measured
   at K <= 1024 on Gaussian data).  CENSUS_FRAC below is about twice the largest share measured in the census.

2. Coverage guard (CPU).  The model graph runs with the emulated launchers of test_model_wiring.py and every `ops`
   function it calls must be checked here (CHECKED) or named in COVERED_ELSEWHERE with an existing test.

3. Sequence.  With IGGT_STREAMK=0 every launch feeding depth, points, confidences, poses and tracks accumulates in a
   fixed order, so the forward is a pure function of its inputs bit for bit: PDL on and off, two eager forwards, and
   eager and CUDA-graph replay must agree exactly.  The switches are read once per process, so each setting runs in a
   child process.  The exception is part_feat: channel_mean (csrc/part.cu) sums with float atomicAdd, whose order
   varies from run to run; it is held to the 1e-4 relative L2 of test_fullsize_gpu.py.

Measured on an H100 80GB HBM3 (700 W power limit, 1980 MHz maximum SM clock); -s prints these per configuration:
* distinct signatures c2_fp16 36, c2_bf16 36, iggt_532 84, demo 108, every one checked; no 16-bit output outside its
  interval (0 ulp) anywhere; fp32 outputs at most 0.99 of their bound (gemm_resid32), attention at most 0.45 of bound 1,
  the DPT tail 0.011, store32 0.47; every exact-operand launch bit-exact (GELU within 0.9993 of its bound);
* share off RN16, fp16: 1.1-1.3 % at K = 2048 / 2304 (head projections and convs), 3.4 % at K = 9216 (the stride-2
  conv as GEMM and the Cin = 1024 layer_rn convs: 1.8 %); bf16: 0.18 % at K = 2304, 0.50 % at K = 9216; bf16 GELU
  (track corr MLP, K = 576): 13 %.  CENSUS_FRAC is about twice these;
* the negative controls fail on 99 % (bias dropped), 79 % (resid2 dropped), 53 % (neighbouring tile column) and 32-90 %
  (keys of another view; bf16 trunk 32 %) of the elements;
* mutants of gemm.cuh that no synthetic store16 or conv test sees each fail this file at C2: a channel-major k-block
  order, the bias zeroed for consumer warpgroup 1, resid2 skipped by consumer warpgroup 1;
* the file takes about 5.7 minutes, peak device memory 27 GB;
* the sequence: every output bit-identical for PDL on / off, two eager forwards and graph replay (c2_fp16 and demo);
  part_feat was bit-identical too in that run.
"""
import ast
import re
import inspect
import math
import os
import subprocess
import sys
import time

import pytest
import torch

from launch_refs import ACC, GELU_ERR, act_interval, check_tail, conv64, gelu64, gemm_plan, qk64, y64
from ulp_bounds import _interval_distance, check_attn_bound1, rn16, ulp16, ulp_distance

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")

CHECKED = ("gemm_store16", "gemm_store32", "gemm_resid32", "gemm_qkv", "conv_nhwc", "attention", "dpt_tail_fused")
# launchers of the forward whose element-wise statement lives in another file
COVERED_ELSEWHERE = {
    "layernorm": "test_epilogues_gpu.py::test_layernorm",
    "layernorm16": "test_heads_bounds_gpu.py::test_layernorm16",
    "layernorm_rows": "test_track_bounds_gpu.py::test_layernorm_rows",
    "patchify": "test_kernels_gpu.py::test_patchify_and_assemble",
    "dino_assemble": "test_kernels_gpu.py::test_patchify_and_assemble",
    "special_tokens": "test_kernels_gpu.py::test_patchify_and_assemble",
    "upsample_bilinear": "test_heads_bounds_gpu.py::test_upsample_bilinear_ladder",
    "deconv_shuffle": "test_heads_bounds_gpu.py::test_deconv_shuffle_bit_exact",
    "im2col3x3_s2": "test_heads_bounds_gpu.py::test_im2col3x3_s2_bit_exact",
    "col2im_k4s2p1": "test_heads_bounds_gpu.py::test_col2im_k4s2p1",
    "dpt_tail": "test_heads_bounds_gpu.py::test_dpt_tail",
    "skinny_gemm": "test_heads_bounds_gpu.py::test_skinny_gemm",
    "small_attention": "test_heads_bounds_gpu.py::test_small_attention",
    "camera_head": "test_heads_bounds_gpu.py::test_camera_head_phases",
    "ocab_attention": "test_heads_bounds_gpu.py::test_window_attention_ocab",
    "window_attention": "test_heads_bounds_gpu.py::test_window_attention_hab",
    "channel_mean": "test_heads_bounds_gpu.py::test_channel_mean",
    "se_scale_add": "test_heads_bounds_gpu.py::test_se_scale_add",
    "avgpool2_nhwc": "test_track_bounds_gpu.py::test_avgpool2",
    "sample_bilinear_nhwc": "test_track_bounds_gpu.py::test_sample_bilinear",
    "corr_sample": "test_track_bounds_gpu.py::test_corr_sample",
    "track_input": "test_track_bounds_gpu.py::test_track_input",
}

CONFIGS = {
    "c2_fp16": dict(model="VGGT", S=8, H=518, W=518, trunk=torch.float16, head=None, points=0),
    "c2_bf16": dict(model="VGGT", S=8, H=518, W=518, trunk=torch.bfloat16, head=None, points=0),
    "iggt_532": dict(model="IGGT", S=8, H=532, W=532, trunk=torch.float16, head=None, points=0),
    "demo": dict(model="IGGT", S=3, H=336, W=504, trunk=torch.float16, head=torch.bfloat16, points=64),
}
WSEED, ISEED = 7, 11
# share of 16-bit outputs allowed off RN16 of the float64 value, by dtype and reduction length K (module docstring):
# FRAC up to K = 1024, then about twice the largest share the census measured in each band
CENSUS_FRAC = {torch.float16: ((1024, 0.01), (4096, 0.026), (16384, 0.07)),
               torch.bfloat16: ((1024, 0.002), (4096, 0.004), (16384, 0.01))}
# GELU: fp16 as FRAC_GELU; bf16 outputs in the negative tail are many bf16 ulps off exact-erf GELU while inside the
# pinned absolute bound (test_epilogues_gpu.py::test_gelu_exhaustive), and real activations put many inputs there
CENSUS_FRAC_GELU = {torch.float16: 0.02, torch.bfloat16: 0.26}
ROWS = 4096                                           # rows of a GEMM reference built at a time


def _report(what, value):
    print(f"[census] {what}: {value}")


def _frac(dtype, K, act):
    if act == 1:
        return CENSUS_FRAC_GELU[dtype]
    return next(f for k, f in CENSUS_FRAC[dtype] if K <= k)


# ============================================================================================== coverage guard (CPU)
def test_census_covers_every_launcher_of_the_forward(monkeypatch):
    """Runs the IGGT graph (part path) and the track head with the emulated launchers and records which `ops`
    functions they call; each must be checked by the census or by a named test that exists.  camera_head (the fused
    camera head runs on the GPU only) is listed in COVERED_ELSEWHERE too."""
    sys.path.insert(0, TESTS)
    import emu_ops
    from test_model_wiring import EMU
    from iggt_official_b200 import ops
    from iggt_official_b200.models import aggregator as agg_mod
    from iggt_official_b200.models.vggt import IGGT
    from oracle import weights
    emu = dict(EMU)
    for name in ("layernorm_rows", "avgpool2_nhwc", "sample_bilinear_nhwc", "corr_sample", "track_input"):
        emu[name] = getattr(emu_ops, name)
    called = set()
    launchers = [n for n, f in vars(ops).items() if callable(f) and not n.startswith("_") and
                 getattr(f, "__module__", None) == ops.__name__]

    def recorder(name):
        fn = emu.get(name)

        def f(*a, **k):
            called.add(name)
            if fn is None:
                raise AssertionError(f"ops.{name} has no emulated statement")
            return fn(*a, **k)
        return f

    for name in launchers:
        monkeypatch.setattr(ops, name, recorder(name))
    monkeypatch.setattr(agg_mod, "_require_cuda", lambda images: None)
    m = IGGT()
    m.load_state_dict(weights.make_state_dict(3, "stress"), strict=False)
    m.eval()
    m.compute_dtype = m.head_dtype = torch.float32
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        m(torch.rand(1, 2, 3, 28, 56, generator=g))
        fmaps = torch.randn(2, 64, 64, 128, generator=g)
        m.track_head.track(fmaps, torch.rand(1, 5, 2, generator=g) * 120, 1, 2, 1, torch.float32)
    assert {"gemm_qkv", "conv_nhwc", "attention", "dpt_tail_fused", "corr_sample", "channel_mean"} <= called
    missing = sorted(n for n in called if n not in CHECKED and n not in COVERED_ELSEWHERE)
    assert not missing, f"launchers of the forward with no element-wise test: {missing}"
    for name, where in COVERED_ELSEWHERE.items():
        fname, test = where.split("::")
        tree = ast.parse(open(os.path.join(TESTS, fname)).read())
        names = {n.name for n in tree.body if isinstance(n, ast.FunctionDef)}
        assert test in names, f"COVERED_ELSEWHERE[{name!r}] names {where}, which does not exist"
        assert name in launchers, f"COVERED_ELSEWHERE names ops.{name}, which does not exist"
    _report("launchers called by the forward", sorted(called))


# ============================================================================================== recording (GPU)
def _desc(v):
    if torch.is_tensor(v):
        return ("T", tuple(v.shape), tuple(v.stride()), str(v.dtype))
    if v is None or isinstance(v, (bool, int, float, str)):
        return v
    return type(v).__name__


def _keep(v):
    if torch.is_tensor(v):
        return v.detach().clone()
    if isinstance(v, tuple):
        return tuple(_keep(t) for t in v)
    return v


def _schedule(ops, name, a):
    if name in ("gemm_store16", "gemm_store32", "gemm_resid32"):
        M, K = a["a"].shape
        p = gemm_plan(M, a["w"].shape[0], K, {"gemm_store16": 0, "gemm_resid32": 1, "gemm_store32": 3}[name])
        return (p["bn"], p["stream_k"], p["grid"])
    if name == "gemm_qkv":
        p = gemm_plan(a["a"].shape[0], 3 * a["C"], a["a"].shape[1], 2)
        return (p["bn"], p["stream_k"], p["grid"])
    if name == "attention":
        return a["splits"] if a["splits"] is not None else ops.attention_plan(a["num_seq"], a["Lq"], a["Lk"], a["H"])[0]
    if name == "conv_nhwc":
        _, H, W, _ = a["x"].shape
        return (-(-W // 16), -(-H // 8))                      # spatial tiles of 8 x 16 pixels (x, y)
    return None


class Census:
    def __init__(self, ops):
        self.ops = ops
        self.orig = {n: getattr(ops, n) for n in CHECKED}
        self.sigs = {}

    def install(self, monkeypatch):
        for n in CHECKED:
            monkeypatch.setattr(self.ops, n, self._wrap(n))

    def _wrap(self, name):
        fn = self.orig[name]
        sig = inspect.signature(fn)

        def f(*args, **kw):
            b = sig.bind(*args, **kw)
            b.apply_defaults()
            a = dict(b.arguments)
            key = (name,) + tuple((k, _desc(v)) for k, v in a.items()) + (("schedule", _schedule(self.ops, name, a)),)
            pre = {k: _keep(v) for k, v in a.items()}
            res = fn(*args, **kw)
            rec = self.sigs.setdefault(key, dict(name=name, count=0, first=None, last=None))
            cap = dict(args=pre, out=_keep(res))
            rec["first" if rec["first"] is None else "last"] = cap
            rec["count"] += 1
            return res
        return f


# ============================================================================================== per-element tallies
class Tally16:
    """check16 (tests/ulp_bounds.py) accumulated over chunks of one launch's output."""

    def __init__(self, dtype):
        self.dtype, self.n, self.off, self.worst, self.beyond, self.where = dtype, 0, 0, 0, 0, ""

    def add(self, out, ref, lo=None, hi=None, max_ulps=1, tag=""):
        exact = ulp_distance(out, ref, self.dtype)
        dist = exact
        if lo is not None:
            lo16 = rn16(torch.minimum(lo, hi), self.dtype)
            hi16 = rn16(torch.maximum(lo, hi), self.dtype)
            dist = torch.minimum(_interval_distance(out, lo16, hi16), exact)
        self.n += out.numel()
        self.off += int((exact != 0).sum())
        self.beyond += int((dist > max_ulps).sum())
        w = int(dist.max()) if out.numel() else 0
        if w > self.worst or not self.where:
            i = int(dist.reshape(-1).argmax())
            self.where = (f"{tag} out {out.reshape(-1)[i].item()!r} ref {ref.reshape(-1)[i].item()!r} ({w} ulp)")
            self.worst = max(self.worst, w)

    def share(self):
        return self.off / max(self.n, 1)

    def verdict(self, max_ulps, frac):
        if self.worst > max_ulps or self.off > frac * self.n:
            return (f"{self.beyond} of {self.n} beyond {max_ulps} ulp, {self.share():.3%} off RN16 (limit {frac:.2%}); "
                    f"worst {self.where}")
        return None


class Tally32:
    """check32 accumulated over chunks: |out - [lo, hi]| <= bound per element, NaN positions equal."""

    def __init__(self):
        self.worst, self.bad, self.n, self.where = 0.0, 0, 0, ""

    def add(self, out, ref, bound, lo=None, hi=None, tag=""):
        o = out.double()
        lo, hi = (ref, ref) if lo is None else (torch.minimum(lo, hi), torch.maximum(lo, hi))
        err = torch.clamp(torch.maximum(lo - o, o - hi), min=0)
        err = torch.where(o == ref, torch.zeros_like(err), err)
        nan_o, nan_r = torch.isnan(o), torch.isnan(ref)
        if not torch.equal(nan_o, nan_r):
            self.bad += int((nan_o != nan_r).sum())
            self.worst = math.inf
            self.where = f"{tag} NaN positions differ"
        err = torch.where(nan_o | nan_r, torch.zeros_like(err), err)
        ratio = torch.where(err > 0, err / bound, torch.zeros_like(err))
        self.n += out.numel()
        self.bad += int((err > bound).sum())
        w = float(ratio.max()) if ratio.numel() else 0.0
        if w > self.worst:
            i = int(ratio.reshape(-1).argmax())
            self.worst = w
            self.where = f"{tag} out {o.reshape(-1)[i].item()!r} ref {ref.reshape(-1)[i].item()!r} ({w:.3g} x bound)"

    def verdict(self):
        return f"{self.bad} of {self.n} beyond the bound; worst {self.where}" if self.bad else None


# ============================================================================================== statements
def _vec(v, n, dev):
    return v.double() if v is not None else torch.zeros(n, dtype=torch.float64, device=dev)


def _store16_chunks(a, w, bias, act, addend, add_rows, dtype):
    """(rows, ref, lo, hi) of gemm_store16 by blocks of rows."""
    M, N = a.shape[0], w.shape[0]
    b = _vec(bias, N, a.device)
    for r0 in range(0, M, ROWS):
        r1 = min(M, r0 + ROWS)
        acc, mag = _gemm64(a[r0:r1], w)
        y = acc + b
        ref, lo, hi = act_interval(act, y, ACC * (mag + b.abs()), dtype)
        if addend is not None:
            ad = addend.double()[torch.arange(r0, r1, device=a.device) % add_rows]
            s2 = 2.0 ** -23 * (ref.abs() + ad.abs())              # the addend joins in fp32 after the activation
            ref, lo, hi = ref + ad, lo + ad - s2, hi + ad + s2
        yield slice(r0, r1), ref, lo, hi


def _gemm64(a, w):
    a64, w64 = a.double(), w.double()
    return a64 @ w64.t(), a64.abs() @ w64.abs().t()


def check_store16(cap, bias_dropped=False):
    a = cap["args"]
    dtype = a["a"].dtype
    out = cap["out"]
    t = Tally16(dtype)
    for rows, ref, lo, hi in _store16_chunks(a["a"], a["w"], None if bias_dropped else a["bias"], a["act"],
                                             a["addend"], a["add_rows"], dtype):
        t.add(out[rows], ref, lo, hi, tag=f"rows {rows.start}..")
    return t, _frac(dtype, a["a"].shape[1], a["act"])


def check_store32(cap):
    a = cap["args"]
    out, act = cap["out"], a["act"]
    N = a["w"].shape[0]
    b = _vec(a["bias"], N, out.device)
    t = Tally32()
    for r0 in range(0, out.shape[0], ROWS):
        r1 = min(out.shape[0], r0 + ROWS)
        acc, mag = _gemm64(a["a"][r0:r1], a["w"])
        y = acc + b
        s = ACC * (mag + b.abs())
        if act == 1:
            g_lo, g_hi = gelu64(y - s), gelu64(y + s)
            t.add(out[r0:r1], gelu64(y), (GELU_ERR / 2 + 2.0 ** -24) * y.abs(), torch.minimum(g_lo, g_hi),
                  torch.maximum(g_lo, g_hi))
        else:
            assert act == 0, act
            t.add(out[r0:r1], y, s)
    return t


def check_resid32(cap, stream_k):
    a = cap["args"]
    x0all, out = a["x"], cap["out"]
    dtype = a["a"].dtype
    N = a["w"].shape[0]
    b = _vec(a["bias"], N, out.device)
    g64 = a["gamma"].double() if a["gamma"] is not None else torch.ones(N, dtype=torch.float64, device=out.device)
    t = Tally32()
    for r0 in range(0, out.shape[0], ROWS):
        r1 = min(out.shape[0], r0 + ROWS)
        acc, mag = _gemm64(a["a"][r0:r1], a["w"])
        x0 = x0all[r0:r1].double()
        y = acc + b
        if a["round_out16"] and not stream_k:
            # whole tiles: x + gamma RN16(acc + b); after the rounding one multiply and one add, 2^-22 of the scale
            _, lo, hi = act_interval(0, y, ACC * (mag + b.abs()), dtype)
            r, r_lo, r_hi = (rn16(v, dtype).double() for v in (y, lo, hi))
            t.add(out[r0:r1], x0 + g64 * r, 2.0 ** -22 * (x0.abs() + g64 * r.abs()), x0 + g64 * r_lo, x0 + g64 * r_hi)
        else:
            t.add(out[r0:r1], x0 + g64 * y, ACC * (x0.abs() + g64 * (mag + b.abs())))
    return t


def check_qkv(cap):
    a = cap["args"]
    out = cap["out"]
    dtype = a["a"].dtype
    C = a["C"]
    bias = a["bias"] if a["bias"] is not None else torch.zeros(3 * C, device=out.device)
    t_v, t_qk = Tally16(dtype), Tally16(dtype)
    M = out.shape[0]
    step = ROWS if not a["qk_norm"] else a["T"] * max(1, ROWS // a["T"])     # whole views: RoPE positions are row % T
    for r0 in range(0, M, step):
        r1 = min(M, r0 + step)
        y, mag = y64(a["a"][r0:r1], a["w"], bias)
        sy = ACC * mag
        o = out[r0:r1]
        if not a["qk_norm"]:
            t_v.add(o, y, y - sy, y + sy, max_ulps=0)
            continue
        u = rn16(y, dtype).double()
        u_lo, u_hi = rn16(y - sy, dtype).double(), rn16(y + sy, dtype).double()
        amb = torch.maximum((u_hi - u).abs(), (u - u_lo).abs())
        t_v.add(o[:, 2 * C:], y[:, 2 * C:], y[:, 2 * C:] - sy[:, 2 * C:], y[:, 2 * C:] + sy[:, 2 * C:], max_ulps=0)
        norm = (a["qn_w"], a["qn_b"], a["kn_w"], a["kn_b"])
        ref, sr = qk64(u, C, a["T"], norm, a["rope_cos"], a["rope_sin"], a["pos_yx"], amb)
        fin = torch.isfinite(ref) & torch.isfinite(sr)
        t_qk.add(o[:, :2 * C], ref, torch.where(fin, ref - sr, ref), torch.where(fin, ref + sr, ref), max_ulps=0)
    return t_v, t_qk


def _conv_statement(x, wp, bias, act, r1, r2, act_post, taps, dtype, drop_resid2=False):
    """(ref, lo, hi) [H, W, Cout] of one image of conv_nhwc."""
    acc, mag = conv64(x, wp, taps)
    b = _vec(bias, wp.shape[0], x.device)
    y = acc + b
    ref, lo, hi = act_interval(act, y, ACC * (mag + b.abs()), dtype)
    if r2 is not None and drop_resid2:
        r2 = None
    if r1 is not None or r2 is not None:
        add = sum(r.double() for r in (r1, r2) if r is not None)
        ref = ref + add
        s2 = 2.0 ** -23 * (sum(r.double().abs() for r in (r1, r2) if r is not None) + ref.abs())   # two fp32 adds
        lo, hi = lo + add - s2, hi + add + s2
    if act_post:
        f = {2: torch.relu, 3: lambda v: torch.where(v > 0, v, 0.01 * v)}[act_post]
        ref, lo, hi = f(ref), f(lo), f(hi)
    return ref, lo, hi


def check_conv(cap, images=None, drop_resid2=False, shift=0):
    a = cap["args"]
    x, out = a["x"], cap["out"]
    dtype = x.dtype
    t = Tally16(dtype)
    for i in (range(x.shape[0]) if images is None else images):
        r1 = a["resid"][i] if a["resid"] is not None else None
        r2 = a["resid2"][i] if a["resid2"] is not None else None
        ref, lo, hi = _conv_statement(x[i], a["wp"], a["bias"], a["act"], r1, r2, a["act_post"], a["taps"], dtype,
                                      drop_resid2)
        if shift:                                          # the statement of the pixel `shift` columns to the right
            W = ref.shape[1]
            ref, lo, hi = (v[:, shift:] for v in (ref, lo, hi))
            t.add(out[i][:, :W - shift], ref, lo, hi, tag=f"image {i}")
        else:
            t.add(out[i], ref, lo, hi, tag=f"image {i}")
    return t, _frac(dtype, a["wp"].shape[1], a["act"])


def check_attention(cap, k_roll=0):
    a = cap["args"]
    k = a["k"]
    if k_roll:
        k = k.view(a["num_seq"], a["Lk"], -1).roll(k_roll, 1).reshape(k.shape)
    return check_attn_bound1(cap["out"], a["q"], k, a["v"], a["num_seq"], a["Lq"], a["Lk"], a["H"], a["q"].dtype,
                             scale=a["scale"], what="attention")


def check_tail_launch(cap):
    a = cap["args"]
    x, wp, bias, w2, b2, mode = a["x"], a["wp"], a["bias"], a["w2"], a["b2"], a["mode"]
    main, conf = cap["out"]
    worst = 0.0
    for i in range(x.shape[0]):
        z, sz = conv64(x[i], wp, 9)
        z, sz = z + bias.double(), sz + bias.double().abs()
        o64 = torch.relu(z) @ w2.double().t() + b2.double()
        A = sz @ w2.double().abs().t() + b2.double().abs()
        worst = max(worst, check_tail(main[i:i + 1], None if conf is None else conf[i:i + 1], o64[None], A[None],
                                      mode, 2.0 ** -18, f"dpt_tail_fused image {i}"))
        del z, sz, o64, A
    return worst


# ============================================================================================== exact operands
def _like(shape, stride, make):
    """A tensor of `shape` whose row pitch is stride[0] (2-D) filled by make(full_shape)."""
    if len(shape) == 2 and stride[0] != shape[1]:
        return make((shape[0], stride[0]))[:, :shape[1]]
    return make(shape)


def _exact_e(K):
    assert K * 8 * 64 < 2 ** 24, K
    return round(math.log2(math.sqrt(K) * 4.9 * 37.2 / 8))          # y about 8 in size


def _ints(lo, hi, dev, g):
    return lambda shape: torch.randint(lo, hi + 1, shape, device=dev, generator=g).double()


def _exact_epilogue(acc, b, act, adds, act_post, dtype):
    """The kernel's fp32 epilogue in torch on the exact fp32 acc: acc + b, act, + each addend in order, act_post, RN16.
    act 1 returns (x16 of the GELU input, None)."""
    v = acc.float() + b.float()
    if act == 1:
        assert not adds and not act_post
        return rn16(v, dtype), None
    if act == 2:
        v = torch.relu(v)
    elif act == 3:
        v = torch.where(v > 0, v, v * 0.01)
    for t in adds:
        v = v + t.float()
    if act_post == 2:
        v = torch.relu(v)
    return None, v.to(dtype)


def _exact_compare(out, x16, ref16, dtype, what):
    if ref16 is not None:
        d = ulp_distance(out, ref16.double(), dtype)                  # +0 and -0 are the same point
        n = int((d != 0).sum())
        assert n == 0, f"{what}: {n} of {out.numel()} elements differ from the fp32 epilogue (worst {int(d.max())} ulp)"
        return 0.0
    x = x16.double()
    ref = gelu64(x)
    delta = x.abs() / 2 * GELU_ERR
    ratio = ((out.double() - ref).abs() / (0.5 * ulp16(ref.abs() + delta, dtype) + delta)).max().item()
    assert ratio <= 1.0, f"{what}: GELU of the exact 16-bit input off by {ratio:.3g} x its bound"
    return ratio


def exact_store16(orig, key, cap, g):
    a = cap["args"]
    d = dict(key[1:])
    dtype = a["a"].dtype
    dev = a["a"].device
    M, K = a["a"].shape
    N = a["w"].shape[0]
    e = _exact_e(K)
    A = _like(d["a"][1], d["a"][2], lambda s: _ints(-8, 8, dev, g)(s).to(dtype))
    Wt = _like(d["w"][1], d["w"][2], lambda s: (_ints(-64, 64, dev, g)(s) * 2.0 ** -e).to(dtype))
    bias = (_ints(-8 << e, 8 << e, dev, g)((N,)) * 2.0 ** -e).float() if a["bias"] is not None else None
    add = None
    if a["addend"] is not None:
        add = _like(d["addend"][1], d["addend"][2], lambda s: (_ints(-64, 64, dev, g)(s) * 2.0 ** -e).to(dtype))
    out = orig(A, Wt, bias, act=a["act"], addend=add, add_rows=a["add_rows"])
    acc = (A.double() @ Wt.double().t())
    b = bias if bias is not None else torch.zeros(N, device=dev)
    adds = [add.double()[torch.arange(M, device=dev) % a["add_rows"]]] if add is not None else []
    x16, ref16 = _exact_epilogue(acc, b, a["act"], adds, 0, dtype)
    return _exact_compare(out, x16, ref16, dtype, "store16 exact")


def exact_conv(orig, key, cap, g):
    a = cap["args"]
    x0, wp0 = a["x"], a["wp"]
    dtype, dev = x0.dtype, x0.device
    NB, H, W, Cin = x0.shape
    Cout, taps = wp0.shape[0], a["taps"]
    e = _exact_e(taps * Cin)
    x = _ints(-8, 8, dev, g)(x0.shape).to(dtype)
    wp = (_ints(-64, 64, dev, g)(wp0.shape) * 2.0 ** -e).to(dtype)
    bias = (_ints(-8 << e, 8 << e, dev, g)((Cout,)) * 2.0 ** -e).float() if a["bias"] is not None else None
    res = [(_ints(-64, 64, dev, g)(r.shape) * 2.0 ** -e).to(dtype) if r is not None else None
           for r in (a["resid"], a["resid2"])]
    out = orig(x, wp, bias, act=a["act"], resid=res[0], taps=taps, resid2=res[1], act_post=a["act_post"])
    b = bias if bias is not None else torch.zeros(Cout, device=dev)
    worst = 0.0
    for i in range(NB):
        acc, _ = conv64(x[i], wp, taps)
        x16, ref16 = _exact_epilogue(acc, b, a["act"], [r[i] for r in res if r is not None], a["act_post"], dtype)
        worst = max(worst, _exact_compare(out[i], x16, ref16, dtype, f"conv exact image {i}"))
    return worst


# ============================================================================================== the census
def _build(cfg, dev="cuda"):
    from iggt_official_b200.models.vggt import IGGT, VGGT
    from oracle import weights
    m = (IGGT if cfg["model"] == "IGGT" else VGGT)()
    m.load_state_dict(weights.make_state_dict(WSEED, "stress"), strict=False)
    m.eval().to(dev)
    m.compute_dtype = cfg["trunk"]
    m.head_dtype = cfg["head"]
    g = torch.Generator().manual_seed(ISEED)
    images = torch.rand(1, cfg["S"], 3, cfg["H"], cfg["W"], generator=g).to(dev)
    qp = None
    if cfg["points"]:
        qp = (torch.rand(1, cfg["points"], 2, generator=g) * torch.tensor([cfg["W"] - 1.0, cfg["H"] - 1.0])).to(dev)
    return m, images, qp


def _stat(stats, name, key, value):
    s = stats.setdefault(name, {})
    s[key] = max(s.get(key, 0.0), value)


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(CONFIGS))
def test_launch_census(monkeypatch, config):
    from iggt_official_b200 import ops
    t0 = time.time()
    cfg = CONFIGS[config]
    census = Census(ops)
    census.install(monkeypatch)
    m, images, qp = _build(cfg)
    with torch.no_grad():
        m(images, query_points=qp)
    torch.cuda.synchronize()
    del m
    monkeypatch.undo()
    torch.cuda.empty_cache()
    t_fwd = time.time() - t0
    failures = []
    counts = {}
    controls = {}
    stats = {}
    g = torch.Generator(device="cuda").manual_seed(17)
    for key, rec in census.sigs.items():
        name = rec["name"]
        counts[name] = counts.get(name, 0) + 1
        desc = ", ".join(f"{k}={v[1] if isinstance(v, tuple) and v and v[0] == 'T' else v}" for k, v in key[1:]
                         if k not in ("out",))
        for which in ("first", "last"):
            cap = rec[which]
            if cap is None:
                continue
            tag = f"{config} {name}({desc}) [{which} of {rec['count']}]"
            a0 = cap["args"]
            try:
                if name in ("gemm_store16", "conv_nhwc"):
                    t, frac = (check_store16 if name == "gemm_store16" else check_conv)(cap)
                    dt = a0["x" if name == "conv_nhwc" else "a"].dtype
                    K = a0["wp"].shape[1] if name == "conv_nhwc" else a0["a"].shape[1]
                    band = next(k for k, _ in CENSUS_FRAC[dt] if K <= k)
                    kind = "gelu" if a0["act"] == 1 else f"K<={band}"
                    _stat(stats, f"{name} {str(dt)[6:]} {kind}", "ulps", t.worst)
                    _stat(stats, f"{name} {str(dt)[6:]} {kind}", "share", t.share())
                    v = t.verdict(1, frac)
                    assert v is None, v
                elif name == "gemm_store32":
                    t = check_store32(cap)
                    _stat(stats, name, "err/bound", t.worst)
                    assert t.verdict() is None, t.verdict()
                elif name == "gemm_resid32":
                    t = check_resid32(cap, dict(key[1:])["schedule"][1])
                    _stat(stats, name, "err/bound", t.worst)
                    assert t.verdict() is None, t.verdict()
                elif name == "gemm_qkv":
                    t_v, t_qk = check_qkv(cap)
                    dt = cap["args"]["a"].dtype
                    _stat(stats, f"{name} {str(dt)[6:]}", "ulps", max(t_v.worst, t_qk.worst))
                    _stat(stats, f"{name} {str(dt)[6:]}", "share", max(t_v.share(), t_qk.share()))
                    for t in (t_v, t_qk):
                        v = t.verdict(0, _frac(dt, cap["args"]["a"].shape[1], 0))
                        assert v is None, v
                elif name == "attention":
                    _stat(stats, name, "err/bound", check_attention(cap))
                elif name == "dpt_tail_fused":
                    _stat(stats, name, "err/bound", check_tail_launch(cap))
            except AssertionError as e:
                failures.append(f"{tag}: {str(e).splitlines()[0][:400]}")
        # exact operands, once per signature
        if name in ("gemm_store16", "conv_nhwc"):
            try:
                f = exact_store16 if name == "gemm_store16" else exact_conv
                _stat(stats, name + " exact", "gelu err/bound", f(census.orig[name], key, rec["first"], g))
            except AssertionError as e:
                failures.append(f"{config} {name}({desc}) exact operands: {str(e).splitlines()[0][:400]}")
        # negative controls, at the first signature that has what each one removes
        cap = rec["first"]
        a = cap["args"]
        if name == "gemm_store16" and "bias dropped" not in controls and a["bias"] is not None and a["act"] == 0 \
                and a["addend"] is None and float(a["bias"].abs().max()) > 0:
            t, frac = check_store16(cap, bias_dropped=True)
            controls["bias dropped"] = (t.verdict(1, frac), t.beyond / t.n, desc)
        if name == "conv_nhwc" and "resid2 dropped" not in controls and a["resid2"] is not None:
            t, frac = check_conv(cap, images=[0], drop_resid2=True)
            controls["resid2 dropped"] = (t.verdict(1, frac), t.beyond / t.n, desc)
        if name == "conv_nhwc" and "neighbouring tile column" not in controls and a["x"].shape[2] > 32 \
                and a["taps"] == 9:
            t, frac = check_conv(cap, images=[0], shift=16)
            controls["neighbouring tile column"] = (t.verdict(1, frac), t.beyond / t.n, desc)
        if name == "attention" and "keys of another view" not in controls and a["num_seq"] == 1 \
                and a["Lk"] == cfg["S"] * (5 + (cfg["H"] // 14) * (cfg["W"] // 14)):
            try:
                check_attention(cap, k_roll=a["Lk"] // cfg["S"])
                controls["keys of another view"] = (None, 0.0, desc)
            except AssertionError as e:
                msg = str(e).splitlines()[0]
                bad, total = (int(v) for v in re.search(r"(\d+) of (\d+) elements", msg).groups())
                controls["keys of another view"] = (msg[:160], bad / total, desc)
        rec["first"] = rec["last"] = None
        torch.cuda.empty_cache()
    _report(f"{config}: distinct signatures per launcher (all checked)", counts)
    _report(f"{config}: total signatures", len(census.sigs))
    for name in sorted(stats):
        _report(f"{config}: worst {name}", stats[name])
    for c, (verdict, share, desc) in controls.items():
        _report(f"{config}: control '{c}' fails on {share:.2%} of the elements ({desc})", verdict)
    _report(f"{config}: peak device memory GB", torch.cuda.max_memory_allocated() / 2 ** 30)
    _report(f"{config}: seconds (forward + recording, total)", (round(t_fwd, 1), round(time.time() - t0, 1)))
    assert {"gemm_store16", "gemm_resid32", "gemm_qkv", "conv_nhwc", "attention", "dpt_tail_fused"} <= set(counts)
    if cfg["points"]:
        assert "gemm_store32" in counts
    for c in ("bias dropped", "resid2 dropped", "neighbouring tile column", "keys of another view"):
        assert c in controls, f"no signature for the control '{c}'"
        assert controls[c][0] is not None, f"the control '{c}' passed: the check cannot see that error"
    assert not failures, f"{len(failures)} launches failed their statement:\n" + "\n".join(failures)


# ============================================================================================== the sequence, bit for bit
CHILD = r'''
import os, sys, torch
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
import test_launch_census_gpu as T
from iggt_official_b200.graphs import GraphedForward
cfg = T.CONFIGS[sys.argv[2]]
m, images, qp = T._build(cfg)
fn = lambda im: m(im, query_points=qp)

def host(out):
    r = {}
    for k, v in out.items():
        if k == "images":
            continue
        r[k] = torch.stack(v).cpu() if isinstance(v, (list, tuple)) else v.cpu()
    return r

with torch.no_grad():
    runs = {"eager1": host(fn(images)), "eager2": host(fn(images))}
    graphed = GraphedForward(fn, model=m)
    graphed(images)
    runs["graph"] = host(graphed(images))
torch.cuda.synchronize()
torch.save(runs, sys.argv[3])
'''

TOL_ATOMIC = 1e-4                   # part_feat: channel_mean's float atomicAdd order (test_fullsize_gpu.py's tolerance)


def _l2(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["c2_fp16", "demo"])
def test_launch_sequence_is_bit_exact(config, tmp_path):
    runs = {}
    for pdl in (1, 0):
        path = str(tmp_path / f"pdl{pdl}.pt")
        env = dict(os.environ, IGGT_STREAMK="0", IGGT_PDL=str(pdl))
        r = subprocess.run([sys.executable, "-c", CHILD, ROOT, config, path], env=env, cwd=ROOT,
                           capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stderr[-4000:]
        runs[pdl] = torch.load(path)
    ref = runs[1]["eager1"]
    pairs = [("PDL on: eager 2", runs[1]["eager2"]), ("PDL on: graph replay", runs[1]["graph"]),
             ("PDL off: eager 1", runs[0]["eager1"]), ("PDL off: eager 2", runs[0]["eager2"]),
             ("PDL off: graph replay", runs[0]["graph"])]
    diffs = []
    for what, run in pairs:
        assert set(run) == set(ref)
        for k in sorted(ref):
            if k == "part_feat":
                e = _l2(run[k], ref[k])
                assert e < TOL_ATOMIC, (what, k, e)
                _report(f"sequence {config} {what} part_feat rel-L2 (float atomics)", e)
                continue
            if not torch.equal(run[k], ref[k]):
                diffs.append(f"{what}: {k} differs in {int((run[k] != ref[k]).sum())} of {ref[k].numel()} elements")
    _report(f"sequence {config}: outputs compared bit for bit", sorted(k for k in ref if k != "part_feat"))
    assert not diffs, "\n".join(diffs)
