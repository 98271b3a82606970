"""Thin tensor-level wrappers over the C-ABI launchers (device pointers + current CUDA stream).

Every function asserts CUDA tensors and raises if the native library is unavailable; there is no
eager-PyTorch fallback on this path.
"""
import torch

from . import _lib

F16, BF16 = 0, 1


def _dt(t: torch.Tensor) -> int:
    if t.dtype == torch.float16:
        return F16
    if t.dtype == torch.bfloat16:
        return BF16
    raise TypeError(f"expected a 16-bit tensor, got {t.dtype}")


def _ptr(t):
    return 0 if t is None else t.data_ptr()


class _StreamArg:
    """placeholder for "the current stream of the launch device", resolved inside _call (after the device switch)"""


_STREAM = _StreamArg()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _chk2d(t):
    assert t.is_cuda and t.dim() == 2 and t.stride(1) == 1, "expect a CUDA row-major 2-D tensor"




# ---------------------------------------------------------------------------------------------------
# Launch accounting: every C-ABI launch goes through _call().  STATS counts launches (bench.py reports
# them as `gpu_launches`); when TRACE is a list, each launch is bracketed by CUDA events on the launching
# stream together with its algorithmic FLOPs / bytes (bench.py's roofline numbers).
STATS = {"launches": 0}
TRACE = None


def _call(ref, name, flops, nbytes, *args):
    """Launch C-ABI entry point `name` on the device that owns `ref` (one of the launch's tensors) and on that device's
    current stream: `model.to("cuda:1")` works without `torch.cuda.set_device(1)`, like the reference's torch modules."""
    if not ref.is_cuda:
        raise RuntimeError(f"{name}: expected CUDA tensors (there is no CPU fallback on this path)")
    if ref.device.index != torch.cuda.current_device():
        with torch.cuda.device(ref.device):
            return _call(ref, name, flops, nbytes, *args)
    args = [(_stream() if a is _STREAM else a) for a in args]
    fn = getattr(_lib.load(), name)
    STATS["launches"] += 1
    if TRACE is None:
        st = fn(*args)
    else:
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        st = fn(*args)
        e1.record()
        TRACE.append((name, float(flops), float(nbytes), e0, e1, tuple(a for a in args if isinstance(a, int) and 0 < a < (1 << 24))[:8]))
    _lib.check(st, name)


def gemm_store16(a, w, bias=None, act=0, addend=None, add_rows=0, out=None):
    """out16[M,N] = act(a @ w.T + bias) (+ addend[row % add_rows])."""
    _chk2d(a); _chk2d(w)
    M, K = a.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=a.dtype, device=a.device)
    _chk2d(out)
    _call(a, "iggt_gemm_store16", 2.0 * M * N * K, 2.0 * (M * K + N * K + M * N),
          a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0), out.data_ptr(),
                                       out.stride(0), M, N, K, _dt(a), _ptr(bias), act, _ptr(addend),
                                       add_rows if addend is not None else 0,
                                       addend.stride(0) if addend is not None else 0, _STREAM)
    return out


def gemm_store32(a, w, bias=None, act=0, out=None):
    _chk2d(a); _chk2d(w)
    M, K = a.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=a.device)
    _call(a, "iggt_gemm_store32", 2.0 * M * N * K, 2.0 * (M * K + N * K) + 4.0 * M * N,
          a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0), out.data_ptr(),
                                       out.stride(0), M, N, K, _dt(a), _ptr(bias), act, _STREAM)
    return out


def gemm_resid32(a, w, x, bias=None, gamma=None, round_out16=False):
    """x32[M,N] += gamma * (a @ w.T + bias), in place."""
    _chk2d(a); _chk2d(w); _chk2d(x)
    assert x.dtype == torch.float32
    M, K = a.shape
    N = w.shape[0]
    _call(a, "iggt_gemm_resid32", 2.0 * M * N * K, 2.0 * (M * K + N * K) + 8.0 * M * N,
          a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0), x.data_ptr(),
                                       x.stride(0), M, N, K, _dt(a), _ptr(bias), _ptr(gamma),
                                       1 if round_out16 else 0, _STREAM)
    return x


def gemm_qkv(a, w, bias, C, qk_norm=False, qn_w=None, qn_b=None, kn_w=None, kn_b=None, rope_cos=None,
             rope_sin=None, pos_yx=None, T=0, out=None, gather_maps=None, n_gather=0, gather_rows=0):
    _chk2d(a); _chk2d(w)
    M, K = a.shape
    if out is None:
        out = torch.empty((M, 3 * C), dtype=a.dtype, device=a.device)
    _call(a, "iggt_gemm_qkv", 6.0 * M * C * K, 2.0 * (M * K + 3 * C * K + 3 * M * C),
          a.data_ptr(), a.stride(0), w.data_ptr(), w.stride(0), out.data_ptr(),
                                   out.stride(0), M, C, K, _dt(a), _ptr(bias), 1 if qk_norm else 0,
                                   _ptr(qn_w), _ptr(qn_b), _ptr(kn_w), _ptr(kn_b), _ptr(rope_cos),
                                   _ptr(rope_sin), _ptr(pos_yx), T, _ptr(gather_maps), n_gather, gather_rows, _STREAM)
    return out


def kv_gather_maps(dst_windows, rows, cols, ld, scenes, scene_ld, dtype, device):
    """Device array of 3-D tensor maps {cols, rows, scenes} for the fused K|V gather: dst_windows[i] = THIS rank's first row
    inside rank i's gathered buffer (row pitch ld, scene pitch scene_ld elements), as a (peer-mapped) CUDA tensor or an
    integer device address."""
    import ctypes
    n = len(dst_windows)
    ptrs = (ctypes.c_void_p * n)(*[d if isinstance(d, int) else d.data_ptr() for d in dst_windows])
    dev = torch.empty(n * 136 + 16, dtype=torch.uint8, device=device)     # maps | raw pointers | ld, scene_ld
    with torch.cuda.device(device):
        st = _lib.load().iggt_kv_gather_maps(ctypes.cast(ptrs, ctypes.c_void_p), n, rows, cols, ld, scenes, scene_ld,
                                            F16 if dtype == torch.float16 else BF16, dev.data_ptr())
    _lib.check(st, "iggt_kv_gather_maps")
    return dev


def conv_nhwc(x, wp, bias=None, act=0, resid=None, taps=9, out=None, resid2=None, act_post=0):
    """x: [NB,H,W,Cin] 16-bit NHWC contiguous; wp: [Cout, taps*Cin] tap-major packed."""
    assert x.is_cuda and x.dim() == 4 and x.is_contiguous()
    NB, H, W, Cin = x.shape
    Cout = wp.shape[0]
    assert wp.shape[1] == taps * Cin and wp.is_contiguous()
    if out is None:
        out = torch.empty((NB, H, W, Cout), dtype=x.dtype, device=x.device)
    if resid is not None:
        assert resid.shape == out.shape and resid.is_contiguous()
    _call(x, "iggt_conv_nhwc", 2.0 * NB * H * W * Cout * taps * Cin, 2.0 * (NB * H * W * (Cin + Cout) + Cout * taps * Cin),
          x.data_ptr(), wp.data_ptr(), out.data_ptr(), NB, H, W, Cin, Cout, taps,
                                    _dt(x), _ptr(bias), act, _ptr(resid), _ptr(resid2), act_post, _STREAM)
    return out


_ATTN_PLANS = {}


def attention_plan(num_seq, Lq, Lk, H, sms=0):
    """(kv splits, workspace bytes) the library picks for this shape (host-side, cached): > 1 only when the launch has
    too few (sequence, head, query-tile) items for the SMs - the view-sharded global attention."""
    import ctypes
    key = (num_seq, Lq, Lk, H, sms)
    if key not in _ATTN_PLANS:
        s, b = ctypes.c_int(0), ctypes.c_int64(0)
        _lib.check(_lib.load().iggt_attention_plan(num_seq, Lq, Lk, H, sms, ctypes.addressof(s), ctypes.addressof(b)),
                   "iggt_attention_plan")
        _ATTN_PLANS[key] = (s.value, b.value)
    return _ATTN_PLANS[key]


def attention(q, k, v, num_seq, Lq, Lk, H, scale=0.125, out=None, splits=None):
    """q/k/v: 2-D (possibly column-sliced) views [rows, H*64] with unit inner stride.  `splits` (None = the library's
    plan) > 1 runs the split-KV form with a torch-allocated fp32 workspace."""
    for t in (q, k, v):
        _chk2d(t)
    if out is None:
        out = torch.empty((num_seq * Lq, H * 64), dtype=q.dtype, device=q.device)
    if splits is None:
        splits, ws_bytes = attention_plan(num_seq, Lq, Lk, H)
    else:
        ws_bytes = splits * num_seq * Lq * H * 66 * 4 if splits > 1 else 0
    flops, nbytes = 4.0 * num_seq * Lq * Lk * H * 64, 2.0 * num_seq * H * 64 * (2 * Lq + 2 * Lk)
    if splits <= 1:
        _call(q, "iggt_attention_fwd", flops, nbytes,
              q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(),
              v.stride(0), out.data_ptr(), out.stride(0), num_seq, Lq, Lk, H, 64,
              float(scale), _dt(q), _STREAM)
    else:
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=q.device)
        _call(q, "iggt_attention_fwd_ws", flops, nbytes + 2.0 * ws_bytes,
              q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(),
              v.stride(0), out.data_ptr(), out.stride(0), num_seq, Lq, Lk, H, 64,
              float(scale), _dt(q), splits, ws.data_ptr(), ws_bytes, _STREAM)
    return out


_KIND = {torch.float16: 0, torch.bfloat16: 1, torch.float32: 2}


def layernorm(x, w, b, eps, out, groups=None, rows_out=None, rows_in=None, in_off=0, out_rows_per_group=None,
              out_off=0):
    """Row-remapped LayerNorm: out[g*orpg + out_off + i] = LN(x[g*rows_in + in_off + i]), i < rows_out."""
    _chk2d(x); _chk2d(out)
    assert x.dtype == torch.float32
    C = x.shape[1]
    if groups is None:
        groups, rows_out, rows_in = 1, x.shape[0], x.shape[0]
    if out_rows_per_group is None:
        out_rows_per_group = rows_out
    _call(x, "iggt_layernorm", 0, groups * rows_out * C * (4 + out.element_size()),
          x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), C, _ptr(w),
                                    _ptr(b), float(eps), groups, rows_out, rows_in, in_off,
                                    out_rows_per_group, out_off, _KIND[out.dtype], _STREAM)
    return out


def patchify(images, KP, dtype):
    """images [NI,3,H,W] fp32 -> [NI*gh*gw, KP] 16-bit normalised im2col."""
    assert images.is_cuda and images.dtype == torch.float32 and images.is_contiguous()
    NI, _, H, W = images.shape
    A = torch.empty((NI * (H // 14) * (W // 14), KP), dtype=dtype, device=images.device)
    _call(images, "iggt_patchify", 0, images.numel() * 4 + A.numel() * 2,
          images.data_ptr(), A.data_ptr(), NI, H, W, KP, _KIND[dtype], _STREAM)
    return A


def dino_assemble(pe16, cls, reg, pos, x, NI, P, R, C):
    _call(pe16, "iggt_dino_assemble", 0, x.numel() * 4 + pe16.numel() * 2,
          pe16.data_ptr(), cls.data_ptr(), reg.data_ptr(), pos.data_ptr(),
                                        x.data_ptr(), NI, P, R, C, _dt(pe16), _STREAM)
    return x


def special_tokens(cam, reg, x, NI, T, R, C, S_loc, view_offset):
    _call(cam, "iggt_special_tokens", 0, NI * (1 + R) * C * 4,
          cam.data_ptr(), reg.data_ptr(), x.data_ptr(), NI, T, R, C, S_loc,
                                         view_offset, _STREAM)
    return x


def upsample_bilinear(x, H, W, tabx=None, taby=None, out=None):
    """[NB,h,w,C] 16-bit NHWC -> [NB,H,W,C], align_corners=True (+ optional split pos-embed tables)."""
    assert x.is_cuda and x.dim() == 4 and x.is_contiguous()
    NB, h, w, C = x.shape
    if out is None:
        out = torch.empty((NB, H, W, C), dtype=x.dtype, device=x.device)
    _call(x, "iggt_upsample_bilinear_nhwc", 0, 2.0 * (x.numel() + out.numel()),
          x.data_ptr(), out.data_ptr(), NB, h, w, H, W, C, _ptr(tabx),
                                                 _ptr(taby), _dt(x), _STREAM)
    return out


def deconv_shuffle(y, NB, h, w, C, k):
    out = torch.empty((NB, h * k, w * k, C), dtype=y.dtype, device=y.device)
    _call(y, "iggt_deconv_shuffle", 0, 4.0 * y.numel(),
          y.data_ptr(), out.data_ptr(), NB, h, w, C, k, _STREAM)
    return out


def im2col3x3_s2(x):
    NB, h, w, C = x.shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    A = torch.empty((NB * ho * wo, 9 * C), dtype=x.dtype, device=x.device)
    _call(x, "iggt_im2col3x3_s2", 0, 2.0 * (x.numel() + A.numel()),
          x.data_ptr(), A.data_ptr(), NB, h, w, C, _STREAM)
    return A, ho, wo


def dpt_tail(x, w, b, mode):
    """x [NB,H,W,32] 16-bit -> (main, conf) fp32; mode 0 depth, 1 points, 2 part (channels-first, conf None)."""
    NB, H, W, _ = x.shape
    OC = w.shape[0]
    if mode == 2:
        main = torch.empty((NB, OC, H, W), dtype=torch.float32, device=x.device)
        conf = None
    else:
        main = torch.empty((NB, H, W, OC - 1), dtype=torch.float32, device=x.device)
        conf = torch.empty((NB, H, W), dtype=torch.float32, device=x.device)
    _call(x, "iggt_dpt_tail", 2.0 * NB * H * W * 32 * OC, NB * H * W * (64 + 4 * OC),
          x.data_ptr(), w.data_ptr(), b.data_ptr(), main.data_ptr(), _ptr(conf), NB, H, W,
                                   OC, mode, _dt(x), _STREAM)
    return main, conf


def dpt_tail_fused(x, wp, bias, w2, b2, mode):
    """x [NB,H,W,128] 16-bit NHWC -> 3x3 conv (wp [32, 9*128] tap-major) + bias + ReLU -> 1x1 (w2 [OC,32] fp32) ->
    head activation, one launch (csrc/tailconv.cu).  Returns (main, conf) like `dpt_tail`."""
    assert x.is_cuda and x.dim() == 4 and x.is_contiguous() and x.shape[3] == 128
    assert wp.shape == (32, 9 * 128) and wp.is_contiguous() and wp.dtype == x.dtype
    NB, H, W, _ = x.shape
    OC = w2.shape[0]
    if mode == 2:
        main = torch.empty((NB, OC, H, W), dtype=torch.float32, device=x.device)
        conf = None
    else:
        main = torch.empty((NB, H, W, OC - 1), dtype=torch.float32, device=x.device)
        conf = torch.empty((NB, H, W), dtype=torch.float32, device=x.device)
    _call(x, "iggt_dpt_tail_fused", 2.0 * NB * H * W * 32 * (9 * 128 + OC), NB * H * W * (256.0 + 4 * OC),
          x.data_ptr(), wp.data_ptr(), bias.data_ptr(), w2.data_ptr(), b2.data_ptr(), main.data_ptr(), _ptr(conf), 0,
          NB, H, W, OC, mode, _dt(x), _STREAM)
    return main, conf


def conv3x3_c128_relu(x, wp, bias):
    """The unfused form of `dpt_tail_fused` (same kernel, stores the 32-channel ReLU map): for A/B checks."""
    assert x.is_cuda and x.dim() == 4 and x.is_contiguous() and x.shape[3] == 128 and wp.shape == (32, 9 * 128)
    NB, H, W, _ = x.shape
    out = torch.empty((NB, H, W, 32), dtype=x.dtype, device=x.device)
    _call(x, "iggt_dpt_tail_fused", 2.0 * NB * H * W * 32 * 9 * 128, NB * H * W * (256.0 + 64),
          x.data_ptr(), wp.data_ptr(), bias.data_ptr(), 0, 0, 0, 0, out.data_ptr(), NB, H, W, 0, 0, _dt(x), _STREAM)
    return out


def skinny_gemm(x, w, bias=None, act=0, gamma=None, resid=None, out=None):
    """fp32 x [M<=32, K] times 16-bit w [N, K]^T -> fp32 [M, N]."""
    _chk2d(x); _chk2d(w)
    assert x.dtype == torch.float32
    M, K = x.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=torch.float32, device=x.device)
    _call(x, "iggt_skinny_gemm", 2.0 * M * N * K, 2.0 * N * K + 4.0 * M * (K + N),
          x.data_ptr(), x.stride(0), w.data_ptr(), w.stride(0), _ptr(bias), _ptr(gamma),
                                      _ptr(resid), resid.stride(0) if resid is not None else 0, out.data_ptr(),
                                      out.stride(0), M, N, K, act, _dt(w), _STREAM)
    return out


def small_attention(qkv, B, N, H, d):
    if N > 256 or (2 * N * d + 4 * N) * 4 > 200 * 1024:
        raise ValueError(f"the camera head's token attention keeps all {N} views' keys and values of a head in shared memory "
                         f"(<= 256 views, <= {200 * 1024 // (8 * d + 16)} at head dim {d}); split the scene into fewer views per call")
    out = torch.empty((B * N, H * d), dtype=torch.float32, device=qkv.device)
    _call(qkv, "iggt_small_attention", 4.0 * B * N * N * H * d, 16.0 * B * N * H * d,
          qkv.data_ptr(), out.data_ptr(), B, N, H, d, float(d) ** -0.5, _STREAM)
    return out


def camera_head(weights, keepalive, tokens, B, S, iters, dtype, return_workspace=False):
    """The whole camera head in one persistent launch (csrc/camera.cu).  `weights`: a filled `_lib.CameraWeights`,
    `keepalive`: the tensors it points to; `tokens`: fp32 camera-token rows [B*S, 2048] (any row pitch).  Returns
    the activated pose encodings fp32 [iters, B*S, 9]."""
    import ctypes
    assert tokens.is_cuda and tokens.dtype == torch.float32 and tokens.dim() == 2 and tokens.shape[1] == 2048 and tokens.stride(1) == 1
    M = B * S
    assert tokens.shape[0] == M
    ws_bytes = int(_lib.load().iggt_camera_head_workspace(M))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=tokens.device)
    out = torch.empty((iters, M, 9), dtype=torch.float32, device=tokens.device)
    wbytes = 2.0 * (2048 * 16 + 6144 * 2048 + 4 * (6144 * 2048 + 2048 * 2048 + 2 * 8192 * 2048) + 1024 * 2048 + 9 * 1024)
    _call(tokens, "iggt_camera_head", 2.0 * M * iters * wbytes / 2, iters * wbytes,
          ctypes.addressof(weights), tokens.data_ptr(), tokens.stride(0), out.data_ptr(), ws.data_ptr(), ws_bytes, B, S,
          iters, F16 if dtype == torch.float16 else BF16, _STREAM)
    return (out, ws) if return_workspace else out


def layernorm16(x, w, b, eps=1e-5, out=None):
    """LayerNorm over the last dim (64 / 128 / 256) of a contiguous 16-bit tensor."""
    assert x.is_cuda and x.is_contiguous()
    C = x.shape[-1]
    rows = x.numel() // C
    if out is None:
        out = torch.empty_like(x)
    _call(x, "iggt_layernorm16", 0, 4.0 * x.numel(), x.data_ptr(), out.data_ptr(), rows, C, w.data_ptr(), b.data_ptr(),
          float(eps), _dt(x), _STREAM)
    return out


def col2im_k4s2p1(y, bias, NB, h, w, C):
    out = torch.empty((NB, 2 * h, 2 * w, C), dtype=y.dtype, device=y.device)
    _call(y, "iggt_col2im_k4s2p1", 0, 2.0 * (y.numel() + out.numel()), y.data_ptr(), bias.data_ptr(), out.data_ptr(),
          NB, h, w, C, _dt(y), _STREAM)
    return out


def ocab_attention(q, k, v, table, rpi):
    """q, k, v: [NB,h,w,256] contiguous 16-bit; table [361,4] fp32; rpi [64,144] int32 in [0,361)."""
    NB, h, w, C = q.shape
    assert C == 256 and q.is_contiguous() and k.is_contiguous() and v.is_contiguous()
    out = torch.empty_like(q)
    _call(q, "iggt_ocab_attention", 4.0 * NB * (h // 8) * (w // 8) * 4 * 64 * 144 * 64, 8.0 * q.numel(),
          q.data_ptr(), k.data_ptr(), v.data_ptr(), table.data_ptr(), rpi.data_ptr(), out.data_ptr(), NB, h, w,
          _dt(q), _STREAM)
    return out


def window_attention(qkv):
    """qkv [NB,h,w,384] contiguous 16-bit -> [NB,h,w,128]."""
    NB, h, w, C3 = qkv.shape
    assert C3 == 384 and qkv.is_contiguous()
    out = torch.empty((NB, h, w, 128), dtype=qkv.dtype, device=qkv.device)
    _call(qkv, "iggt_window_attention", 4.0 * NB * (h // 8) * (w // 8) * 4 * 64 * 64 * 32, 2.0 * (qkv.numel() + out.numel()),
          qkv.data_ptr(), out.data_ptr(), NB, h, w, _dt(qkv), _STREAM)
    return out


def channel_mean(x):
    """x [NB,h,w,C] 16-bit -> [NB,C] fp32 spatial means."""
    NB, h, w, C = x.shape
    mean = torch.empty((NB, C), dtype=torch.float32, device=x.device)
    _call(x, "iggt_channel_mean", 0, 2.0 * x.numel(), x.data_ptr(), mean.data_ptr(), NB, h * w, C, _dt(x), _STREAM)
    return mean


def se_scale_add(y0, cx, mean, w1, b1, w2, b2, alpha):
    NB, h, w, C = y0.shape
    out = torch.empty_like(y0)
    _call(y0, "iggt_se_scale_add", 0, 6.0 * y0.numel(), y0.data_ptr(), cx.data_ptr(), mean.data_ptr(), w1.data_ptr(),
          b1.data_ptr(), w2.data_ptr(), b2.data_ptr(), out.data_ptr(), NB, h * w, C, w1.shape[0], float(alpha),
          _dt(y0), _STREAM)
    return out


def pose_to_cameras(pose_enc, H, W, build_intrinsics=True):
    """pose_enc [..., 9] fp32 -> (extrinsics [..., 3, 4], intrinsics [..., 3, 3] or None)."""
    assert pose_enc.is_cuda and pose_enc.dtype == torch.float32 and pose_enc.shape[-1] == 9
    p = pose_enc.contiguous()
    n = p.numel() // 9
    extr = torch.empty(p.shape[:-1] + (3, 4), dtype=torch.float32, device=p.device)
    intr = torch.empty(p.shape[:-1] + (3, 3), dtype=torch.float32, device=p.device) if build_intrinsics else None
    _call(pose_enc, "iggt_pose_to_cameras", 0, 30.0 * 4 * n, p.data_ptr(), extr.data_ptr(), _ptr(intr), n, H, W, _STREAM)
    return extr, intr


def unproject_depth(depth, extrinsics, intrinsics, eps=1e-8, z_far=100.0, with_mask=True):
    """depth [n,H,W] (or [n,H,W,1]) fp32, cameras per view -> (world [n,H,W,3], mask [n,H,W] bool or None)."""
    if depth.dim() == 4:
        depth = depth[..., 0]
    d = depth.contiguous()
    n, H, W = d.shape
    e = extrinsics.reshape(n, 3, 4).contiguous()
    k = intrinsics.reshape(n, 3, 3).contiguous()
    world = torch.empty((n, H, W, 3), dtype=torch.float32, device=d.device)
    mask = torch.empty((n, H, W), dtype=torch.uint8, device=d.device) if with_mask else None
    _call(depth, "iggt_unproject_depth", 0, 17.0 * d.numel(), d.data_ptr(), e.data_ptr(), k.data_ptr(), world.data_ptr(),
          _ptr(mask), n, H, W, float(eps), float(z_far), _STREAM)
    return world, (mask.bool() if mask is not None else None)


def resample_bicubic_u8(src, kk_h, bounds_h, kk_v, bounds_v, out, oy0=0):
    """Pillow-exact 8-bit bicubic resize + ToTensor.  src u8 [Hin, Win, 3] (CUDA);  kk_* int32 [size, ksize] and
    bounds_* int32 [size, 2] are the fixed-point tap tables of each pass (load_fn.precompute_coeffs);  out is a
    planar fp32 view [3, rows, Wout] (any plane / row stride, unit column stride) that receives output rows
    [oy0, oy0 + rows) of the resized image divided by 255."""
    assert src.is_cuda and src.dtype == torch.uint8 and src.dim() == 3 and src.shape[2] == 3 and src.is_contiguous()
    assert out.is_cuda and out.dtype == torch.float32 and out.dim() == 3 and out.shape[0] == 3 and out.stride(2) == 1
    for t in (kk_h, bounds_h, kk_v, bounds_v):
        assert t.is_cuda and t.dtype == torch.int32 and t.is_contiguous()
    h_in, w_in, _ = src.shape
    w_out, rows = kk_h.shape[0], out.shape[1]
    assert out.shape[2] == w_out and oy0 >= 0 and oy0 + rows <= kk_v.shape[0]
    bv = bounds_v[oy0:oy0 + rows].cpu()
    first = int(bv[0, 0])                                  # source rows the vertical pass of this window touches
    last = int(bv[-1, 0] + bv[-1, 1])
    assert 0 <= first < last <= h_in
    tmp = torch.empty((last - first, w_out, 3), dtype=torch.uint8, device=src.device)
    _call(src, "iggt_resample_h_u8", 0, float((last - first) * 3 * (w_in + w_out)), src[first:].data_ptr(), w_in * 3,
          last - first, w_out, kk_h.data_ptr(), bounds_h.data_ptr(), kk_h.shape[1], tmp.data_ptr(), _STREAM)
    _call(src, "iggt_resample_v_u8_f32", 0, float(tmp.numel() + out.numel() * 4), tmp.data_ptr(), w_out, kk_v.data_ptr(),
          bounds_v.data_ptr(), kk_v.shape[1], first, oy0, rows, out.data_ptr(), out.stride(0), out.stride(1), _STREAM)
    return out


def knn_mean_features(points, feats, k, return_graph=False, stats=None):
    """points [n,3] fp32, feats [n,F] fp32 (or None) -> mean over each point's k nearest OTHER points of their feature
    rows [n,F] (and, with return_graph, (idx [n,k] int32, d2 [n,k])).  Exact; the only library call is the radix sort
    of the Morton codes (the search is exact for any ordering, the curve only tightens the tile boxes)."""
    assert points.is_cuda and points.dtype == torch.float32 and points.dim() == 2 and points.shape[1] == 3
    pts = points.contiguous()
    n = pts.shape[0]
    assert 0 < n < 2 ** 31 and 0 < k <= 32
    dev = pts.device
    lo, hi = pts.amin(0).contiguous(), pts.amax(0).contiguous()
    codes = torch.empty(n, dtype=torch.int64, device=dev)
    _call(points, "iggt_knn_morton", 0, 20.0 * n, pts.data_ptr(), n, lo.data_ptr(), hi.data_ptr(), codes.data_ptr(), _STREAM)
    order = torch.argsort(codes)
    nblocks = (n + 255) // 256
    sorted4 = torch.empty((n, 4), dtype=torch.float32, device=dev)
    aabb = torch.empty((nblocks, 6), dtype=torch.float32, device=dev)
    _call(points, "iggt_knn_reorder", 0, 36.0 * n, pts.data_ptr(), order.data_ptr(), n, sorted4.data_ptr(), aabb.data_ptr(),
          _STREAM)
    out = None
    F = 0
    if feats is not None:
        assert feats.is_cuda and feats.dtype == torch.float32 and feats.dim() == 2 and feats.shape[0] == n
        feats = feats.contiguous()
        F = feats.shape[1]
        out = torch.empty_like(feats)
    idx = torch.empty((n, k), dtype=torch.int32, device=dev) if return_graph else None
    d2 = torch.empty((n, k), dtype=torch.float32, device=dev) if return_graph else None
    _call(points, "iggt_knn_mean_features", 0, float(n) * (16 + 4 * F * (k + 1)), sorted4.data_ptr(), aabb.data_ptr(), n, k,
          _ptr(feats), F, _ptr(out), _ptr(idx), _ptr(d2), _ptr(stats), _STREAM)
    return (out, idx, d2) if return_graph else out


# ---------------------------------------------------------------------------------------------------
# HDBSCAN of the instance features (csrc/cluster.cu)
def cluster_prepare(x):
    """x [n,8] fp32 -> (sorted8 [n,8], orig [n] int32, box [ceil(n/256),16]): Morton order (stable library sort) and
    the bounding box of every tile of 256 sorted points."""
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.shape[1] == 8
    x = x.contiguous()
    n = x.shape[0]
    assert 0 < n < 2 ** 31
    lo, hi = x.amin(0).contiguous(), x.amax(0).contiguous()
    codes = torch.empty(n, dtype=torch.int64, device=x.device)
    _call(x, "iggt_cluster_morton", 0, 72.0 * n, x.data_ptr(), n, lo.data_ptr(), hi.data_ptr(), codes.data_ptr(), _STREAM)
    order = torch.sort(codes, stable=True).indices
    sorted8 = torch.empty_like(x)
    orig = torch.empty(n, dtype=torch.int32, device=x.device)
    box = torch.empty(((n + 255) // 256, 16), dtype=torch.float32, device=x.device)
    _call(x, "iggt_cluster_reorder", 0, 76.0 * n, x.data_ptr(), order.data_ptr(), n, sorted8.data_ptr(), orig.data_ptr(),
          box.data_ptr(), _STREAM)
    return sorted8, orig, box


def cluster_core(sorted8, box, k):
    """Squared distance of every sorted point to its k-th nearest other point -> core2 [n] (sorted order)."""
    n = sorted8.shape[0]
    assert 1 <= k <= 512 and k < n
    core2 = torch.empty(n, dtype=torch.float32, device=sorted8.device)
    _call(sorted8, "iggt_cluster_core", 0, 36.0 * n, sorted8.data_ptr(), box.data_ptr(), n, int(k), core2.data_ptr(),
          _STREAM)
    return core2


def cluster_mst(sorted8, box, orig, core2):
    """Minimum spanning tree of the mutual-reachability graph -> (a [n-1] int32, b [n-1] int32, w2 [n-1] squared
    weights, rounds): unsorted edges between original point indices."""
    import ctypes
    n = sorted8.shape[0]
    assert n >= 2
    ws_bytes = ctypes.c_int64()
    _lib.check(_lib.load().iggt_cluster_mst_workspace(n, ctypes.byref(ws_bytes)), "iggt_cluster_mst_workspace")
    ws = torch.empty(ws_bytes.value, dtype=torch.uint8, device=sorted8.device)
    a = torch.empty(n - 1, dtype=torch.int32, device=sorted8.device)
    b = torch.empty_like(a)
    w2 = torch.empty(n - 1, dtype=torch.float32, device=sorted8.device)
    rounds = ctypes.c_int32(0)
    _call(sorted8, "iggt_cluster_mst", 0, 48.0 * n, sorted8.data_ptr(), box.data_ptr(), orig.data_ptr(), core2.data_ptr(),
          n, ws.data_ptr(), a.data_ptr(), b.data_ptr(), w2.data_ptr(), ctypes.byref(rounds), _STREAM)
    return a, b, w2, rounds.value


def hdbscan_labels(mst, n, min_cluster_size, eps):
    """Host (no GPU): mst [n-1,3] float64 (a, b, weight) sorted by weight -> labels [n] int64 (-1 = noise), numbered
    as scikit-learn's tree_to_labels numbers them."""
    import numpy as np
    mst = np.ascontiguousarray(mst, dtype=np.float64)
    assert mst.shape == (n - 1, 3)
    labels = np.empty(n, dtype=np.int64)
    _lib.check(_lib.load().iggt_hdbscan_labels(mst.ctypes.data, int(n), int(min_cluster_size), float(eps),
                                               labels.ctypes.data), "iggt_hdbscan_labels")
    return labels


def mst_orient(mst, root=0):
    """Host (no GPU): orients the rows (a, b, weight) of mst [n-1,3] float64 in place from parent to child of the tree
    rooted at point `root` - the orientation scikit-learn's Prim MST from point 0 records."""
    import numpy as np
    assert isinstance(mst, np.ndarray) and mst.dtype == np.float64 and mst.flags.c_contiguous and mst.shape[1] == 3
    _lib.check(_lib.load().iggt_mst_orient(mst.ctypes.data, mst.shape[0] + 1, int(root)), "iggt_mst_orient")
    return mst


def cluster_fill(sorted8, box, orig, label_sorted, palette=None):
    """label_sorted [n] int32 (sorted order, -1 = noise, at least one labelled point) -> (labels [n] int64, rgb [n,3]
    uint8 or None) at the original indices: noise points take the label of their nearest labelled point."""
    n = sorted8.shape[0]
    assert label_sorted.dtype == torch.int32 and label_sorted.shape == (n,)
    dev = sorted8.device
    tile_count = torch.empty((n + 255) // 256, dtype=torch.int32, device=dev)
    out = torch.empty(n, dtype=torch.int64, device=dev)
    rgb = None
    if palette is not None:
        assert palette.dtype == torch.uint8 and palette.is_cuda and palette.dim() == 2 and palette.shape[1] == 3
        palette = palette.contiguous()
        rgb = torch.empty((n, 3), dtype=torch.uint8, device=dev)
    _call(sorted8, "iggt_cluster_fill", 0, 48.0 * n, sorted8.data_ptr(), box.data_ptr(), orig.data_ptr(),
          label_sorted.data_ptr(), n, tile_count.data_ptr(), _ptr(palette), out.data_ptr(), _ptr(rgb), _STREAM)
    return out, rgb


# ---------------------------------------------------------------------------------------------------
# PCA feature colours and exact quantiles (csrc/pca.cu)
class PcaBasis:
    """Device outputs of iggt_pca_basis: moments [C + C(C+1)/2] f64, cov [C,C] f64, evals [C] f64, evecs [C,C] f64,
    V [C,3] fp32 (the first three eigenvectors) and nonfinite [1] int64."""

    def __init__(self, C, device):
        f64 = dict(dtype=torch.float64, device=device)
        self.moments = torch.empty(C + C * (C + 1) // 2, **f64)
        self.cov = torch.empty((C, C), **f64)
        self.evals = torch.empty(C, **f64)
        self.evecs = torch.empty((C, C), **f64)
        self.V = torch.empty((C, 3), dtype=torch.float32, device=device)
        self.nonfinite = torch.empty(1, dtype=torch.int64, device=device)


def _workspace(query, *args):
    import ctypes
    nbytes = ctypes.c_int64()
    _lib.check(getattr(_lib.load(), query)(*args, ctypes.byref(nbytes)), query)
    return nbytes.value


def pca_basis(x):
    """x [n,C] fp32 (3 <= C <= 8) -> PcaBasis: fixed-order fp64 moments, the sample covariance and its Jacobi
    eigendecomposition, all on the device (no host synchronisation)."""
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and 3 <= x.shape[1] <= 8
    x = x.contiguous()
    n, C = x.shape
    assert n > 0
    ws = torch.empty(_workspace("iggt_pca_basis_workspace", C), dtype=torch.uint8, device=x.device)
    b = PcaBasis(C, x.device)
    _call(x, "iggt_pca_basis", 3.0 * n * C * (C + 3), 4.0 * n * C, x.data_ptr(), n, C, ws.data_ptr(), b.moments.data_ptr(),
          b.cov.data_ptr(), b.evals.data_ptr(), b.evecs.data_ptr(), b.V.data_ptr(), b.nonfinite.data_ptr(), _STREAM)
    return b


def pca_project(x, V):
    """x [n,C] fp32, V [C,3] fp32 -> y [3,n] fp32 = (x @ V).T (fp32 fmas in channel order).  The rows of y are
    padded to a multiple of 4 floats (16-byte aligned rows for the later stages)."""
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and 3 <= x.shape[1] <= 8
    x = x.contiguous()
    n, C = x.shape
    assert V.dtype == torch.float32 and V.shape == (C, 3)
    V = V.contiguous()
    ldy = (n + 3) // 4 * 4
    y = torch.empty((3, ldy), dtype=torch.float32, device=x.device)
    _call(x, "iggt_pca_project", 6.0 * n * C, 4.0 * n * (C + 3), x.data_ptr(), n, C, V.data_ptr(), y.data_ptr(), ldy,
          _STREAM)
    return y[:, :n]


def quantile(y, q):
    """y [rows,n] fp32 (unit column stride), q: sequence of floats in [0, 1] -> [rows, len(q)] fp32, equal to
    torch.quantile(y[r], q[i]) bit for bit (linear interpolation; a row with a NaN gives NaN), for any n < 2^32."""
    import ctypes
    assert y.is_cuda and y.dtype == torch.float32 and y.dim() == 2 and y.stride(1) == 1
    rows, n = y.shape
    q = [float(v) for v in q]
    assert 0 < rows <= 65535 and 0 < n < 2 ** 32 and len(q) > 0 and all(0.0 <= v <= 1.0 for v in q)
    ws = torch.empty(_workspace("iggt_quantile_workspace", rows), dtype=torch.uint8, device=y.device)
    out = torch.empty((rows, len(q)), dtype=torch.float32, device=y.device)
    qa = (ctypes.c_float * len(q))(*q)
    passes = 3 * ((len(q) + 1) // 2)                      # three radix passes per pair of quantiles
    _call(y, "iggt_quantile", 0, 4.0 * rows * n * passes, y.data_ptr(), rows, n, y.stride(0), qa, len(q), ws.data_ptr(),
          out.data_ptr(), _STREAM)
    return out


def pca_stretch(y, qv):
    """y [3,n] fp32 (unit column stride), qv [3,2] fp32 (lo, hi) -> out [n,3] fp32 =
    clamp((y.T - lo) / (hi - lo), 0, 1), 0.5 in a channel whose hi <= lo."""
    assert y.is_cuda and y.dtype == torch.float32 and y.dim() == 2 and y.shape[0] == 3 and y.stride(1) == 1
    assert qv.is_cuda and qv.dtype == torch.float32 and qv.shape == (3, 2)
    qv = qv.contiguous()
    n = y.shape[1]
    out = torch.empty((n, 3), dtype=torch.float32, device=y.device)
    _call(y, "iggt_pca_stretch", 3.0 * n, 24.0 * n, y.data_ptr(), n, y.stride(0), qv.data_ptr(), out.data_ptr(), _STREAM)
    return out


def sym_eig(a):
    """Host (no GPU): a [C,C] float64 symmetric (1 <= C <= 8) -> (evals [C] descending, evecs [C,C] with eigenvector j
    in column j, its largest-magnitude component positive) by the cyclic Jacobi code iggt_pca_basis runs."""
    import numpy as np
    a = np.ascontiguousarray(a, dtype=np.float64)
    C = a.shape[0]
    assert a.shape == (C, C) and 1 <= C <= 8
    evals = np.empty(C, np.float64)
    evecs = np.empty((C, C), np.float64)
    _lib.check(_lib.load().iggt_sym_eig(a.ctypes.data, C, evals.ctypes.data, evecs.ctypes.data), "iggt_sym_eig")
    return evals, evecs


# ---------------------------------------------------------------------------------------------------
# Track head (csrc/track.cu)
def avgpool2_nhwc(x):
    """[NB,H,W,C] 16-bit -> [NB,H//2,W//2,C]."""
    assert x.is_cuda and x.is_contiguous() and x.dim() == 4
    NB, H, W, C = x.shape
    y = torch.empty((NB, H // 2, W // 2, C), dtype=x.dtype, device=x.device)
    _call(x, "iggt_avgpool2_nhwc", 0, 2.0 * (x.numel() + y.numel()), x.data_ptr(), y.data_ptr(), NB, H, W, C, _dt(x), _STREAM)
    return y


def sample_bilinear_nhwc(x, coords):
    """x [NB,H,W,C] 16-bit, coords [NB,R,2] fp32 (x,y) pixels -> [NB,R,C] fp32 (border padding, align_corners)."""
    assert x.is_cuda and x.is_contiguous() and coords.dtype == torch.float32
    NB, H, W, C = x.shape
    coords = coords.contiguous()
    R = coords.shape[1]
    out = torch.empty((NB, R, C), dtype=torch.float32, device=x.device)
    _call(x, "iggt_sample_bilinear_nhwc", 0, 12.0 * out.numel(), x.data_ptr(), coords.data_ptr(), out.data_ptr(), NB, R, H, W,
          C, _dt(x), _STREAM)
    return out


def corr_sample(levels, targets, coords, B, N, S, ldo=576):
    """levels: 7 NHWC [B*S,H_l,W_l,128] 16-bit maps; targets [B*N*S,128], coords [B*N*S,2] fp32 in (b,n,s) row order
    -> [B*N*S, ldo] 16-bit (7 x 81 correlations, zero padded: the A operand of the corr MLP)."""
    import ctypes
    assert len(levels) == 7 and all(l.is_cuda and l.is_contiguous() and l.shape[-1] == 128 for l in levels)
    assert targets.dtype == torch.float32 and targets.is_contiguous() and coords.dtype == torch.float32
    coords = coords.contiguous()
    rows = B * N * S
    out = torch.empty((rows, ldo), dtype=levels[0].dtype, device=targets.device)
    ptrs = (ctypes.c_void_p * 7)(*[l.data_ptr() for l in levels])
    Hs = (ctypes.c_int * 7)(*[l.shape[1] for l in levels])
    Ws = (ctypes.c_int * 7)(*[l.shape[2] for l in levels])
    _call(targets, "iggt_corr_sample", 2.0 * rows * 7 * 100 * 128, rows * 7.0 * 100 * 256,
          ctypes.cast(ptrs, ctypes.c_void_p), ctypes.cast(Hs, ctypes.c_void_p), ctypes.cast(Ws, ctypes.c_void_p),
          targets.data_ptr(), coords.data_ptr(), out.data_ptr(), B, N, S, ldo, _dt(levels[0]), _STREAM)
    return out


def track_input(coords, fcorr, tfeat, pos, ref_tok, ln_w, ln_b, S, dtype, ldo=392, want_raw=False):
    """Rows (b,n,s): coords [rows,2], fcorr / tfeat [rows,128], pos [B*N,388], ref_tok [2,388] (all fp32) ->
    LayerNorm(388)'d transformer input [rows, ldo] 16-bit (and the fp32 pre-norm rows when want_raw)."""
    rows = coords.shape[0]
    for t in (coords, fcorr, tfeat, pos, ref_tok, ln_w, ln_b):
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
    out = torch.empty((rows, ldo), dtype=dtype, device=coords.device)
    raw = torch.empty((rows, 388), dtype=torch.float32, device=coords.device) if want_raw else None
    _call(coords, "iggt_track_input", 0, rows * (388.0 * 6 + 2 * ldo), coords.data_ptr(), fcorr.data_ptr(), tfeat.data_ptr(),
          pos.data_ptr(), ref_tok.data_ptr(), ln_w.data_ptr(), ln_b.data_ptr(), out.data_ptr(), _ptr(raw), rows, S, ldo,
          1e-5, F16 if dtype == torch.float16 else BF16, _STREAM)
    return (out, raw) if want_raw else out


def layernorm_rows(x, w, b, eps=1e-5, out32=None, out16=None):
    """LayerNorm of fp32 rows x [rows,C] (last-dim stride 1, any row pitch) into out32 [rows,C] and / or out16 [rows,>=C]."""
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
    rows, C = x.shape
    assert out32 is not None or out16 is not None
    if out32 is not None:
        assert out32.dtype == torch.float32 and out32.is_contiguous() and tuple(out32.shape) == (rows, C)
    ld16, dt = 0, 0
    if out16 is not None:
        assert out16.is_contiguous() and out16.shape[0] == rows and out16.shape[1] >= C
        ld16, dt = out16.shape[1], _dt(out16)
    _call(x, "iggt_layernorm_rows", 0, rows * C * 10.0, x.data_ptr(), x.stride(0), C, w.data_ptr(), b.data_ptr(), float(eps),
          rows, _ptr(out32), _ptr(out16), ld16, dt, _STREAM)
    return out32, out16
