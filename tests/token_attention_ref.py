"""The token attention of the camera head for scenes of any number of views (csrc/heads.cu, `token_attention_kernel`):
a float64 reference, an fp32 torch statement of the kernel's tile walk, and the per-element error bound derived from
the kernel's operation order.  Shared by tests/test_many_views_cpu.py (which shows the bound accepts the tile walk and
rejects a walk with one rescale skipped) and tests/test_many_views_gpu.py (which holds the kernel to it)."""
import math

import torch

U24 = 2.0 ** -24
KT = 64                         # keys per tile (TA_KT)


def split(qkv, B, N, H, d):
    """qkv [B*N, 3*H*d] -> q, k, v [B, H, N, d]"""
    return qkv.view(B, N, 3, H, d).permute(2, 0, 3, 1, 4)


def flat(t):
    """[B, H, N, d] -> [B*N, H*d], the layout of the kernel's output"""
    B, H, N, d = t.shape
    return t.transpose(1, 2).reshape(B * N, H * d)


def tile_walk(qkv, B, N, H, d, skip_rescale_at=None):
    """fp32 statement of the kernel: key tiles of KT in order, a running max m and sum l per query row, acc and l
    rescaled by exp(m_old - m_new), p = exp(s - m_new), l = l * alpha + sum(p), acc = acc * alpha + p v, out = acc * (1 / l).
    `skip_rescale_at`: the tile whose rescale is left out (a broken walk, for showing that the bound rejects it)."""
    q, k, v = split(qkv.float(), B, N, H, d)
    scale = d ** -0.5
    m = torch.full(q.shape[:-1] + (1,), -math.inf, dtype=torch.float32)
    l = torch.zeros_like(m)
    acc = torch.zeros_like(q)
    for t, t0 in enumerate(range(0, N, KT)):
        s = (q @ k[..., t0:t0 + KT, :].transpose(-1, -2)) * scale
        mn = torch.maximum(m, s.amax(-1, keepdim=True))
        alpha = torch.exp(m - mn)
        if t == skip_rescale_at:
            alpha = torch.ones_like(alpha)
        p = torch.exp(s - mn)
        l = l * alpha + p.sum(-1, keepdim=True)
        acc = acc * alpha + p @ v[..., t0:t0 + KT, :]
        m = mn
    return flat(acc * (1.0 / l))


def reference_and_bound(qkv, B, N, H, d):
    """float64 attention O64 [B*N, H*d] and the per-element bound |O - O64| of the kernel.  In the kernel's order:
      s = fmaf chain over d (d 2^-24 of scale |q|.|k|), * RN(scale) (2 roundings: 2^-23 |s|);
      p = expf(s - m_t), m_t the running max after the key's tile t: the subtraction 2^-24 |s - m_t|, expf 2^-22;
      every later tile t' multiplies the key's weight by alpha = expf(m_t'-1 - m_t'): 2^-24 |m_t'-1 - m_t'| + 2^-22, and
      acc * alpha rounds once more (2^-24) - the running maxima cancel in the normalisation, their roundings do not;
      -> weight error dd_j.  l: per tile (p0 + p1) and a 5-level butterfly, then one fmaf with l * alpha: (T + 6) 2^-24
      relative for T tiles; P V: N sequential fmaf (N 2^-24 of P @ |V|); acc * (1 / l): 2 roundings.
      |O - O64| <= (P dd) @ |V| + |O| (sum P dd + (T + 8) 2^-24) + N 2^-24 P @ |V|."""
    q, k, v = split(qkv.double(), B, N, H, d)
    scale = d ** -0.5
    s = q @ k.transpose(-1, -2) * scale
    p = torch.softmax(s, -1)
    o64 = p @ v
    T = -(-N // KT)
    # running max after each tile, and the rescale allowance R_t summed over the tiles after t
    tmax = torch.stack([s[..., t * KT:(t + 1) * KT].amax(-1) for t in range(T)], -1)        # [B, H, N, T]
    run = torch.cummax(tmax, -1).values
    step = torch.zeros_like(run)
    step[..., 1:] = U24 * (run[..., 1:] - run[..., :-1]) + 2.0 ** -22 + U24
    later = step.flip(-1).cumsum(-1).flip(-1) - step                                       # sum over t' > t
    tile_of = torch.arange(N, device=s.device) // KT
    m_t = run[..., tile_of]                                                                 # [B, H, N, N]
    R = later[..., tile_of]
    dd = (d * U24 * scale * (q.abs() @ k.abs().transpose(-1, -2)) + 2.0 ** -23 * s.abs() + U24 * (s - m_t).abs()
          + 2.0 ** -22 + R)
    pd = p * dd
    va = v.abs()
    bound = pd @ va + o64.abs() * (pd.sum(-1, keepdim=True) + (T + 8) * U24) + N * U24 * (p @ va)
    return flat(o64), flat(bound)


def worst_ratio(out, o64, bound):
    """max |out - O64| / bound over the elements (<= 1 is inside the bound)"""
    return ((out.double().cpu() - o64.cpu()).abs() / bound.cpu()).max().item()


def random_qkv(B, N, H, d, seed, logit_sd=8.0, device="cpu"):
    """logits q.k / sqrt(d) of standard deviation ~logit_sd, as in the small_attention test"""
    g = torch.Generator(device=device).manual_seed(seed)
    qkv = torch.randn(B * N, 3 * H * d, device=device, generator=g)
    qkv[:, :2 * H * d] *= math.sqrt(logit_sd)
    return qkv


def logits_qkv(B, N, H, d, logits, seed, device="cpu"):
    """qkv whose logits are `logits` [N] (the same for every query row, scene and head) plus a small random part:
    column 0 of q is sqrt(d) and column 0 of k_j is logits[j], the other columns are random at 1 / 8 of the scale."""
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, N, H, d, generator=g) * 0.125
    k = torch.randn(B, N, H, d, generator=g) * 0.125
    v = torch.randn(B, N, H, d, generator=g)
    q[..., 0] = math.sqrt(d)
    k[..., 0] = logits.float().view(1, N, 1)
    return torch.stack([q, k, v], 2).reshape(B * N, 3 * H * d).to(device)


def adversarial_logits(kind, N, seed=0):
    """[N] logits that stress the online softmax:
      increasing: every tile raises the max (and rescales);  last_tile: the largest logit is the last key (in the
      ragged last tile);  dominant: one key 30 above the rest (softmax close to one-hot);  plus80 / minus80: around +-80
      (expf of an unshifted logit overflows)."""
    g = torch.Generator().manual_seed(seed)
    noise = torch.randn(N, generator=g, dtype=torch.float64)
    if kind == "increasing":
        return torch.linspace(-40.0, 40.0, N, dtype=torch.float64) + 0.5 * noise
    if kind == "last_tile":
        x = 4.0 * noise
        x[-1] = x.max() + 12.0
        return x
    if kind == "dominant":
        x = 2.0 * noise
        x[N // 3] = x.max() + 30.0
        return x
    if kind == "plus80":
        return 80.0 + 8.0 * noise
    if kind == "minus80":
        return -80.0 + 8.0 * noise
    raise ValueError(kind)


ADVERSARIAL = ["increasing", "last_tile", "dominant", "plus80", "minus80"]
