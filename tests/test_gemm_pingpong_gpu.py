"""GEMM schedules that stress the ping-pong consumers of gemm_wgmma_kernel (GPU): the two consumer warpgroups take
alternate work segments of a CTA and follow each other around the shared stage ring, so segments shorter than the ring
(1 or 2 k-blocks against 3 or 6 stages) and CTAs with odd and even segment counts must still give exact tiles."""
import ctypes
import math

import pytest
import torch

from iggt_official_b200 import _lib
from launch_refs import ACC, FRAC, gemm64
from ulp_bounds import around, check16, check32

pytestmark = pytest.mark.gpu

STORE16, RESID32 = 0, 1


def plan(epi, M, N, K):
    out = (ctypes.c_int * 7)()
    assert _lib.load().iggt_gemm_plan(epi, M, N, K, ctypes.cast(out, ctypes.c_void_p)) == 0
    return dict(zip(["bn", "pair", "stream_k", "m_tiles", "n_tiles", "k_blocks", "grid"], list(out)))


@pytest.fixture(scope="module")
def ops():
    from iggt_official_b200 import ops as _ops
    return _ops


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_resid32_stream_k_segments_shorter_than_the_ring(ops, dtype):
    # 34 x 8 tiles of 2 k-blocks cut into ranges of 5 k-blocks: segments of 1 and 2 k-blocks, 3 or 4 per CTA
    M, N, K = 34 * 128, 1024, 128
    p = plan(RESID32, M, N, K)
    assert p["stream_k"] == 1 and p["k_blocks"] == 2
    g = torch.Generator(device="cuda").manual_seed(11)
    a = torch.randn(M, K, device="cuda", generator=g).to(dtype)
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).to(dtype)
    bias = torch.randn(N, device="cuda", generator=g)
    gamma = torch.rand(N, device="cuda", generator=g) + 0.5
    x = torch.randn(M, N, device="cuda", generator=g)
    x0 = x.double()
    ops.gemm_resid32(a, w, x, bias, gamma)
    torch.cuda.synchronize()
    # stream-K: x + gamma * (acc + b) per element, within ACC of x's and the product's magnitude sum
    acc, mag = gemm64(a, w)
    b64, g64 = bias.double(), gamma.double()
    check32(x, x0 + g64 * (acc + b64), x0.abs() + g64 * (mag + b64.abs()), ACC, what="resid32 stream-K short segments")


@pytest.mark.parametrize("M,N", [(50 * 128, 768), (300 * 128 - 5, 64)])   # BN = 128 (3 stages) / BN = 64 (6 stages)
def test_store16_one_k_block_tiles(ops, M, N):
    # K = 64: every tile is one k-block; 300 tiles on a 132-CTA grid give CTAs 2 or 3 tiles
    K = 64
    p = plan(STORE16, M, N, K)
    assert p["k_blocks"] == 1 and p["stream_k"] == 0
    g = torch.Generator(device="cuda").manual_seed(M + N)
    a = torch.randn(M, K, device="cuda", generator=g).half()
    w = (torch.randn(N, K, device="cuda", generator=g) / math.sqrt(K)).half()
    bias = torch.randn(N, device="cuda", generator=g)
    out = ops.gemm_store16(a, w, bias, act=0)
    torch.cuda.synchronize()
    # RN16 of the ACC interval per element, 1 ulp, the store16 share off RN16 (test_epilogues_gpu.py)
    acc, mag = gemm64(a, w)
    y = acc + bias.double()
    lo, hi = around(y, ACC * (mag + bias.double().abs()))
    check16(out, y, torch.float16, 1, FRAC[torch.float16], lo, hi, what="store16 one-k-block tiles")
