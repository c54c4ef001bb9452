"""GPU parity of the fused attention at the lengths BASELINE.json quotes (16K, 128K) and beyond 2^31 elements.

The fp32 oracle of the whole [S, S] problem does not finish in seconds at these lengths, so parity is checked two ways:
  * SAMPLED ROWS vs the oracle: `oracle.ops.attention` on a few hundred query rows (first / last rows, both sides of
    every kind of tile boundary, random rows) against ALL keys they may see, with their true global positions -
    output (excess over the bf16 floor < 2e-3, the bound of tests/test_gpu_attention.py) and fp32 log-sum-exp (1e-4);
  * FULL TENSOR vs a live flash-attn 2.8 run (the kernel the reference calls, dot_product_attention.py:374-390) on the
    same device tensors: two independent bf16 flash attentions differ by their two P-rounding errors and two output
    roundings (measured 2.6e-3 .. 3.0e-3 relative Frobenius); an indexing / masking / scheduling mistake anywhere in
    the tensor shows up as O(1).
What these lengths exercise that S = 4096 does not: the head-major work order (`block_major = 0`, chosen when K/V of
all kv heads exceed 64 MB), thousands of key tiles per work item, the boustrophedon sweep over > 10^4 items, 64-bit
row offsets (the last test), and the zig-zag query segments of a context-parallel rank at their global positions
(training/utils.py:329-341).
"""
import math

import pytest
import torch

from oracle import ops as O
from tests.attn_grad_ref import _sample_rows
from tests.util import rel_fro

pytestmark = pytest.mark.gpu

TOL_EXCESS = 2e-3     # same bound as tests/test_gpu_attention.py
TOL_LSE = 1e-4
TOL_VS_FLASH = 4e-3   # two independent bf16 flash attentions (see module docstring)


@pytest.fixture(scope="module")
def L(lib_built):
    from long_vita_b200 import ops

    return ops


def _device_inputs(S, hq, hkv, d, seed, sq=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    sq = S if sq is None else sq
    q = torch.randn((1, sq, hq, d), generator=g, device="cuda", dtype=torch.float32).to(torch.bfloat16)
    k = torch.randn((1, S, hkv, d), generator=g, device="cuda", dtype=torch.float32).to(torch.bfloat16)
    v = torch.randn((1, S, hkv, d), generator=g, device="cuda", dtype=torch.float32).to(torch.bfloat16)
    return q, k, v


def _check_rows(out, lse, q, k, v, rows, q_pos_of_row):
    """out [1, sq, hq, d] (device), lse [1, hq, sq]; oracle on `rows` (local indices) at global positions."""
    qs = q[:, rows.cuda()].cpu()
    kc, vc = k.cpu(), v.cpu()
    ref, lse_ref = O.attention(qs, kc, vc, causal=True, q_pos=q_pos_of_row, head_chunk=5)
    got = out[:, rows.cuda()].cpu()
    e_total = rel_fro(got, ref)
    e_floor = rel_fro(ref.to(torch.bfloat16), ref)
    excess = math.sqrt(max(e_total ** 2 - e_floor ** 2, 0.0))
    e_lse = float((lse[:, :, rows.cuda()].cpu() - lse_ref).abs().max())
    # per-row check as well: one wrong row must not hide inside a Frobenius norm over hundreds of good ones
    per_row = ((got.float() - ref).norm(dim=(2, 3)) / ref.norm(dim=(2, 3))).view(-1)
    assert excess < TOL_EXCESS and e_lse < TOL_LSE and float(per_row.max()) < 6e-3, (excess, e_total, e_floor, e_lse, float(per_row.max()))
    return excess, e_lse


def _vs_flash(out, q, k, v):
    fa = pytest.importorskip("flash_attn")
    theirs = fa.flash_attn_func(q, k, v, causal=True)
    num, den = 0.0, 0.0
    for s0 in range(0, out.shape[1], 8192):        # chunked: fp32 copies of a 128K x 40 x 128 tensor are 2.7 GB each
        a, b = out[:, s0 : s0 + 8192].float(), theirs[:, s0 : s0 + 8192].float()
        num += float((a - b).pow(2).sum())
        den += float(b.pow(2).sum())
    e = math.sqrt(num / den)
    assert e < TOL_VS_FLASH, e
    return e


@pytest.mark.parametrize("S", [16384, 131072])
def test_attention_forward_at_baseline_lengths(L, S):
    """LLM geometry 40:8 x 128, causal.  16 384: globally longest-first order; 131 072: head-major order."""
    hq, hkv, d = 40, 8, 128
    q, k, v = _device_inputs(S, hq, hkv, d, seed=S)
    out, lse = L.attention_fwd(q, k, v, causal=True, return_lse=True)
    rows = _sample_rows(256, S, seed=S)
    _check_rows(out, lse, q, k, v, rows, rows)
    _vs_flash(out, q, k, v)


@pytest.mark.parametrize("S,cp,rank", [(16384, 8, 5), (131072, 8, 0), (131072, 4, 3)])
def test_zigzag_segments_at_baseline_lengths(L, S, cp, rank):
    """A context-parallel rank's two query segments (chunks r and 2cp-1-r) against the whole K/V at its global
    positions - the single-device form of what lv_attn_cp_fwd computes (q_seg_len / q_seg_pos / kv_pos arithmetic)."""
    hq, hkv, d = 40, 8, 128
    c = S // (2 * cp)
    q, k, v = _device_inputs(S, hq, hkv, d, seed=S + rank, sq=2 * c)
    pos = O.zigzag_positions(S, cp, rank)
    out, lse = L.attention_fwd(q, k, v, causal=True, return_lse=True, q_seg_len=c, q_seg_pos=(rank * c, (2 * cp - 1 - rank) * c))
    rows = _sample_rows(192, 2 * c, seed=rank, boundaries=(128, 256, c))
    _check_rows(out, lse, q, k, v, rows, pos[rows])


def test_attention_forward_beyond_2_31_elements(L):
    """S = 425 984 (3328 x 128): Q and O hold 2.18e9 elements each, so row offsets need 64 bits; 1.9 PFLOP."""
    S, hq, hkv, d = 425984, 40, 8, 128
    assert S * hq * d > 2 ** 31
    q, k, v = _device_inputs(S, hq, hkv, d, seed=7)
    out, lse = L.attention_fwd(q, k, v, causal=True, return_lse=True)
    rows = torch.tensor(sorted({0, 127, 128, 255, 256, S // 2, S - 257, S - 256, S - 129, S - 128, S - 2, S - 1}
                               | {int(x) for x in torch.randint(S // 2, S, (36,), generator=torch.Generator().manual_seed(7))}))
    _check_rows(out, lse, q, k, v, rows, rows)
