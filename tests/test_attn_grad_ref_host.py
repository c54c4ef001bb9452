"""Pins the float64 attention-gradient reference (tests/attn_grad_ref.py) on the CPU, before any GPU test relies on it:
full mode equals fp32 autograd of the oracle attention, and sampled rows equal the matching slices of full mode."""
import math

import pytest
import torch

from oracle import ops as O
from tests.attn_grad_ref import attention_grads
from tests.util import seeded

# (sq, sk, hq, hkv, d, causal, q_pos, kv_pos0, scale); q_pos "zz" = zig-zag chunks (1, 2) of 4 chunks of 24 keys
CASES = [
    (37, 37, 2, 2, 16, True, None, 0, None),
    (37, 37, 2, 2, 16, False, None, 0, None),
    (40, 40, 10, 2, 16, True, None, 0, None),        # GQA 5:1
    (33, 33, 8, 1, 32, False, None, 0, None),        # GQA 8:1
    (20, 70, 5, 1, 16, True, None, 0, None),         # sk > sq, bottom-right aligned
    (50, 20, 2, 1, 16, True, None, 0, None),         # sq > sk: the first 30 rows see no key
    (48, 96, 5, 1, 16, True, "zz", 0, None),         # a context-parallel rank's two query segments
    (40, 40, 2, 2, 16, True, None, 13, None),        # kv_pos0 > 0: early rows see nothing, late keys are unseen
    (30, 45, 4, 2, 16, False, None, 0, 0.3),         # explicit scale
    (30, 30, 8, 8, 16, True, None, 0, 0.05),
]


def _inputs(sq, sk, hq, hkv, d, seed, b=2):
    g = seeded(seed)
    q = torch.randn((b, sq, hq, d), generator=g).to(torch.bfloat16)
    k = torch.randn((b, sk, hkv, d), generator=g).to(torch.bfloat16)
    v = torch.randn((b, sk, hkv, d), generator=g).to(torch.bfloat16)
    do = torch.randn((b, sq, hq, d), generator=g).to(torch.bfloat16)
    return q, k, v, do


def _positions(sq, sk, q_pos, kv_pos0):
    if q_pos == "zz":
        c = sq // 2
        qp = torch.cat([torch.arange(c, 2 * c), torch.arange(2 * c, 3 * c) + c])
    else:
        qp = torch.arange(sq) + (sk - sq)
    return qp, torch.arange(sk) + kv_pos0


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300))


@pytest.mark.parametrize("sq,sk,hq,hkv,d,causal,q_pos,kv_pos0,scale", CASES)
def test_full_mode_equals_fp32_autograd_of_the_oracle(sq, sk, hq, hkv, d, causal, q_pos, kv_pos0, scale):
    q, k, v, do = _inputs(sq, sk, hq, hkv, d, seed=sq * 7 + sk)
    qp, kp = _positions(sq, sk, q_pos, kv_pos0)
    ref = O.attention_grads(q, k, v, do, causal=causal, scale=scale, q_pos=qp, kv_pos=kp)
    got = attention_grads(q, k, v, do, causal=causal, scale=scale, q_pos=qp, kv_pos=kp)
    for name, a, r in zip(("dq", "dk", "dv"), got, ref):
        assert a.dtype == torch.float64 and torch.isfinite(a).all(), name
        r = torch.nan_to_num(r)
        assert _rel(a, r) < 1e-5, (name, _rel(a, r))
    if causal:
        blind = qp < kp[0]                                   # query rows that see no key
        assert not got[0][:, blind].any()
        unseen = kp > qp.max()                               # key rows no query sees
        assert not got[1][:, unseen].any() and not got[2][:, unseen].any()


def test_rows_that_see_no_key_get_zero_and_no_nan():
    q, k, v, do = _inputs(50, 20, 2, 1, 16, seed=3)
    dq, dk, dv = attention_grads(q, k, v, do, causal=True)
    assert torch.isfinite(dq).all() and torch.isfinite(dk).all() and torch.isfinite(dv).all()
    # row 30 sees one key, so P = 1 and dS = dP - delta = 0 there as well; rows 31.. see two or more
    assert not dq[:, :31].any() and dq[:, 31:].abs().amax(dim=(0, 2, 3)).min() > 0


@pytest.mark.parametrize("sq,sk,hq,hkv,d,causal,q_pos,kv_pos0,scale", [CASES[2], CASES[4], CASES[6], CASES[7], CASES[8]])
def test_sampled_rows_equal_the_slices_of_full_mode(sq, sk, hq, hkv, d, causal, q_pos, kv_pos0, scale):
    q, k, v, do = _inputs(sq, sk, hq, hkv, d, seed=sq + sk)
    qp, kp = _positions(sq, sk, q_pos, kv_pos0)
    kw = dict(causal=causal, scale=scale, q_pos=qp, kv_pos=kp)
    fq, fk, fv = attention_grads(q, k, v, do, **kw)
    rows = torch.tensor(sorted({0, 1, sq // 2, sq - 2, sq - 1}))
    keys = torch.tensor(sorted({0, sk // 3, sk - 3, sk - 1}))
    sq_, sk_, sv_ = attention_grads(q, k, v, do, q_rows=rows, kv_rows=keys, **kw)
    assert torch.allclose(sq_, fq[:, rows], rtol=1e-12, atol=1e-14)
    assert torch.allclose(sk_, fk[:, keys], rtol=1e-12, atol=1e-14)
    assert torch.allclose(sv_, fv[:, keys], rtol=1e-12, atol=1e-14)
    # dQ only / dK, dV only
    oq, ok, ov = attention_grads(q, k, v, do, q_rows=rows, kv_rows=torch.tensor([], dtype=torch.int64), **kw)
    assert torch.allclose(oq, sq_, rtol=1e-12, atol=1e-14) and ok.shape[1] == 0 and ov.shape[1] == 0
    nq, nk, nv = attention_grads(q, k, v, do, q_rows=torch.tensor([], dtype=torch.int64), kv_rows=keys, **kw)
    assert nq.shape[1] == 0 and torch.allclose(nk, sk_, rtol=1e-12, atol=1e-14) and torch.allclose(nv, sv_, rtol=1e-12, atol=1e-14)


def test_chunking_does_not_change_the_result():
    """A score block of a few hundred bytes forces one query row per block; the arithmetic per row is the same."""
    q, k, v, do = _inputs(48, 96, 5, 1, 16, seed=11)
    qp, kp = _positions(48, 96, "zz", 0)
    big = attention_grads(q, k, v, do, causal=True, q_pos=qp, kv_pos=kp)
    small = attention_grads(q, k, v, do, causal=True, q_pos=qp, kv_pos=kp, block_bytes=256)
    for a, b in zip(big, small):
        assert torch.allclose(a, b, rtol=1e-12, atol=1e-14)


def test_default_scale_is_one_over_sqrt_d():
    q, k, v, do = _inputs(20, 20, 2, 2, 16, seed=5, b=1)
    a = attention_grads(q, k, v, do, causal=True)
    b = attention_grads(q, k, v, do, causal=True, scale=1 / math.sqrt(16))
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_delta_from_a_given_forward_output():
    """`out` = the exact O reproduces full mode; a bf16-rounded O changes delta, hence dQ / dK, but never dV."""
    q, k, v, do = _inputs(40, 40, 10, 2, 16, seed=13)
    exact = attention_grads(q, k, v, do, causal=True)
    o, _ = O.attention(q, k, v, causal=True)
    same = attention_grads(q, k, v, do, causal=True, out=o)
    for a, b in zip(exact, same):
        assert _rel(a, b) < 1e-6
    rounded = attention_grads(q, k, v, do, causal=True, out=o.to(torch.bfloat16))
    assert _rel(rounded[0], exact[0]) > 1e-4 and _rel(rounded[1], exact[1]) > 1e-4
    assert torch.equal(rounded[2], exact[2])
