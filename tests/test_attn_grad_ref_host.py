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


# ------------------------------------------------------------------------------------------------ documents, terms
from tests.attn_fwd_ref import doc_lo  # noqa: E402
from tests.attn_grad_ref import (check_attn_bwd, check_planted_pairs, edge_targets, plant_edge_pairs,  # noqa: E402
                                 plant_pairs)

LOG2E = 1.4426950408889634


def _cu(sq, seed, lengths=()):
    """Boundaries of a packed row: the given document lengths first, then random ones up to sq."""
    g = seeded(seed)
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    while cu[-1] < sq:
        cu.append(min(sq, cu[-1] + int(torch.randint(1, 40, (1,), generator=g))))
    return torch.tensor(cu)


def _hidden(sq, sk, causal, q_pos, kv_pos, kv_lo=None):
    """[sq, sk] True = key hidden from the row."""
    h = kv_pos[None, :] > q_pos[:, None] if causal else torch.zeros((sq, sk), dtype=torch.bool)
    if kv_lo is not None:
        h = h | (torch.arange(sk)[None, :] < torch.as_tensor(kv_lo)[:, None])
    return h


def _bhsd(t, G=1):
    return t.double().repeat_interleave(G, 2).permute(0, 2, 1, 3)


def _direct(q, k, v, do, hidden, scale=None, out=None):
    """Every output of attention_grads(terms=True) by its dense float64 formula, under an arbitrary mask [sq, sk]."""
    b, sq, hq, d = q.shape
    hkv = k.shape[2]
    G = hq // hkv
    scale = 1 / math.sqrt(d) if scale is None else scale
    qf, kf, vf, dof = _bhsd(q), _bhsd(k, G), _bhsd(v, G), _bhsd(do)
    s = (qf @ kf.transpose(-1, -2) * scale).masked_fill(hidden, float("-inf"))
    lse = torch.logsumexp(s, -1, keepdim=True)
    p = torch.nan_to_num(torch.exp(s - lse), nan=0.0)
    o = p @ vf if out is None else _bhsd(out)
    delta = (dof * o).sum(-1, keepdim=True)
    dp = dof @ vf.transpose(-1, -2)
    ds = p * (dp - delta)
    e = p * (dof.abs() @ vf.abs().transpose(-1, -2) + (dof * o).abs().sum(-1, keepdim=True))

    def qside(x):                                       # [b, hq, sq, d] -> [b, sq, hq, d]
        return x.permute(0, 2, 1, 3)

    def kside(x):                                       # [b, hq, sk, d], summed over each group -> [b, sk, hkv, d]
        return x.view(b, hkv, G, *x.shape[2:]).sum(2).permute(0, 2, 1, 3)

    pt, at = p.transpose(-1, -2), (p * (dp - delta).abs()).transpose(-1, -2)
    return {
        "dq": qside(scale * ds @ kf), "dk": kside(scale * ds.transpose(-1, -2) @ qf), "dv": kside(pt @ dof),
        "A_q": qside(scale * (p * (dp - delta).abs()) @ kf.abs()), "E_q": qside(scale * e @ kf.abs()),
        "sig_q": qside(scale * (ds.square() @ kf.square()).sqrt()),
        "A_k": kside(scale * at @ qf.abs()), "E_k": kside(scale * e.transpose(-1, -2) @ qf.abs()),
        "sig_k": scale * kside(ds.square().transpose(-1, -2) @ qf.square()).sqrt(),
        "A_v": kside(pt @ dof.abs()), "sig_v": kside(p.square().transpose(-1, -2) @ dof.square()).sqrt(),
        "n_q": (~hidden).sum(-1), "n_k": (~hidden).sum(0), "lse": lse[..., 0],
    }


def test_kv_lo_equals_one_call_per_document_and_the_fp32_oracle():
    sq = 300
    cu = _cu(sq, 3, lengths=(1, 63, 64, 65))
    q, k, v, do = _inputs(sq, sq, 10, 2, 16, seed=7, b=1)
    got = attention_grads(q, k, v, do, causal=True, kv_lo=doc_lo(cu, sq))
    for a, e in zip(cu[:-1].tolist(), cu[1:].tolist()):
        sl = slice(a, e)
        one = attention_grads(q[:, sl], k[:, sl], v[:, sl], do[:, sl], causal=True)
        fp32 = O.attention_grads(q[:, sl], k[:, sl], v[:, sl], do[:, sl], causal=True)
        for name, x, y, z in zip(("dq", "dk", "dv"), got, one, fp32):
            assert torch.allclose(x[:, sl], y, rtol=1e-12, atol=1e-14), (name, a, e)
            if e - a > 1:
                assert _rel(x[:, sl], z) < 1e-5, (name, a, e, _rel(x[:, sl], z))


TERM_CASES = [   # (sq, sk, hq, hkv, causal, q_pos, kv_pos0, docs)
    (40, 40, 10, 2, True, None, 0, False),
    (48, 96, 4, 2, True, "zz", 0, False),
    (40, 40, 2, 2, True, None, 13, False),
    (30, 45, 4, 2, False, None, 0, False),
    (90, 90, 4, 1, True, None, 0, True),
]


@pytest.mark.parametrize("sq,sk,hq,hkv,causal,q_pos,kv_pos0,docs", TERM_CASES)
def test_terms_equal_their_direct_formulas(sq, sk, hq, hkv, causal, q_pos, kv_pos0, docs):
    q, k, v, do = _inputs(sq, sk, hq, hkv, 16, seed=sq + hq)
    qp, kp = _positions(sq, sk, q_pos, kv_pos0)
    lo = doc_lo(_cu(sq, 5, lengths=(1, 7, 8, 9)), sq) if docs else None
    out = O.attention(q, k, v, causal=causal, q_pos=qp, kv_pos=kp)[0].to(torch.bfloat16)
    kw = dict(causal=causal, q_pos=qp, kv_pos=kp, kv_lo=lo, out=out)
    ref = attention_grads(q, k, v, do, terms=True, **kw)
    direct = _direct(q, k, v, do, _hidden(sq, sk, causal, qp, kp, lo), out=out)
    for name, x in direct.items():
        y = ref[name]
        if x.dtype == torch.int64:
            assert torch.equal(y, x), name
        elif name == "lse":
            assert torch.equal(torch.isinf(y), torch.isinf(x)) and torch.allclose(y[torch.isfinite(y)], x[torch.isfinite(x)])
        else:
            assert torch.allclose(y, x, rtol=1e-10, atol=1e-12), (name, float((y - x).abs().max()))
    assert ref["n_max"] == int(direct["n_q"].max()) and ref["lse_max"] == pytest.approx(
        float(direct["lse"][torch.isfinite(direct["lse"])].abs().max()))
    # sampled rows and keys, one row per score block: the slices of full mode
    rows = torch.tensor(sorted({0, 1, sq // 2, sq - 2, sq - 1}))
    keys = torch.tensor(sorted({0, sk // 3, sk // 2, sk - 3, sk - 1}))
    part = attention_grads(q, k, v, do, terms=True, q_rows=rows, kv_rows=keys, block_bytes=256, **kw)
    for name in ("dq", "A_q", "E_q", "sig_q", "n_q"):
        assert torch.allclose(part[name].double(), ref[name][:, rows].double() if name != "n_q" else ref[name][rows].double(),
                              rtol=1e-12, atol=1e-14), name
    for name in ("dk", "dv", "A_k", "E_k", "sig_k", "A_v", "sig_v", "n_k"):
        full = ref[name][keys] if name == "n_k" else ref[name][:, keys]
        assert torch.allclose(part[name].double(), full.double(), rtol=1e-12, atol=1e-14), name


# ------------------------------------------------------------------------------------------------ a correct backward
def _forward(q, k, v, hidden, scale=None):
    """A correct forward's results: the exact output rounded to bf16, the exact lse rounded to fp32."""
    b, sq, hq, d = q.shape
    G = hq // k.shape[2]
    scale = 1 / math.sqrt(d) if scale is None else scale
    s = (_bhsd(q) @ _bhsd(k, G).transpose(-1, -2) * scale).masked_fill(hidden, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.nan_to_num(torch.exp(s - lse[..., None]), nan=0.0)
    return (p @ _bhsd(v, G)).permute(0, 2, 1, 3).to(torch.bfloat16), lse.float()


def _emulate(q, k, v, do, out, lse, hid_a, hid_b, scale=None):
    """fp32 flash backward as a correct tensor-core kernel computes it, with the mask of pass A (dK / dV) and of pass B
    (dQ) given separately ([sq, sk] or [hq, sq, sk], True = hidden): P from the forward's lse, delta from its bf16
    output, bf16 P and dS, fp32 accumulation per 64-key tile (dQ) and per 64-row query tile of each head (dK, dV)."""
    b, sq, hq, d = q.shape
    sk, hkv = k.shape[1], k.shape[2]
    G = hq // hkv
    scale = 1 / math.sqrt(d) if scale is None else scale
    qf, dof = q.float().permute(0, 2, 1, 3), do.float().permute(0, 2, 1, 3)
    kf, vf = (t.float().repeat_interleave(G, 2).permute(0, 2, 1, 3) for t in (k, v))
    x = qf @ kf.transpose(-1, -2)
    dp = dof @ vf.transpose(-1, -2)
    delta = (dof * out.float().permute(0, 2, 1, 3)).sum(-1, keepdim=True)
    p = torch.exp2(x * torch.tensor(scale * LOG2E, dtype=torch.float32) - (lse * LOG2E)[..., None])
    ds = p * (dp - delta) * scale
    zero = torch.zeros((), dtype=torch.float32)
    dsb = torch.where(hid_b, zero, ds).to(torch.bfloat16).float()
    pa = torch.where(hid_a, zero, p).to(torch.bfloat16).float()
    dsa = torch.where(hid_a, zero, ds).to(torch.bfloat16).float()
    dq = torch.zeros_like(qf)
    for j0 in range(0, sk, 64):
        dq += dsb[..., j0 : j0 + 64] @ kf[:, :, j0 : j0 + 64]
    dk = torch.zeros((b, hkv, sk, d))
    dv = torch.zeros((b, hkv, sk, d))
    for h in range(hkv):
        for hh in range(h * G, (h + 1) * G):
            for i0 in range(0, sq, 64):
                rs = slice(i0, i0 + 64)
                dv[:, h] += pa[:, hh, rs].transpose(-1, -2) @ dof[:, hh, rs]
                dk[:, h] += dsa[:, hh, rs].transpose(-1, -2) @ qf[:, hh, rs]
    return tuple(t.permute(0, 2, 1, 3).to(torch.bfloat16) for t in (dq, dk, dv))


def _zz_pos(sq):
    c = sq // 2
    return torch.cat([torch.arange(c, 2 * c), torch.arange(3 * c, 4 * c)])


TWINS = {   # every path's small-size twin: (b, sq, sk, hq, hkv, d, causal, q_pos, kv_pos0, docs, scale)
    "decoder ragged": (1, 300, 300, 10, 2, 128, True, None, 0, None, None),
    "decoder GQA 8": (2, 193, 193, 16, 2, 64, True, None, 0, None, None),
    "zig-zag rank": (1, 256, 512, 10, 2, 128, True, "zz", 0, None, None),
    "documents": (1, 700, 700, 10, 2, 128, True, None, 0, (300, 1, 63, 64, 65, 127, 128, 129), None),
    "kv_pos0": (1, 256, 256, 4, 2, 128, True, None, 37, None, None),
    "sq > sk": (2, 300, 100, 10, 2, 128, True, None, 0, None, None),
    "sk > sq": (1, 100, 612, 10, 2, 128, True, None, 0, None, None),
    "vit": (2, 257, 257, 16, 16, 64, False, None, 0, None, None),
    "scale": (1, 333, 333, 10, 2, 64, True, None, 0, None, 0.05),
}


def _twin(name, seed=0):
    b, sq, sk, hq, hkv, d, causal, q_pos, kv_pos0, docs, scale = TWINS[name]
    q, k, v, do = _inputs(sq, sk, hq, hkv, d, seed=seed + sq + hq, b=b)
    qp = _zz_pos(sq) if q_pos == "zz" else torch.arange(sq) + (sk - sq)
    kp = torch.arange(sk) + kv_pos0
    lo = doc_lo(_cu(sq, 1, lengths=docs), sq) if docs else None
    planted = None
    if causal:
        rows = torch.arange(sq)
        targets = edge_targets(rows, qp, kv_pos0)
        if docs:   # even rows of a document: the previous document's last key; odd rows: the document's first key
            targets = torch.where(rows % 2 == 0, lo - 1, lo)
        planted = plant_edge_pairs(q, k, rows, targets, q_pos=qp, kv_pos=kp, kv_lo=lo, scale=scale)
    hid = _hidden(sq, sk, causal, qp, kp, lo)
    kw = dict(causal=causal, q_pos=qp, kv_pos=kp, kv_lo=lo, scale=scale)
    return q, k, v, do, hid, kw, planted


@pytest.mark.parametrize("name", list(TWINS))
def test_a_correct_flash_backward_passes_at_the_gpu_limits(name):
    q, k, v, do, hid, kw, planted = _twin(name)
    out, lse = _forward(q, k, v, hid, kw["scale"])
    ref = attention_grads(q, k, v, do, out=out, terms=True, **kw)
    if planted is not None:
        check_planted_pairs(q, k, ref, planted, scale=kw["scale"], label=name)
    st = check_attn_bwd(_emulate(q, k, v, do, out, lse, hid, hid, kw["scale"]), ref, label=name)
    assert st["z_row_dq"] > 0.3 and st["z_row_dk"] > 0.3        # the emulation does round


# ------------------------------------------------------------------------------------------------ defects
S, HQ, HKV, D = 2048, 2, 1, 128
TILE = torch.arange(1024, 1152)          # the planted query tile: crosses the diagonal at 64- and 128-row boundaries


@pytest.fixture(scope="module")
def dense():
    q, k, v, do = _inputs(S, S, HQ, HKV, D, seed=23, b=1)
    pos = torch.arange(S)
    planted = plant_edge_pairs(q, k, TILE, edge_targets(TILE, pos), q_pos=pos, kv_pos=pos)
    hid = _hidden(S, S, True, pos, pos)
    out, lse = _forward(q, k, v, hid)
    ref = attention_grads(q, k, v, do, causal=True, out=out, terms=True)
    check_planted_pairs(q, k, ref, planted)
    got = _emulate(q, k, v, do, out, lse, hid, hid)
    check_attn_bwd(got, ref, label="dense")
    return q, k, v, do, out, lse, hid, ref, got


def _rejects(got, ref, what):
    with pytest.raises(AssertionError) as e:
        check_attn_bwd(got, ref, label=what)
    return str(e.value)


def _mutate(hid, rows, keys, value):
    bad = hid.clone()
    bad[..., rows, keys] = value
    return bad


LEAK = (torch.arange(1024, 1088), torch.arange(1025, 1089))    # rows 1024 .. 1087 also see key i + 1
DIAG = (torch.arange(1024, 1088), torch.arange(1024, 1088))    # ... or lose their diagonal key


@pytest.mark.parametrize("defect", ["leak", "diagonal"])
def test_rejects_pass_a_with_one_key_wrong_for_one_tile(dense, defect):
    q, k, v, do, out, lse, hid, ref, _ = dense
    rows, keys = LEAK if defect == "leak" else DIAG
    bad = _mutate(hid, rows, keys, defect != "leak")
    msg = _rejects(_emulate(q, k, v, do, out, lse, bad, hid), ref, "pass A " + defect)
    assert "'dk'" in msg or "'dv'" in msg


@pytest.mark.parametrize("defect", ["leak", "diagonal"])
def test_rejects_pass_b_with_one_key_wrong_for_one_tile(dense, defect):
    """Caught through the paired plants: with the forward's saturating plants (P = 1 on the target) dQ would not
    depend on the key at all."""
    q, k, v, do, out, lse, hid, ref, _ = dense
    rows, keys = LEAK if defect == "leak" else DIAG
    bad = _mutate(hid, rows, keys, defect != "leak")
    msg = _rejects(_emulate(q, k, v, do, out, lse, hid, bad), ref, "pass B " + defect)
    assert "'dq'" in msg and "elementwise" in msg


def test_rejects_one_interior_key_tile_missing_from_one_query_tiles_dq(dense):
    q, k, v, do, out, lse, hid, ref, _ = dense
    bad = hid.expand(HQ, S, S).clone()
    bad[1, 1536:1600, 512:576] = True
    msg = _rejects(_emulate(q, k, v, do, out, lse, hid, bad), ref, "key tile")
    assert "'dq'" in msg


def test_rejects_one_query_tile_of_one_head_missing_from_dk_dv(dense):
    q, k, v, do, out, lse, hid, ref, _ = dense
    bad = hid.expand(HQ, S, S).clone()
    bad[1, 1536:1600] = True
    msg = _rejects(_emulate(q, k, v, do, out, lse, bad, hid), ref, "head tile")
    assert "'dk'" in msg or "'dv'" in msg


def test_rejects_two_heads_dq_swapped(dense):
    _, _, _, _, _, _, _, ref, (dq, dk, dv) = dense
    bad = dq.clone()
    bad[:, :, 0], bad[:, :, 1] = dq[:, :, 1], dq[:, :, 0]
    _rejects((bad, dk, dv), ref, "heads swapped")


def test_rejects_inexact_edges(dense):
    """A blind row's dQ and an unseen key's dK / dV must be exactly 0; nothing may be NaN."""
    q, k, v, do = _inputs(50, 20, 2, 1, 16, seed=29, b=1)
    hid = _hidden(50, 20, True, torch.arange(50) - 30, torch.arange(20))
    out, lse = _forward(q, k, v, hid)
    ref = attention_grads(q, k, v, do, causal=True, out=out, terms=True)
    dq, dk, dv = _emulate(q, k, v, do, out, lse, hid, hid)
    check_attn_bwd((dq, dk, dv), ref)
    bad = dq.clone()
    bad[0, 3, 0, 0] = 1e-30
    assert "exactly 0" in _rejects((bad, dk, dv), ref, "blind row")
    _, _, _, _, _, _, _, ref2, (dq2, dk2, dv2) = dense
    bad = dv2.clone()
    bad[0, 2047, 0, 5] = float("nan")
    assert "non-finite" in _rejects((dq2, dk2, bad), ref2, "nan")


@pytest.mark.parametrize("which", ["A", "B"])
def test_rejects_a_document_boundary_off_by_one_in_one_pass(which):
    """~100 documents in 2048 rows; in one pass only, every row of one document also sees the previous document's
    last key.  The document's rows are planted at its start."""
    sq = 2048
    cu = _cu(sq, 31)
    q, k, v, do = _inputs(sq, sq, HQ, HKV, D, seed=31, b=1)
    lo = doc_lo(cu, sq)
    pos = torch.arange(sq)
    i = int(torch.searchsorted(cu, 1000))
    a, e = int(cu[i]), int(cu[i + 1])
    rows = torch.arange(a, e)
    planted = plant_edge_pairs(q, k, rows, torch.where(rows % 2 == 0, a - 1, a), q_pos=pos, kv_pos=pos, kv_lo=lo)
    hid = _hidden(sq, sq, True, pos, pos, lo)
    out, lse = _forward(q, k, v, hid)
    ref = attention_grads(q, k, v, do, causal=True, kv_lo=lo, out=out, terms=True)
    check_planted_pairs(q, k, ref, planted)
    check_attn_bwd(_emulate(q, k, v, do, out, lse, hid, hid), ref)
    bad_lo = lo.clone()
    bad_lo[a:e] -= 1
    bad = _hidden(sq, sq, True, pos, pos, bad_lo)
    got = _emulate(q, k, v, do, out, lse, bad, hid) if which == "A" else _emulate(q, k, v, do, out, lse, hid, bad)
    msg = _rejects(got, ref, "document boundary " + which)
    assert ("'dq'" in msg) == (which == "B")


def test_rejects_the_second_segment_position_off_by_64():
    """A zig-zag rank (segments of 256 rows at chunks 1 and 2 of 4): both passes place segment 1 64 rows late."""
    sq, sk = 512, 1024
    q, k, v, do = _inputs(sq, sk, HQ, HKV, D, seed=37, b=1)
    pos, kp = _zz_pos(sq), torch.arange(sk)
    rows = torch.cat([torch.arange(256, 384), torch.arange(384, 512)])
    planted = plant_edge_pairs(q, k, rows, edge_targets(rows, pos), q_pos=pos, kv_pos=kp)
    hid = _hidden(sq, sk, True, pos, kp)
    out, lse = _forward(q, k, v, hid)
    ref = attention_grads(q, k, v, do, causal=True, q_pos=pos, out=out, terms=True)
    check_planted_pairs(q, k, ref, planted)
    check_attn_bwd(_emulate(q, k, v, do, out, lse, hid, hid), ref)
    bad_pos = pos.clone()
    bad_pos[256:] += 64
    bad = _hidden(sq, sk, True, bad_pos, kp)
    _rejects(_emulate(q, k, v, do, out, lse, bad, bad), ref, "q_seg_pos[1] + 64")


def test_rejects_kv_pos0_off_by_one():
    sq = sk = 512
    kv_pos0 = 100
    q, k, v, do = _inputs(sq, sk, HQ, HKV, D, seed=41, b=1)
    pos, kp = torch.arange(sq), torch.arange(sk) + kv_pos0
    rows = torch.arange(64, 256)
    planted = plant_edge_pairs(q, k, rows, edge_targets(rows, pos, kv_pos0), q_pos=pos, kv_pos=kp)
    hid = _hidden(sq, sk, True, pos, kp)
    out, lse = _forward(q, k, v, hid)
    ref = attention_grads(q, k, v, do, causal=True, kv_pos=kp, out=out, terms=True)
    check_planted_pairs(q, k, ref, planted)
    check_attn_bwd(_emulate(q, k, v, do, out, lse, hid, hid), ref)
    for off in (1, -1):
        bad = _hidden(sq, sk, True, pos, kp + off)
        _rejects(_emulate(q, k, v, do, out, lse, bad, bad), ref, f"kv_pos0 {off:+d}")


def test_paired_plants_hold_their_weights_at_every_head_dim():
    for d, scale in ((64, None), (128, None), (128, 0.05)):
        q, k, v, do = _inputs(600, 600, 10, 2, d, seed=d, b=1)
        rows = torch.tensor([5, 127, 128, 300, 599, 64, 65])
        targets = torch.tensor([5, 127, 129, 300, 599, 65, 66])
        pos = torch.arange(600)
        planted = plant_edge_pairs(q, k, rows, targets, q_pos=pos, kv_pos=pos, scale=scale)
        assert planted["visible"][0].numel() == 4 and planted["hidden"][0].numel() == 3
        ref = attention_grads(q, k, v, do, causal=True, scale=scale, q_rows=rows.sort().values, kv_rows=torch.tensor([], dtype=torch.int64), terms=True)
        check_planted_pairs(q, k, ref, planted, scale=scale)
    with pytest.raises(AssertionError):
        plant_pairs(q, k, [3], [2], [2])
