"""Pins the float64 attention-forward reference and its checker (tests/attn_fwd_ref.py) on the CPU, before any GPU test
relies on them: the reference equals the fp32 oracle and a direct float64 softmax, sampled rows equal slices of full
mode, `kv_lo` equals one call per document; an fp32 emulation of a correct flash forward passes the checker at the GPU
limits, and corruptions of correct results of the kind a mask or indexing bug produces each fail it."""
import math

import pytest
import torch

from oracle import ops as O
from tests.attn_fwd_ref import attention_fwd_ref, check_attn_fwd, check_planted, doc_lo, plant_keys
from tests.util import seeded

LN2 = math.log(2.0)


def _inputs(b, sq, sk, hq, hkv, d, seed):
    g = seeded(seed)
    q = torch.randn((b, sq, hq, d), generator=g).to(torch.bfloat16)
    k = torch.randn((b, sk, hkv, d), generator=g).to(torch.bfloat16)
    v = torch.randn((b, sk, hkv, d), generator=g).to(torch.bfloat16)
    return q, k, v


def _hidden(sq, sk, causal, q_pos=None, kv_pos=None, kv_lo=None):
    """[sq, sk] True = key hidden from the row."""
    qp = torch.arange(sq) + (sk - sq) if q_pos is None else torch.as_tensor(q_pos)
    kp = torch.arange(sk) if kv_pos is None else torch.as_tensor(kv_pos)
    h = kp[None, :] > qp[:, None] if causal else torch.zeros((sq, sk), dtype=torch.bool)
    if kv_lo is not None:
        h = h | (torch.arange(sk)[None, :] < torch.as_tensor(kv_lo)[:, None])
    return h


def _direct(q, k, v, hidden, scale=None):
    """Textbook float64 softmax attention under an arbitrary mask `hidden` [sq, sk] or [hq, sq, sk]."""
    G = q.shape[2] // k.shape[2]
    scale = 1.0 / math.sqrt(q.shape[-1]) if scale is None else scale
    kf, vf = k.double().repeat_interleave(G, 2), v.double().repeat_interleave(G, 2)
    s = torch.einsum("bqhd,bkhd->bhqk", q.double(), kf) * scale
    s = s.masked_fill(hidden, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.nan_to_num(torch.exp(s - lse[..., None]), nan=0.0)
    return torch.einsum("bhqk,bkhd->bqhd", p, vf), lse


def _emulate(q, k, v, hidden, scale=None, tile=128):
    """fp32 flash forward as a correct tensor-core kernel computes it: 128-key tiles, running max in the log2 domain,
    P rounded to bf16 for P V, l summed from the unrounded P, out rounded once to bf16."""
    G = q.shape[2] // k.shape[2]
    scale = 1.0 / math.sqrt(q.shape[-1]) if scale is None else scale
    sl2 = torch.tensor(scale * 1.4426950408889634, dtype=torch.float32)
    qf = q.float().permute(0, 2, 1, 3)
    kf = k.float().repeat_interleave(G, 2).permute(0, 2, 1, 3)
    vf = v.float().repeat_interleave(G, 2).permute(0, 2, 1, 3)
    b, hq, sq, d = qf.shape
    m = torch.full((b, hq, sq, 1), float("-inf"))
    l = torch.zeros((b, hq, sq, 1))
    o = torch.zeros((b, hq, sq, d))
    for j0 in range(0, kf.shape[2], tile):
        s = torch.matmul(qf, kf[:, :, j0 : j0 + tile].transpose(-1, -2))
        s = s.masked_fill(hidden[..., j0 : j0 + tile], float("-inf"))
        mn = torch.maximum(m, s.amax(-1, keepdim=True) * sl2)
        ms = torch.where(mn == float("-inf"), torch.zeros_like(mn), mn)
        alpha = torch.exp2(m - ms)
        p = torch.exp2(s * sl2 - ms)
        l = l * alpha + p.sum(-1, keepdim=True)
        o = o * alpha + torch.matmul(p.to(torch.bfloat16).float(), vf[:, :, j0 : j0 + tile])
        m = mn
    inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
    out = (o * inv).to(torch.bfloat16).permute(0, 2, 1, 3)
    lse = torch.where(l > 0, (m + torch.log2(l)) * LN2, torch.full_like(l, float("-inf")))[..., 0]
    return out, lse


def _zz(sq):
    """Zig-zag query positions: chunks 1 and 2 of four chunks of sq / 2 keys (sk = 2 sq)."""
    c = sq // 2
    return torch.cat([torch.arange(c, 2 * c), torch.arange(2 * c, 3 * c) + c])


# (b, sq, sk, hq, hkv, d, causal, q_pos, kv_pos0, scale)
CASES = [
    (2, 37, 37, 2, 2, 16, True, None, 0, None),
    (1, 37, 37, 2, 2, 16, False, None, 0, None),
    (2, 40, 40, 10, 2, 16, True, None, 0, None),     # GQA 5:1
    (1, 33, 33, 8, 1, 32, False, None, 0, None),     # GQA 8:1
    (1, 20, 70, 5, 1, 16, True, None, 0, None),      # sk > sq, bottom-right aligned
    (2, 50, 20, 2, 1, 16, True, None, 0, None),      # sq > sk: the first 30 rows see no key
    (1, 48, 96, 5, 1, 16, True, "zz", 0, None),      # a context-parallel rank's two query segments
    (1, 40, 40, 2, 2, 16, True, None, 13, None),     # kv_pos0 > 0: early rows see nothing
    (1, 30, 45, 4, 2, 16, False, None, 0, 0.3),      # explicit scale
]


def _pos(sq, sk, q_pos, kv_pos0):
    qp = _zz(sq) if q_pos == "zz" else torch.arange(sq) + (sk - sq)
    return qp, torch.arange(sk) + kv_pos0


@pytest.mark.parametrize("b,sq,sk,hq,hkv,d,causal,q_pos,kv_pos0,scale", CASES)
def test_reference_equals_the_fp32_oracle_and_a_direct_softmax(b, sq, sk, hq, hkv, d, causal, q_pos, kv_pos0, scale):
    q, k, v = _inputs(b, sq, sk, hq, hkv, d, seed=sq * 3 + sk)
    qp, kp = _pos(sq, sk, q_pos, kv_pos0)
    ref = attention_fwd_ref(q, k, v, causal=causal, scale=scale, q_pos=qp, kv_pos=kp)
    o32, l32 = O.attention(q, k, v, causal=causal, scale=scale, q_pos=qp, kv_pos=kp)
    assert ref["out"].dtype == torch.float64 and torch.isfinite(ref["out"]).all()
    assert float((ref["out"] - o32.double()).abs().max()) < 1e-5
    fin = torch.isfinite(l32)
    assert torch.equal(torch.isfinite(ref["lse"]), fin)
    assert float((ref["lse"][fin] - l32.double()[fin]).abs().max()) < 1e-5
    do, dl = _direct(q, k, v, _hidden(sq, sk, causal, qp, kp), scale)
    assert torch.allclose(ref["out"], do, rtol=1e-12, atol=1e-13)
    assert torch.equal(ref["lse"] == float("-inf"), dl == float("-inf"))
    assert torch.allclose(ref["lse"][fin], dl[fin], rtol=1e-12, atol=1e-13)
    blind = ref["n_keys"] == 0
    assert not ref["out"][:, blind].any() and not ref["A"][:, blind].any()
    assert torch.equal(ref["n_keys"], (~_hidden(sq, sk, causal, qp, kp)).sum(-1))


def test_a_and_sigma_are_the_magnitudes_of_p_v():
    q, k, v = _inputs(1, 30, 30, 4, 2, 16, seed=5)
    ref = attention_fwd_ref(q, k, v, causal=True)
    hid = _hidden(30, 30, True)
    kf, vf = k.double().repeat_interleave(2, 2), v.double().repeat_interleave(2, 2)
    s = torch.einsum("bqhd,bkhd->bhqk", q.double(), kf).masked_fill(hid, float("-inf")) / 4
    p = torch.softmax(s, -1)
    assert torch.allclose(ref["A"], torch.einsum("bhqk,bkhd->bqhd", p, vf.abs()), rtol=1e-12)
    assert torch.allclose(ref["sigma"], torch.einsum("bhqk,bkhd->bqhd", p * p, vf * vf).sqrt(), rtol=1e-12)
    assert torch.allclose(ref["M"], torch.where(hid, 0.0, s.abs()).amax(-1), rtol=1e-12)


@pytest.mark.parametrize("case", [CASES[2], CASES[4], CASES[5], CASES[6], CASES[7]])
def test_sampled_rows_equal_the_slices_of_full_mode(case):
    b, sq, sk, hq, hkv, d, causal, q_pos, kv_pos0, scale = case
    q, k, v = _inputs(b, sq, sk, hq, hkv, d, seed=sq + sk)
    qp, kp = _pos(sq, sk, q_pos, kv_pos0)
    kw = dict(causal=causal, scale=scale, q_pos=qp, kv_pos=kp)
    full = attention_fwd_ref(q, k, v, **kw)
    rows = torch.tensor(sorted({0, 1, sq // 2, sq - 2, sq - 1}))
    for bb in (1 << 30, 64):                       # a tiny score block: one row per block
        part = attention_fwd_ref(q, k, v, q_rows=rows, block_bytes=bb, **kw)
        for name in ("out", "A", "sigma"):
            assert torch.allclose(part[name], full[name][:, rows], rtol=1e-12, atol=1e-14), name
        for name in ("lse", "M"):
            assert torch.equal(part[name] == float("-inf"), full[name][:, :, rows] == float("-inf"))
            f = torch.isfinite(part[name])
            assert torch.allclose(part[name][f], full[name][:, :, rows][f], rtol=1e-12, atol=1e-14), name
        assert torch.equal(part["n_keys"], full["n_keys"][rows])


def _docs(sq, seed, lengths=()):
    """Boundaries of a packed row: the given document lengths first, then random ones up to sq."""
    g = seeded(seed)
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    while cu[-1] < sq:
        cu.append(min(sq, cu[-1] + int(torch.randint(1, 40, (1,), generator=g))))
    return torch.tensor(cu)


def test_kv_lo_equals_one_call_per_document():
    sq = 300
    cu = _docs(sq, 3, lengths=(1, 63, 64, 65))
    q, k, v = _inputs(1, sq, sq, 10, 2, 16, seed=7)
    ref = attention_fwd_ref(q, k, v, causal=True, kv_lo=doc_lo(cu, sq))
    for a, e in zip(cu[:-1].tolist(), cu[1:].tolist()):
        one = attention_fwd_ref(q[:, a:e], k[:, a:e], v[:, a:e], causal=True)
        assert torch.allclose(ref["out"][:, a:e], one["out"], rtol=1e-12, atol=1e-14)
        assert torch.allclose(ref["lse"][:, :, a:e], one["lse"], rtol=1e-12, atol=1e-14)
        assert torch.equal(ref["n_keys"][a:e], torch.arange(1, e - a + 1))


def _check_emulated(q, k, v, hidden, ref, scale=None, label=""):
    out, lse = _emulate(q, k, v, hidden, scale)
    return check_attn_fwd(out, lse, ref, label=label), out, lse


@pytest.mark.parametrize("case", CASES)
def test_a_correct_flash_forward_passes_at_the_gpu_limits(case):
    b, sq, sk, hq, hkv, d, causal, q_pos, kv_pos0, scale = case
    q, k, v = _inputs(b, sq, sk, hq, hkv, d, seed=sq * 5 + d)
    qp, kp = _pos(sq, sk, q_pos, kv_pos0)
    ref = attention_fwd_ref(q, k, v, causal=causal, scale=scale, q_pos=qp, kv_pos=kp)
    _check_emulated(q, k, v, _hidden(sq, sk, causal, qp, kp), ref, scale)


# One long causal sequence that the corruptions below start from: 2048 rows, GQA 2:1, d = 64.
S, HQ, HKV, D = 2048, 4, 2, 64


@pytest.fixture(scope="module")
def long_case():
    q, k, v = _inputs(1, S, S, HQ, HKV, D, seed=11)
    # planted keys: row 1500 wants its hidden key 1501, row 1700 its diagonal key 1700
    plant_keys(q, k, [1500, 1700], [1501, 1700])
    hid = _hidden(S, S, True)
    ref = attention_fwd_ref(q, k, v, causal=True)
    stats, out, lse = _check_emulated(q, k, v, hid, ref)
    check_planted(ref, v, [1500], [1501], visible=False)
    check_planted(ref, v, [1700], [1700], visible=True)
    return q, k, v, hid, ref, out, lse


def _splice(out, lse, q, k, v, hidden, rows, heads=None):
    """Correct (out, lse) with rows (and heads) replaced by the bf16 / fp32 rounding of a direct softmax under `hidden`."""
    o, l = _direct(q, k, v, hidden)
    out, lse = out.clone(), lse.clone()
    hs = slice(None) if heads is None else heads
    out[:, rows, hs] = o[:, rows, hs].to(torch.bfloat16)
    lse[:, hs, rows] = l[:, hs, rows].float()
    return out, lse


def _rejects(out, lse, ref, what):
    with pytest.raises(AssertionError) as e:
        check_attn_fwd(out, lse, ref, label=what)
    return str(e.value)


def test_rejects_one_key_leaked_past_the_diagonal(long_case):
    q, k, v, hid, ref, out, lse = long_case
    bad = hid.clone()
    bad[1500, 1501] = False
    _rejects(*_splice(out, lse, q, k, v, bad, [1500]), ref, "leak")


def test_rejects_the_diagonal_key_dropped(long_case):
    q, k, v, hid, ref, out, lse = long_case
    bad = hid.clone()
    bad[1700, 1700] = True
    _rejects(*_splice(out, lse, q, k, v, bad, [1700]), ref, "diagonal dropped")


def test_rejects_one_key_tile_missing_for_one_tile_and_head(long_case):
    q, k, v, hid, ref, out, lse = long_case
    bad = hid.expand(HQ, S, S).clone()
    bad[1, 512:640, 256:384] = True
    _rejects(*_splice(out, lse, q, k, v, bad, list(range(512, 640)), heads=[1]), ref, "tile missing")


def test_rejects_a_row_shifted_by_one(long_case):
    _, _, _, _, ref, out, lse = long_case
    bad = out.clone()
    bad[:, 1000] = out[:, 1001]
    _rejects(bad, lse, ref, "row shift")


def test_rejects_two_heads_of_one_group_swapped(long_case):
    _, _, _, _, ref, out, lse = long_case
    bad = out.clone()
    bad[:, :, 0], bad[:, :, 1] = out[:, :, 1], out[:, :, 0]
    _rejects(bad, lse, ref, "heads swapped")


def test_rejects_an_lse_with_one_extra_key(long_case):
    """Row i's lse also counts key i + 1 (hidden): it moves by exp(s - lse) ~ 1/n, caught by the lse bound alone."""
    q, k, v, hid, ref, out, lse = long_case
    s = torch.einsum("bqhd,bqhd->bhq", q[:, 1000:1999].double(), k[:, 1001:2000].double().repeat_interleave(2, 2)) / 8
    h, r = divmod(int(s[0].argmax()), s.shape[-1])
    r += 1000
    bad = lse.clone()
    bad[0, h, r] = float(torch.logaddexp(lse[0, h, r].double(), s[0, h, r - 1000]))
    msg = _rejects(out, bad, ref, "lse extra key")
    assert "lse" in msg


def test_rejects_an_unmasked_ragged_tail():
    """Non-causal, sk = 200: the second 64-row half of each query tile also weighs the 56 zero-filled keys past sk."""
    q, k, v = _inputs(1, 200, 200, 4, 2, 64, seed=13)
    ref = attention_fwd_ref(q, k, v, causal=False)
    hid = _hidden(200, 200, False)
    out, lse = _emulate(q, k, v, hid)
    check_attn_fwd(out, lse, ref)
    zk = torch.cat([k, torch.zeros((1, 56, 2, 64), dtype=k.dtype)], 1)
    zv = torch.cat([v, torch.zeros((1, 56, 2, 64), dtype=v.dtype)], 1)
    o, l = _direct(q, zk, zv, torch.zeros((200, 256), dtype=torch.bool))
    bad, badl = out.clone(), lse.clone()
    rows = list(range(64, 128)) + list(range(192, 200))
    bad[:, rows], badl[:, :, rows] = o[:, rows].to(torch.bfloat16), l[:, :, rows].float()
    _rejects(bad, badl, ref, "ragged tail")


def test_rejects_a_document_boundary_off_by_one():
    """~250 documents in 4096 rows; in one of them every row also sees the last key of the previous document."""
    sq = 4096
    cu = _docs(sq, 17)
    assert cu.numel() > 200
    q, k, v = _inputs(1, sq, sq, 4, 2, 64, seed=17)
    lo = doc_lo(cu, sq)
    ref = attention_fwd_ref(q, k, v, causal=True, kv_lo=lo)
    out, lse = _emulate(q, k, v, _hidden(sq, sq, True, kv_lo=lo))
    check_attn_fwd(out, lse, ref)
    i = 137
    a, e = int(cu[i]), int(cu[i + 1])
    bad_lo = lo.clone()
    bad_lo[a:e] -= 1
    badref = attention_fwd_ref(q, k, v, causal=True, kv_lo=bad_lo, q_rows=torch.arange(a, e))
    bad, badl = out.clone(), lse.clone()
    bad[:, a:e], badl[:, :, a:e] = badref["out"].to(torch.bfloat16), badref["lse"].float()
    _rejects(bad, badl, ref, "document boundary")


def test_exact_edges_are_exact():
    """A row that sees no key must give 0 and -inf exactly, and a zero V column exactly 0."""
    q, k, v = _inputs(1, 50, 20, 2, 1, 16, seed=19)
    v[..., 12:] = 0
    ref = attention_fwd_ref(q, k, v, causal=True)
    out, lse = _emulate(q, k, v, _hidden(50, 20, True))
    check_attn_fwd(out, lse, ref)
    bad = out.clone()
    bad[0, 3, 0, 0] = 1e-30                        # a blind row
    _rejects(bad, lse, ref, "blind row")
    bad = out.clone()
    bad[0, 40, 1, 13] = 1e-30                      # a zero V column
    _rejects(bad, lse, ref, "zero column")
    badl = lse.clone()
    badl[0, 0, 3] = -1e30
    _rejects(out, badl, ref, "blind lse")
    bad = out.clone()
    bad[0, 40, 1, 0] = float("nan")
    _rejects(bad, lse, ref, "nan")


def test_planted_keys_dominate_their_rows_at_every_head_dim():
    for d, scale in ((64, None), (128, None), (128, 72 ** -0.5)):
        q, k, v = _inputs(1, 600, 600, 10, 2, d, seed=d)
        rows = torch.tensor([5, 127, 128, 300, 599])
        plant_keys(q, k, rows, rows, scale=scale)
        ref = attention_fwd_ref(q, k, v, causal=True, scale=scale, q_rows=rows)
        check_planted(ref, v, range(5), rows, visible=True)
        # the planted key beats every other logit of its row by the planted gap
        sc = 1 / math.sqrt(d) if scale is None else scale
        kf = k.double().repeat_interleave(5, 2)
        s = torch.einsum("bqhd,bkhd->bhqk", q[:, rows].double(), kf) * sc
        s_t = s[0, :, torch.arange(5), rows]
        s[0, :, torch.arange(5), rows] = float("-inf")
        assert float((s_t - s[0].amax(-1)).min()) >= 15
