"""Pins the float64 reference of the FP8 attention forward and its checker (tests/attn_fp8_ref.py) on the CPU, before any
GPU test relies on them, at the calls a filled K/V cache makes (sq < sk, the diagonal at any offset inside a 128-key
tile and a 64-row Q group) and at the ABI's edges (GQA 5:1, 8:8 and 64:8, batch 2, an explicit scale).

* `reference` equals a textbook float64 softmax over the dequantised operands, its mask built from the positions
  row + sk - sq and its Q quantised group by group here; `q_rows` results, D and SV equal those rows of the full result.
* An fp32 emulation of the kernel's arithmetic (csrc/attn_fwd_fp8.cu: 128-key tiles, a log2-domain online softmax with
  the combined scale s_q s_k scale log2(e) floored at FLT_MIN, l from the unrounded p, e4m3(p 2^8) 2^-8 for P V, the V
  scale applied per tile) passes `check` at the committed LSE_RATIO / Z_ROW on every shape, and with an all-zero Q
  group on a diagonal tile, an all-zero K block and a Q group holding one 1000x row.
* Each corruption of that emulation of the kind an indexing bug produces makes `check` raise, on a batch-2 call with
  sq < sk whose rows are all planted (tests/attn_fwd_ref.py, `plant_keys`): the mask shifted by +1 or -1 key, the Q
  groups aligned to key positions instead of query row 0, a K or V scale read from the neighbouring block, the ragged
  last key tile dropped, the batch entries' K / V swapped, an explicit scale ignored, the FLT_MIN floor removed (NaN on a
  zero Q group at a mask edge), and one tile's V scale omitted.
"""
import math

import pytest
import torch

from tests import attn_fp8_ref as R
from tests.attn_fwd_ref import check_planted, plant_keys
from tests.fp8_ref import quant_rows_ref

D = 128
LOG2E = 1.4426950408889634
LN2 = math.log(2.0)
FLT_MIN = torch.finfo(torch.float32).tiny


def _inputs(b, sq, sk, hq, hkv, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn((b, sq, hq, D), generator=g).to(torch.bfloat16)
    k = torch.randn((b, sk, hkv, D), generator=g).to(torch.bfloat16)
    v = torch.randn((b, sk, hkv, D), generator=g).to(torch.bfloat16)
    return q, k, v


def _plant_all_rows(q, k, scale=None):
    """Plant every row of every batch entry (bottom-right aligned positions): in entry e, rows i with (i + e) even want
    their first hidden key (position + 1, when it exists), the others their diagonal key, so the two entries' plants
    differ.  Returns [(hidden rows, targets, visible rows, targets)] per entry."""
    sq, sk = q.shape[1], k.shape[1]
    rows = torch.arange(sq)
    pos = rows + (sk - sq)
    out = []
    for e in range(q.shape[0]):
        hid = ((rows + e) % 2 == 0) & (pos + 1 < sk)
        plant_keys(q[e:e + 1], k[e:e + 1], torch.cat([rows[hid], rows[~hid]]), torch.cat([pos[hid] + 1, pos[~hid]]),
                   scale=scale)
        out.append((rows[hid], pos[hid] + 1, rows[~hid], pos[~hid]))
    return out


def _check_plants(ref, k, v, planted, skip=()):
    """Each plant still dominates (or stays hidden) after quantisation, judged on the reference over the dequantised V;
    rows in `skip` ((entry, row) pairs whose Q was overwritten) are left out."""
    k8, vt8, ks, vs = R.quant_kv(k, v)
    _, vf = R.dequant_kv(k8, vt8, ks, vs, k.shape[1])
    for e, (rh, th, rv, tv) in enumerate(planted):
        one = {"out": ref["out"][e:e + 1]}
        for rows, tgt, vis in ((rh, th, False), (rv, tv, True)):
            keep = torch.tensor([(e, int(r)) not in skip for r in rows], dtype=torch.bool)
            if keep.any():
                check_planted(one, vf[e:e + 1], rows[keep], tgt[keep], visible=vis)


# ------------------------------------------------------------------------------------------------ direct float64
def _direct_q(q):
    """The kernel's Q rule written out group by group: per (batch, head), rows [64 g, 64 g + 64) are one e4m3 row of
    csrc/fp8_core.h; returns float(q8) s_q (the fp32 product, as dequant_kv forms K and V) [b, sq, hq, d] float64."""
    b, sq, hq, d = q.shape
    out = torch.zeros(q.shape, dtype=torch.float64)
    for e in range(b):
        for h in range(hq):
            for r0 in range(0, sq, R.QROWS):
                x = q[e, r0:r0 + R.QROWS, h]
                codes, s = quant_rows_ref(x.reshape(1, -1))
                out[e, r0:r0 + R.QROWS, h] = (codes.view(R.FP8).float() * s).view(x.shape).double()
    return out


def _direct(q, k, v, scale=None):
    """Textbook float64 causal softmax over the dequantised operands, query row i at position i + sk - sq; returns
    (out, lse, hidden [sq, sk], qf, kf, vf)."""
    sq, sk = q.shape[1], k.shape[1]
    G = q.shape[2] // k.shape[2]
    scale = 1.0 / math.sqrt(q.shape[-1]) if scale is None else scale
    kf, vf = R.dequant_kv(*R.quant_kv(k, v), sk)
    qf = _direct_q(q)
    kr, vr = kf.double().repeat_interleave(G, 2), vf.double().repeat_interleave(G, 2)
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kr) * scale
    hidden = torch.arange(sk)[None, :] > (torch.arange(sq) + (sk - sq))[:, None]
    s = s.masked_fill(hidden, float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    return torch.einsum("bhqk,bkhd->bqhd", p, vr), lse, hidden, qf, kf, vf


# (b, sq, sk, hq, hkv, scale): sq < sk with sk - sq = 1, 63, 64, 65, 127 (mod 128) and the offsets a cache makes
# (33, 129); sq == sk on both sides of 64 and 128; an explicit scale; batch 2
SHAPES = [
    (1, 200, 457, 5, 1, None),       # 257
    (1, 100, 163, 8, 8, None),       # 63
    (2, 37, 229, 5, 1, None),        # 192
    (1, 300, 365, 5, 1, None),       # 65
    (1, 3, 130, 64, 8, None),        # 127
    (1, 300, 333, 5, 1, None),       # 33
    (1, 1, 130, 5, 1, None),         # 129
    (1, 129, 129, 5, 1, None),
    (1, 1, 1, 8, 8, None),
    (1, 63, 63, 5, 1, None),
    (2, 64, 64, 5, 1, None),
    (1, 65, 65, 64, 8, None),
    (1, 127, 127, 5, 1, None),
    (1, 128, 128, 8, 8, None),
    (1, 129, 200, 5, 1, 0.02),
    (2, 200, 457, 10, 2, 0.5),
]


def _ids(shapes):
    return [f"b{b}-{sq}x{sk}-{hq}:{hkv}" + ("" if s is None else f"-scale{s}") for b, sq, sk, hq, hkv, s in shapes]


@pytest.mark.parametrize("b,sq,sk,hq,hkv,scale", SHAPES, ids=_ids(SHAPES))
def test_reference_equals_a_direct_float64_softmax(b, sq, sk, hq, hkv, scale):
    q, k, v = _inputs(b, sq, sk, hq, hkv, seed=sq * 7 + sk)
    ref = R.reference(q, k, v, scale=scale)
    do, dl, hidden, qf, kf, vf = _direct(q, k, v, scale)
    assert torch.equal(R.quant_q(q).double(), qf)
    assert torch.allclose(ref["out"], do, rtol=1e-12, atol=1e-13)
    assert torch.allclose(ref["lse"], dl, rtol=1e-12, atol=1e-13)
    assert torch.equal(ref["n_keys"], (~hidden).sum(-1))
    # the bound terms: D = scale |q8 s_q| max_j |k8_j s_k| over the kv head, SV = sum of |v| over the visible keys
    G = hq // hkv
    sc = 1.0 / math.sqrt(D) if scale is None else scale
    kmax = kf.double().norm(dim=-1).amax(1).repeat_interleave(G, -1)                       # [b, hq]
    assert torch.allclose(ref["D"], (sc * qf.norm(dim=-1) * kmax[:, None]).permute(0, 2, 1), rtol=1e-12)
    sv = torch.einsum("qk,bkhd->bqhd", (~hidden).double(), vf.double().abs()).repeat_interleave(G, 2)
    assert torch.allclose(ref["SV"], sv, rtol=1e-6)                # an fp32 prefix sum: a bound term
    # sampled rows are the rows of the full result (their Q groups quantised alone)
    rows = torch.tensor(sorted({r for r in (0, 1, 62, 63, 64, 65, 127, 128, sq // 2, sq - 1) if r < sq}))
    part = R.reference(q, k, v, q_rows=rows, scale=scale)
    for name in ("out", "A", "sigma", "SV"):
        assert torch.allclose(part[name], ref[name][:, rows], rtol=1e-12, atol=1e-14), name
    for name in ("lse", "M", "D"):
        assert torch.allclose(part[name], ref[name][:, :, rows], rtol=1e-12, atol=1e-14), name
    assert torch.equal(part["n_keys"], ref["n_keys"][rows])


# ------------------------------------------------------------------------------------------------ fp32 emulation
def _q_codes(q, off=0):
    """Q's e4m3 codes [b, hq, sq, d] float32 and each row's group scale [b, hq, sq]; the 64-row groups start at query
    row -off (off = 0 is the kernel's rule: groups aligned to query row 0 of the call)."""
    b, sq, hq, d = q.shape
    qp = torch.cat([torch.zeros((b, off, hq, d), dtype=q.dtype), q], 1)
    qb, ng = R._blocks(qp, R.QROWS)
    codes, s = quant_rows_ref(qb)
    codes = codes.view(R.FP8).float().view(b, hq, ng * R.QROWS, d)[:, :, off:off + sq]
    return codes, s.repeat_interleave(R.QROWS, -1)[..., off:off + sq]


def _emulate(q, k, v, *, scale=None, mask_shift=0, q_off=0, k_scale_nb=False, v_scale_nb=False, drop_ragged=False,
             kv_swap=False, floor=True, v_scale_skip=None):
    """The FP8 kernel's arithmetic in fp32: (out [b, sq, hq, d] bf16, lse [b, hq, sq] fp32).  The keyword arguments
    other than `scale` are corruptions (all off: the correct kernel)."""
    b, sq, hq, d = q.shape
    sk, hkv = k.shape[1], k.shape[2]
    G = hq // hkv
    scale = 1.0 / math.sqrt(d) if scale is None else scale
    scale_log2 = torch.tensor(scale, dtype=torch.float32) * torch.tensor(LOG2E, dtype=torch.float32)
    k8, vt8, ks, vs = R.quant_kv(k, v)
    nt = ks.shape[-1]
    one = torch.ones_like(ks)
    kc, vc = R.dequant_kv(k8, vt8, one, one, nt * R.BLOCK)          # e4m3 codes [b, nt * 128, hkv, d], padding 0
    kc, vc = (t.repeat_interleave(G, 2).permute(0, 2, 1, 3) for t in (kc, vc))
    ks, vs = ks.repeat_interleave(G, 1), vs.repeat_interleave(G, 1)  # [b, hq, nt]
    if kv_swap:
        kc, vc, ks, vs = (t.flip(0) for t in (kc, vc, ks, vs))
    qc, qs = _q_codes(q, q_off)
    qs_log2 = (qs * scale_log2)[..., None]                            # [b, hq, sq, 1]
    qpos = torch.arange(sq) + (sk - sq) + mask_shift
    hidden = (torch.arange(nt * R.BLOCK)[None, :] > qpos[:, None]) | (torch.arange(nt * R.BLOCK)[None, :] >= sk)
    m = torch.full((b, hq, sq, 1), float("-inf"))
    l = torch.zeros((b, hq, sq, 1))
    o = torch.zeros((b, hq, sq, d))
    n_tiles = nt - 1 if drop_ragged and sk % R.BLOCK else nt
    nb = lambda j: j + 1 if j + 1 < nt else j - 1                     # noqa: E731
    for j in range(n_tiles):
        cols = slice(j * R.BLOCK, (j + 1) * R.BLOCK)
        cs = qs_log2 * ks[..., nb(j) if k_scale_nb else j][..., None, None]
        if floor:
            cs = cs.clamp_min(FLT_MIN)
        s = torch.matmul(qc, kc[:, :, cols].transpose(-1, -2))         # e4m3 products are exact in fp32
        s = s.masked_fill(hidden[:, cols], float("-inf"))
        mn = torch.fmax(m, s.amax(-1, keepdim=True) * cs)              # fmaxf: a NaN operand is ignored
        ms = torch.where(mn == float("-inf"), torch.zeros_like(mn), mn)
        alpha = torch.exp2(m - ms)
        p = torch.exp2(s * cs - ms)
        l = l * alpha + p.sum(-1, keepdim=True)
        acc = torch.matmul((p * 256.0).to(R.FP8).float(), vc[:, :, cols])
        sv = 1.0 if v_scale_skip == j else vs[..., nb(j) if v_scale_nb else j][..., None, None]
        o = alpha * o + (sv / 256.0) * acc
        m = mn
    inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
    out = (o * inv).to(torch.bfloat16).permute(0, 2, 1, 3)
    lse = torch.where(l > 0, (m + torch.log2(l)) * LN2, torch.full_like(l, float("-inf")))[..., 0]
    return out, lse


@pytest.mark.parametrize("b,sq,sk,hq,hkv,scale", SHAPES, ids=_ids(SHAPES))
def test_a_correct_emulation_passes_at_the_gpu_limits(b, sq, sk, hq, hkv, scale):
    """Every row planted (a plant needs sq <= sk): the rows hold near one-hot softmaxes next to the diagonal."""
    q, k, v = _inputs(b, sq, sk, hq, hkv, seed=sq * 11 + sk)
    planted = _plant_all_rows(q, k, scale)
    ref = R.reference(q, k, v, scale=scale)
    _check_plants(ref, k, v, planted)
    out, lse = _emulate(q, k, v, scale=scale)
    st = R.check(out, lse, ref, label="emulation")
    assert st["lse_ratio"] <= R.LSE_RATIO / 2 and st["z_row"] <= R.Z_ROW / 2, st


EDGES = ["zero_q_group", "zero_k_block", "outlier_row"]


@pytest.mark.parametrize("edge", EDGES)
@pytest.mark.parametrize("sq,sk", [(200, 457), (300, 300)])
def test_a_correct_emulation_passes_at_the_scale_edges(edge, sq, sk):
    """An all-zero Q group on a diagonal tile (scale 0: the FLT_MIN floor keeps the masked keys at -inf), an all-zero K
    block (logits exactly 0), and a Q group whose scale is set by one row 1000x larger than the rest (their codes
    mostly subnormal or zero)."""
    q, k, v = _inputs(2, sq, sk, 10, 2, seed=sq + sk + len(edge))
    _plant_all_rows(q, k)
    if edge == "zero_q_group":
        q[1, 128:192, 3] = 0
        q[0, 64:128] = 0
    elif edge == "zero_k_block":
        k[0, 128:256, 1] = 0
        k[1, 256:384] = 0
    else:
        q[0, 70, 4] = (q[0, 70, 4].float() * 1000).to(torch.bfloat16)
    ref = R.reference(q, k, v)
    R.check(*_emulate(q, k, v), ref, label=edge)


# ------------------------------------------------------------------------------------------------ corruptions
@pytest.fixture(scope="module")
def cache_call():
    """Batch 2, 10:2 heads, 200 new rows over 457 keys (sk - sq = 257: 1 mod 128 and mod 64, a ragged last key tile of
    73 keys), every row planted, entry 1 head 3 rows 64..127 all zero (a zero Q group across the diagonal)."""
    q, k, v = _inputs(2, 200, 457, 10, 2, seed=457)
    planted = _plant_all_rows(q, k)
    q[1, 64:128, 3] = 0
    ref = R.reference(q, k, v)
    _check_plants(ref, k, v, planted, skip={(1, r) for r in range(64, 128)})
    R.check(*_emulate(q, k, v), ref, label="clean")
    return q, k, v, ref


CORRUPTIONS = {
    "mask_plus_one": dict(mask_shift=1),
    "mask_minus_one": dict(mask_shift=-1),
    "q_groups_at_key_positions": dict(q_off=257 % R.QROWS),
    "k_scale_of_next_block": dict(k_scale_nb=True),
    "v_scale_of_next_block": dict(v_scale_nb=True),
    "ragged_key_tile_dropped": dict(drop_ragged=True),
    "batch_kv_swapped": dict(kv_swap=True),
    "zero_scale_not_floored": dict(floor=False),
    "v_scale_omitted_on_tile_1": dict(v_scale_skip=1),
}


@pytest.mark.parametrize("name", list(CORRUPTIONS))
def test_check_rejects(cache_call, name):
    q, k, v, ref = cache_call
    out, lse = _emulate(q, k, v, **CORRUPTIONS[name])
    with pytest.raises(AssertionError):
        R.check(out, lse, ref, label=name)


def test_check_rejects_an_ignored_scale():
    """scale = 0.02 (plants at that scale): a kernel that used 1/sqrt(d) instead."""
    q, k, v = _inputs(1, 129, 200, 5, 1, seed=2)
    _plant_all_rows(q, k, scale=0.02)
    ref = R.reference(q, k, v, scale=0.02)
    R.check(*_emulate(q, k, v, scale=0.02), ref, label="scale 0.02")
    with pytest.raises(AssertionError):
        R.check(*_emulate(q, k, v), ref, label="scale ignored")


def test_the_zero_scale_floor_matters_only_at_a_mask_edge(cache_call):
    """Without the floor the zero Q group's rows are NaN (-inf * 0 on their masked keys); every other row is unchanged."""
    q, k, v, _ = cache_call
    good, _ = _emulate(q, k, v)
    bad, _ = _emulate(q, k, v, floor=False)
    nan = bad.isnan().any(-1)
    assert bool(nan[1, 64:128, 3].all())
    nan[1, 64:128, 3] = False
    assert not nan.any()
    keep = torch.ones(bad.shape[:3], dtype=torch.bool)
    keep[1, 64:128, 3] = False
    assert torch.equal(bad[keep], good[keep])
