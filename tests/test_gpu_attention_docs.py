"""GPU parity of document-masked attention over one packed row (lv_attn_docs_fwd / lv_attn_docs_bwd).

1. One document is today's causal kernel, bit for bit.
2. Documents whose lengths are multiples of 128 give, row for row, exactly what a standalone causal call on each
   document gives: the tile walks coincide, so any difference is a range or a mask bug.
3. Unaligned and edge documents: the forward against the fp32 oracle with the tolerances of the dense kernels (output
   excess < 2e-3, lse < 1e-4), the gradients against the float64 reference of tests/attn_grad_ref.py through
   `check_attn_bwd`, with the first rows of documents planted at their start (`plant_pairs`: the previous document's
   last key hidden, the document's first key visible); and within 1.25x of flash_attn_varlen_func where installed.
4. Two backward runs are bit-identical.
"""
import math

import pytest
import torch

from oracle import ops as O
from tests import packed_oracle as PO
from tests.attn_fwd_ref import doc_lo
from tests.attn_grad_ref import check_rows, plant_edge_pairs
from tests.util import randn_bf16, rel_fro, seeded

pytestmark = pytest.mark.gpu


def excess(out, ref):
    e, f = rel_fro(out, ref), rel_fro(ref.to(torch.bfloat16), ref)
    return math.sqrt(max(e * e - f * f, 0.0))


def cu_of(lengths):
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    return cu


def inputs(S, hq, hkv, d, seed):
    g = seeded(seed)
    q, k, v = randn_bf16((1, S, hq, d), g), randn_bf16((1, S, hkv, d), g), randn_bf16((1, S, hkv, d), g)
    return q, k, v, randn_bf16((1, S, hq, d), g)


def run_docs(q, k, v, do, cu):
    """(out, lse, dq, dk, dv) of the document kernels."""
    from long_vita_b200 import ops

    qc, kc, vc, doc = (t.cuda() for t in (q, k, v, do))
    cut = torch.tensor(cu, dtype=torch.int32, device="cuda")
    out, lse = ops.attention_fwd(qc, kc, vc, causal=True, return_lse=True, cu_seqlens=cut)
    dq, dk, dv = ops.attention_bwd(doc, qc, kc, vc, out, lse, causal=True, cu_seqlens=cut)
    return out, lse, dq, dk, dv


def run_causal(q, k, v, do):
    from long_vita_b200 import ops

    qc, kc, vc, doc = (t.cuda() for t in (q, k, v, do))
    out, lse = ops.attention_fwd(qc, kc, vc, causal=True, return_lse=True)
    dq, dk, dv = ops.attention_bwd(doc, qc, kc, vc, out, lse, causal=True)
    return out, lse, dq, dk, dv


def oracle_per_doc(q, k, v, do, cu):
    """fp32 oracle, one causal call per document (documents are independent by definition)."""
    outs, lses, dqs, dks, dvs = [], [], [], [], []
    for a, b in zip(cu, cu[1:]):
        sl = slice(a, b)
        o, l = O.attention(q[:, sl], k[:, sl], v[:, sl], causal=True)
        gq, gk, gv = O.attention_grads(q[:, sl], k[:, sl], v[:, sl], do[:, sl], causal=True)
        outs.append(o), lses.append(l), dqs.append(gq), dks.append(gk), dvs.append(gv)
    return (torch.cat(outs, 1), torch.cat(lses, 2), torch.cat(dqs, 1), torch.cat(dks, 1), torch.cat(dvs, 1))


@pytest.mark.parametrize("S,hq,hkv,d", [(1000, 40, 8, 128), (16384, 40, 8, 128), (1000, 16, 16, 64)])
def test_one_document_is_the_causal_kernel_bit_for_bit(lib_built, S, hq, hkv, d):
    q, k, v, do = inputs(S, hq, hkv, d, seed=S + d)
    got = run_docs(q, k, v, do, [0, S])
    ref = run_causal(q, k, v, do)
    for name, a, r in zip(("out", "lse", "dq", "dk", "dv"), got, ref):
        assert torch.equal(a, r), name


@pytest.mark.parametrize("lengths,hq,hkv,d", [
    ([512, 128, 1024, 384, 256], 40, 8, 128),
    ([128, 640, 256, 128], 5, 1, 128),
    ([384, 128, 512], 16, 16, 64),
])
def test_aligned_documents_equal_separate_calls_bit_for_bit(lib_built, lengths, hq, hkv, d):
    cu = cu_of(lengths)
    q, k, v, do = inputs(cu[-1], hq, hkv, d, seed=len(lengths) + hq)
    out, lse, dq, dk, dv = run_docs(q, k, v, do, cu)
    for a, b in zip(cu, cu[1:]):
        sl = slice(a, b)
        r = run_causal(q[:, sl].contiguous(), k[:, sl].contiguous(), v[:, sl].contiguous(), do[:, sl].contiguous())
        assert torch.equal(out[:, sl], r[0]), ("out", a, b)
        assert torch.equal(lse[:, :, sl], r[1]), ("lse", a, b)
        assert torch.equal(dq[:, sl], r[2]), ("dq", a, b)
        assert torch.equal(dk[:, sl], r[3]), ("dk", a, b)
        assert torch.equal(dv[:, sl], r[4]), ("dv", a, b)


def _short_docs(S, seed):
    g = torch.Generator().manual_seed(seed)
    lengths = []
    while sum(lengths) < S:
        lengths.append(int(torch.randint(20, 81, (1,), generator=g)))
    lengths[-1] -= sum(lengths) - S
    if lengths[-1] == 0:
        lengths.pop()
    return lengths


EDGE = [1, 63, 64, 65, 127, 128, 129, 30, 90, 200, 45, 17]   # boundaries inside both 64-row halves; ragged end


@pytest.mark.parametrize("lengths,hq,hkv", [
    (EDGE, 40, 8),
    (EDGE, 5, 1),
    ([700, 3, 5, 1000, 260, 77], 5, 1),
    (_short_docs(16384, 7), 40, 8),       # ~300 documents of ~50 tokens
    (_short_docs(16384, 8), 5, 1),
])
def test_unaligned_documents_against_the_oracle(lib_built, lengths, hq, hkv):
    cu = cu_of(lengths)
    d = 128
    S = cu[-1]
    q, k, v, do = inputs(S, hq, hkv, d, seed=len(lengths) * 3 + hq)
    lo = doc_lo(cu, S)
    rows = torch.cat([torch.arange(a, min(e, a + 130)) for a, e in zip(cu[1:], cu[2:])])
    planted = plant_edge_pairs(q, k, rows, torch.where(rows % 2 == 0, lo[rows] - 1, lo[rows]), q_pos=torch.arange(S),
                               kv_pos=torch.arange(S), kv_lo=lo)
    got = run_docs(q, k, v, do, cu)
    ref = oracle_per_doc(q, k, v, do, cu)
    for t in got:
        assert torch.isfinite(t).all()
    assert excess(got[0], ref[0]) < 2e-3, excess(got[0], ref[0])
    assert float((got[1].cpu() - ref[1]).abs().max()) < 1e-4
    check_rows(got[2:], *(t.cuda() for t in (q, k, v, do)), got[0], causal=True, kv_lo=lo.cuda(), planted=planted,
               label=f"documents {len(lengths)} x {hq}:{hkv}")
    if sum(lengths) <= 2048:     # the per-document oracle is the definition; cross-check with the explicit mask once
        o_m, l_m = PO.attention(q, k, v, cu)
        assert torch.allclose(o_m, ref[0], atol=1e-5) and torch.allclose(l_m, ref[1], atol=1e-5)


def test_unaligned_documents_vs_flash_attn_varlen(lib_built):
    fa = pytest.importorskip("flash_attn")
    lengths = EDGE + [1500, 900]
    cu = cu_of(lengths)
    q, k, v, do = inputs(cu[-1], 40, 8, 128, seed=77)
    got = run_docs(q, k, v, do, cu)
    ref = oracle_per_doc(q, k, v, do, cu)
    qf, kf, vf = (t[0].cuda().requires_grad_(True) for t in (q, k, v))
    cut = torch.tensor(cu, dtype=torch.int32, device="cuda")
    m = max(lengths)
    of = fa.flash_attn_varlen_func(qf, kf, vf, cut, cut, m, m, causal=True)
    of.backward(do[0].cuda())
    assert excess(got[0], ref[0]) < 1.25 * excess(of.unsqueeze(0), ref[0]) + 2e-4
    for a, f, r in zip(got[2:], (qf.grad, kf.grad, vf.grad), ref[2:]):
        assert excess(a, r) < 1.25 * excess(f.unsqueeze(0), r) + 2e-4, (excess(a, r), excess(f.unsqueeze(0), r))


def test_document_backward_is_deterministic(lib_built):
    cu = cu_of(_short_docs(4096, 3) + [1000, 2000])
    q, k, v, do = inputs(cu[-1], 40, 8, 128, seed=11)
    a = run_docs(q, k, v, do, cu)
    b = run_docs(q, k, v, do, cu)
    for name, x, y in zip(("out", "lse", "dq", "dk", "dv"), a, b):
        assert torch.equal(x, y), name


def test_packed_cu_seqlens_on_the_device(lib_built):
    """The helper's tensor drives the kernels without a further host check, and the autograd twin saves it."""
    from long_vita_b200 import ops

    lengths = [300, 45, 700]
    cu = cu_of(lengths)
    pos = torch.cat([torch.arange(n) for n in lengths]).view(1, -1).cuda()
    cut = ops.packed_cu_seqlens(pos)
    assert cut.dtype == torch.int32 and cut.is_cuda and cut.tolist() == cu
    q, k, v, do = inputs(cu[-1], 10, 2, 128, seed=5)
    qg, kg, vg = (t.cuda().requires_grad_(True) for t in (q, k, v))
    out = ops.attention(qg, kg, vg, causal=True, cu_seqlens=cut)
    out.backward(do.cuda())
    ref = run_docs(q, k, v, do, cu)
    assert torch.equal(out, ref[0]) and torch.equal(qg.grad, ref[2]) and torch.equal(kg.grad, ref[3])
    assert torch.equal(vg.grad, ref[4])
