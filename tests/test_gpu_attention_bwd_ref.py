"""The attention backward (`lv_attn_bwd`, `lv_attn_docs_bwd`) against the float64 reference of tests/attn_grad_ref.py,
on one H100, on the paths the other backward files do not hold to its checker: the decoder at 16 897 tokens (a ragged
last 128-row tile and 64-row half), a packed row of ~2 000 documents with edge lengths at 131 072 tokens (sampled),
and InternViT's 64 frames through `ops.vit_attention`'s strided dQKV buffer.  tests/test_gpu_attention_bwd_long.py,
tests/test_gpu_attention_bwd_edges.py and tests/test_gpu_attention_docs.py run the rest of the decoder,
context-parallel, ABI and document cases through the same checker.

Each result goes through `check_attn_bwd` (exact edges, elementwise bound, per-row Z, excess).  Paired plants
(`plant_pairs`) sit on every row of the query tiles that cross a mask edge - the diagonal at 64- and 128-row tile
boundaries, a document start (the previous document's last key hidden, the document's first key visible) - so a mask
off by one key in either pass is an O(1) error.  Large cases run twice and must be bit-identical.  Inputs are generated
on the device from seeds and the reference runs on the device.  The figures are printed (`pytest -s`); DESIGN.md lists
the worst ones against the limits.
"""
import pytest
import torch

from tests.attn_fwd_ref import doc_lo
from tests.attn_grad_ref import _sample_rows, check_rows, edge_targets, plant_edge_pairs

pytestmark = pytest.mark.gpu

HQ, HKV, D = 40, 8, 128
WORST = {}


@pytest.fixture(scope="module")
def L(lib_built):
    from long_vita_b200 import ops

    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    yield ops
    print(f"\n[attn_bwd_ref] worst figures {({k: round(v, 4) for k, v in WORST.items()})}; "
          f"peak extra device memory {(torch.cuda.max_memory_allocated() - base) / 2**30:.1f} GiB")


def _inputs(b, sq, sk, hq, hkv, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)

    def rnd(*shape):
        return torch.randn(shape, generator=g, device="cuda", dtype=torch.float32).to(torch.bfloat16)

    return rnd(b, sq, hq, d), rnd(b, sk, hkv, d), rnd(b, sk, hkv, d), rnd(b, sq, hq, d)


def _tile_rows(tiles, sq, tile=128):
    return torch.cat([torch.arange(t * tile, min(sq, (t + 1) * tile)) for t in tiles])


def _fwd_bwd(L, q, k, v, do, **kw):
    out, lse = L.attention_fwd(q, k, v, causal=True, return_lse=True, **kw)
    return out, L.attention_bwd(do, q, k, v, out, lse, causal=True, **kw)


def test_decoder_16897_full_tensor(L):
    """40:8 x 128 causal, every gradient element: the last 128-row tile has one row and its 64-row halves are ragged.
    The first, middle and last two query tiles are planted on every row (first hidden key or diagonal)."""
    T = 16897
    q, k, v, do = _inputs(1, T, T, HQ, HKV, D, seed=T)
    n_t = (T + 127) // 128
    rows = _tile_rows([0, n_t // 2, n_t - 2, n_t - 1], T)
    pos = torch.arange(T)
    planted = plant_edge_pairs(q, k, rows, edge_targets(rows, pos), q_pos=pos, kv_pos=pos)
    out, got = _fwd_bwd(L, q, k, v, do)
    check_rows(got, q, k, v, do, out, causal=True, planted=planted, worst=WORST, label=f"decoder {T}")
    _, again = _fwd_bwd(L, q, k, v, do)
    assert all(torch.equal(a, b) for a, b in zip(got, again))


def _doc_targets(cu, docs, rows_per_doc=256):
    """Every row of the first `rows_per_doc` of each document in `docs`: even rows want the previous document's last key
    (hidden), odd rows the document's first key (visible)."""
    rows, targets = [], []
    for i in docs:
        a, e = int(cu[i]), int(cu[i + 1])
        r = torch.arange(a, min(e, a + rows_per_doc))
        rows.append(r)
        targets.append(torch.where(r % 2 == 0, a - 1, a))
    return torch.cat(rows), torch.cat(targets)


def _cu(lengths):
    cu = [0]
    for n in lengths:
        cu.append(cu[-1] + n)
    return torch.tensor(cu)


def test_documents_131k_sampled(L):
    """131 072 tokens, ~2 000 documents: edge lengths 1, 63, 64, 65, 127, 128, 129 whose starts and ends fall on and
    beside 64- and 128-row tile boundaries, one of 40 000, the rest 1 .. 89.  dQ on the planted rows (every row of the
    edge documents and the first 256 of the long one), the rows at every document edge and random rows; dK / dV on
    the 128-key tiles holding the edge documents and the long one's first and last, each against every query that sees
    them."""
    S = 131072
    g = torch.Generator().manual_seed(5)
    lengths = [128, 1, 63, 64, 65, 127, 128, 129, 40000]   # starts at 128, 129, 192, 256, 321, 448, 576, 705
    while sum(lengths) < S:
        lengths.append(int(torch.randint(1, 90, (1,), generator=g)))
    lengths[-1] -= sum(lengths) - S
    cu = _cu(lengths)
    assert 1900 < len(lengths) < 2200 and int(cu[-1]) == S
    q, k, v, do = _inputs(1, S, S, HQ, HKV, D, seed=2001)
    lo = doc_lo(cu, S, "cuda")
    prow, targets = _doc_targets(cu, range(1, 9))
    pos = torch.arange(S)
    planted = plant_edge_pairs(q, k, prow, targets, q_pos=pos, kv_pos=pos, kv_lo=lo.cpu())
    cut = cu.to("cuda", torch.int32)
    out, got = _fwd_bwd(L, q, k, v, do, cu_seqlens=cut)
    starts = cu[:-1]
    edges = torch.cat([starts, starts + 1, cu[1:] - 1, cu[1:] - 2]).clamp(0, S - 1)
    pick = torch.randperm(edges.numel(), generator=g)[:600]
    rows = torch.unique(torch.cat([edges[pick], prow, _sample_rows(64, S, seed=9)]))
    tiles = sorted({int(cu[i]) // 128 for i in range(1, 10)} | {int(cu[9]) // 128 - 1, S // 128 - 1})
    keys = _tile_rows(tiles, S)
    check_rows(got, q, k, v, do, out, causal=True, kv_lo=lo, q_rows=rows, kv_rows=keys, planted=planted, worst=WORST,
               label="documents 131072")
    _, again = _fwd_bwd(L, q, k, v, do, cu_seqlens=cut)
    assert all(torch.equal(a, b) for a, b in zip(got, again))


def test_internvit_64_frames(L):
    """InternViT: 64 frames x 1025 tokens x 16 heads x 64, non-causal, through ops.vit_attention's autograd: q / k / v
    strided views of the QKV GEMM output ([H, 3, D] columns), dQ / dK / dV written through the same strides into one
    dQKV buffer.  Every gradient element."""
    n, S, H, d = 64, 1025, 16, 64
    g = torch.Generator(device="cuda").manual_seed(65)
    qkv = torch.randn((n, S, 3 * H * d), generator=g, device="cuda").to(torch.bfloat16)
    do = torch.randn((n, S, H * d), generator=g, device="cuda").to(torch.bfloat16)
    x = qkv.clone().requires_grad_(True)
    out = L.vit_attention(x, H)
    out.backward(do)
    g5 = x.grad.view(n, S, H, 3, d)
    v5 = qkv.view(n, S, H, 3, d)
    check_rows((g5[:, :, :, 0], g5[:, :, :, 1], g5[:, :, :, 2]), v5[:, :, :, 0], v5[:, :, :, 1], v5[:, :, :, 2],
               do.view(n, S, H, d), out.detach().view(n, S, H, d), causal=False, worst=WORST, label="internvit 64x1025")
    x2 = qkv.clone().requires_grad_(True)
    L.vit_attention(x2, H).backward(do)
    assert torch.equal(x2.grad, x.grad)
