"""The attention forward (`attn_fwd_kernel`) against the float64 reference of tests/attn_fwd_ref.py, on one H100.

Every path that runs the forward kernel is here at the shapes it runs: the decoder prefill (40:8 x 128, causal) on
both sides of the block-major / head-major switch, at the bench length and with a ragged last tile, sampled rows at
131 072 and 425 984; a context-parallel rank's zig-zag segments; InternViT through `ops.vit_attention`'s strided views
and SigLIP's zero-padded heads; a packed row of ~2 000 documents (`lv_attn_docs_fwd`); flash-decoding
(`ops.attention_decode`) with every split count and a NaN-filled cache tail; and the ABI's edges (ragged lengths,
GQA 1 / 5 / 8, batch > 1, sk > sq, sq > sk, kv_pos0, explicit scales, large logits, layouts, strided views).

Each result goes through `check_attn_fwd` (exact edges, lse bound, elementwise bound, per-row Z, excess).  Planted keys
(`plant_keys`) sit on every row of query tiles that cross a mask edge - a diagonal, a zig-zag segment start or end, a
document start, kv_pos0, a decode split border - so a mask off by one key there is an O(1) error at any length.  Large
cases run twice and must be bit-identical (the schedule is static), and `return_lse=False` must not change a bit.
All inputs are generated on the device from seeds and the reference runs on the device.  The figures are printed
(`pytest -s`); DESIGN.md lists the worst ones against the limits.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.attn_fwd_ref import (PLANT_GAP, _sample_rows, attention_fwd_ref, check_attn_fwd, check_planted, doc_lo,
                                plant_keys)

pytestmark = pytest.mark.gpu

HQ, HKV, D = 40, 8, 128
WORST = {}


@pytest.fixture(scope="module")
def L(lib_built):
    from long_vita_b200 import ops

    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    yield ops
    print(f"\n[attn_fwd_ref] worst figures {({k: round(v, 4) for k, v in WORST.items()})}; "
          f"peak extra device memory {(torch.cuda.max_memory_allocated() - base) / 2**30:.1f} GiB")


def _randn(shape, g, scale=1.0):
    return (torch.randn(shape, generator=g, device="cuda", dtype=torch.float32) * scale).to(torch.bfloat16)


def _inputs(b, sq, sk, hq, hkv, d, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return _randn((b, sq, hq, d), g), _randn((b, sk, hkv, d), g), _randn((b, sk, hkv, d), g)


def _check(out, lse, q, k, v, *, causal, rows=None, label, merged=False, **kw):
    """Reference on `rows` (None = all) and check_attn_fwd of the kernel's result there; records the worst figures."""
    ref = attention_fwd_ref(q, k, v, causal=causal, q_rows=rows, **kw)
    if rows is not None:
        r = rows.to(out.device)
        out, lse = out[:, r], (None if lse is None else lse[:, :, r])
    st = check_attn_fwd(out, lse, ref, merged=merged, label=label)
    print(label, {k_: f"{v_:.3g}" for k_, v_ in st.items()})
    for k_, v_ in st.items():
        WORST[k_] = max(WORST.get(k_, 0.0), v_)
    return ref


def _plant_edge_rows(q, k, rows, qpos, kv_pos0=0, n_keys=None):
    """Plant every row in `rows` (local indices, global positions qpos[rows]): even ones want their first hidden key
    (position + 1, if it exists), odd ones their diagonal key.  Returns (hidden rows, targets, visible rows, targets)."""
    rows = torch.as_tensor(rows, dtype=torch.int64)
    n_keys = k.shape[1] if n_keys is None else n_keys
    diag = qpos[rows] - kv_pos0
    hid = (torch.arange(rows.numel()) % 2 == 0) & (diag + 1 < n_keys) & (diag + 1 >= 0)
    vis = ~hid & (diag >= 0) & (diag < n_keys)
    plant_keys(q, k, torch.cat([rows[hid], rows[vis]]), torch.cat([diag[hid] + 1, diag[vis]]))
    return rows[hid], diag[hid] + 1, rows[vis], diag[vis]


def _check_plants(ref, rows, v, planted):
    rh, th, rv, tv = planted
    if rh.numel():
        check_planted(ref, v, torch.searchsorted(rows, rh), th, visible=False)
    if rv.numel():
        check_planted(ref, v, torch.searchsorted(rows, rv), tv, visible=True)


def _tile_rows(tiles, sq, tile=128):
    return torch.cat([torch.arange(t * tile, min(sq, (t + 1) * tile)) for t in tiles])


# ------------------------------------------------------------------------------------------------ decoder prefill
@pytest.mark.parametrize("T", [18432, 16897, 2304, 6144, 6272])
def test_decoder_prefill_full_tensor(L, T):
    """40:8 x 128 causal over every row.  18 432 is the bench length (head-major order), 16 897 has a one-row last
    tile; 6144 is the last length in block-major order (sk hkv d 4 = 24 MB), 6272 the first in head-major order."""
    q, k, v = _inputs(1, T, T, HQ, HKV, D, seed=T)
    n_t = (T + 127) // 128
    planted = _plant_edge_rows(q, k, _tile_rows([0, n_t // 2, n_t - 1], T), torch.arange(T))
    out, lse = L.attention_fwd(q, k, v, causal=True, return_lse=True)
    ref = _check(out, lse, q, k, v, causal=True, label=f"prefill {T}")
    _check_plants(ref, torch.arange(T), v, planted)
    del ref
    assert torch.equal(L.attention_fwd(q, k, v, causal=True), out)          # return_lse=False: same bits
    out2, lse2 = L.attention_fwd(q, k, v, causal=True, return_lse=True)
    assert torch.equal(out2, out) and torch.equal(lse2, lse)


@pytest.mark.parametrize("T", [131072, 425984])
def test_decoder_prefill_sampled_rows(L, T):
    """Sampled rows (ends, both sides of 128 / 256-row tile boundaries, random) plus fully planted diagonal tiles.
    At 425 984 Q and O hold more than 2^31 elements."""
    q, k, v = _inputs(1, T, T, HQ, HKV, D, seed=T + 1)
    n_t = T // 128
    prow = _tile_rows([0, 1, n_t // 2, n_t - 1], T)
    planted = _plant_edge_rows(q, k, prow, torch.arange(T))
    out, lse = L.attention_fwd(q, k, v, causal=True, return_lse=True)
    rows = torch.unique(torch.cat([_sample_rows(160, T, seed=T), prow]))
    ref = _check(out, lse, q, k, v, causal=True, rows=rows, label=f"prefill {T} sampled")
    _check_plants(ref, rows, v, planted)
    del ref
    out2, lse2 = L.attention_fwd(q, k, v, causal=True, return_lse=True)
    assert torch.equal(out2, out) and torch.equal(lse2, lse)


@pytest.mark.parametrize("cp,rank", [(8, 0), (8, 5), (4, 3)])
def test_zigzag_segments(L, cp, rank):
    """A context-parallel rank's local queries (chunks r and 2cp-1-r of S = 131 072) against the whole K/V: the first
    and last query tile of each segment are planted (first hidden key = position + 1, or the diagonal)."""
    S = 131072
    c = S // (2 * cp)
    q, k, v = _inputs(1, 2 * c, S, HQ, HKV, D, seed=cp * 10 + rank)
    pos = torch.cat([torch.arange(rank * c, (rank + 1) * c), torch.arange((2 * cp - 1 - rank) * c, (2 * cp - rank) * c)])
    tiles = [0, c // 128 - 1, c // 128, 2 * c // 128 - 1]
    prow = _tile_rows(tiles, 2 * c)
    planted = _plant_edge_rows(q, k, prow, pos)
    out, lse = L.attention_fwd(q, k, v, causal=True, return_lse=True, q_seg_len=c,
                               q_seg_pos=(rank * c, (2 * cp - 1 - rank) * c))
    rows = torch.unique(torch.cat([_sample_rows(128, 2 * c, seed=rank, boundaries=(128, 256, c)), prow]))
    ref = _check(out, lse, q, k, v, causal=True, rows=rows, q_pos=pos, label=f"zigzag cp{cp} r{rank}")
    _check_plants(ref, rows, v, planted)
    out2, _ = L.attention_fwd(q, k, v, causal=True, return_lse=True, q_seg_len=c,
                              q_seg_pos=(rank * c, (2 * cp - 1 - rank) * c))
    assert torch.equal(out2, out)


# ------------------------------------------------------------------------------------------------ edges
RAGGED = [
    (1, 128, True, 1), (1, 64, False, 5), (63, 64, True, 5), (63, 128, False, 1),
    (64, 128, True, 8), (64, 64, False, 1), (65, 64, True, 5), (65, 128, True, 1),
    (127, 128, False, 5), (127, 64, True, 8), (128, 64, True, 1), (128, 128, False, 8),
    (129, 128, True, 5), (129, 64, False, 8), (191, 64, True, 1), (191, 128, True, 8),
    (193, 128, False, 8), (193, 64, True, 5),
]


@pytest.mark.parametrize("s,d,causal,G", RAGGED)
def test_ragged_lengths(L, s, d, causal, G):
    """sq = sk on both sides of the 64-row halves and 128-row tiles; GQA 1 / 5 / 8; batch 2 or 3.  Causal cases have
    every row planted."""
    b, hkv = 3 if s % 2 else 2, 2
    q, k, v = _inputs(b, s, s, G * hkv, hkv, d, seed=s * 10 + G)
    planted = _plant_edge_rows(q, k, torch.arange(s), torch.arange(s)) if causal else None
    out, lse = L.attention_fwd(q, k, v, causal=causal, return_lse=True)
    ref = _check(out, lse, q, k, v, causal=causal, label=f"ragged {s} d{d} G{G} {'causal' if causal else 'full'}")
    if planted is not None:
        _check_plants(ref, torch.arange(s), v, planted)


@pytest.mark.parametrize("sq,sk", [(100, 612), (65, 1000), (1, 300), (2, 4097), (3, 129), (4, 2048)])
@pytest.mark.parametrize("causal", [True, False])
def test_cross_lengths_sk_above_sq(L, sq, sk, causal):
    """Bottom-right aligned (query i at position i + sk - sq); sq = 2..4 is the multi-token decode step of
    hf/modeling.attention_step.  Causal: every row planted."""
    d = 64 if sq == 65 else 128
    q, k, v = _inputs(1, sq, sk, 10, 2, d, seed=sq + sk)
    planted = _plant_edge_rows(q, k, torch.arange(sq), torch.arange(sq) + sk - sq) if causal else None
    out, lse = L.attention_fwd(q, k, v, causal=causal, return_lse=True)
    ref = _check(out, lse, q, k, v, causal=causal, label=f"cross {sq}x{sk} {'causal' if causal else 'full'}")
    if planted is not None:
        _check_plants(ref, torch.arange(sq), v, planted)


@pytest.mark.parametrize("sq,sk,d", [(300, 100, 128), (257, 64, 64), (700, 129, 128)])
def test_causal_sq_above_sk_blind_rows(L, sq, sk, d):
    """The first sq - sk rows see no key: out = 0 and lse = -inf exactly (whole work items among them)."""
    q, k, v = _inputs(2, sq, sk, 10, 2, d, seed=sq)
    out, lse = L.attention_fwd(q, k, v, causal=True, return_lse=True)
    _check(out, lse, q, k, v, causal=True, label=f"blind {sq}x{sk}")


@pytest.mark.parametrize("sq,sk,kv_pos0,d", [(384, 384, 100, 128), (200, 500, 37, 64), (256, 256, 64, 128),
                                             (512, 512, 300, 128)])
def test_kv_pos0(L, sq, sk, kv_pos0, d):
    """Keys at kv_pos0 + j.  The row just before kv_pos0 wants key 0 (hidden), the row at kv_pos0 key 0 (visible), and
    the tiles around them are planted.  (512, 300): the first two query tiles are work items with no visible key."""
    q, k, v = _inputs(1, sq, sk, 10, 2, d, seed=kv_pos0 + sq)
    qpos = torch.arange(sq) + (sk - sq)
    r0 = kv_pos0 - (sk - sq)                    # local row at position kv_pos0
    t0 = max(r0, 0) // 128
    prow = _tile_rows(sorted({max(t0 - 1, 0), t0}), sq)
    planted = _plant_edge_rows(q, k, prow, qpos, kv_pos0)
    extra = [r for r in (r0 - 1,) if 0 <= r and r not in set(prow.tolist())]
    if extra:
        plant_keys(q, k, extra, [0])
    out, lse = L.attention_fwd(q, k, v, causal=True, return_lse=True, kv_pos0=kv_pos0)
    ref = _check(out, lse, q, k, v, causal=True, kv_pos=torch.arange(sk) + kv_pos0, label=f"kv_pos0 {sq}x{sk}+{kv_pos0}")
    _check_plants(ref, torch.arange(sq), v, planted)
    if r0 >= 1:
        assert not out[:, : r0].any() and bool((lse[:, :, :r0] == float("-inf")).all())


@pytest.mark.parametrize("scale", [0.05, 0.3, 72 ** -0.5])
@pytest.mark.parametrize("d", [64, 128])
def test_explicit_scale(L, scale, d):
    q, k, v = _inputs(1, 333, 333, 10, 2, d, seed=int(scale * 1000) + d)
    q = (q.float() * 3).to(torch.bfloat16)
    out, lse = L.attention_fwd(q, k, v, causal=True, scale=scale, return_lse=True)
    _check(out, lse, q, k, v, causal=True, scale=scale, label=f"scale {scale:.4f} d{d}")


@pytest.mark.parametrize("causal", [True, False])
def test_large_logit_ramp(L, causal):
    """q and k scaled by 3, keys by a 0.2 -> 6 ramp: logits of a few tens that grow across key tiles, so the running
    max and the rescale of O change on almost every tile."""
    g = torch.Generator(device="cuda").manual_seed(77)
    sq = 1100
    q, k, v = _randn((1, sq, 10, D), g, 3.0), _randn((1, sq, 2, D), g, 3.0), _randn((1, sq, 2, D), g)
    k = (k.float() * torch.linspace(0.2, 6.0, sq, device="cuda").view(1, sq, 1, 1)).to(torch.bfloat16)
    out, lse = L.attention_fwd(q, k, v, causal=causal, return_lse=True)
    _check(out, lse, q, k, v, causal=causal, label=f"large logits {'causal' if causal else 'full'}")


def test_ragged_tail_against_zero_filled_keys(L):
    """Non-causal, sk = 1025 and 200: rows whose every real logit is below -15, so an unmasked zero-filled key past sk
    (s = 0) would dominate them.  Rows in both 64-row halves of every query tile."""
    for sk, d in ((1025, 64), (200, 128)):
        g = torch.Generator(device="cuda").manual_seed(sk)
        e = torch.zeros(d, device="cuda")
        e[0] = 1.0
        k = (torch.randn((2, sk, 2, d), generator=g, device="cuda") + 12.0 * e).to(torch.bfloat16)
        v = _randn((2, sk, 2, d), g)
        q = _randn((2, sk, 10, d), g)
        rows = torch.cat([torch.arange(t, sk, 128) for t in (5, 37, 64 + 5, 64 + 40)])
        q[:, rows] = (-4.0 * math.sqrt(d) * e).to(torch.bfloat16)             # logits -4 k[0], k[0] = 12 +- 4: < -30
        out, lse = L.attention_fwd(q, k, v, causal=False, return_lse=True)
        ref = _check(out, lse, q, k, v, causal=False, label=f"ragged tail {sk}")
        assert float(ref["lse"][:, :, rows].max()) < -10


@pytest.mark.parametrize("layout", ["bshd", "sbhd", "bhsd"])
def test_layouts(L, layout):
    perm = {"bshd": (0, 1, 2, 3), "sbhd": (1, 0, 2, 3), "bhsd": (0, 2, 1, 3)}[layout]
    inv = [perm.index(i) for i in range(4)]
    q, k, v = _inputs(2, 389, 389, 10, 2, D, seed=31)
    out = L.attention_fwd(*(t.permute(inv).contiguous() for t in (q, k, v)), causal=True, layout=layout)
    out_b, lse = L.attention_fwd(q, k, v, causal=True, return_lse=True)
    assert torch.equal(out.permute(perm), out_b)
    _check(out_b, lse, q, k, v, causal=True, label=f"layout {layout}")


@pytest.mark.parametrize("layout", ["megatron", "decoder"])
def test_fused_qkv_strided_views(L, layout):
    """Q / K / V as strided views of one fused QKV buffer (megatron: [s, b, ng, (G + 2) d] with ng = 1; decoder:
    [s, b, (hq + 2 hkv) d]), read in place: bit-identical to contiguous copies."""
    s, b, G = 389, 2, 5
    hkv = 1 if layout == "megatron" else 2
    hq = G * hkv
    g = torch.Generator(device="cuda").manual_seed(21)
    fused = _randn((s, b, (hq + 2 * hkv) * D), g)
    q = fused[..., : hq * D].unflatten(-1, (hq, D)).permute(1, 0, 2, 3)
    k = fused[..., hq * D : (hq + hkv) * D].unflatten(-1, (hkv, D)).permute(1, 0, 2, 3)
    v = fused[..., (hq + hkv) * D :].unflatten(-1, (hkv, D)).permute(1, 0, 2, 3)
    assert not any(t.is_contiguous() for t in (q, k, v))
    out, lse = L.attention_fwd(q, k, v, causal=True, return_lse=True)
    qc, kc, vc = (t.contiguous() for t in (q, k, v))
    out_c, lse_c = L.attention_fwd(qc, kc, vc, causal=True, return_lse=True)
    assert torch.equal(out, out_c) and torch.equal(lse, lse_c)
    _check(out_c, lse_c, qc, kc, vc, causal=True, label=f"fused qkv {layout}")


def test_out_view_leaves_the_rest_of_the_buffer_unchanged(L):
    """out= a strided view of a sentinel-filled buffer (rows offset, heads a slice, ragged last tile): every element
    outside the view keeps its sentinel, the view gets the bits of a plain call."""
    q, k, v = _inputs(2, 193, 193, 10, 2, D, seed=41)
    buf = torch.full((2, 200, 12, D), 7.0, dtype=torch.bfloat16, device="cuda")
    view = buf[:, 3:196, 1:11]
    L.attention_fwd(q, k, v, causal=True, out=view)
    ref_out = L.attention_fwd(q, k, v, causal=True)
    assert torch.equal(view, ref_out)
    mask = torch.ones(buf.shape, dtype=torch.bool, device="cuda")
    mask[:, 3:196, 1:11] = False
    assert bool((buf[mask] == 7.0).all())


# ------------------------------------------------------------------------------------------------ vision
def test_internvit_64_frames(L):
    """InternViT: 64 frames x 1025 tokens x 16 heads x 64, non-causal, through ops.vit_attention's strided
    [n, S, H, 3, D] views of the QKV GEMM output: 9 216 work items, ~70 rounds per CTA on the 4-stage ring."""
    n, S, H, d = 64, 1025, 16, 64
    g = torch.Generator(device="cuda").manual_seed(64)
    qkv = _randn((n, S, 3 * H * d), g)
    out = L.vit_attention(qkv, H)
    v5 = qkv.view(n, S, H, 3, d)
    q, k, v = v5[:, :, :, 0], v5[:, :, :, 1], v5[:, :, :, 2]
    _check(out.view(n, S, H, d), None, q, k, v, causal=False, label="internvit 64x1025")
    _, lse = L.attention_fwd(q, k, v, causal=False, return_lse=True)
    ref = attention_fwd_ref(q[:4], k[:4], v[:4], causal=False)
    check_attn_fwd(out.view(n, S, H, d)[:4], lse[:4], ref, label="internvit lse")
    assert torch.equal(L.vit_attention(qkv, H), out)


def test_siglip_zero_padded_heads(L):
    """SigLIP as hf/siglip.py runs it: 1024 tokens, 16 heads of 72 zero-padded to 128, scale 72^-0.5; the padded
    output columns are exactly 0."""
    n, S, H, hn = 8, 1024, 16, 72
    g = torch.Generator(device="cuda").manual_seed(72)
    qkv = F.pad(_randn((n, S, H * 3 * hn), g).view(n, S, H, 3, hn), (0, 128 - hn))
    q, k, v = qkv[:, :, :, 0], qkv[:, :, :, 1], qkv[:, :, :, 2]
    out, lse = L.attention_fwd(q, k, v, causal=False, scale=hn ** -0.5, return_lse=True)
    assert not out[..., hn:].any()
    _check(out, lse, q, k, v, causal=False, scale=hn ** -0.5, label="siglip")


# ------------------------------------------------------------------------------------------------ documents
def test_documents_packed_row(L):
    """131 072 tokens, ~2 000 documents: lengths 1, 63, 64, 65, 127, 128, 129, one of 40 000, the rest random.  Rows
    at every kind of document edge are checked; the tiles holding the starts of the edge documents are planted (first
    hidden key doc_start - 1, or the document's first key doc_start)."""
    S = 131072
    g = torch.Generator().manual_seed(5)
    lengths = [300, 1, 63, 64, 65, 127, 128, 129, 40000]
    while sum(lengths) < S:
        lengths.append(int(torch.randint(1, 90, (1,), generator=g)))
    lengths[-1] -= sum(lengths) - S
    cu = [0]
    for n_ in lengths:
        cu.append(cu[-1] + n_)
    assert 1900 < len(lengths) < 2200 and cu[-1] == S
    cu_t = torch.tensor(cu)
    q, k, v = _inputs(1, S, S, HQ, HKV, D, seed=2000)
    # planted: every row of the documents 1 .. 8 (the edge lengths and the start of the long one) and the last tile of
    # the long one
    starts = cu_t[:-1]
    rows_p, targets, vis = [], [], []
    for i in range(1, 9):
        a, e = cu[i], cu[i + 1]
        for j, r in enumerate(range(a, min(e, a + 256))):
            rows_p.append(r)
            hidden = j % 2 == 0
            targets.append(a - 1 if hidden else a)
            vis.append(not hidden)
    a = cu[8]
    for j, r in enumerate(range(cu[9] - 128, cu[9])):
        rows_p.append(r)
        targets.append(a - 1 if j % 2 == 0 else a)
        vis.append(j % 2 == 1)
    plant_keys(q, k, rows_p, targets)
    cu_dev = L.packed_cu_seqlens(actual_seq_len=cu[1:], device="cuda", seq_len=S)
    out, lse = L.attention_fwd(q, k, v, causal=True, return_lse=True, cu_seqlens=cu_dev)
    edges = torch.cat([starts, starts + 1, cu_t[1:] - 1, cu_t[1:] - 2]).clamp(0, S - 1)
    pick = torch.randperm(edges.numel(), generator=g)[:600]
    rows = torch.unique(torch.cat([edges[pick], torch.tensor(rows_p), _sample_rows(64, S, seed=9)]))
    ref = _check(out, lse, q, k, v, causal=True, rows=rows, kv_lo=doc_lo(cu_t, S, "cuda"), label="documents 131072")
    rp, tp, vp = torch.tensor(rows_p), torch.tensor(targets), torch.tensor(vis)
    check_planted(ref, v, torch.searchsorted(rows, rp[~vp]), tp[~vp], visible=False)
    check_planted(ref, v, torch.searchsorted(rows, rp[vp]), tp[vp], visible=True)
    out2, lse2 = L.attention_fwd(q, k, v, causal=True, return_lse=True, cu_seqlens=cu_dev)
    assert torch.equal(out2, out) and torch.equal(lse2, lse)


# ------------------------------------------------------------------------------------------------ decode
def _plant_decode(q, k, targets):
    """plant_keys for one query token whose heads want different keys: q [hq, d], k [cap, hkv, d], {head: key}."""
    G = q.shape[0] // k.shape[1]
    for h, t in targets.items():
        kt = k[t, h // G].float()
        k[t, h // G] = (kt * (2 * math.sqrt(D) / kt.norm())).to(k.dtype)
    for h, t in targets.items():                 # after every rescale: two heads of a group may share a key
        kt = k[t, h // G].float()
        nrm = kt.norm()
        q[h] = (PLANT_GAP / (D ** -0.5 * nrm * (nrm - 7.0)) * kt).to(q.dtype)


@pytest.mark.parametrize("length", [1, 127, 128, 129, 2047, 2048, 2049, 33000, 131072, 131073])
def test_decode(L, length):
    """One token against a 40:8 x 128 cache for every split count: the cache rows at and past `length` are NaN (never
    read); the even heads want a key on a split border (the last key of one split, the first of the next), so a split
    that drops or repeats its border key is an O(1) error; out and the merged lse against float64."""
    g = torch.Generator(device="cuda").manual_seed(length)
    cap = length + 300
    q = _randn((HQ, D), g)
    kc, vc = _randn((cap, HKV, D), g), _randn((cap, HKV, D), g)
    kc[length:] = float("nan")
    vc[length:] = float("nan")
    G = HQ // HKV
    for n_splits in (None, 1, 16, 64):
        ns = n_splits if n_splits is not None else max(1, L._sm_count(q.device) // HKV)
        chunk = max(128, (-(-length // ns) + 127) // 128 * 128)
        borders = sorted({t for c0 in range(chunk, length, chunk) for t in (c0 - 1, c0)} | {0, length - 1})
        qq, kk = q.clone(), kc.clone()
        targets = {h: borders[(h // 2) % len(borders)] for h in range(0, HQ, 2)}
        _plant_decode(qq, kk, targets)
        out, lse = L.attention_decode(qq, kk, vc, length, n_splits=n_splits, return_lse=True)
        ref = _check(out.view(1, 1, HQ, D), lse.view(1, HQ, 1), qq.view(1, 1, HQ, D), kk[:length].unsqueeze(0),
                     vc[:length].unsqueeze(0), causal=False, merged=True, label=f"decode {length} splits {n_splits}")
        hs = torch.tensor(sorted(targets))
        vt = vc[torch.tensor([targets[h] for h in hs.tolist()]), hs // G].double()
        dist = (ref["out"][0, 0, hs] - vt).norm(dim=-1) / vt.norm(dim=-1)
        assert float(dist.max()) < 1e-2, ("decode plant", length, n_splits, float(dist.max()))
