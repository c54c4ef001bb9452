"""Pins the float64 token-wise references and their checker (tests/tokenwise_ref.py) on the CPU, before any GPU test
relies on them: each reference equals a direct float64 restatement and agrees with the CPU oracle / fp32 autograd,
slabbing does not change the reductions, the checker accepts bf16(r) and an fp32 emulation of each kernel's
arithmetic, and it rejects, at the flip limits the GPU tests use, each kind of wrong result built here from correct
data."""
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import ops as O
from tests.tokenwise_ref import (FLIPS, bias_gelu_ref, check_tokenwise, check_untouched, decode_merge_ref, edge_groups,
                                 edge_op, edge_rows, flip_limits,
                                 gelu_bwd_ref, layernorm_bwd_ref, layernorm_dwdb_ref, layernorm_ref, ls_residual_bwd_ref,
                                 ls_residual_ref, residual_sum, rmsnorm_bwd_ref, rmsnorm_dw_ref, rmsnorm_ref, rope_bwd_ref,
                                 rope_ref, rope_table_ref, swiglu_bwd_ref, swiglu_ref)
from tests.util import randn_bf16, seeded

BF, f64 = torch.bfloat16, torch.float64
ROWS, COLS = 256, 5120


def _chk(op, y, ref, name=""):
    return check_tokenwise(y, *ref, name=name or op, **flip_limits(op, y.shape[-1] if y.dim() else 1))


def _norm_inputs(rows=ROWS, cols=COLS, seed=1, scale=1.0, mean=0.0):
    g = seeded(seed)
    x = (torch.randn((rows, cols), generator=g) * scale + mean).to(BF)
    w = (1 + 0.1 * torch.randn(cols, generator=g)).to(BF)
    return x, w, randn_bf16((cols,), g, 0.1), randn_bf16((rows, cols), g), randn_bf16((rows, cols), g)


# ------------------------------------------------------------------------------------------------
# fp32 emulations of the kernels' arithmetic (and the mutations of them)
# ------------------------------------------------------------------------------------------------
def emu_rmsnorm(x, w, eps, *, drop_last=False, div=None):
    s = x.float()
    ss = (s[:, :-8] if drop_last else s).square().sum(-1, keepdim=True)
    rstd = torch.rsqrt(ss / (div or x.shape[-1]) + eps)
    return ((s * rstd).to(BF).float() * w.float()).to(BF)


def emu_layernorm(x, w, b, eps, *, one_pass=False):
    v = x.float()
    m = v.mean(-1, keepdim=True)
    var = (v.square().mean(-1, keepdim=True) - m * m) if one_pass else (v - m).square().mean(-1, keepdim=True)
    return ((v - m) * torch.rsqrt(var + eps) * w.float() + b.float()).to(BF)


def emu_rmsnorm_bwd(x, w, dy, eps, add_in=None, parts=16, drop_part=None):
    """fp32 as the kernel: dw partial rows p hold the rows r = p mod parts in order (the grid stride), summed after."""
    v, g, wf = x.float(), dy.float(), w.float()
    rstd = torch.rsqrt(v.square().mean(-1, keepdim=True) + eps)
    xh = v * rstd
    dot = (g * wf * xh).sum(-1, keepdim=True) / x.shape[-1]
    dx = rstd * (g * wf - xh * dot) + (0 if add_in is None else add_in.float())
    part = torch.zeros((parts, x.shape[-1]))
    for r in range(x.shape[0]):
        part[r % parts] += g[r] * xh[r]
    if drop_part is not None:
        part[drop_part] = 0
    return dx.to(BF), part.sum(0).to(BF)


def emu_rope(x, cos, sin, *, swap_halves=False, sin_sign=1.0):
    h = x.shape[-1] // 2
    xf, c, s = x.float(), cos.float()[:, None], sin_sign * sin.float()[:, None]
    o1 = (xf[..., :h] * c[..., :h]).to(BF).float() + (-xf[..., h:] * s[..., :h]).to(BF).float()
    o2 = (xf[..., h:] * c[..., h:]).to(BF).float() + (xf[..., :h] * s[..., h:]).to(BF).float()
    return torch.cat([o2, o1] if swap_halves else [o1, o2], -1).to(BF)


def emu_swiglu(gu, *, swap=False):
    i = gu.shape[-1] // 2
    g, u = gu[..., :i].float(), gu[..., i:].float()
    if swap:
        g, u = u, g
    return (F.silu(g).to(BF).float() * u).to(BF)


def emu_decode_merge(o, lse, *, skip=None):
    n, G, hkv, d = o.shape
    l = lse.permute(1, 2, 0).reshape(hkv * G, n).clone()
    if skip is not None:
        l[:, skip] = -math.inf
    m = l.max(-1, keepdim=True).values
    w = torch.exp(l - m)
    acc = (w[..., None] * o.float().permute(2, 1, 0, 3).reshape(hkv * G, n, d)).sum(1)
    return (acc / w.sum(-1, keepdim=True)).to(BF)


# ------------------------------------------------------------------------------------------------
# the references against direct restatements, the oracle and fp32 autograd
# ------------------------------------------------------------------------------------------------
def test_norm_references_are_the_float64_restatements():
    x, w, b, dy, a = _norm_inputs(64, 1024, seed=2)
    s = residual_sum(x, a)
    assert torch.equal(s, x + a)                               # the oracle's bf16 add
    xd, wd = s.double(), w.double()
    want = (xd * torch.rsqrt(xd.square().mean(-1, keepdim=True) + 1e-6)).to(BF).double() * wd
    torch.testing.assert_close(rmsnorm_ref(x, w, 1e-6, a).r, want, rtol=1e-14, atol=0)
    want = F.layer_norm(x.double(), (1024,), wd, b.double(), 1e-5)
    torch.testing.assert_close(layernorm_ref(x, w, b, 1e-5).r, want, rtol=1e-12, atol=1e-12)
    # the backward references against float64 autograd of the same definitions (the inner bf16 rounding as identity)
    xg, wg = x.double().requires_grad_(True), wd.clone().requires_grad_(True)
    (xg * torch.rsqrt(xg.square().mean(-1, keepdim=True) + 1e-6) * wg).backward(dy.double())
    dx, dw = rmsnorm_bwd_ref(x, w, dy, 1e-6, a), rmsnorm_dw_ref(x, w, dy, 1e-6)
    torch.testing.assert_close(dx.r, xg.grad + a.double(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(dw.r, wg.grad, rtol=1e-12, atol=1e-12)
    xg, wg, bg = x.double().requires_grad_(True), wd.clone().requires_grad_(True), b.double().requires_grad_(True)
    F.layer_norm(xg, (1024,), wg, bg, 1e-5).backward(dy.double())
    dx, (dw, db) = layernorm_bwd_ref(x, w, dy, 1e-5), layernorm_dwdb_ref(x, w, dy, 1e-5)
    for got, want in ((dx.r, xg.grad), (dw.r, wg.grad), (db.r, bg.grad)):
        torch.testing.assert_close(got, want, rtol=1e-10, atol=1e-10)


def test_norm_references_agree_with_the_oracle():
    x, w, b, _, a = _norm_inputs(64, 1024, seed=3)
    for got, want in ((rmsnorm_ref(x, w, 1e-6, a).r, O.rmsnorm(x + a, w, 1e-6)),
                      (layernorm_ref(x, w, b, 1e-6).r, O.layernorm(x, w, b, 1e-6))):
        assert float((got.to(BF) != want).double().mean()) < 2e-3


def test_activation_and_rope_references():
    g = seeded(4)
    gu, dh = randn_bf16((64, 2 * 512), g, 2.0), randn_bf16((64, 512), g)
    gd, ud = gu[:, :512].double(), gu[:, 512:].double()
    torch.testing.assert_close(swiglu_ref(gu).r, F.silu(gd).to(BF).double() * ud, rtol=1e-14, atol=0)
    assert float((swiglu_ref(gu).r.to(BF) != O.swiglu(gu)).double().mean()) < 1e-2
    gg = gu.double().requires_grad_(True)
    (F.silu(gg[:, :512]) * gg[:, 512:]).backward(dh.double())
    torch.testing.assert_close(swiglu_bwd_ref(gu, dh).r, gg.grad, rtol=1e-12, atol=1e-300)
    x, b = randn_bf16((64, 512), g, 2.0), randn_bf16((512,), g)
    for approx in ("none", "tanh"):
        pre = (x.float() + b.float()).to(BF).double()
        torch.testing.assert_close(bias_gelu_ref(x, b, approx).r, F.gelu(pre, approximate=approx), rtol=1e-14, atol=0)
        ref = bias_gelu_ref(x, b, approx)             # fp32 cancels in the negative tail: compare outside it
        fp32 = O.bias_gelu(pre.float(), None, approx).to(BF)
        assert float(((ref.r.to(BF) != fp32) & ~ref.skip).double().mean()) < 1e-2
        pg = x.double().requires_grad_(True)
        F.gelu(pg, approximate=approx).backward(dh.double())
        torch.testing.assert_close(gelu_bwd_ref(x, dh, approx).r, pg.grad, rtol=1e-10, atol=1e-13)
    y, ls = randn_bf16((64, 512), g), randn_bf16((512,), g)
    assert torch.equal(ls_residual_ref(x, y, ls, b).r.to(BF), O.ls_residual(x, y, ls, b))
    yg, lg = y.double().requires_grad_(True), ls.double().requires_grad_(True)
    (x.double() + yg * lg).backward(dh.double())
    dy, dls = ls_residual_bwd_ref(dh, y, ls)
    torch.testing.assert_close(dy.r, yg.grad, rtol=0, atol=0)
    torch.testing.assert_close(dls.r, lg.grad, rtol=1e-12, atol=1e-12)
    # RoPE: bit-exact with the oracle; the backward is the float64 autograd of the unrounded rotation
    t = randn_bf16((100, 6, 64), g)
    pos = torch.randint(0, 1 << 17, (100,), generator=g)
    inv = O.rope_inv_freq(64, 1e6)
    cos, sin = O.rope_tables(pos, inv)
    assert torch.equal(rope_ref(t, cos, sin).r.to(BF), O.rope_apply(t, cos, sin))
    tg, dyr = t.double().requires_grad_(True), randn_bf16((100, 6, 64), g)
    O.rope_apply(tg, cos.double(), sin.double()).backward(dyr.double())
    torch.testing.assert_close(rope_bwd_ref(dyr, cos, sin).r, tg.grad, rtol=1e-14, atol=0)
    rc, rs = rope_table_ref(pos, inv)
    ang = (pos.float()[:, None] * inv[None]).double()
    assert torch.equal(rc.r, ang.cos()) and torch.equal(rs.r, ang.sin())
    assert float((rc.r.to(BF) != cos[:, :32]).double().mean()) < 2e-3


def test_decode_merge_reference():
    g = seeded(5)
    n, G, hkv, d = 7, 5, 2, 64
    o = randn_bf16((n, G, hkv, d), g)
    lse = torch.rand((n, hkv, G), generator=g) * 160 - 80
    lse[3] = -math.inf
    lse[:, 1, 4] = -math.inf
    ref, L, bound = decode_merge_ref(o, lse)
    l = lse.double().permute(1, 2, 0).reshape(hkv * G, n)
    p = torch.softmax(l, -1)
    want = torch.einsum("hs,shd->hd", p, o.double().permute(0, 2, 1, 3).reshape(n, hkv * G, d))
    h = 1 * G + 4                                               # the all -inf head
    keep = torch.arange(hkv * G) != h
    torch.testing.assert_close(ref.r[keep], want[keep], rtol=1e-12, atol=1e-12)
    assert not bool(ref.r[h].any()) and bool(torch.isneginf(L[h])) and bool((bound[keep] > 0).all())
    torch.testing.assert_close(L[keep], torch.logsumexp(l, -1)[keep], rtol=1e-14, atol=0)


def test_slabbing_does_not_change_the_reductions():
    x, w, _, dy, a = _norm_inputs(300, 256, seed=6)
    whole = [rmsnorm_dw_ref(x, w, dy, 1e-6), *layernorm_dwdb_ref(x, w, dy, 1e-6), ls_residual_bwd_ref(dy, x, w)[1]]
    slabbed = [rmsnorm_dw_ref(x, w, dy, 1e-6, slab_bytes=8 * 4 * 256 * 7),
               *layernorm_dwdb_ref(x, w, dy, 1e-6, slab_bytes=8 * 6 * 256 * 5),
               ls_residual_bwd_ref(dy, x, w, slab_bytes=8 * 2 * 256 * 3)[1]]
    for p, q in zip(whole, slabbed):
        torch.testing.assert_close(q.r, p.r, rtol=1e-13, atol=1e-13)
        torch.testing.assert_close(q.d, p.d, rtol=1e-12, atol=1e-300)
    # the dx references are row-independent: a slab of rows gives the same rows of the whole
    for ref in (rmsnorm_bwd_ref, layernorm_bwd_ref):
        torch.testing.assert_close(ref(x[100:170], w, dy[100:170], 1e-6, a[100:170]).r, ref(x, w, dy, 1e-6, a).r[100:170],
                                   rtol=0, atol=0)


# ------------------------------------------------------------------------------------------------
# acceptance: bf16(r) and fp32 emulations of the kernels
# ------------------------------------------------------------------------------------------------
def test_checker_accepts_the_rounded_reference_and_fp32_emulations():
    x, w, b, dy, a = _norm_inputs()
    ref = rmsnorm_ref(x, w, 1e-6)
    res = check_tokenwise(ref.r.to(BF), *ref)
    assert res["flip_frac"] == 0 and res["max_ulps"] <= 1.0
    _chk("rmsnorm", emu_rmsnorm(x, w, 1e-6), ref)
    xs = (x.float() * 1e-3).to(BF)
    _chk("rmsnorm", emu_rmsnorm(xs, w, 1e-6), rmsnorm_ref(xs, w, 1e-6))
    xm, *_ = _norm_inputs(seed=7, scale=0.5, mean=40.0)
    for op, xx in (("layernorm", x), ("layernorm_offset", xm)):
        _chk(op, emu_layernorm(xx, w, b, 1e-6), layernorm_ref(xx, w, b, 1e-6))
    dx, dw = emu_rmsnorm_bwd(x, w, dy, 1e-6, a)
    rdx, rdw = rmsnorm_bwd_ref(x, w, dy, 1e-6, a), rmsnorm_dw_ref(x, w, dy, 1e-6)
    _chk("rmsnorm_bwd", dx, rdx)
    _chk("norm_dw", dw, rdw)
    xg = xm.float().requires_grad_(True)
    wg, bg = w.float().requires_grad_(True), b.float().requires_grad_(True)
    F.layer_norm(xg, (COLS,), wg, bg, 1e-6).backward(dy.float())
    rdx, (rdw, rdb) = layernorm_bwd_ref(xm, w, dy, 1e-6), layernorm_dwdb_ref(xm, w, dy, 1e-6)
    _chk("layernorm_bwd", xg.grad.to(BF), rdx)
    _chk("norm_dw", wg.grad.to(BF), rdw)
    _chk("norm_dw", bg.grad.to(BF), rdb)
    g = seeded(8)
    gu, dh = randn_bf16((64, 2 * 2048), g, 2.0), randn_bf16((64, 2048), g)
    _chk("swiglu", emu_swiglu(gu), swiglu_ref(gu))
    gf = gu.float().requires_grad_(True)
    O.swiglu(gf).backward(dh.float())
    _chk("swiglu_bwd", gf.grad.to(BF), swiglu_bwd_ref(gu, dh))
    xa = randn_bf16((64, 2048), g, 3.0)
    for approx in ("none", "tanh"):
        _chk("gelu", F.gelu(xa.float(), approximate=approx).to(BF), bias_gelu_ref(xa, None, approx))
        xf = xa.float().requires_grad_(True)
        F.gelu(xf, approximate=approx).backward(dh.float())
        _chk("gelu_bwd", xf.grad.to(BF), gelu_bwd_ref(xa, dh, approx))
    t = randn_bf16((64, 8, 128), g)
    cos, sin = O.rope_tables(torch.arange(64) * 1000, O.rope_inv_freq(128, 1e6))
    _chk("exact", emu_rope(t, cos, sin), rope_ref(t, cos, sin))
    dyr = randn_bf16((64, 8, 128), g)
    _chk("rope_bwd", emu_rope(dyr, cos, -sin), rope_bwd_ref(dyr, cos, sin))
    o = randn_bf16((150, 5, 8, 128), g)
    lse = torch.rand((150, 8, 5), generator=g) * 160 - 80
    ref, _, _ = decode_merge_ref(o, lse)
    _chk("decode_merge", emu_decode_merge(o, lse), ref)


def test_checker_demands_bit_exactness_where_the_kernel_is_exact():
    t = randn_bf16((16, 8, 64), seeded(9))
    cos, sin = O.rope_tables(torch.arange(16), O.rope_inv_freq(64, 1e6))
    y = emu_rope(t, cos, sin)
    y.view(-1)[77] = (y.view(-1)[77].float() * (1 + 2 ** -7)).to(BF)   # one element one ulp off
    with pytest.raises(AssertionError, match="elementwise|flip"):
        _chk("exact", y, rope_ref(t, cos, sin))


# ------------------------------------------------------------------------------------------------
# rejections: each wrong result is built on the CPU from correct data
# ------------------------------------------------------------------------------------------------
REJECT = "flip fraction|flipped roundings|elementwise"


@pytest.mark.parametrize("mutation", ["drop_last_vector", "cols_minus_8"])
def test_rejects_an_rmsnorm_statistic_off_by_one_vector(mutation):
    x, w, *_ = _norm_inputs()
    kw = {"drop_last": True} if mutation == "drop_last_vector" else {"div": COLS - 8}
    with pytest.raises(AssertionError, match=REJECT):
        _chk("rmsnorm", emu_rmsnorm(x, w, 1e-6, **kw), rmsnorm_ref(x, w, 1e-6))


def test_rejects_a_one_pass_variance_on_mean_offset_rows():
    x, w, b, *_ = _norm_inputs(seed=7, scale=0.5, mean=40.0)
    with pytest.raises(AssertionError, match=REJECT):
        _chk("layernorm_offset", emu_layernorm(x, w, b, 1e-6, one_pass=True), layernorm_ref(x, w, b, 1e-6))


def _edge_inputs(cols, seed):
    g = seeded(seed)
    x = edge_rows(cols, lambda shape, scale, mean: (torch.randn(shape, generator=g) * scale + mean).to(BF), "cpu")
    w = (1 + 0.1 * torch.randn(cols, generator=g)).to(BF)
    return x, w, randn_bf16((cols,), g, 0.1)


@pytest.mark.parametrize("cols", [1024, 5120])
@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_edge_rows_tell_a_one_pass_variance_from_the_two_pass_one(cols, seed):
    """The GPU's edge-row layout, each group checked as a tensor of its own with its own limits: the two-pass fp32
    LayerNorm passes on every group, the one-pass one is rejected on the mean-offset rows."""
    x, w, b = _edge_inputs(cols, seed)
    for eps in (1e-6, 1e-5):
        good, bad = emu_layernorm(x, w, b, eps), emu_layernorm(x, w, b, eps, one_pass=True)
        for group, sl in edge_groups():
            _chk(edge_op("layernorm", group), good[sl], layernorm_ref(x[sl], w, b, eps), f"layernorm {group}")
        sl = dict(edge_groups())["offset"]
        with pytest.raises(AssertionError, match=REJECT):
            _chk(edge_op("layernorm", "offset"), bad[sl], layernorm_ref(x[sl], w, b, eps))


@pytest.mark.parametrize("cols", [1024, 5120, 16384])
def test_rejects_one_rmsnorm_row_with_the_cols_minus_8_divisor(cols):
    """One wrong row among 64 correct ones is rejected: 4 % (16 384 columns) to 66 % (1024) of its roundings flip.
    The rows have scale 3: with rstd close to 1, s rstd lies within about one bf16 ulp of s, and an rstd off by
    2.4e-4 (cols - 8 at 16 384 columns) can leave every product on its side of the ties."""
    x, w, *_ = _norm_inputs(rows=64, cols=cols, seed=13, scale=3.0)
    y = emu_rmsnorm(x, w, 1e-6)
    y[37] = emu_rmsnorm(x[37:38], w, 1e-6, div=cols - 8)[0]
    with pytest.raises(AssertionError, match=REJECT):
        _chk("rmsnorm", y, rmsnorm_ref(x, w, 1e-6))


def test_rejects_eps_ignored_on_small_rows():
    x, w, *_ = _norm_inputs(scale=1e-3)
    with pytest.raises(AssertionError, match=REJECT):
        _chk("rmsnorm", emu_rmsnorm(x, w, 0.0), rmsnorm_ref(x, w, 1e-6))


def test_rejects_dw_missing_one_ctas_partial_row():
    x, w, _, dy, _ = _norm_inputs(rows=2112)
    _, dw = emu_rmsnorm_bwd(x, w, dy, 1e-6, parts=264, drop_part=100)
    with pytest.raises(AssertionError, match=REJECT):
        _chk("norm_dw", dw, rmsnorm_dw_ref(x, w, dy, 1e-6))


def test_rejects_one_output_row_shifted():
    x, w, *_ = _norm_inputs()
    y = emu_rmsnorm(x, w, 1e-6)
    y[200] = y[201]
    with pytest.raises(AssertionError, match=REJECT):
        _chk("rmsnorm", y, rmsnorm_ref(x, w, 1e-6))


@pytest.mark.parametrize("mutation", [{"swap_halves": True}, {"sin_sign": -1.0}])
def test_rejects_rope_halves_swapped_or_sin_of_the_wrong_sign(mutation):
    t = randn_bf16((64, 8, 128), seeded(10))
    cos, sin = O.rope_tables(torch.arange(64) * 37, O.rope_inv_freq(128, 1e6))
    with pytest.raises(AssertionError, match=REJECT):
        _chk("exact", emu_rope(t, cos, sin, **mutation), rope_ref(t, cos, sin))


def test_rejects_swiglu_gate_and_up_swapped():
    gu = randn_bf16((64, 2 * 1024), seeded(11), 2.0)
    with pytest.raises(AssertionError, match=REJECT):
        _chk("swiglu", emu_swiglu(gu, swap=True), swiglu_ref(gu))


def test_rejects_a_decode_merge_that_skips_one_split():
    g = seeded(12)
    o = randn_bf16((150, 5, 8, 128), g)
    lse = torch.randn((150, 8, 5), generator=g)                # comparable splits: each weighs about 1 / 150
    ref, _, _ = decode_merge_ref(o, lse)
    with pytest.raises(AssertionError, match=REJECT):
        _chk("decode_merge", emu_decode_merge(o, lse, skip=77), ref)


def test_check_untouched():
    buf = torch.full((4, 6, 24), 7.0, dtype=BF)
    view = buf[:, 1:5, 8:16]
    view.fill_(1)
    check_untouched(buf, view, 7.0)
    buf[3, 5, 0] = 0
    with pytest.raises(AssertionError, match="outside the view"):
        check_untouched(buf, view, 7.0)


def test_flip_limits_cover_every_op_the_tests_name():
    assert flip_limits("exact", 1024) == {"flip_frac": 0.0, "flip_row": 0}
    for op, (frac, row) in FLIPS.items():
        assert op == "rope_bwd" or (0 <= frac <= 0.05 and 0 <= row <= 0.1), op


def test_near_tie():
    from tests.tokenwise_ref import near_tie

    v = torch.tensor([1.0 + 2.0 ** -8, 1.0 + 2.0 ** -8 + 2.0 ** -22, 1.0 + 2.0 ** -8 + 2.0 ** -17, 1.0, -3.0 - 2.0 ** -7],
                     dtype=torch.float64)
    assert near_tie(v).tolist() == [True, True, False, False, True]
