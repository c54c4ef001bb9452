"""GPU parity: token-wise operators through the C ABI vs the CPU oracle on identical bf16 inputs.
Permutation / index operators must be bit-exact; arithmetic operators are compared against the
oracle evaluated in bf16 (the reference's eager sequence) and must agree to 1e-3 relative
Frobenius error with at most a small fraction of 1-ulp differences."""
import pytest
import torch

from oracle import ops as O
from tests.util import mismatch_fraction, randn_bf16, rel_fro, seeded

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L(lib_built):
    from long_vita_b200 import ops

    return ops


@pytest.mark.parametrize("rows,cols", [(1, 5120), (37, 5120), (300, 1024), (64, 4096), (5, 1152), (3, 8192)])
def test_rmsnorm(L, rows, cols):
    g = seeded(1)
    x, w = randn_bf16((rows, cols), g), (1 + 0.1 * torch.randn(cols, generator=g)).to(torch.bfloat16)
    y = L.rmsnorm(x.cuda(), w.cuda(), 1e-6)
    ref = O.rmsnorm(x, w, 1e-6)
    assert rel_fro(y, ref) < 1e-3 and mismatch_fraction(y, ref) < 0.01


def test_rmsnorm_fused_residual(L):
    g = seeded(2)
    x, r, w = randn_bf16((130, 5120), g), randn_bf16((130, 5120), g), randn_bf16((5120,), g)
    y, s = L.rmsnorm(x.cuda(), w.cuda(), 1e-6, residual=r.cuda())
    s_ref = x + r
    assert torch.equal(s.cpu(), s_ref)
    ref = O.rmsnorm(s_ref, w, 1e-6)
    assert rel_fro(y, ref) < 1e-3 and mismatch_fraction(y, ref) < 0.01


@pytest.mark.parametrize("rows,cols,eps", [(1025 * 2, 1024, 1e-6), (256, 4096, 1e-5), (7, 1152, 1e-6), (37, 5120, 1e-6),
                                          (3, 8192, 1e-6)])
def test_layernorm(L, rows, cols, eps):
    g = seeded(3)
    x = randn_bf16((rows, cols), g)
    w, b = randn_bf16((cols,), g), randn_bf16((cols,), g, 0.1)
    y = L.layernorm(x.cuda(), w.cuda(), b.cuda(), eps)
    ref = O.layernorm(x, w, b, eps)
    assert rel_fro(y, ref) < 1e-3 and mismatch_fraction(y, ref) < 0.01


def test_rope_table_and_apply(L):
    g = seeded(4)
    n, hq, hkv, d = 515, 40, 8, 128
    pos = torch.cat([torch.arange(0, 300), torch.arange(1_000_000, 1_000_000 + n - 300)]).to(torch.int64)
    inv = O.rope_inv_freq(d, 1e6)
    cos, sin = L.rope_table(pos.cuda(), inv.cuda())
    cos_r, sin_r = O.rope_tables(pos, inv)
    # libm sincosf vs torch differ by <= 2 ulp fp32, so a bf16 rounding boundary is rarely crossed
    assert mismatch_fraction(cos, cos_r) < 2e-3 and mismatch_fraction(sin, sin_r) < 2e-3
    assert rel_fro(cos, cos_r) < 1e-4
    # apply on a strided view of a fused qkv buffer [n, hkv, (5 q + k + v), d] as Megatron lays it out
    qkv = randn_bf16((n, hkv, 7, d), g)
    q = qkv[:, :, :5].reshape(n, hq, d)            # copy (non-viewable), like Megatron's reshape
    k = qkv[:, :, 5]                               # strided view
    qg, kg = q.cuda(), qkv.cuda()[:, :, 5]
    oq = L.rope(qg, cos_r.cuda(), sin_r.cuda())
    ok = L.rope(kg, cos_r.cuda(), sin_r.cuda())
    assert torch.equal(oq.cpu(), O.rope_apply(q, cos_r, sin_r))
    assert torch.equal(ok.cpu(), O.rope_apply(k, cos_r, sin_r))


def test_rope_kernel_reproduces_the_references_megatron_rope_bit_exactly(L):
    """lv_rope on the angles' bf16 cos / sin against the committed output of the reference's own
    apply_rotary_pos_emb_bshd (tests/golden/ref_megatron_rope.pt, generated from /root/reference)."""
    import os
    import sys

    gold_dir = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    sys.path.insert(0, gold_dir)
    from make_golden import rope_golden_input

    gold = torch.load(os.path.join(gold_dir, "ref_megatron_rope.pt"))
    t = rope_golden_input()[:, 0]                                   # [S, heads, 128]
    ang = gold["emb"].view(gold["S"], 128)
    cos, sin = torch.cos(ang).to(torch.bfloat16), torch.sin(ang).to(torch.bfloat16)     # :200-201
    out = L.rope(t.cuda(), cos.cuda(), sin.cuda())
    assert torch.equal(out.cpu(), gold["applied"][:, 0])


def test_swiglu(L):
    g = seeded(5)
    gu = randn_bf16((77, 2 * 13824), g, 2.0)
    y = L.swiglu(gu.cuda())
    ref = O.swiglu(gu)
    assert rel_fro(y, ref) < 1e-3 and mismatch_fraction(y, ref) < 0.01


@pytest.mark.parametrize("approx", ["none", "tanh"])
def test_bias_gelu(L, approx):
    g = seeded(6)
    x, b = randn_bf16((129, 4096), g, 2.0), randn_bf16((4096,), g)
    y = L.bias_gelu(x.cuda(), b.cuda(), approx)
    ref = O.bias_gelu(x, b, approx)
    # 1 + erf(x / sqrt 2) cancels catastrophically in the far negative tail (|gelu| < 1e-5 there), so
    # libm-vs-libdevice ulp differences flip bf16 roundings of those tiny values: bound the error
    # in norm and absolutely instead of counting flipped elements
    assert rel_fro(y, ref) < 1e-3
    assert float((y.float().cpu() - ref.float()).abs().max()) < 2e-2 * float(ref.float().abs().max()) * 2 ** -7


def test_ls_residual(L):
    g = seeded(7)
    x, y, ls, b = randn_bf16((1025, 1024), g), randn_bf16((1025, 1024), g), randn_bf16((1024,), g), randn_bf16((1024,), g)
    out = L.ls_residual(x.cuda(), y.cuda(), ls.cuda(), b.cuda())
    assert torch.equal(out.cpu(), O.ls_residual(x, y, ls, b))
    out = L.ls_residual(x.cuda(), y.cuda())
    assert torch.equal(out.cpu(), x + y)


def test_pixel_shuffle_bit_exact(L):
    g = seeded(8)
    n, hw, c = 3, 32, 1024
    x = randn_bf16((n, 1 + hw * hw, c), g)
    out = L.pixel_shuffle(x.cuda(), hw, has_cls=True)
    ref = O.pixel_shuffle_half(x[:, 1:].reshape(n, hw, hw, c)).reshape(n, -1, 4 * c)
    assert torch.equal(out.cpu(), ref)
    out = L.pixel_shuffle(x[:, 1:].contiguous().cuda(), hw, has_cls=False)
    assert torch.equal(out.cpu(), ref)


def test_embed_scatter_bit_exact(L):
    g = seeded(9)
    vocab, hidden, n_tok, n_img = 1000, 5120, 2048, 3
    table = randn_bf16((vocab, hidden), g)
    ids = torch.randint(0, vocab, (n_tok,), generator=g)
    feat = randn_bf16((n_img, 256, hidden), g)
    dst = torch.stack([torch.arange(10 + i * 300, 10 + i * 300 + 256) for i in range(n_img)]).view(-1)
    out = L.embed_scatter(ids.cuda(), table.cuda(), feat.cuda(), dst.cuda())
    assert torch.equal(out.cpu(), O.embed_scatter(ids, table, feat, dst))
    # src/tgt index mode used under context parallelism (language_model_embedding.py:127-130)
    src = torch.randperm(n_img * 256, generator=g)[:200]
    dst2 = torch.randperm(n_tok, generator=g)[:200]
    out = L.embed_scatter(ids.cuda(), table.cuda(), feat.cuda(), dst2.cuda(), src.cuda())
    assert torch.equal(out.cpu(), O.embed_scatter(ids, table, feat, dst2, src))
    # no features at all
    out = L.embed_scatter(ids.cuda(), table.cuda())
    assert torch.equal(out.cpu(), table[ids])


def test_row_gather_scatter_bit_exact(L):
    g = seeded(10)
    x = randn_bf16((4096, 5120), g)
    mask = torch.rand(4096, generator=g) < 0.1
    idx = mask.nonzero().view(-1)
    sel = L.row_gather(x.cuda(), idx.cuda())
    assert torch.equal(sel.cpu(), x[mask])
    back = L.row_scatter_zero(sel, idx.cuda(), 4096)
    ref = torch.zeros_like(x)
    ref[mask] = x[mask]
    assert torch.equal(back.cpu(), ref)
    empty = L.row_gather(x.cuda(), idx[:0].cuda())
    assert empty.shape == (0, 5120)


def test_rmsnorm_backward(L):
    g = seeded(31)
    for rows, cols in ((300, 5120), (77, 640), (1000, 1024), (129, 2048), (33, 8192)):
        x, dy = randn_bf16((rows, cols), g, 2.0), randn_bf16((rows, cols), g)
        w = (1 + 0.1 * torch.randn(cols, generator=g)).to(torch.bfloat16)
        add = randn_bf16((rows, cols), g)
        xf, wf = x.float().requires_grad_(True), w.float().requires_grad_(True)
        (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-6) * wf).backward(dy.float())
        dx, dw = L.rmsnorm_bwd(x.cuda(), w.cuda(), dy.cuda(), 1e-6)
        assert rel_fro(dx, xf.grad) < 4e-3 and rel_fro(dw, wf.grad) < 4e-3, (rows, cols, rel_fro(dx, xf.grad), rel_fro(dw, wf.grad))
        dx2, _ = L.rmsnorm_bwd(x.cuda(), w.cuda(), dy.cuda(), 1e-6, add_in=add.cuda())
        assert rel_fro(dx2, xf.grad + add.float()) < 4e-3
    # through the autograd function, fused residual form
    x, r = randn_bf16((64, 640), g).cuda().requires_grad_(True), randn_bf16((64, 640), g).cuda().requires_grad_(True)
    w = torch.ones(640, dtype=torch.bfloat16, device="cuda", requires_grad=True)
    y, s = L.rmsnorm_autograd(x, w, 1e-6, residual=r)
    (y.float().sum() + 2 * s.float().sum()).backward()
    assert torch.equal(x.grad, r.grad) and x.grad.shape == x.shape and w.grad.shape == w.shape


def test_swiglu_backward(L):
    g = seeded(32)
    gu, dh = randn_bf16((257, 2 * 1024), g, 2.0), randn_bf16((257, 1024), g)
    guf = gu.float().requires_grad_(True)
    O.swiglu(guf).backward(dh.float())
    d = L.swiglu_bwd(gu.cuda(), dh.cuda())
    assert rel_fro(d, guf.grad) < 4e-3, rel_fro(d, guf.grad)


def test_linear_and_rope_autograd(L):
    g = seeded(33)
    x, w, b = randn_bf16((203, 640), g), randn_bf16((384, 640), g, 0.05), randn_bf16((384,), g)
    dy = randn_bf16((203, 384), g)
    xg, wg, bg = (t.cuda().requires_grad_(True) for t in (x, w, b))
    L.linear_autograd(xg, wg, bg).backward(dy.cuda())
    xf, wf, bf_ = (t.float().requires_grad_(True) for t in (x, w, b))
    (xf @ wf.t() + bf_).backward(dy.float())
    assert rel_fro(xg.grad, xf.grad) < 3e-3 and rel_fro(wg.grad, wf.grad) < 3e-3 and rel_fro(bg.grad, bf_.grad) < 3e-3
    t = randn_bf16((128, 5, 128), g)
    inv = O.rope_inv_freq(128, 1e6)
    cos, sin = O.rope_tables(torch.arange(128), inv, torch.bfloat16)
    tg = t.cuda().requires_grad_(True)
    dyr = randn_bf16((128, 5, 128), g)
    L.rope_autograd(tg, cos.cuda(), sin.cuda()).backward(dyr.cuda())
    tf = t.float().requires_grad_(True)
    O.rope_apply(tf, cos.float(), sin.float()).backward(dyr.float())
    assert rel_fro(tg.grad, tf.grad) < 4e-3
