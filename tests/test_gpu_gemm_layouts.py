"""GPU: the wgmma GEMM with MN-major (transposed, read in place) operands, and the backward passes built on it.

Every layout result must be bit-identical to the K-major kernel run on materialised transposed copies (same values,
same k-block order, same zero tails) and within 1e-3 relative Frobenius of an fp32 reference rounded once to bf16.
The backward call sites (`_LinearFn`, `linear_wgrad`, `lm_head_ce_bwd`, the patch-embedding weight gradient) must
give the gradients of the transposed-copy composition they replaced, which is restated here.
"""
import pytest
import torch
import torch.nn.functional as F

from tests.util import randn_bf16, rel_fro, seeded

pytestmark = pytest.mark.gpu

ACTS = {0: None, 1: "gelu", 2: "gelu_tanh", 3: "swiglu"}


@pytest.fixture(scope="module")
def L(lib_built):
    from long_vita_b200 import ops

    return ops


def _operand(t, mn_major, pad):
    """t [rows, K] fp32 -> (bf16 storage, leading dimension) in the requested layout, rows padded by `pad` elements of
    storage (a non-dense leading dimension)."""
    rows, K = t.shape
    if mn_major:
        ld = (rows + 7) // 8 * 8 + pad
        s = torch.zeros((K, ld), dtype=torch.bfloat16, device="cuda")
        s[:, :rows] = t.t()
    else:
        ld = K + pad
        s = torch.zeros((rows, ld), dtype=torch.bfloat16, device="cuda")
        s[:, :K] = t
    return s, ld


def _gemm_ex(a, w, a_mn, w_mn, bias, act, pad):
    from long_vita_b200 import _lib, ops

    M, K = a.shape
    N = w.shape[0]
    sa, lda = _operand(a, a_mn, pad)
    sw, ldw = _operand(w, w_mn, pad)
    n_out = N // 2 if act == 3 else N
    ldc = n_out + pad
    c = torch.full((M, ldc), 7.0, dtype=torch.bfloat16, device="cuda")
    _lib.check(_lib.lib().lv_gemm_ex(sa.data_ptr(), sw.data_ptr(), ops._ptr(bias), c.data_ptr(), M, N, K, lda, ldw, ldc,
                                     int(a_mn), int(w_mn), act, ops._stream()), "lv_gemm_ex")
    if pad:
        assert torch.all(c[:, n_out:] == 7.0), "wrote past the row"
    return c[:, :n_out]


def _kmajor_copy(t):
    """[rows, K] -> contiguous bf16 [rows, K8], K rounded up to a multiple of 8 with zero columns."""
    rows, K = t.shape
    out = torch.zeros((rows, (K + 7) // 8 * 8), dtype=torch.bfloat16, device="cuda")
    out[:, :K] = t
    return out


def _ref(a, w, bias, act):
    y = a.double() @ w.double().t()
    if bias is not None:
        y = y + bias.double()
    if act == 3:
        g, u = y[:, 0::2].to(torch.bfloat16).float(), y[:, 1::2].to(torch.bfloat16).float()
        return (F.silu(g).to(torch.bfloat16).float() * u).to(torch.bfloat16)
    if act:
        y = F.gelu(y.to(torch.bfloat16).float(), approximate="tanh" if act == 2 else "none")
    return y.to(torch.bfloat16)


def _check(L, M, N, K, a_mn, w_mn, act, with_bias, pad, seed):
    g = seeded(seed)
    a = randn_bf16((M, K), g).cuda()
    w = randn_bf16((N, K), g, 1.0 / max(1.0, K ** 0.5)).cuda()
    bias = randn_bf16((N,), g, 0.5).cuda() if with_bias else None
    got = _gemm_ex(a, w, a_mn, w_mn, bias, act, pad)
    ak = _kmajor_copy(a)
    if M <= 4 and (a_mn or w_mn):
        # the MN-major call runs the tensor-core kernel at any M; K-major copies of M <= 4 rows would take the GEMV, so
        # the comparison runs them with zero rows appended (rows are independent in the tensor-core kernel)
        ak = torch.cat([ak, torch.zeros((8 - M, ak.shape[1]), dtype=ak.dtype, device=ak.device)])
    want = L.linear(ak, _kmajor_copy(w), bias, act=ACTS[act])[:M]
    assert torch.equal(got, want), (M, N, K, a_mn, w_mn, act, (got.float() - want.float()).abs().max().item())
    assert rel_fro(got, _ref(a, w, bias, act)) < 1e-3


LAYOUTS = [(False, False), (True, False), (False, True), (True, True)]


@pytest.mark.parametrize("a_mn,w_mn", LAYOUTS)
@pytest.mark.parametrize("K", [1, 7, 63, 64, 1025, 65600])
def test_contraction_lengths(L, a_mn, w_mn, K):
    if (not a_mn or not w_mn) and K % 8:
        K = (K + 7) // 8 * 8          # a K-major operand has rows of whole 16-byte vectors
    _check(L, 300, 520, K, a_mn, w_mn, 0, True, 0, seed=K)


@pytest.mark.parametrize("a_mn,w_mn", LAYOUTS)
@pytest.mark.parametrize("act", [0, 1, 2, 3])
def test_epilogues_with_tails_and_strided_leading_dimensions(L, a_mn, w_mn, act):
    _check(L, 131, 784, 328, a_mn, w_mn, act, act != 3, 24, seed=10 + act)


@pytest.mark.parametrize("a_mn,w_mn", LAYOUTS)
@pytest.mark.parametrize("M", [1, 3, 4])
def test_small_m(L, a_mn, w_mn, M):
    # M <= 4 takes the GEMV path only with both operands K-major; otherwise the tensor-core kernel
    _check(L, M, 1040, 512, a_mn, w_mn, 0, True, 8, seed=M)


def test_ops_linear_reads_transposed_views(L):
    g = seeded(5)
    dy, x, w = randn_bf16((1001, 264), g).cuda(), randn_bf16((1001, 136), g).cuda(), randn_bf16((264, 136), g).cuda()
    assert torch.equal(L.linear(dy, w.t()), L.linear(dy, w.t().contiguous()))
    assert torch.equal(L.linear(dy.t(), x.t()), L.linear(_kmajor_copy(dy.t()), _kmajor_copy(x.t())))


# ------------------------------------------------------------------------------------------------
# backward call sites against the transposed-copy composition they replaced
# ------------------------------------------------------------------------------------------------
def _old_kmajor(t):
    rows, cols = t.shape
    if rows % 8 == 0:
        return t.t().contiguous()
    out = torch.zeros((cols, (rows + 7) // 8 * 8), dtype=t.dtype, device=t.device)
    out[:, :rows] = t.t()
    return out


@pytest.fixture
def old_composition(L, monkeypatch):
    """Within the test, the backward call sites run the previous transposed-copy composition."""

    def linear_wgrad(dy2, x2):
        if dy2.shape[0] == 0:
            return torch.zeros((dy2.shape[1], x2.shape[1]), dtype=dy2.dtype, device=dy2.device)
        return L.linear(_old_kmajor(dy2), _old_kmajor(x2))

    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        n_out, k_in = weight.shape
        dy2 = dy.reshape(-1, n_out).contiguous()
        x2 = x.reshape(-1, k_in)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = L.linear(dy2, _old_kmajor(weight)).view(x.shape)
        if ctx.needs_input_grad[1]:
            dw = linear_wgrad(dy2, x2)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy2.float().sum(dim=0).to(dy2.dtype)
        return dx, dw, db

    def lm_head_ce_bwd(sel, weight, labels, lse, dloss, need_dsel=True, need_dw=False, vocab_chunk=16384):
        M, c = sel.shape
        V = weight.shape[0]
        dsel = torch.zeros((M, c), dtype=torch.float32, device=sel.device) if need_dsel else None
        dw = torch.empty((V, c), dtype=torch.bfloat16, device=sel.device) if need_dw else None
        if M == 0:
            if dw is not None:
                dw.zero_()
            return (None if dsel is None else dsel.to(torch.bfloat16)), dw
        labels, dloss = labels.contiguous(), dloss.contiguous().float()
        chunks = L._ce_chunks(V, vocab_chunk)
        buf = torch.empty((M, chunks[0][1] - chunks[0][0]), dtype=torch.bfloat16, device=sel.device)
        st = _old_kmajor(sel) if need_dw else None
        for v0, v1 in chunks:
            lg = L.ce_grad(L.linear(sel, weight[v0:v1], out=buf[:, : v1 - v0]), labels, lse, dloss, v0)
            if need_dsel:
                dsel += L.linear(lg, _old_kmajor(weight[v0:v1])).float()
            if need_dw:
                L.linear(_old_kmajor(lg), st, out=dw[v0:v1])
        return (None if dsel is None else dsel.to(torch.bfloat16)), dw

    def use():
        monkeypatch.setattr(L, "linear_wgrad", linear_wgrad)
        monkeypatch.setattr(L._LinearFn, "backward", staticmethod(backward))
        monkeypatch.setattr(L, "lm_head_ce_bwd", lm_head_ce_bwd)

    return use


def _grads(fn, leaves):
    for t in leaves:
        t.grad = None
    fn()
    return [None if t.grad is None else t.grad.clone() for t in leaves]


@pytest.mark.parametrize("N,K,with_bias", [(7168, 5120, True), (5120, 5120, False), (27648, 5120, False),
                                           (5120, 13824, False)])
def test_linear_autograd_at_the_decoder_shapes(L, old_composition, N, K, with_bias):
    T = 1037            # a reduced token count, not a multiple of 8
    g = seeded(N + K)
    x = randn_bf16((T, K), g).cuda().requires_grad_(True)
    w = randn_bf16((N, K), g, K ** -0.5).cuda().requires_grad_(True)
    b = randn_bf16((N,), g).cuda().requires_grad_(True) if with_bias else None
    dy = randn_bf16((T, N), g).cuda()
    leaves = [x, w] + ([b] if with_bias else [])
    run = lambda: L.linear_autograd(x, w, b).backward(dy)
    new = _grads(run, leaves)
    old_composition()
    old = _grads(run, leaves)
    for n, o in zip(new, old):
        assert torch.equal(n, o)


@pytest.mark.parametrize("M", [0, 3, 2000])
def test_masked_lm_head_ce_gradients(L, old_composition, M):
    s, c, V = 2500, 5120, 2 * 16384 + 1000
    g = seeded(M + 1)
    h = randn_bf16((s, 1, c), g).cuda().requires_grad_(True)
    w = randn_bf16((V, c), g, c ** -0.5).cuda().requires_grad_(True)
    mask = torch.zeros((1, s), dtype=torch.bool)
    mask[0, torch.randperm(s, generator=g)[:M]] = True
    labels = torch.randint(0, V, (1, M), generator=g)
    if M:
        labels[0, 0] = -1           # one ignored row
    mask, labels = mask.cuda(), labels.cuda()
    dloss = randn_bf16((1, M), g).float().cuda()
    run = lambda: L.masked_lm_head_ce(h, w, mask, labels).backward(dloss)
    new = _grads(run, [h, w])
    old_composition()
    old = _grads(run, [h, w])
    assert torch.equal(new[1], old[1])
    if M <= 4:
        # d_sel of M <= 4 rows: the transposed-copy composition ran the GEMV (a different fp32 summation order), the
        # MN-major weight view runs the tensor-core kernel
        assert rel_fro(new[0], old[0]) < 2e-3
    else:
        assert torch.equal(new[0], old[0])


@pytest.mark.parametrize("freeze", [False, True])
def test_vision_model_gradients(L, old_composition, freeze):
    from long_vita_b200.config import LongVITAConfig
    from tests.test_gpu_vision_train import _model, _run, _weights

    cfg = LongVITAConfig.tiny(layers=1, vit_layers=2)
    w = _weights(cfg, seed=83)
    g = seeded(84)
    images, d_out = randn_bf16((2, 3, 448, 448), g), randn_bf16((2, 256, cfg.hidden_size), g)
    m = _model(cfg, w, vision_model_freeze=freeze)
    out_new, g_new = _run(m, images, d_out)
    g_new = {k: None if t is None else t.clone() for k, t in g_new.items()}
    m.zero_grad(set_to_none=True)
    old_composition()
    out_old, g_old = _run(m, images, d_out)
    assert torch.equal(out_new, out_old)
    assert g_new.keys() == g_old.keys()
    assert any(t is not None for t in g_new.values())
    for k in g_new:
        assert (g_new[k] is None) == (g_old[k] is None), k
        if g_new[k] is not None:
            assert torch.equal(g_new[k], g_old[k]), k
