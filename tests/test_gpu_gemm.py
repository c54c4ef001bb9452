"""GPU parity: wgmma GEMM (+bias, +GELU) and patch embedding vs the CPU oracle."""
import pytest
import torch
import torch.nn.functional as F

from oracle import ops as O
from tests.util import max_rel, randn_bf16, rel_fro, seeded

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L(lib_built):
    from long_vita_b200 import ops

    return ops


def ref_linear(x, w, b=None, act=None):
    y = x.float() @ w.float().t()
    if b is not None:
        y = y + b.float()
    y = y.to(torch.bfloat16)
    if act == "gelu":
        y = F.gelu(y)
    elif act == "gelu_tanh":
        y = F.gelu(y, approximate="tanh")
    return y


@pytest.mark.parametrize(
    "M,N,K",
    [(128, 256, 64), (128, 256, 512), (256, 512, 5120), (1025, 3072, 1024), (300, 1024, 4096), (2, 2048, 5120),
     (1, 256, 5120), (777, 5120, 13824), (2050, 4096, 1024), (64, 1000, 328)],
)
def test_gemm_shapes(L, M, N, K):
    g = seeded(M * 7 + N)
    x, w = randn_bf16((M, K), g), randn_bf16((N, K), g, 0.05)
    y = L.linear(x.cuda(), w.cuda())
    ref = ref_linear(x, w)
    assert y.shape == (M, N)
    assert rel_fro(y, ref) < 1e-3, (rel_fro(y, ref), max_rel(y, ref))


@pytest.mark.parametrize("act", [None, "gelu", "gelu_tanh"])
def test_gemm_bias_act(L, act):
    g = seeded(11)
    M, N, K = 515, 4096, 1024
    x, w, b = randn_bf16((M, K), g), randn_bf16((N, K), g, 0.05), randn_bf16((N,), g)
    y = L.linear(x.cuda(), w.cuda(), b.cuda(), act)
    ref = ref_linear(x, w, b, act)
    assert rel_fro(y, ref) < 1.5e-3, rel_fro(y, ref)


def test_gemm_strided_rows(L):
    g = seeded(12)
    big = randn_bf16((200, 3 * 1024), g)
    w = randn_bf16((512, 1024), g, 0.05)
    xs = big.cuda()[:, 1024:2048]                 # row stride 3072, 16-byte aligned
    y = L.linear(xs, w.cuda())
    assert rel_fro(y, ref_linear(big[:, 1024:2048], w)) < 1e-3


def test_patch_embed(L):
    g = seeded(13)
    n, size, ps, C = 3, 448, 14, 1024
    img = randn_bf16((n, 3, size, size), g)
    w = randn_bf16((C, 3, ps, ps), g, 0.02)
    b = randn_bf16((C,), g, 0.02)
    cls = randn_bf16((1, 1, C), g)
    pos = randn_bf16((1, 1 + (size // ps) ** 2, C), g)
    out = L.patch_embed(img.cuda(), L.pad_patch_weight(w.cuda()), b.cuda(), cls.cuda(), pos.cuda(), ps)
    ref = O.patch_embed(img.float(), w.float(), b.float(), cls.float(), pos.float())
    assert out.shape == ref.shape
    assert rel_fro(out, ref) < 3e-3, rel_fro(out, ref)
    # class-token row is an exact bf16 add
    assert torch.equal(out[:, 0].cpu(), (cls + pos[:, :1]).expand(n, 1, C)[:, 0])


def test_logit_masked_lm_head_forward_and_dgrad(L):
    """a12: masked_select + GEMM (layers.py:402-409) and its input gradient (layers.py:443-451)."""
    g = seeded(14)
    s, c, vocab = 700, 640, 2048
    h = randn_bf16((s, 1, c), g)
    w = randn_bf16((vocab, c), g, 0.05)
    mask = torch.rand(1, s, generator=g) < 0.05
    mask[0, -1] = True
    hg = h.cuda().requires_grad_(True)
    out = L.masked_linear(hg, w.cuda(), mask.cuda())
    ref = O.masked_linear_fwd(h.float(), w.float(), mask)
    assert out.shape == ref.shape
    assert rel_fro(out, ref.to(torch.bfloat16)) < 1e-3          # vs the oracle rounded once to bf16, like the other GEMM tests
    go = randn_bf16(tuple(ref.shape), g)
    out.backward(go.cuda())
    gx = hg.grad
    gx_ref, _ = O.masked_linear_bwd(go.float(), h.float(), w.float(), mask)
    assert gx.shape == (s, 1, c)
    assert rel_fro(gx, gx_ref.to(torch.bfloat16)) < 1e-3
    # rows outside the mask are exactly zero (masked_scatter into zeros)
    assert torch.equal(gx.cpu()[~mask[0]], torch.zeros_like(gx.cpu()[~mask[0]]))


def test_gemm_fused_swiglu_epilogue_is_bit_exact_with_unfused_pair(L):
    g = seeded(15)
    M, H, I = 700, 1024, 2304
    x = randn_bf16((M, H), g)
    gate, up = randn_bf16((I, H), g, 0.05), randn_bf16((I, H), g, 0.05)
    unfused = L.swiglu(L.linear(x.cuda(), torch.cat([gate, up]).cuda()))
    fused = L.linear(x.cuda(), L.interleave_gate_up(gate.cuda(), up.cuda()), act="swiglu")
    assert fused.shape == (M, I)
    assert torch.equal(fused, unfused)
    ref = O.swiglu(ref_linear(x, torch.cat([gate, up])))
    assert rel_fro(fused, ref) < 1.5e-3


@pytest.mark.parametrize("M", [1, 2, 3, 4])
@pytest.mark.parametrize("act", [None, "gelu", "swiglu"])
def test_small_m_weight_stream_path(L, M, act):
    """M <= 4 (decode) runs the HBM-bound GEMV kernel instead of a 128-row tensor-core tile; same epilogue
    arithmetic.  N = 1000 / 1008 and K = 328 exercise the odd-column tail and a K that is not a multiple of
    the 256-element warp stride."""
    g = seeded(50 + M)
    for N, K in ((5120, 5120), (1008 if act == "swiglu" else 1000, 328)):
        x, w = randn_bf16((M, K), g), randn_bf16((N, K), g, 0.05)
        b = None if act == "swiglu" else randn_bf16((N,), g)
        y = L.linear(x.cuda(), w.cuda(), None if b is None else b.cuda(), act)
        if act == "swiglu":
            full = (x.float() @ w.float().t()).to(torch.bfloat16)
            ref = (F.silu(full[:, 0::2].float()).to(torch.bfloat16).float() * full[:, 1::2].float()).to(torch.bfloat16)
            assert y.shape == (M, N // 2)
        else:
            ref = ref_linear(x, w, b, act)
        assert rel_fro(y, ref) < 2e-3, (N, K, rel_fro(y, ref))
