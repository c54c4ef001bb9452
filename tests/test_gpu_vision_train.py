"""GPU parity of the vision-side training path: the backward kernels of the ViT / projector operators against fp32
autograd, the ViT attention backward into one dQKV buffer, and the whole trainable tower + projector
(`B200VisionModel`) against fp32 autograd of the oracle at the tiny and at the real InternViT-300M geometry.
Tolerances: token-wise backward 1e-3 relative Frobenius (DESIGN §2), attention the excess bound of
tests/test_gpu_attention_bwd.py, the composed model 8e-3 on features and 1e-2 on every parameter gradient or 1.25x
the error of eager bf16 autograd where that is larger (see the test)."""
import math

import pytest
import torch
import torch.nn.functional as F

from long_vita_b200.config import LongVITAConfig
from long_vita_b200.megatron import checkpoint as CK
from long_vita_b200.weights import global_weights, vit_layer_weights
from oracle import model as OM
from oracle import ops as O
from tests.util import randn_bf16, rel_fro, seeded

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L(lib_built):
    from long_vita_b200 import ops

    return ops


def r16(out, ref):
    """Relative Frobenius error against the fp32 oracle rounded once to bf16, the dtype of the result (DESIGN §2: a
    bf16 rounding of any result alone costs ~1.6e-3 against the unrounded value)."""
    return rel_fro(out, ref.to(torch.bfloat16))


def excess(out, ref):
    e, f = rel_fro(out, ref), rel_fro(ref.to(torch.bfloat16), ref)
    return math.sqrt(max(e * e - f * f, 0.0))


# ------------------------------------------------------------------------------------------------
# single operators
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("has_cls", [True, False])
def test_pixel_shuffle_bwd_inverts_forward_bit_exact(L, has_cls):
    g = seeded(1)
    x = randn_bf16((3, 32 * 32 + (1 if has_cls else 0), 1024), g).cuda()
    dx = L.pixel_shuffle_bwd(L.pixel_shuffle(x, 32, has_cls), 32, has_cls)
    assert dx.shape == x.shape
    if has_cls:
        assert torch.equal(dx[:, 1:], x[:, 1:]) and torch.equal(dx[:, 0], torch.zeros_like(x[:, 0]))
    else:
        assert torch.equal(dx, x)


def test_patch_im2col_matches_unfold_bit_exact(L):
    g = seeded(2)
    images = randn_bf16((2, 3, 448, 448), g)
    col = L.patch_im2col(images.cuda(), 14, 640).cpu()
    ref = F.unfold(images.float(), 14, stride=14).transpose(1, 2).reshape(2 * 1024, 588).to(torch.bfloat16)
    assert torch.equal(col[:, :588], ref) and not col[:, 588:].any()


@pytest.mark.parametrize("rows,cols,eps,with_add", [(2 * 1025, 1024, 1e-6, True), (2 * 1025, 1024, 1e-6, False),
                                                    (512, 4096, 1e-5, False), (37, 4096, 1e-5, True), (3, 8192, 1e-6, False)])
def test_layernorm_bwd(L, rows, cols, eps, with_add):
    g = seeded(rows + cols)
    x = randn_bf16((rows, cols), g, 2.0) + 0.5
    w = (1 + 0.2 * torch.randn(cols, generator=g)).to(torch.bfloat16)
    b = randn_bf16((cols,), g, 0.1)
    dy = randn_bf16((rows, cols), g)
    add = randn_bf16((rows, cols), g) if with_add else None
    xf, wf, bf = (t.float().requires_grad_(True) for t in (x, w, b))
    F.layer_norm(xf, (cols,), wf, bf, eps).backward(dy.float())
    ref_dx = xf.grad + (add.float() if with_add else 0)
    dx, dw, db = L.layernorm_bwd(x.cuda(), w.cuda(), dy.cuda(), eps, add_in=None if add is None else add.cuda())
    assert r16(dx, ref_dx) < 1e-3, r16(dx, ref_dx)
    assert r16(dw, wf.grad) < 1e-3 and r16(db, bf.grad) < 1e-3, (r16(dw, wf.grad), r16(db, bf.grad))
    if not with_add:                      # weight / bias gradients only: the same partial sums, no dx written
        none, dw2, db2 = L.layernorm_bwd(x.cuda(), w.cuda(), dy.cuda(), eps, need_dx=False)
        assert none is None and torch.equal(dw2, dw) and torch.equal(db2, db)


@pytest.mark.parametrize("approximate", ["none", "tanh"])
def test_gelu_bwd(L, approximate):
    g = seeded(3)
    pre, dy = randn_bf16((2 * 1025, 4096), g, 2.0), randn_bf16((2 * 1025, 4096), g)
    pf = pre.float().requires_grad_(True)
    F.gelu(pf, approximate=approximate).backward(dy.float())
    dx = L.gelu_bwd(pre.cuda(), dy.cuda(), approximate)
    assert r16(dx, pf.grad) < 1e-3, r16(dx, pf.grad)


@pytest.mark.parametrize("rows,cols", [(4 * 1025, 1024), (5, 1024), (300, 640)])
def test_ls_residual_bwd(L, rows, cols):
    g = seeded(rows)
    dout, y, ls = randn_bf16((rows, cols), g), randn_bf16((rows, cols), g), randn_bf16((cols,), g, 0.3)
    dy, dls = L.ls_residual_bwd(dout.cuda(), y.cuda(), ls.cuda())
    assert r16(dy, dout.float() * ls.float()) < 1e-3
    ref = (dout.float() * y.float()).sum(0)
    assert r16(dls, ref) < 1e-3, r16(dls, ref)


def test_vit_attention_backward_into_one_dqkv_buffer(L):
    """4 frames of the ViT geometry (16 heads x 64, S = 1025): q / k / v are strided views of the QKV GEMM output in
    Megatron's [H, 3, D] column order, and their gradients land in one buffer through the same strides."""
    g = seeded(4)
    n, S, H, D = 4, 1025, 16, 64
    qkv = randn_bf16((n, S, 3 * H * D), g)
    do = randn_bf16((n, S, H * D), g)
    v5 = qkv.view(n, S, H, 3, D)
    rq, rk, rv = O.attention_grads(v5[:, :, :, 0], v5[:, :, :, 1], v5[:, :, :, 2], do.view(n, S, H, D), causal=False)
    x = qkv.cuda().requires_grad_(True)
    out = L.vit_attention(x, H, D ** -0.5)
    assert out.shape == (n, S, H * D)
    out.backward(do.cuda())
    g5 = x.grad.view(n, S, H, 3, D)
    for name, a, r in (("dq", g5[:, :, :, 0], rq), ("dk", g5[:, :, :, 1], rk), ("dv", g5[:, :, :, 2], rv)):
        assert torch.isfinite(a).all(), name
        assert excess(a, r) < 3e-3, (name, excess(a, r))


# ------------------------------------------------------------------------------------------------
# the whole tower + projector
# ------------------------------------------------------------------------------------------------
def _weights(cfg, seed, layer_scale=None):
    """Synthetic weights (perturbed biases / norms).  `layer_scale` resets ls1 / ls2 to that value with 10 % jitter (the
    synthetic default is ~1)."""
    w = global_weights(cfg, seed, "cpu", torch.float32, perturb=True, with_lm=False)
    for i in range(cfg.visual.num_hidden_layers):
        w.update(vit_layer_weights(cfg, i, seed, "cpu", torch.float32, perturb=True))
    if layer_scale is not None:
        g = seeded(seed + 1)
        for k in w:
            if k.endswith((".ls1", ".ls2")):
                w[k] = layer_scale * (1 + 0.1 * torch.randn(w[k].shape, generator=g))
    return {k: t.to(torch.bfloat16) for k, t in w.items()}


def _model(cfg, w, **flags):
    from long_vita_b200.megatron.vision_model import B200VisionModel

    m = B200VisionModel(cfg.hidden_size, cfg.visual, device="cuda", **flags)
    m.load_state_dict({k[len(CK.EFM):]: t for k, t in CK.hf_to_mcore(w, cfg).items()}, strict=True)
    return m


def _oracle(cfg, w, images, d_out):
    """fp32 autograd of oracle.model on the GPU (TF32 off) with the same bf16 weights."""
    tf = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        leaves = {k: t.cuda().float().requires_grad_(True) for k, t in w.items()}
        vit = OM.vit_forward(cfg, leaves, images.cuda().float())
        out = OM.projector_forward(cfg, leaves, vit[:, 1:, :])
        out.backward(d_out.cuda().float())
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = tf
    return out.detach(), {k: t.grad for k, t in leaves.items()}


def _eager_bf16(cfg, w, images, d_out):
    """The same oracle autograd in bf16: the eager rounding sequence the reference's own bf16 training executes."""
    leaves = {k: t.cuda().requires_grad_(True) for k, t in w.items()}
    vit = OM.vit_forward(cfg, leaves, images.cuda())
    out = OM.projector_forward(cfg, leaves, vit[:, 1:, :])
    out.backward(d_out.cuda())
    return out.detach(), {k: t.grad for k, t in leaves.items()}


def _run(m, images, d_out):
    out = m(images=images.cuda())
    out.backward(d_out.cuda())
    grads = {CK.EFM + k: p.grad for k, p in m.named_parameters()}
    return out.detach(), grads


@pytest.mark.parametrize("geometry", ["tiny", "internvit_300m"])
def test_tower_and_projector_against_fp32_oracle_autograd(lib_built, geometry):
    """Features <= 8e-3 and every parameter gradient <= 1e-2 relative Frobenius against fp32 autograd, or - where
    bf16 arithmetic itself cannot get that close - within 1.25x of the error of eager bf16 autograd of the same
    oracle on the same inputs (the yardstick flash-attn is for the attention tests).  On the synthetic weights
    (layer scales ~1, N(0, 1) position embeddings) the eager bf16 sequence is at ~1.3e-2 on the 24-layer features and
    up to ~2.5e-2 on token-summed gradients (biases, norm weights, layer scales)."""
    cfg = LongVITAConfig.tiny(layers=1, vit_layers=2) if geometry == "tiny" else LongVITAConfig()
    w = _weights(cfg, seed=77)
    g = seeded(78)
    images = randn_bf16((2, 3, 448, 448), g)
    d_out = randn_bf16((2, 256, cfg.hidden_size), g)
    m = _model(cfg, w)
    out, grads = _run(m, images, d_out)
    hf = CK.mcore_to_hf(grads, cfg)
    del m, grads
    ref_out, ref_grads = _oracle(cfg, w, images, d_out)
    eager_out, eager_grads = _eager_bf16(cfg, w, images, d_out)
    e, floor = rel_fro(out, ref_out), rel_fro(eager_out, ref_out)
    assert e <= max(8e-3, 1.25 * floor), (e, floor)
    assert set(hf) == set(ref_grads)
    bad = {}
    for k in ref_grads:
        e, floor = rel_fro(hf[k], ref_grads[k]), rel_fro(eager_grads[k], ref_grads[k])
        if e > max(1e-2, 1.25 * floor):
            bad[k] = (e, floor)
    assert not bad, bad


def test_tower_and_projector_strict_bounds_at_realistic_layer_scales(lib_built):
    """The composed-model bounds of DESIGN §2 (stated for the tiny geometry) without any allowance: features <= 8e-3
    and every parameter gradient <= 1e-2 relative Frobenius against fp32 autograd, with layer scales ~0.1 (the order
    of a trained InternViT's; the synthetic ~1 above makes every branch as large as the residual stream).  Over the 24
    layers of the real geometry the bf16 residual stream alone costs more than that - eager bf16 autograd of the same
    oracle measures 1.25e-2 on the features and up to 5.5e-2 on token-summed gradients at these scales - so there the
    test above holds this build to that floor instead."""
    cfg = LongVITAConfig.tiny(layers=1, vit_layers=2)
    w = _weights(cfg, seed=91, layer_scale=0.1)
    g = seeded(92)
    images = randn_bf16((2, 3, 448, 448), g)
    d_out = randn_bf16((2, 256, cfg.hidden_size), g)
    m = _model(cfg, w)
    out, grads = _run(m, images, d_out)
    hf = CK.mcore_to_hf(grads, cfg)
    del m, grads
    ref_out, ref_grads = _oracle(cfg, w, images, d_out)
    e = rel_fro(out, ref_out)
    assert e <= 8e-3, e
    errs = {k: rel_fro(hf[k], ref_grads[k]) for k in ref_grads}
    worst = max(errs, key=errs.get)
    assert errs[worst] <= 1e-2, (worst, errs[worst], sorted(errs.values())[-5:])


def test_backward_is_bit_reproducible(lib_built):
    cfg = LongVITAConfig.tiny(layers=1, vit_layers=2)
    w = _weights(cfg, seed=79)
    g = seeded(80)
    images, d_out = randn_bf16((3, 3, 448, 448), g), randn_bf16((3, 256, cfg.hidden_size), g)
    m = _model(cfg, w)
    out1, g1 = _run(m, images, d_out)
    g1 = {k: t.clone() for k, t in g1.items()}
    m.zero_grad(set_to_none=True)
    out2, g2 = _run(m, images, d_out)
    assert torch.equal(out1, out2)
    for k in g1:
        assert torch.equal(g1[k], g2[k]), k


def test_vision_model_freeze_launches_no_vit_backward(L):
    cfg = LongVITAConfig.tiny(layers=1, vit_layers=2)
    w = _weights(cfg, seed=81)
    g = seeded(82)
    images, d_out = randn_bf16((2, 3, 448, 448), g), randn_bf16((2, 256, cfg.hidden_size), g)
    m = _model(cfg, w, vision_model_freeze=True)
    out = m(images=images.cuda())
    torch.cuda.synchronize()
    n0 = L.launch_count()
    out.backward(d_out.cuda())
    torch.cuda.synchronize()
    launches = L.launch_count() - n0
    # projector only: LayerNorm backward, GELU backward, and dX + dW GEMMs of linear_fc1 and linear_fc2
    assert launches == 6, launches
    assert all(p.grad is None for k, p in m.named_parameters() if k.startswith("vit."))
    assert all(p.grad is not None for k, p in m.named_parameters() if not k.startswith("vit."))
