"""Gradient-accumulation fusion (Megatron's `config.gradient_accumulation_fusion`) on a box without a GPU.

Under the CPU oracle forms of the operators (tests/hostlogic.py, tests/vision_oracle.py), with the one new operator,
`ops.linear_wgrad_accumulate`, restated here in float64 and recording its calls: the gradient each autograd function
returns for a weight whose gradient went to `main_grad` (long_vita_megatron/core/tensor_parallel/layers.py:486-518),
the errors for a missing or non-fp32 main_grad, the vocabulary-chunk row slices of the LM head, the patch-embedding
columns, the plumbing of the flag through the three training surfaces, and that with the flag absent or off no surface
calls the new operator.  Also the argument checks of `lv_gemm_wgrad_acc_f32`.
"""
from __future__ import annotations

import os
import sys
import types

import pytest
import torch

from long_vita_b200 import ops
from long_vita_b200.config import LongVITAConfig
from long_vita_b200.megatron import checkpoint as CK
from tests import vision_oracle as VO
from tests.hostlogic import oracle_ops

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))

from make_vit_grad_golden import golden_inputs  # noqa: E402

bf16, f32 = torch.bfloat16, torch.float32
FUSED_SUFFIXES = ("conv1.weight", "linear_qkv.weight", "linear_proj.weight", "linear_fc1.weight", "linear_fc2.weight")


@pytest.fixture
def acc_calls(monkeypatch):
    """ops.linear_wgrad_accumulate restated (main_grad += dY^T X in float64, rounded once to fp32); returns the calls as
    (main_grad shape, main_grad data_ptr, main_grad row stride, T)."""
    calls = []

    def restated(dy2, x2, main_grad):
        assert main_grad.dtype == f32 and main_grad.shape == (dy2.shape[1], x2.shape[1])
        calls.append((tuple(main_grad.shape), main_grad.data_ptr(), main_grad.stride(0), dy2.shape[0]))
        main_grad.copy_((main_grad.double() + dy2.double().t() @ x2.double()).float())
        return main_grad

    monkeypatch.setattr(ops, "linear_wgrad_accumulate", restated)
    return calls


def _linear_case(seed=1, T=24, n_in=32, n_out=16):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, n_in, generator=g).to(bf16)
    w = (torch.randn(n_out, n_in, generator=g) * 0.2).to(bf16)
    b = torch.randn(n_out, generator=g).to(bf16)
    dy = torch.randn(T, n_out, generator=g).to(bf16)
    return x, w, b, dy


def _run_linear(x, w, b, dy, fuse):
    xd, wd, bd = x.clone().requires_grad_(True), w, b.clone().requires_grad_(True)
    with oracle_ops():
        ops.linear_autograd(xd, wd, bd, accumulate_wgrad=fuse).backward(dy)
    return xd.grad, bd.grad


@pytest.mark.parametrize("attrs", [{}, {"grad_added_to_main_grad": False},
                                   {"grad_added_to_main_grad": False, "zero_out_wgrad": True},
                                   {"grad_added_to_main_grad": False, "zero_out_wgrad": False}])
def test_linear_dummy_gradient_rules(acc_calls, attrs):
    x, w, b, dy = _linear_case()
    wf = w.clone().requires_grad_(True)
    wf.main_grad = torch.full(w.shape, 0.5, dtype=f32)
    for k, v in attrs.items():
        setattr(wf, k, v)
    dx, db = _run_linear(x, wf, b, dy, True)
    assert len(acc_calls) == 1 and acc_calls[0][0] == tuple(w.shape) and acc_calls[0][3] == x.shape[0]
    assert torch.equal(wf.main_grad, (0.5 + dy.double().t() @ x.double()).float())
    if "grad_added_to_main_grad" not in attrs:
        assert wf.grad is None                                   # layers.py:517-518
    else:
        assert wf.grad_added_to_main_grad is True
        assert wf.grad.shape == w.shape and wf.grad.dtype == bf16
        if attrs.get("zero_out_wgrad"):
            assert torch.equal(wf.grad, torch.zeros_like(wf.grad))
    # dX and the bias gradient are those of the un-fused path
    wu = w.clone().requires_grad_(True)
    dx_u, db_u = _run_linear(x, wu, b, dy, False)
    assert torch.equal(dx, dx_u) and torch.equal(db, db_u)


def test_linear_fusion_errors(acc_calls):
    x, w, b, dy = _linear_case()
    wf = w.clone().requires_grad_(True)
    with pytest.raises(RuntimeError, match="main_grad"):
        _run_linear(x, wf, b, dy, True)
    wf.main_grad = torch.zeros(w.shape, dtype=bf16)
    with pytest.raises(NotImplementedError, match="fp32"):
        _run_linear(x, wf, b, dy, True)
    assert not acc_calls


def test_frozen_weight_is_untouched(acc_calls):
    x, w, b, dy = _linear_case()
    _run_linear(x, w, b, dy, True)                               # w does not require grad and has no main_grad
    assert not acc_calls and w.grad is None


def test_lm_head_chunks_accumulate_into_row_slices(acc_calls):
    g = torch.Generator().manual_seed(12)
    s, c, V = 40, 64, 200          # 200 = 3 chunks of 64 + a ragged 8
    h = torch.randn(s, 1, c, generator=g).to(bf16)
    w = (torch.randn(V, c, generator=g) * 0.2).to(bf16)
    mask = torch.rand(1, s, generator=g) < 0.4
    M = int(mask.sum())
    labels = torch.randint(0, V, (1, M), generator=g)
    up = torch.randn(1, M, generator=g)
    grads = {}
    for fuse in (False, True):
        hd, wd = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
        if fuse:
            wd.main_grad = torch.zeros((V, c), dtype=f32)
            wd.grad_added_to_main_grad = False
        with oracle_ops():
            ops.masked_lm_head_ce(hd, wd, mask, labels, vocab_chunk=64, accumulate_wgrad=fuse).backward(up)
        grads[fuse] = (hd.grad, wd.grad if not fuse else wd.main_grad)
        if fuse:
            assert wd.grad_added_to_main_grad is True and wd.grad.shape == (V, c)
    base = grads[True][1].data_ptr()
    assert [(shape, (ptr - base) // (4 * c), ld, T) for shape, ptr, ld, T in acc_calls] == \
        [((64, c), 0, c, M), ((64, c), 64, c, M), ((64, c), 128, c, M), ((8, c), 192, c, M)]
    assert torch.equal(grads[True][0], grads[False][0])
    assert (grads[True][1].to(bf16).float() - grads[False][1].float()).abs().max() <= \
        2.0 ** -7 * grads[False][1].float().abs().max()


def test_masked_linear_passes_the_flag(acc_calls):
    g = torch.Generator().manual_seed(13)
    h = torch.randn(10, 1, 32, generator=g).to(bf16).requires_grad_(True)
    w = torch.randn(24, 32, generator=g).to(bf16).requires_grad_(True)
    w.main_grad = torch.zeros((24, 32), dtype=f32)
    mask = torch.zeros(1, 10, dtype=torch.bool)
    mask[0, 3:7] = True
    with oracle_ops():
        ops.masked_linear(h, w, mask, accumulate_wgrad=True).backward(torch.ones(4, 1, 24, dtype=bf16))
    assert [cl[0] for cl in acc_calls] == [(24, 32)] and acc_calls[0][3] == 4 and w.grad is None


# ------------------------------------------------------------------------------------------------
# surfaces
# ------------------------------------------------------------------------------------------------
def _attach(params):
    for p in params:
        p.main_grad = torch.zeros(p.shape, dtype=f32)
        p.grad_added_to_main_grad = False


def _layer(fuse):
    from long_vita_b200.megatron.transformer_layer import B200TransformerLayer
    from long_vita_b200.weights import llm_layer_weights

    cfg = LongVITAConfig.tiny(layers=1)
    mc = CK.hf_to_mcore(llm_layer_weights(cfg, 0, seed=5, dtype=bf16, perturb=True), cfg)
    mcfg = types.SimpleNamespace(hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_attention_heads,
                                 num_query_groups=cfg.num_key_value_heads, kv_channels=cfg.head_dim,
                                 ffn_hidden_size=cfg.intermediate_size, layernorm_epsilon=cfg.rms_norm_eps,
                                 hidden_dropout=0.0, attention_dropout=0.0, params_dtype=bf16)
    if fuse != "absent":
        mcfg.gradient_accumulation_fusion = fuse
    layer = B200TransformerLayer(mcfg, layer_number=1)
    layer.load_state_dict({k[len("decoder.layers.0."):]: v for k, v in mc.items()}, strict=True)
    for p in layer.parameters():
        p.requires_grad_(True)
    return cfg, layer


def _train_layer(cfg, layer):
    s = 32
    g = torch.Generator().manual_seed(6)
    x = torch.randn(s, 1, cfg.hidden_size, generator=g).to(bf16).requires_grad_(True)
    with oracle_ops():
        out, _ = layer(hidden_states=x, attention_mask=None, rotary_pos_emb=None)
        out.backward(torch.randn(s, 1, cfg.hidden_size, generator=g).to(bf16))
    return out.detach(), x.grad


@pytest.mark.parametrize("fuse", ["absent", False])
def test_transformer_layer_without_the_flag_never_calls_the_new_op(acc_calls, fuse):
    cfg, layer = _layer(fuse)
    _train_layer(cfg, layer)
    assert not acc_calls and all(p.grad is not None for p in layer.parameters())


def test_transformer_layer_with_fusion_accumulates_its_four_weights(acc_calls):
    cfg, layer = _layer(True)
    fused = {n: p for n, p in layer.named_parameters() if n.endswith(FUSED_SUFFIXES)}
    assert sorted(fused) == ["mlp.linear_fc1.weight", "mlp.linear_fc2.weight", "self_attention.linear_proj.weight",
                             "self_attention.linear_qkv.weight"]
    _attach(fused.values())
    out, dx = _train_layer(cfg, layer)
    assert sorted(cl[0] for cl in acc_calls) == sorted(tuple(p.shape) for p in fused.values())
    _, ref = _layer(False)
    out_u, dx_u = _train_layer(cfg, ref)
    assert torch.equal(out, out_u) and torch.equal(dx, dx_u)
    ref_params = dict(ref.named_parameters())
    for n, p in layer.named_parameters():
        if n in fused:
            assert p.grad_added_to_main_grad is True
            d = (p.main_grad - ref_params[n].grad.float()).abs().max()
            assert d <= 2.0 ** -7 * ref_params[n].grad.float().abs().max(), n
        else:                                                    # norm weights and the qkv bias: unchanged path
            assert torch.equal(p.grad, ref_params[n].grad), n


def _vision(fuse, freeze=False):
    from long_vita_b200.megatron.vision_model import B200VisionModel

    cfg, w, images, d_out = golden_inputs()
    m = B200VisionModel(cfg.hidden_size, cfg.visual, params_dtype=f32, device="cpu", vision_model_freeze=freeze,
                        gradient_accumulation_fusion=fuse)
    m.load_state_dict({k[len(CK.EFM):]: t for k, t in CK.hf_to_mcore(w, cfg).items()}, strict=True)
    return m, images[:1], d_out[:1]


@pytest.mark.parametrize("freeze", [False, True])
def test_vision_model_with_fusion(acc_calls, freeze):
    m, images, d_out = _vision(True, freeze)
    assert m.gradient_accumulation_fusion
    params = dict(m.named_parameters())
    fused = [n for n in params if n.endswith(FUSED_SUFFIXES)]
    assert len(fused) == 1 + 4 * len(m.vit.decoder.layers) + 2
    _attach(params[n] for n in fused)
    with VO.vision_oracle_ops():
        m(images=images).backward(d_out)
    ref, _, _ = _vision(False, freeze)
    with VO.vision_oracle_ops():
        ref(images=images).backward(d_out)
    ref_params = dict(ref.named_parameters())
    C = params["vit.conv1.weight"].shape[0]
    shapes = [cl[0] for cl in acc_calls]
    assert ((C, 588) in shapes) != freeze                        # the 588 real im2col columns, not the padded 640
    for n in fused:
        p = params[n]
        if freeze and n.startswith("vit."):
            assert p.grad is None and p.grad_added_to_main_grad is False and not bool(p.main_grad.any()), n
            continue
        assert p.grad_added_to_main_grad is True and p.grad.shape == p.shape, n
        want = ref_params[n].grad
        assert (p.main_grad - want).abs().max() <= 1e-5 * want.abs().max(), n
    for n, p in params.items():
        if n not in fused:
            g, want = p.grad, ref_params[n].grad
            assert (g is None and want is None) or torch.equal(g, want), n


def test_vision_model_without_fusion_never_calls_the_new_op(acc_calls):
    m, images, d_out = _vision(False)
    assert not m.gradient_accumulation_fusion
    with VO.vision_oracle_ops():
        m(images=images).backward(d_out)
    assert not acc_calls


def test_vision_provider_reads_the_flag():
    from long_vita_b200.megatron.vision_model import b200_vision_model_provider

    base = dict(hidden_size=640, vision_model_type="intern_300m", add_class_token=True, vision_projector_pre_norm=True,
                vision_downsample_ratio=0.5, vision_model_freeze=True, vision_projector_freeze=False,
                norm_epsilon=1e-6, image_size=448)
    cfg = types.SimpleNamespace(params_dtype=bf16)
    assert not b200_vision_model_provider(cfg, args=types.SimpleNamespace(**base)).gradient_accumulation_fusion
    for v in (False, None):
        a = types.SimpleNamespace(**base, gradient_accumulation_fusion=v)
        assert not b200_vision_model_provider(cfg, args=a).gradient_accumulation_fusion
    a = types.SimpleNamespace(**base, gradient_accumulation_fusion=True)
    assert b200_vision_model_provider(cfg, args=a).gradient_accumulation_fusion


@pytest.mark.parametrize("fused_loss", [True, False])
def test_gptvl_output_layer(acc_calls, monkeypatch, fused_loss):
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel
    from long_vita_b200.weights import synthetic_state_dict

    cfg = LongVITAConfig.tiny(layers=1, vit_layers=1)
    mc = CK.hf_to_mcore(synthetic_state_dict(cfg, seed=7, dtype=bf16, perturb=True), cfg)
    seen = []
    real_ce, real_ml = ops.masked_lm_head_ce, ops.masked_linear
    monkeypatch.setattr(ops, "masked_lm_head_ce",
                        lambda *a, **k: seen.append(("ce", k.get("accumulate_wgrad"))) or real_ce(*a, **k))
    monkeypatch.setattr(ops, "masked_linear",
                        lambda *a, **k: seen.append(("linear", k.get("accumulate_wgrad"))) or real_ml(*a, **k))
    s = 24
    g = torch.Generator().manual_seed(8)
    ids = torch.randint(0, cfg.vocab_size, (1, s), generator=g)
    labels = torch.randint(0, cfg.vocab_size, (1, s), generator=g)
    mask = torch.zeros(1, s, dtype=torch.bool)
    mask[0, 10:20] = True
    pos = torch.arange(s).unsqueeze(0)
    for fuse in (None, False, True):
        kw = {} if fuse is None else {"gradient_accumulation_fusion": fuse}
        model = B200GPTVLModel(cfg, mc, **kw)
        model.fused_loss = fused_loss
        assert model.gradient_accumulation_fusion is bool(fuse)
        model.output_weight = model.output_weight.detach().clone().requires_grad_(True)
        if fuse:
            _attach([model.output_weight])
        acc_calls.clear()
        seen.clear()
        with oracle_ops():
            loss = model(ids, pos, None, labels=labels, logit_mask=mask)
            loss.sum().backward()
        assert seen == [("ce" if fused_loss else "linear", bool(fuse))]
        if fuse:
            assert [cl[0] for cl in acc_calls] == [tuple(model.output_weight.shape)]
            assert model.output_weight.grad_added_to_main_grad is True and bool(model.output_weight.main_grad.any())
        else:
            assert not acc_calls and model.output_weight.grad is not None


# ------------------------------------------------------------------------------------------------
# C ABI argument checks
# ------------------------------------------------------------------------------------------------
def test_lv_gemm_wgrad_acc_f32_rejects_bad_arguments_without_a_gpu(lib_built):
    from long_vita_b200 import _lib

    h = _lib.lib()

    def acc(*a):
        return h.lv_gemm_wgrad_acc_f32(*a, None), h.lv_last_error()

    P = 256          # a 16-byte aligned fake address: every case fails its checks (or returns) before touching memory
    rc, msg = acc(None, P, P, 64, 64, 16, 64, 64, 64, 1, 1)
    assert rc == -1 and b"null pointer" in msg
    rc, msg = acc(P, P, None, 64, 64, 16, 64, 64, 64, 1, 1)
    assert rc == -1 and b"null pointer" in msg
    rc, msg = acc(P, P, P, 64, 64, 16, 64, 64, 64, 2, 1)
    assert rc == -1 and b"must be 0 or 1" in msg
    for a_mn, w_mn in ((0, 0), (0, 1), (1, 0)):
        rc, msg = acc(P, P, P, 64, 64, 16, 64, 64, 64, a_mn, w_mn)
        assert rc == -1 and b"only MN-major" in msg
    rc, msg = acc(P, P, P, 64, 0, 16, 64, 64, 64, 1, 1)
    assert rc == -1 and b"bad shape" in msg
    rc, msg = acc(P, P, P, -1, 64, 16, 64, 64, 64, 1, 1)
    assert rc == -1 and b"bad shape" in msg
    rc, msg = acc(P, P, P, 64, 1 << 31, 16, 64, 1 << 31, 1 << 31, 1, 1)
    assert rc == -1 and b"too large" in msg
    rc, msg = acc(P, P, P, 64, 62, 16, 64, 64, 64, 1, 1)
    assert rc == -1 and b"N=62" in msg
    rc, msg = acc(P, P, P, 64, 64, 16, 60, 64, 64, 1, 1)
    assert rc == -1 and b"lda=60" in msg
    rc, msg = acc(P, P, P, 64, 64, 16, 68, 64, 64, 1, 1)
    assert rc == -1 and b"lda=68" in msg
    rc, msg = acc(P, P, P, 64, 64, 16, 64, 56, 64, 1, 1)
    assert rc == -1 and b"ldw=56" in msg and b"N=64" in msg
    rc, msg = acc(P, P, P, 64, 64, 16, 64, 64, 66, 1, 1)
    assert rc == -1 and b"ldc=66" in msg
    rc, msg = acc(P, P, P, 64, 64, 16, 64, 64, 60, 1, 1)
    assert rc == -1 and b"ldc=60" in msg
    rc, msg = acc(P, P, P + 8, 64, 64, 16, 64, 64, 64, 1, 1)
    assert rc == -1 and b"16-byte aligned" in msg
    rc, msg = acc(P, P + 2, P, 64, 64, 16, 64, 64, 64, 1, 1)
    assert rc == -1 and b"16-byte aligned" in msg
    # nothing to add: no launch, success
    assert acc(P, P, P, 64, 64, 0, 64, 64, 64, 1, 1)[0] == 0
    assert acc(P, P, P, 0, 64, 16, 8, 64, 64, 1, 1)[0] == 0
