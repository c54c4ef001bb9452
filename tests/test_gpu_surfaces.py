"""GPU tests of the reference-facing operator surfaces: Megatron `core_attention` slot and patch
wrapper (through the Megatron-free stub), HF AttentionInterface function, InternAttention.inner_attn
replacement."""
import math

import pytest
import torch

from oracle import ops as O
from tests.util import randn_bf16, rel_fro, seeded

pytestmark = pytest.mark.gpu


def _excess(out, ref):
    e, f = rel_fro(out, ref), rel_fro(ref.to(torch.bfloat16), ref)
    return math.sqrt(max(e * e - f * f, 0.0))


def _qkv_sbhd(s, b, np_, ng, hn, seed):
    g = seeded(seed)
    return randn_bf16((s, b, np_, hn), g), randn_bf16((s, b, ng, hn), g), randn_bf16((s, b, ng, hn), g)


def test_core_attention_slot_llm_and_vit(lib_built):
    from long_vita_b200.megatron import stub
    from long_vita_b200.megatron.core_attention import B200DotProductAttention

    cfg = stub.TransformerConfig(hidden_size=1280, num_attention_heads=10, num_query_groups=2)
    spec = stub.ModuleSpec(module=B200DotProductAttention)
    attn = stub.build_module(spec, config=cfg, layer_number=1, attn_mask_type=stub.AttnMaskType.causal,
                             attention_type="self")
    q, k, v = _qkv_sbhd(700, 2, 10, 2, 128, 1)
    out = attn(q.cuda(), k.cuda(), v.cuda(), None, attn_mask_type=stub.AttnMaskType.causal, packed_seq_params=None)
    assert out.shape == (700, 2, 1280)
    ref, _ = O.attention(q.permute(1, 0, 2, 3), k.permute(1, 0, 2, 3), v.permute(1, 0, 2, 3), causal=True)
    assert _excess(out.view(700, 2, 10, 128).permute(1, 0, 2, 3), ref) < 2e-3
    # ViT slot: no_mask, 16 heads x 64
    vcfg = stub.TransformerConfig(hidden_size=1024, num_attention_heads=16, num_query_groups=16)
    vattn = B200DotProductAttention(vcfg, 3, stub.AttnMaskType.no_mask, "self")
    q, k, v = _qkv_sbhd(1025, 2, 16, 16, 64, 2)
    out = vattn(q.cuda(), k.cuda(), v.cuda(), None)
    ref, _ = O.attention(q.permute(1, 0, 2, 3), k.permute(1, 0, 2, 3), v.permute(1, 0, 2, 3), causal=False)
    assert _excess(out.view(1025, 2, 16, 64).permute(1, 0, 2, 3), ref) < 2e-3
    with pytest.raises(AssertionError):
        vattn(q.cuda(), k.cuda(), v.cuda(), None, packed_seq_params=object())


def test_patch_registry_wrapper(lib_built):
    from long_vita_b200.megatron import stub
    from long_vita_b200.megatron.core_attention import b200_dot_product_attention_forward_wrapper

    class Patched(stub.DotProductAttention):
        pass

    stub.apply_reference_style_patch(Patched, "forward", b200_dot_product_attention_forward_wrapper)
    cfg = stub.TransformerConfig(hidden_size=640, num_attention_heads=5, num_query_groups=1)
    mod = Patched(cfg, 1, stub.AttnMaskType.causal)
    q, k, v = _qkv_sbhd(384, 1, 5, 1, 128, 3)
    out = mod.forward(q.cuda(), k.cuda(), v.cuda(), None, stub.AttnMaskType.causal, None)
    ref, _ = O.attention(q.permute(1, 0, 2, 3), k.permute(1, 0, 2, 3), v.permute(1, 0, 2, 3), causal=True)
    assert out.shape == (384, 1, 640)
    assert _excess(out.view(384, 1, 5, 128).permute(1, 0, 2, 3), ref) < 2e-3


def test_hf_attention_interface_function(lib_built):
    from long_vita_b200.hf import attention_interface as AI

    name = AI.register()
    from transformers import AttentionInterface

    assert name in AttentionInterface()._global_mapping or name in dict(AttentionInterface._global_mapping)
    g = seeded(4)
    q, k, v = randn_bf16((2, 10, 300, 128), g), randn_bf16((2, 2, 300, 128), g), randn_bf16((2, 2, 300, 128), g)
    out, w = AI.b200_attention_forward(None, q.cuda(), k.cuda(), v.cuda(), None, dropout=0.0, scaling=128 ** -0.5,
                                       is_causal=True)
    assert w is None and out.shape == (2, 300, 10, 128)
    ref, _ = O.attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), causal=True)
    assert _excess(out, ref) < 2e-3


def test_intern_inner_attn_replacement(lib_built):
    from long_vita_b200.hf.attention_interface import B200FlashAttention

    g = seeded(5)
    qkv = randn_bf16((3, 1025, 3, 16, 64), g)
    out, w = B200FlashAttention(attention_dropout=0.0)(qkv.cuda(), key_padding_mask=None, need_weights=False, causal=False)
    assert w is None and out.shape == (3, 1025, 16, 64)
    ref, _ = O.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], causal=False)
    assert _excess(out, ref) < 2e-3
    with pytest.raises(AssertionError):
        B200FlashAttention()(qkv.float().cuda())


def test_whole_layer_spec_module_matches_oracle_decoder_layer(lib_built):
    """B2: the `--spec` layer with TE state-dict names and Megatron's grouped QKV layout."""
    from types import SimpleNamespace

    from long_vita_b200.config import LongVITAConfig
    from long_vita_b200.megatron import stub
    from long_vita_b200.megatron.transformer_layer import B200TransformerLayer, get_b200_layer_spec
    from long_vita_b200.weights import llm_layer_weights
    from oracle import model as OM

    cfg = LongVITAConfig.tiny(layers=1)
    w = llm_layer_weights(cfg, 0, seed=5, dtype=torch.bfloat16, perturb=True)
    mcfg = SimpleNamespace(hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_attention_heads,
                           num_query_groups=cfg.num_key_value_heads, kv_channels=cfg.head_dim,
                           ffn_hidden_size=cfg.intermediate_size, layernorm_epsilon=cfg.rms_norm_eps,
                           hidden_dropout=0.0, attention_dropout=0.0, params_dtype=torch.bfloat16)
    spec = get_b200_layer_spec()
    layer = stub.build_module(spec, config=mcfg, layer_number=1)
    assert isinstance(layer, B200TransformerLayer)
    names = set(layer.state_dict().keys())
    assert {"self_attention.linear_qkv.layer_norm_weight", "self_attention.linear_qkv.weight",
            "self_attention.linear_qkv.bias", "self_attention.linear_proj.weight", "mlp.linear_fc1.layer_norm_weight",
            "mlp.linear_fc1.weight", "mlp.linear_fc2.weight"} == names
    # HF -> mcore grouped layout (tools/hf2mcore_long_vita.py:599-613)
    p = "model.layers.0."
    ng, g, hn, h = cfg.num_key_value_heads, cfg.num_attention_heads // cfg.num_key_value_heads, cfg.head_dim, cfg.hidden_size
    qw = w[p + "self_attn.q_proj.weight"].view(ng, g, hn, h)
    kw = w[p + "self_attn.k_proj.weight"].view(ng, 1, hn, h)
    vw = w[p + "self_attn.v_proj.weight"].view(ng, 1, hn, h)
    qb = w[p + "self_attn.q_proj.bias"].view(ng, g, hn)
    kb = w[p + "self_attn.k_proj.bias"].view(ng, 1, hn)
    vb = w[p + "self_attn.v_proj.bias"].view(ng, 1, hn)
    sd = {
        "self_attention.linear_qkv.layer_norm_weight": w[p + "input_layernorm.weight"],
        "self_attention.linear_qkv.weight": torch.cat([qw, kw, vw], dim=1).reshape(-1, h),
        "self_attention.linear_qkv.bias": torch.cat([qb, kb, vb], dim=1).reshape(-1),
        "self_attention.linear_proj.weight": w[p + "self_attn.o_proj.weight"],
        "mlp.linear_fc1.layer_norm_weight": w[p + "post_attention_layernorm.weight"],
        "mlp.linear_fc1.weight": torch.cat([w[p + "mlp.gate_proj.weight"], w[p + "mlp.up_proj.weight"]], dim=0),
        "mlp.linear_fc2.weight": w[p + "mlp.down_proj.weight"],
    }
    layer.load_state_dict({k: v.cuda() for k, v in sd.items()}, strict=True)
    s = 515
    g_ = seeded(6)
    x = randn_bf16((s, 1, h), g_)
    inv = O.rope_inv_freq(hn, cfg.rope_theta)
    freqs = torch.outer(torch.arange(s).float(), inv)
    emb = torch.cat((freqs, freqs), dim=-1)[:, None, None, :]            # Megatron RotaryEmbedding.forward output
    out, ctx = layer(hidden_states=x.cuda(), attention_mask=None, context=None, context_mask=None,
                     rotary_pos_emb=emb.cuda(), inference_params=None, packed_seq_params=None)
    assert ctx is None and out.shape == (s, 1, h)
    cos, sin = O.rope_tables(torch.arange(s), inv, torch.bfloat16)
    ref = OM.decoder_layer(cfg, OM.cast_weights(w, torch.float32), 0, x[:, 0].float(), cos.float(), sin.float())
    assert rel_fro(out[:, 0], ref) < 4e-3, rel_fro(out[:, 0], ref)


def test_masked_lm_head_autograd(lib_built):
    """a12 backward on the kernels: dX scatter and dW = dY^T sel through the transposed-operand GEMM (K = M
    padded to 8)."""
    from long_vita_b200 import ops

    g = seeded(12)
    s, c, vocab = 300, 640, 2048
    h = randn_bf16((s, 1, c), g)
    w = randn_bf16((vocab, c), g, scale=0.05)
    mask = torch.zeros(1, s, dtype=torch.bool)
    mask[0, [5, 6, 77, 150, 299]] = True
    dy = randn_bf16((5, 1, vocab), g)
    hg, wg = h.cuda().requires_grad_(True), w.cuda().requires_grad_(True)
    out = ops.masked_linear(hg, wg, mask.cuda())
    out.backward(dy.cuda())
    ref_out = O.masked_linear_fwd(h.float(), w.float(), mask)
    gx, gw = O.masked_linear_bwd(dy.float(), h.float(), w.float(), mask)
    assert rel_fro(out, ref_out) < 4e-3
    assert rel_fro(hg.grad, gx) < 4e-3 and rel_fro(wg.grad, gw) < 4e-3


def test_spec_layer_training_step_matches_oracle_autograd(lib_built):
    """B2 training path on the kernels: forward + backward of the `--spec` layer (RMSNorm / SwiGLU / RoPE backward
    kernels, lv_attn_bwd, GEMM dX / dW) against fp32 autograd through the oracle decoder layer."""
    from types import SimpleNamespace

    from long_vita_b200.config import LongVITAConfig
    from long_vita_b200.megatron import checkpoint as ck
    from long_vita_b200.megatron.transformer_layer import B200TransformerLayer
    from long_vita_b200.weights import llm_layer_weights
    from oracle import model as OM

    cfg = LongVITAConfig.tiny(layers=1)
    hf = llm_layer_weights(cfg, 0, seed=9, dtype=torch.bfloat16, perturb=True)
    mc = ck.hf_to_mcore(hf, cfg)
    mcfg = SimpleNamespace(hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_attention_heads,
                           num_query_groups=cfg.num_key_value_heads, kv_channels=cfg.head_dim,
                           ffn_hidden_size=cfg.intermediate_size, layernorm_epsilon=cfg.rms_norm_eps,
                           hidden_dropout=0.0, attention_dropout=0.0, params_dtype=torch.bfloat16)
    layer = B200TransformerLayer(mcfg, layer_number=1)
    layer.load_state_dict({k[len("decoder.layers.0."):]: v.cuda() for k, v in mc.items()}, strict=True)
    for prm in layer.parameters():
        prm.requires_grad_(True)
    s = 384
    g_ = seeded(10)
    x = randn_bf16((s, 1, cfg.hidden_size), g_).cuda().requires_grad_(True)
    dout = randn_bf16((s, 1, cfg.hidden_size), g_, 0.1)
    inv = O.rope_inv_freq(cfg.head_dim, cfg.rope_theta)
    freqs = torch.outer(torch.arange(s).float(), inv)
    emb = torch.cat((freqs, freqs), dim=-1)[:, None, None, :]
    out, _ = layer(hidden_states=x, attention_mask=None, rotary_pos_emb=emb.cuda())
    out.backward(dout.cuda())
    w32 = {k: v.float().requires_grad_(True) for k, v in hf.items()}
    xr = x.detach().float().cpu()[:, 0].requires_grad_(True)
    cos, sin = O.rope_tables(torch.arange(s), inv, torch.float32)
    ref = OM.decoder_layer(cfg, w32, 0, xr, cos, sin)
    ref.backward(dout.float()[:, 0])
    assert rel_fro(out[:, 0], ref.detach()) < 8e-3
    assert rel_fro(x.grad[:, 0], xr.grad) < 2e-2
    ref_mc = ck.hf_to_mcore({k: v.grad for k, v in w32.items()}, cfg)
    for name, prm in layer.named_parameters():
        assert rel_fro(prm.grad, ref_mc["decoder.layers.0." + name]) < 3e-2, name
