"""GPU composition of packed samples: a packed prompt of three documents through B200GPTVLModel, LongVITAModel and the
`--spec` layer (with `actual_seq_len` published as a Megatron training loop does) gives, per document, what the oracle
model / the same module gives on each document alone."""
import sys
import types

import pytest
import torch

from long_vita_b200.config import LongVITAConfig
from long_vita_b200.megatron import checkpoint as ck
from long_vita_b200.weights import synthetic_state_dict
from oracle import model as OM
from oracle import ops as O
from tests.util import rel_fro

pytestmark = pytest.mark.gpu

LENGTHS = [150, 77, 173]


def _bounds():
    cu = [0]
    for n in LENGTHS:
        cu.append(cu[-1] + n)
    return list(zip(cu, cu[1:]))


def _packed_pos():
    return torch.cat([torch.arange(n) for n in LENGTHS]).view(1, -1).cuda()


@pytest.fixture(scope="module")
def setup(lib_built):
    cfg = LongVITAConfig.tiny(layers=2, vit_layers=1)
    hf = synthetic_state_dict(cfg, seed=77, dtype=torch.bfloat16, perturb=True)
    return cfg, hf


def _check(logits, cfg, hf, ids):
    w32 = OM.cast_weights(hf, torch.float32)
    ref = torch.cat([OM.long_vita_forward(cfg, w32, ids[:, a:b], None, None)[0] for a, b in _bounds()])
    assert rel_fro(logits, ref) < 1.5e-2, rel_fro(logits, ref)
    # random-init tiny model: near-ties flip a few argmax positions under bf16 (tests/test_gpu_megatron_model.py)
    assert float((logits.float().argmax(-1).cpu() == ref.argmax(-1)).float().mean()) > 0.93


def test_gptvl_model_packed_prompt(setup):
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel

    cfg, hf = setup
    model = B200GPTVLModel(cfg, {k: v.cuda() for k, v in ck.hf_to_mcore(hf, cfg).items()})
    ids = torch.randint(0, cfg.vocab_size, (1, sum(LENGTHS)), generator=torch.Generator().manual_seed(1))
    out = model(ids.cuda(), _packed_pos(), None)[0]
    _check(out, cfg, hf, ids)
    alone = torch.cat([model(ids[:, a:b].cuda(), torch.arange(b - a).view(1, -1).cuda(), None)[0] for a, b in _bounds()])
    assert rel_fro(out, alone) < 5e-3      # bf16 GEMMs over a different number of rows, two layers deep


def test_hf_model_packed_prompt(setup):
    from long_vita_b200.hf.modeling import LongVITAForCausalLM

    cfg, hf = setup
    model = LongVITAForCausalLM(cfg, {k: v.cuda() for k, v in hf.items()})
    ids = torch.randint(0, cfg.vocab_size, (1, sum(LENGTHS)), generator=torch.Generator().manual_seed(2))
    out = model(input_ids=ids.cuda(), position_ids=_packed_pos()).logits[0]
    _check(out, cfg, hf, ids)


def test_spec_layer_training_with_actual_seq_len(setup, monkeypatch):
    """Gradients of the packed layer equal those of each document run alone (the tolerances of the training-layer
    test), on the kernels: lv_attn_docs_fwd / lv_attn_docs_bwd inside ops.attention."""
    from long_vita_b200.megatron.transformer_layer import B200TransformerLayer

    cfg, hf = setup
    mc = ck.hf_to_mcore(hf, cfg)
    mcfg = types.SimpleNamespace(hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_attention_heads,
                                 num_query_groups=cfg.num_key_value_heads, kv_channels=cfg.head_dim,
                                 ffn_hidden_size=cfg.intermediate_size, layernorm_epsilon=cfg.rms_norm_eps,
                                 hidden_dropout=0.0, attention_dropout=0.0, params_dtype=torch.bfloat16)
    layer = B200TransformerLayer(mcfg, layer_number=1)
    layer.load_state_dict({k[len("decoder.layers.0."):]: v.cuda() for k, v in mc.items()
                           if k.startswith("decoder.layers.0.")}, strict=True)
    mod = types.ModuleType("long_vita_megatron.training.utils")
    state = {"ends": None}
    mod.get_actual_seq_len = lambda: state["ends"]
    monkeypatch.setitem(sys.modules, "long_vita_megatron.training.utils", mod)
    s = sum(LENGTHS)
    x = torch.randn(s, 1, cfg.hidden_size, generator=torch.Generator().manual_seed(4)).to(torch.bfloat16).cuda()
    dy = torch.randn(s, 1, cfg.hidden_size, generator=torch.Generator().manual_seed(5)).to(torch.bfloat16).cuda()
    inv = O.rope_inv_freq(cfg.head_dim, cfg.rope_theta)
    pos = _packed_pos().view(-1).cpu()

    def rotary(p):
        f = torch.outer(p.float(), inv)
        return torch.cat((f, f), dim=-1).view(-1, 1, 1, cfg.head_dim).cuda()

    def run(xi, p, ends):
        state["ends"] = ends
        xi = xi.clone().requires_grad_(True)
        out, _ = layer(hidden_states=xi, attention_mask=None, context=None, context_mask=None,
                       rotary_pos_emb=rotary(p), inference_params=None, packed_seq_params=None)
        return out, xi

    out, xp = run(x, pos, [b for _, b in _bounds()])
    out.backward(dy)
    outs, grads = [], []
    for a, b in _bounds():
        o, xi = run(x[a:b], pos[a:b], None)
        o.backward(dy[a:b])
        outs.append(o.detach())
        grads.append(xi.grad)
    assert rel_fro(out.detach(), torch.cat(outs)) < 2e-3
    assert rel_fro(xp.grad, torch.cat(grads)) < 1e-2, rel_fro(xp.grad, torch.cat(grads))
