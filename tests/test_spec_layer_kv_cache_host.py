"""CPU tests of Megatron's `--use-kv-cache` protocol on the `--spec` decoder layer (B200TransformerLayer with
`inference_params`).

Megatron's inference loop is restated in a few lines (`_spec_generate`): the layers are built with `build_module`,
each forward calls every layer with the rotary table of `max_sequence_length` positions and the shared
`inference_params`, then the final norm and the LM head, and advances `sequence_len_offset` by the forward's length.

* On the CPU oracle (tests/hostlogic.py), a prompt and 8 greedy steps give logits equal to B200GPTVLModel's on the
  same state dict under the same protocol: device cache, offloaded cache with 1 device layer (whole and streamed
  prefill), FP8 host tier through `config.kv_host_dtype`.
* RoPE takes the table's rows at `sequence_len_offset`.
* The cache's length follows the offset (kv_cache `commit_to`); an offset that moves back or jumps raises.
* Refusals (context parallelism, max_batch_size > 1, packed samples, gradients), with nothing launched.
* With `inference_params=None` the layer makes the same C calls as before, and a cached generation leaves them alone.

The GPU twin is tests/test_gpu_spec_layer_kv_cache.py.
"""
import sys
import types

import pytest
import torch

from long_vita_b200 import ops
from long_vita_b200.config import LongVITAConfig
from long_vita_b200.hf import modeling
from long_vita_b200.kv_cache import KVCache, OffloadedKVCache
from long_vita_b200.megatron import checkpoint as ck
from long_vita_b200.megatron.stub import build_module
from long_vita_b200.megatron.transformer_layer import get_b200_layer_spec
from long_vita_b200.weights import synthetic_state_dict
from tests.hostlogic import oracle_ops
from tests.test_kv_fp8_host import _oracle_fp8_host_tier
from tests.test_offloaded_cache_host import _host_memory, _offload, _oracle_host_tier
from tests.test_ops_args_host import lib  # noqa: F401  (lib is the recording-stub fixture)
from tests.test_stream_layer_host import _constants

FP8 = torch.float8_e4m3fn


def megatron_config(cfg, **kw):
    """The TransformerConfig fields the layer reads, at the geometry of `cfg`."""
    return types.SimpleNamespace(hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_attention_heads,
                                 num_query_groups=cfg.num_key_value_heads, kv_channels=cfg.head_dim,
                                 ffn_hidden_size=cfg.intermediate_size, layernorm_epsilon=cfg.rms_norm_eps,
                                 num_layers=cfg.num_hidden_layers, hidden_dropout=0.0, attention_dropout=0.0,
                                 params_dtype=torch.bfloat16, **kw)


def spec_layers(cfg, mc, **kw):
    """The decoder as Megatron builds it from `--spec`: one B200TransformerLayer per layer_number, loaded with the
    TE-named weights of the mcore state dict."""
    mcfg = megatron_config(cfg, **kw)
    layers = []
    for i in range(cfg.num_hidden_layers):
        layer = build_module(get_b200_layer_spec(), config=mcfg, layer_number=i + 1)
        p = f"decoder.layers.{i}."
        layer.load_state_dict({k[len(p):]: v for k, v in mc.items() if k.startswith(p)}, strict=True)
        layers.append(layer)
    return layers


def rotary_table(cfg, n, device="cpu", shift=0):
    """Megatron's `freqs` [n, 1, 1, d] fp32 for positions shift .. shift + n - 1 (rotary_pos_embedding.py:84-122)."""
    inv = modeling.rope_inv_freq(cfg, device)
    freqs = torch.outer(torch.arange(shift, shift + n, device=device).float(), inv)
    return torch.cat((freqs, freqs), dim=-1).view(n, 1, 1, cfg.head_dim)


def inference_params(capacity):
    """megatron-core 0.7 InferenceParams(max_batch_size=1, max_sequence_length=capacity)."""
    return types.SimpleNamespace(max_batch_size=1, max_sequence_length=capacity, sequence_len_offset=0,
                                 batch_size_offset=0, key_value_memory_dict={})


def spec_forward(layers, head, ids, ip, table):
    """One forward of Megatron's loop over the `--spec` layers: embedding, every layer with inference_params, the
    final norm and the LM head; then sequence_len_offset advances by the forward's length.  Returns logits [s, V]."""
    emb, norm_w, out_w, eps = head
    s = ids.shape[1]
    x = ops.embed_scatter(ids, emb).view(s, 1, -1)
    for layer in layers:
        x, _ = layer(hidden_states=x, attention_mask=None, context=None, context_mask=None, rotary_pos_emb=table,
                     inference_params=ip, packed_seq_params=None)
    logits = ops.linear(ops.rmsnorm(x.view(s, -1), norm_w, eps), out_w)
    ip.sequence_len_offset += s
    return logits


def _spec_generate(cfg, layers, head, ids, steps, capacity, shift=0):
    """The prompt, then `steps` greedy tokens; the rotary table is built anew for every forward, as Megatron does."""
    ip = inference_params(capacity)
    out = [spec_forward(layers, head, ids, ip, rotary_table(cfg, capacity, ids.device, shift))]
    for _ in range(steps):
        tok = out[-1][-1].float().argmax().view(1, 1)
        out.append(spec_forward(layers, head, tok, ip, rotary_table(cfg, capacity, ids.device, shift)))
    return out, ip


def _mirror_generate(model, ids, steps, capacity):
    """The same protocol on B200GPTVLModel: the prompt with its positions, then one token per call."""
    s = ids.shape[1]
    ip = types.SimpleNamespace(key_value_memory_dict={}, max_sequence_length=capacity, use_kv_cache=True)
    out = [model(ids, torch.arange(s).unsqueeze(0), None, inference_params=ip)[0]]
    for i in range(steps):
        tok = out[-1][-1].float().argmax().view(1, 1)
        out.append(model(tok, torch.tensor([[s + i]]), None, inference_params=ip)[0])
    return out, ip


@pytest.fixture(scope="module")
def tiny():
    cfg = LongVITAConfig.tiny(layers=2, vit_layers=1)
    mc = ck.hf_to_mcore(synthetic_state_dict(cfg, seed=41, dtype=torch.bfloat16, perturb=True), cfg)
    return cfg, mc


def _models(cfg, mc, kv_host_dtype=torch.bfloat16):
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel

    with oracle_ops():
        mirror = B200GPTVLModel(cfg, mc, kv_host_dtype=kv_host_dtype)
    kw = {} if kv_host_dtype == torch.bfloat16 else {"kv_host_dtype": kv_host_dtype}
    head = (mirror.word_embeddings, mirror.final_layernorm, mirror.output_weight, cfg.rms_norm_eps)
    return mirror, spec_layers(cfg, mc, **kw), head


def _prompt(cfg, s=300):
    return torch.randint(0, cfg.vocab_size, (1, s), generator=torch.Generator().manual_seed(8))


# ------------------------------------------------------------------------------------------------
# the --spec loop against B200GPTVLModel on the CPU oracle
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tier", ["device", "offloaded", "offloaded-streamed", "fp8-host"])
def test_spec_loop_equals_the_mirror(monkeypatch, tiny, tier):
    cfg, mc = tiny
    steps, s = 8, 300
    ids = _prompt(cfg, s)
    mirror, layers, head = _models(cfg, mc, FP8 if tier == "fp8-host" else torch.bfloat16)
    host = _oracle_fp8_host_tier if tier == "fp8-host" else _oracle_host_tier
    with host(monkeypatch) as host_calls, _constants(256, 128, 256 if tier == "offloaded-streamed" else None):
        if tier != "device":
            _offload(monkeypatch, cfg, 1)
        want, mip = _mirror_generate(mirror, ids, steps, s + steps)
        n_mirror = len(host_calls)
        got, ip = _spec_generate(cfg, layers, head, ids, steps, s + steps)
    cache, ref = ip.key_value_memory_dict["b200_kv_cache"], mip.key_value_memory_dict["b200_kv_cache"]
    assert type(cache) is type(ref) is (KVCache if tier == "device" else OffloadedKVCache)
    if tier != "device":
        assert cache.n_dev == 1 and cache.host_dtype == (FP8 if tier == "fp8-host" else torch.bfloat16)
        assert host_calls[n_mirror:] == host_calls[:n_mirror] and n_mirror >= steps   # the same host-tier calls
    assert [tuple(t.shape) for t in got] == [(s, cfg.vocab_size)] + [(1, cfg.vocab_size)] * steps
    for i, (a, b) in enumerate(zip(got, want)):
        assert torch.equal(a, b), i
    # the last forward's rows are pending, committed by the next forward's first layer; the mirror commits at once
    assert len(cache) == s + steps - 1 and len(ref) == s + steps and ip.sequence_len_offset == s + steps
    cache.commit_to(ip.sequence_len_offset)
    assert len(cache) == s + steps
    if tier == "device":
        for j in range(cfg.num_hidden_layers):
            assert torch.equal(cache.k[j][: s + steps], ref.k[j][: s + steps])
            assert torch.equal(cache.v[j][: s + steps], ref.v[j][: s + steps])
    else:
        assert torch.equal(cache.k[0][: s + steps], ref.k[0][: s + steps])
        assert torch.equal(cache.host[0][: s + steps], ref.host[0][: s + steps])


def test_rope_rows_are_taken_at_the_offset(monkeypatch, tiny):
    cfg, mc = tiny
    s = 300
    ids = _prompt(cfg, s)
    _, layers, head = _models(cfg, mc)
    seen = []
    with oracle_ops() as o:
        rope = o.rope

        def recording(x, cos, sin, out=None):
            seen.append((cos, sin))
            return rope(x, cos, sin, out=out)

        o.rope = recording
        base, _ = _spec_generate(cfg, layers, head, ids, 2, s + 4)
        # every call took the rows [offset, offset + s) of the table, as views of one table shared by the layers
        cos, sin = modeling.ops.rope_table(torch.arange(s + 4), modeling.rope_inv_freq(cfg, "cpu"))
        starts = [0] * 2 * len(layers) + [s] * 2 * len(layers) + [s + 1] * 2 * len(layers)
        assert len(seen) == len(starts)
        for (c, n), r0 in zip(seen, starts):
            assert torch.equal(c, cos[r0 : r0 + c.shape[0]]) and torch.equal(n, sin[r0 : r0 + c.shape[0]])
        step = seen[2 * len(layers):]
        assert all(c._base is step[0][0]._base for c, _ in step[: 2 * len(layers)])
        # the same tokens with every position one further: the table rows move, and so do the logits
        shifted, _ = _spec_generate(cfg, layers, head, ids, 2, s + 4, shift=1)
    assert not torch.equal(base[0], shifted[0]) and not torch.equal(base[1], shifted[1])


# ------------------------------------------------------------------------------------------------
# the cache's length follows sequence_len_offset
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["device", "offloaded"])
def test_commit_to_rule(monkeypatch, kind):
    with _host_memory(monkeypatch):
        c = KVCache(2, 16, 1, 128, "cpu") if kind == "device" else OffloadedKVCache(2, 1, 16, 1, 128, "cpu")
    k = torch.zeros(5, 1, 128, dtype=torch.bfloat16)
    c.commit_to(0)                                           # an empty cache at offset 0
    c.append(0, k, k)
    c.commit_to(0)                                           # a later layer of the same forward
    assert (len(c), c._pending) == (0, 5)
    for bad in (1, 4, 6, 10):                                # neither this forward nor the next
        with pytest.raises(ValueError, match=f"sequence_len_offset {bad} does not follow"):
            c.commit_to(bad)
        assert (len(c), c._pending) == (0, 5)
    c.commit_to(5)                                           # the next forward: the pending rows are committed
    assert (len(c), c._pending) == (5, 0)
    c.commit_to(5)
    for bad in (0, 4, 6):                                    # back, or past the pending rows
        with pytest.raises(ValueError, match="does not follow"):
            c.commit_to(bad)
    assert len(c) == 5


def test_offset_that_moves_back_or_jumps_raises(monkeypatch, tiny):
    cfg, mc = tiny
    s = 300
    ids = _prompt(cfg, s)
    _, layers, head = _models(cfg, mc)
    with oracle_ops():
        out, ip = _spec_generate(cfg, layers, head, ids, 1, s + 8)
        cache = ip.key_value_memory_dict["b200_kv_cache"]
        tok = out[-1][-1].float().argmax().view(1, 1)
        for off in (s - 1, 0, s + 2, s + 5):               # s would re-run the last step, s + 1 is the next
            ip.sequence_len_offset = off
            with pytest.raises(ValueError, match="does not follow"):
                spec_forward(layers, head, tok, ip, rotary_table(cfg, s + 8))
            assert (len(cache), cache._pending) == (s, 1)
        ip.sequence_len_offset = s + 1
        spec_forward(layers, head, tok, ip, rotary_table(cfg, s + 8))
    assert len(cache) == s + 1 and ip.sequence_len_offset == s + 2


# ------------------------------------------------------------------------------------------------
# refusals, nothing launched; inference_params=None unchanged
# ------------------------------------------------------------------------------------------------
def _layer(cfg, mc, **kw):
    return spec_layers(LongVITAConfig.tiny(layers=1, vit_layers=1), mc, **kw)[0]


def test_refusals(lib, monkeypatch, tiny):  # noqa: F811
    cfg, mc = tiny
    s = 16
    x = torch.zeros(s, 1, cfg.hidden_size, dtype=torch.bfloat16)
    table = rotary_table(cfg, 64)

    def call(layer, ip, **kw):
        return layer(hidden_states=kw.pop("x", x), rotary_pos_emb=table, inference_params=ip, **kw)

    cp = _layer(cfg, mc, context_parallel_size=2)
    ip = inference_params(64)
    with pytest.raises(NotImplementedError, match="context parallelism"):
        call(cp, ip)
    layer = _layer(cfg, mc)
    ip.max_batch_size = 2
    with pytest.raises(NotImplementedError, match="max_batch_size 2"):
        call(layer, ip)
    with pytest.raises(NotImplementedError, match="micro-batch 1"):
        call(layer, inference_params(64), x=torch.zeros(s, 2, cfg.hidden_size, dtype=torch.bfloat16))
    with monkeypatch.context() as m:
        m.setitem(sys.modules, "long_vita_megatron.training.utils",
                  types.SimpleNamespace(get_actual_seq_len=lambda: [6, 16]))
        with pytest.raises(NotImplementedError, match="packed samples.*cannot be combined with a KV cache"):
            call(layer, inference_params(64))
    with torch.enable_grad():
        with pytest.raises(NotImplementedError, match="with gradients enabled"):
            call(layer, inference_params(64), x=x.clone().requires_grad_(True))
    with pytest.raises(ValueError, match="rotary_pos_emb has 64 rows"):
        call(layer, types.SimpleNamespace(**{**vars(inference_params(64)), "sequence_len_offset": 60}))
    with pytest.raises(ValueError, match="host dtype"):
        _layer(cfg, mc, kv_host_dtype=torch.float16)
    assert lib.calls == []


def _names(calls):
    return [c[0] for c in calls]


def test_no_inference_params_makes_the_calls_it_made_before(lib, monkeypatch, tiny):  # noqa: F811
    """Without inference_params the layer makes the calls of the prefill-only layer: RMSNorm, the QKV GEMM, RoPE on
    q and k, causal attention over its own rows, the O GEMM, the fused add + RMSNorm, gate|up with SwiGLU, down, and
    the residual add; a cached generation on the same layer does not change them."""
    cfg, mc = tiny
    s = 16
    x = torch.zeros(s, 1, cfg.hidden_size, dtype=torch.bfloat16)
    table = rotary_table(cfg, s)
    layer = _layer(cfg, mc)
    layer(hidden_states=x, rotary_pos_emb=table, inference_params=None)
    before = list(lib.calls)
    assert _names(before) == ["lv_rmsnorm", "lv_gemm_bias_act", "lv_rope", "lv_rope", "lv_attn_fwd",
                              "lv_gemm_bias_act", "lv_rmsnorm", "lv_gemm_bias_act", "lv_gemm_bias_act",
                              "lv_ls_residual"]
    att = before[4][1]._obj
    assert (att.sq, att.sk, att.causal) == (s, s, 1)
    lib.calls.clear()
    ip = inference_params(s + 4)
    layer(hidden_states=x, rotary_pos_emb=rotary_table(cfg, s + 4), inference_params=ip)
    ip.sequence_len_offset += s
    layer(hidden_states=x[:1], rotary_pos_emb=rotary_table(cfg, s + 4), inference_params=ip)
    assert "lv_attn_decode_merge" in _names(lib.calls)        # the decode step ran
    lib.calls.clear()
    layer(hidden_states=x, rotary_pos_emb=table, inference_params=None)
    assert _names(lib.calls) == _names(before)
    assert lib.calls[4][1]._obj.sk == s and lib.calls[2][3:] == before[2][3:]
