"""The row-chunked decoder layer on the H100 (hf.modeling.row_chunks / DecoderLayer.forward).

* Bit-identity: a 4-layer model of the 14B geometry with 64 frames, at T = 18 432 (the bench prompt) and 16 897 (a
  ragged last chunk), with the chunk constants patched down so that each layer runs in five chunks, must give
  torch.equal hidden states and logits, K/V-cache prefill + 8 greedy tokens, a packed row, B200GPTVLModel with a
  logit mask and the `--spec` layer, against the one-chunk run.
* Memory: a text-only 2-layer forward at the 1M bench length (1 058 816 tokens) finishes within the per-token bound of
  the chunked layer (x, QKV, attention output, RoPE tables: 35 328 bytes per token) plus the chunk temporaries, and two
  chunk sizes give bit-identical last-token logits.
* The attention launch the chunked layer makes at that length, beyond the longest length tests/
  test_gpu_attention_fwd_ref.py covers: sampled rows against the float64 reference, diagonal tiles planted.
"""
import dataclasses
from functools import partial

import pytest
import torch

from long_vita_b200.config import LongVITAConfig
from long_vita_b200.synthetic import build_prompt, synthetic_frames
from tests.test_gpu_attention_fwd_ref import D, HKV, HQ, _check, _check_plants, _inputs, _plant_edge_rows, _tile_rows

pytestmark = pytest.mark.gpu

T_1M = 1058816                       # bench.py --frames 4096
ACT_BYTES_PER_TOKEN = 2 * (5120 + 7168 + 5120 + 2 * 128)       # x, QKV, attention output, cos + sin (bf16)


@pytest.fixture
def chunked(monkeypatch):
    """Patches the chunk constants: chunked(threshold, rows)."""
    from long_vita_b200.hf import modeling

    def set_(threshold, rows):
        monkeypatch.setattr(modeling, "ROW_CHUNK_THRESHOLD", threshold)
        monkeypatch.setattr(modeling, "ROW_CHUNK", rows)
    return set_


@pytest.fixture(scope="module")
def M(lib_built):
    from long_vita_b200.hf import modeling

    cfg = dataclasses.replace(LongVITAConfig.long_vita_14b(), num_hidden_layers=4)
    model = modeling.LongVITAForCausalLM.from_synthetic(cfg, seed=7, device="cuda", perturb=True)
    frames = synthetic_frames(cfg, 64, device="cuda")
    yield cfg, model, frames, modeling
    del model, frames
    torch.cuda.empty_cache()


def _prompt(cfg, T):
    ids, idx = build_prompt(cfg, 64, 16, pad_multiple=2048) if T == 18432 else build_prompt(cfg, 64, 385, pad_multiple=1)
    assert ids.shape[1] == T
    return ids.cuda(), idx.cuda()


def _twice(chunked, fn, modeling, T):
    """fn() with one chunk, then with 4096-row chunks (five chunks at both lengths)."""
    whole = fn()
    chunked(4096, 4096)
    assert len(modeling.row_chunks(T)) == 5
    return whole, fn()


def _equal(a, b):
    if isinstance(a, torch.Tensor):
        return torch.equal(a, b)
    return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("T", [18432, 16897])
def test_hidden_states_and_kept_logits(M, chunked, T):
    cfg, model, frames, modeling = M
    ids, idx = _prompt(cfg, T)

    def run():
        a = model(input_ids=ids, images=frames, image_indices=idx, num_logits_to_keep=64, output_hidden_states=True)
        b = model(input_ids=ids, images=frames, image_indices=idx, num_logits_to_keep=64)     # x updated in place
        return a.logits, a.hidden_states, b.logits

    whole, chunk = _twice(chunked, run, modeling, T)
    assert _equal(chunk, whole)
    assert torch.equal(whole[0], whole[2]) and whole[0].float().abs().sum() > 0


def test_cache_prefill_and_greedy_tokens(M, chunked):
    cfg, model, frames, modeling = M
    ids, idx = _prompt(cfg, 18432)

    def run():
        out = model(input_ids=ids, images=frames, image_indices=idx, use_cache=True, num_logits_to_keep=1,
                    max_cache_len=ids.shape[1] + 8)
        cache, logits = out.past_key_values, [out.logits]
        for _ in range(8):
            tok = logits[-1][0, -1].float().argmax().view(1, 1)
            logits.append(model(input_ids=tok, past_key_values=cache, use_cache=True, num_logits_to_keep=1).logits)
        n = len(cache)
        return logits, [c[:n] for c in cache.k], [c[:n] for c in cache.v]

    whole, chunk = _twice(chunked, run, modeling, 18432)
    assert _equal(chunk, whole)


def test_packed_row(M, chunked):
    cfg, model, frames, modeling = M
    ids, idx = _prompt(cfg, 18432)
    pos = torch.cat([torch.arange(9000), torch.arange(18432 - 9000)]).unsqueeze(0).cuda()   # boundary inside a chunk
    whole, chunk = _twice(chunked, lambda: model(input_ids=ids, images=frames, image_indices=idx, position_ids=pos,
                                                 num_logits_to_keep=300).logits, modeling, 18432)
    assert torch.equal(chunk, whole)


def test_megatron_model_with_logit_mask(M, chunked):
    from long_vita_b200.megatron import checkpoint as ck
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel

    cfg, model, frames, modeling = M
    gpt = B200GPTVLModel(cfg, ck.hf_to_mcore(model.state_dict(), cfg))
    ids, idx = _prompt(cfg, 16897)
    s = ids.shape[1]
    mask = torch.zeros(1, s, dtype=torch.bool, device="cuda")
    mask[0, [0, 3455, 3456, 9000, s - 1]] = True
    whole, chunk = _twice(chunked, lambda: gpt(ids, torch.arange(s, device="cuda").unsqueeze(0), None, logit_mask=mask,
                                               external_inputs={"images": frames, "indices": idx}), modeling, s)
    assert whole.shape == (1, 5, cfg.vocab_size) and torch.equal(chunk, whole)


def test_spec_layer(M, chunked):
    import types

    from long_vita_b200.megatron import checkpoint as ck
    from long_vita_b200.megatron.transformer_layer import B200TransformerLayer

    cfg, model, _, modeling = M
    mc = ck.hf_to_mcore(model.state_dict(), cfg)
    mcfg = types.SimpleNamespace(hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_attention_heads,
                                 num_query_groups=cfg.num_key_value_heads, kv_channels=cfg.head_dim,
                                 ffn_hidden_size=cfg.intermediate_size, layernorm_epsilon=cfg.rms_norm_eps,
                                 hidden_dropout=0.0, attention_dropout=0.0, params_dtype=torch.bfloat16)
    layer = B200TransformerLayer(mcfg, layer_number=1).cuda()
    layer.load_state_dict({k[len("decoder.layers.1."):]: v for k, v in mc.items() if k.startswith("decoder.layers.1.")})
    s = 16897
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(s, 1, cfg.hidden_size, generator=g, device="cuda").to(torch.bfloat16)
    keep = x.clone()
    inv = modeling.rope_inv_freq(cfg, "cuda")
    freqs = torch.outer(torch.arange(s, device="cuda").float(), inv)
    rotary = torch.cat((freqs, freqs), dim=-1).view(s, 1, 1, cfg.head_dim)
    with torch.no_grad():
        whole, chunk = _twice(chunked, lambda: layer(hidden_states=x, rotary_pos_emb=rotary)[0], modeling, s)
    assert torch.equal(chunk, whole) and torch.equal(x, keep)


def test_one_million_tokens_text_only_two_layers(lib_built, chunked):
    from long_vita_b200.hf import modeling

    cfg = dataclasses.replace(LongVITAConfig.long_vita_14b(), num_hidden_layers=2)
    model = modeling.LongVITAForCausalLM.from_synthetic(cfg, seed=11, device="cuda")
    ids = torch.randint(0, cfg.vocab_size, (1, T_1M), generator=torch.Generator().manual_seed(2)).cuda()
    logits = []
    for rows in (65536, 40000):
        chunked(262144, rows)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        with torch.no_grad():
            logits.append(model(input_ids=ids, num_logits_to_keep=1).logits)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
        n = len(modeling.row_chunks(T_1M))
        chunk_rows = max(r1 - r0 for r0, r1 in modeling.row_chunks(T_1M))
        # per chunk row: the norm output, the O-projection output, the SwiGLU output and the MLP output
        temp = chunk_rows * 2 * (5120 + 5120 + 13824 + 5120)
        print(f"[1M] {n} chunks of <= {chunk_rows} rows: peak above the resident model and ids {peak / 2**30:.2f} GiB "
              f"= {peak / T_1M:.0f} B/token; bound {ACT_BYTES_PER_TOKEN} B/token + {temp / 2**30:.2f} GiB")
        assert peak <= T_1M * (ACT_BYTES_PER_TOKEN + 64) + temp, peak
    assert torch.equal(logits[0], logits[1]) and torch.isfinite(logits[0].float()).all()
    del model
    torch.cuda.empty_cache()


def test_attention_at_one_million_tokens(lib_built):
    """The decoder's attention call at T = 1 058 816: 40:8 x 128, causal, one launch; sampled rows (ends, tile edges,
    random) and every row of four diagonal tiles planted, against the float64 reference."""
    from long_vita_b200 import ops
    from tests.attn_fwd_ref import _sample_rows

    T = T_1M
    q, k, v = _inputs(1, T, T, HQ, HKV, D, seed=T)
    n_t = T // 128
    prow = _tile_rows([0, 1, n_t // 2, n_t - 1], T)
    planted = _plant_edge_rows(q, k, prow, torch.arange(T))
    out, lse = ops.attention_fwd(q, k, v, causal=True, return_lse=True)
    rows = torch.unique(torch.cat([_sample_rows(160, T, seed=T), prow]))
    ref = _check(out, lse, q, k, v, causal=True, rows=rows, label=f"prefill {T} sampled")
    _check_plants(ref, rows, v, planted)
