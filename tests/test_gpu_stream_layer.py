"""The streamed decoder layer on the H100 (hf.modeling.STREAM_THRESHOLD / DecoderLayer._forward_streamed).

* Bit-identity: a 4-layer model of the 14B geometry with 64 frames, at T = 18 432 (the bench prompt) and 16 897 (a
  ragged last span), with the thresholds patched to 4096 rows so that each layer runs in five spans, must give
  torch.equal hidden states and kept logits (HF), B200GPTVLModel logits under a logit mask and `--spec` layer output,
  streamed against the whole-tensor and the row-chunked runs; inputs_embeds are left as they were.
* Attention: the span calls of a streamed layer, each span's queries over its key prefix, stacked, are torch.equal to
  one whole call, output and LSE.
* The longest launch of the 2M-token prompt: its last span, 63 488 query rows over all 2 115 584 keys (40:8 x 128),
  sampled rows and every row of four planted diagonal tiles against the float64 reference.
* Memory: a 2-layer forward of the 8192-frame bench prompt (2 115 584 tokens, frames on the device) stays within the
  streamed layer's per-token bound (x, K|V, RoPE tables: 14 848 bytes per token) plus the span and ViT-chunk
  temporaries, and two span sizes give bit-identical, finite last-token logits.
"""
import dataclasses
import time

import pytest
import torch

from long_vita_b200.config import LongVITAConfig
from long_vita_b200.synthetic import build_prompt, synthetic_frames
from tests.test_gpu_attention_fwd_ref import D, HKV, HQ, _check, _check_plants, _inputs, _plant_edge_rows, _tile_rows

pytestmark = pytest.mark.gpu

T_2M = 2115584                       # bench.py --frames 8192
STREAM_BYTES_PER_TOKEN = 2 * (5120 + 2 * 1024 + 2 * 128)        # x, K|V, cos + sin (bf16)


@pytest.fixture
def plan(monkeypatch):
    """plan(name): the whole-tensor layer, or 4096-row spans row-chunked or streamed (five spans at both lengths)."""
    from long_vita_b200.hf import modeling

    def set_(name):
        monkeypatch.setattr(modeling, "ROW_CHUNK_THRESHOLD", 262144 if name == "whole" else 4096)
        monkeypatch.setattr(modeling, "ROW_CHUNK", 65536 if name == "whole" else 4096)
        monkeypatch.setattr(modeling, "STREAM_THRESHOLD", 4096 if name == "streamed" else 1179648)
    return set_


def _three(plan, fn, T):
    from long_vita_b200.hf import modeling

    out = {}
    for name in ("whole", "chunked", "streamed"):
        plan(name)
        assert len(modeling.row_chunks(T)) == (1 if name == "whole" else 5)
        assert modeling.streams(T, modeling.attention_step()) == (name == "streamed")
        out[name] = fn()
    return out


def _equal(a, b):
    if isinstance(a, torch.Tensor):
        return torch.equal(a, b)
    return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))


@pytest.fixture(scope="module")
def M(lib_built):
    from long_vita_b200.hf import modeling

    cfg = dataclasses.replace(LongVITAConfig.long_vita_14b(), num_hidden_layers=4)
    model = modeling.LongVITAForCausalLM.from_synthetic(cfg, seed=7, device="cuda", perturb=True)
    model.model.vision_chunk = 16          # four ViT chunks: four per-chunk scatters when streamed
    frames = synthetic_frames(cfg, 64, device="cuda")
    yield cfg, model, frames, modeling
    del model, frames
    torch.cuda.empty_cache()


def _prompt(cfg, T):
    ids, idx = build_prompt(cfg, 64, 16, pad_multiple=2048) if T == 18432 else build_prompt(cfg, 64, 385, pad_multiple=1)
    assert ids.shape[1] == T
    return ids.cuda(), idx.cuda()


@pytest.mark.parametrize("T", [18432, 16897])
def test_hidden_states_and_kept_logits(M, plan, T):
    cfg, model, frames, modeling = M
    ids, idx = _prompt(cfg, T)

    def run():
        a = model(input_ids=ids, images=frames, image_indices=idx, num_logits_to_keep=64, output_hidden_states=True)
        b = model(input_ids=ids, images=frames, image_indices=idx, num_logits_to_keep=64)     # x updated in place
        return a.logits, a.hidden_states, b.logits

    r = _three(plan, run, T)
    assert _equal(r["streamed"], r["whole"]) and _equal(r["chunked"], r["whole"])
    assert torch.equal(r["whole"][0], r["whole"][2]) and r["whole"][0].float().abs().sum() > 0


def test_inputs_embeds_are_not_overwritten(M, plan):
    cfg, model, frames, modeling = M
    g = torch.Generator(device="cuda").manual_seed(3)
    emb = torch.randn(1, 16897, cfg.hidden_size, generator=g, device="cuda").to(torch.bfloat16)
    keep = emb.clone()
    r = _three(plan, lambda: model(inputs_embeds=emb, num_logits_to_keep=64).logits, 16897)
    assert torch.equal(r["streamed"], r["whole"]) and torch.equal(r["chunked"], r["whole"]) and torch.equal(emb, keep)


@pytest.mark.parametrize("via", ["external_inputs", "inference_params"])
def test_megatron_model_with_logit_mask(M, plan, via):
    """Called directly, and as Megatron's generation loop calls it without --use-kv-cache (inputs in
    inference_params, use_kv_cache False)."""
    import types

    from long_vita_b200.megatron import checkpoint as ck
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel

    cfg, model, frames, modeling = M
    gpt = B200GPTVLModel(cfg, ck.hf_to_mcore(model.state_dict(), cfg))
    gpt.vision_chunk = 16
    ids, idx = _prompt(cfg, 16897)
    s = ids.shape[1]
    mask = torch.zeros(1, s, dtype=torch.bool, device="cuda")
    mask[0, [0, 3455, 3456, 9000, s - 1]] = True
    ext = {"images": frames, "indices": idx}
    pos = torch.arange(s, device="cuda").unsqueeze(0)
    if via == "external_inputs":
        run = lambda: gpt(ids, pos, None, logit_mask=mask, external_inputs=ext)             # noqa: E731
    else:
        run = lambda: gpt(ids, pos, None, inference_params=types.SimpleNamespace(                # noqa: E731
            external_inputs=ext, key_value_memory_dict={}, logit_mask=mask, use_kv_cache=False))
    scatters = []
    scatter = modeling.scatter_images

    def counted(*a, **kw):
        scatters.append(1)
        return scatter(*a, **kw)
    modeling.scatter_images = counted
    try:
        r = _three(plan, run, s)
    finally:
        modeling.scatter_images = scatter
    assert len(scatters) == 1                     # the streamed run only
    assert r["whole"].shape == (1, 5, cfg.vocab_size)
    assert torch.equal(r["streamed"], r["whole"]) and torch.equal(r["chunked"], r["whole"])


def test_spec_layer(M, plan):
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
        r = _three(plan, lambda: layer(hidden_states=x, rotary_pos_emb=rotary)[0], s)
    assert torch.equal(r["streamed"], r["whole"]) and torch.equal(r["chunked"], r["whole"]) and torch.equal(x, keep)


def test_span_attention_calls_stack_to_the_whole_call(lib_built, plan):
    from long_vita_b200 import ops
    from long_vita_b200.hf import modeling

    T = 16897
    plan("streamed")
    q, k, v = _inputs(1, T, T, HQ, HKV, D, seed=T + 7)
    out, lse = ops.attention_fwd(q, k, v, causal=True, return_lse=True)
    outs, lses = [], []
    for r0, r1 in modeling.row_chunks(T):
        o, l = ops.attention_fwd(q[:, r0:r1], k[:, :r1], v[:, :r1], causal=True, return_lse=True)
        outs.append(o)
        lses.append(l)
    assert len(outs) == 5
    assert torch.equal(torch.cat(outs, dim=1), out) and torch.equal(torch.cat(lses, dim=2), lse)


def test_last_span_of_the_2m_prompt(lib_built):
    """The longest attention launch of the 8192-frame prompt: its last span's queries over every key."""
    from long_vita_b200 import ops
    from long_vita_b200.hf import modeling
    from tests.attn_fwd_ref import _sample_rows

    r0, r1 = modeling.row_chunks(T_2M)[-1]
    assert r1 == T_2M
    sq = r1 - r0
    q, k, v = _inputs(1, sq, T_2M, HQ, HKV, D, seed=T_2M)
    n_t = sq // 128
    prow = _tile_rows([0, 1, n_t // 2, n_t - 1], sq)
    planted = _plant_edge_rows(q, k, prow, torch.arange(sq) + r0)
    out, lse = ops.attention_fwd(q, k, v, causal=True, return_lse=True)
    rows = torch.unique(torch.cat([_sample_rows(160, sq, seed=sq), prow]))
    ref = _check(out, lse, q, k, v, causal=True, rows=rows, label=f"span [{r0}, {r1}) of {T_2M} sampled")
    _check_plants(ref, rows, v, planted)


def test_8192_frames_two_layers(lib_built, monkeypatch):
    from long_vita_b200.hf import modeling

    cfg = dataclasses.replace(LongVITAConfig.long_vita_14b(), num_hidden_layers=2)
    model = modeling.LongVITAForCausalLM.from_synthetic(cfg, seed=11, device="cuda")
    ids, idx = build_prompt(cfg, 8192, 16, pad_multiple=2048)
    assert ids.shape[1] == T_2M
    ids, idx = ids.cuda(), idx.cuda()
    frames = synthetic_frames(cfg, 8192, device="cuda")
    # the ViT chunk: hidden, norm output, QKV, attention output, projection output, residual sum, fc1 output
    vit_temp = modeling.VISION_CHUNK * 1025 * 2 * (6 * 1024 + 3072 + 4096)
    logits = []
    for rows in (65536, 40000):
        monkeypatch.setattr(modeling, "ROW_CHUNK", rows)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t0 = time.time()
        with torch.no_grad():
            logits.append(model(input_ids=ids, images=frames, image_indices=idx, num_logits_to_keep=1).logits)
        torch.cuda.synchronize()
        secs = time.time() - t0
        peak = torch.cuda.max_memory_allocated() - base
        spans = modeling.row_chunks(T_2M)
        span_rows = max(r1 - r0 for r0, r1 in spans)
        # per span row: the Q span, the attention output, the O-projection output, the norm output, the SwiGLU output
        # and the MLP output
        temp = span_rows * 2 * (5 * 5120 + 13824)
        print(f"[2M] {len(spans)} spans of <= {span_rows} rows, {secs:.1f} s: peak above the resident model, frames "
              f"and ids {peak / 2**30:.2f} GiB = {peak / T_2M:.0f} B/token; bound {STREAM_BYTES_PER_TOKEN} B/token + "
              f"{temp / 2**30:.2f} + {vit_temp / 2**30:.2f} GiB")
        assert peak <= T_2M * (STREAM_BYTES_PER_TOKEN + 64) + temp + vit_temp, peak
    assert torch.equal(logits[0], logits[1]) and torch.isfinite(logits[0].float()).all()
    del model, frames
    torch.cuda.empty_cache()
