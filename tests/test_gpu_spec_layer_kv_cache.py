"""Megatron's `--use-kv-cache` protocol on the `--spec` decoder layer, on the H100.

Megatron's loop is restated as in tests/test_spec_layer_kv_cache_host.py (the layers built with `build_module`, each
called with the shared `inference_params` and the rotary table of `max_sequence_length` positions, then the final norm
and the LM head) and compared with B200GPTVLModel under the same protocol.  Both run the same kernels on the same
re-ordered weights, so their logits are equal, not close.

1. Tiny geometry: the prompt and 16 greedy decode steps, device cache and cache with 1 of 2 layers on the host.
2. 4 layers of the 14B geometry at 18 432 tokens, 2 host layers: the prefill logits equal the `--spec` forward without
   a cache, and 16 teacher-forced decode steps equal the mirror's.
3. 1 058 816 tokens, 2 layers both on the host: the prefill (row-chunked) fits, its logits and the first 2 decode
   steps equal the mirror's; the peak device memory and the pinned bytes are printed (`pytest -s`).
"""
import dataclasses
import gc

import pytest
import torch

from tests.test_gpu_offloaded_cache import ROW, _need_host
from tests.test_spec_layer_kv_cache_host import inference_params, rotary_table, spec_layers

pytestmark = pytest.mark.gpu


def _placed(monkeypatch, n_dev):
    from long_vita_b200 import kv_cache

    monkeypatch.setattr(kv_cache, "device_layers", lambda *a, **kw: n_dev)


def _setup(cfg, seed):
    from long_vita_b200.megatron import checkpoint as ck
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel
    from long_vita_b200.weights import synthetic_state_dict

    mc = ck.hf_to_mcore(synthetic_state_dict(cfg, seed=seed, device="cuda", perturb=True), cfg)
    mirror = B200GPTVLModel(cfg, mc)
    layers = spec_layers(cfg, mc)
    head = (mirror.word_embeddings, mirror.final_layernorm, mirror.output_weight, cfg.rms_norm_eps)
    return mirror, layers, head


def _spec(layers, head, ids, ip, table):
    """One forward of Megatron's loop; logits of the last row [1, V] (the GEMV of a masked LM head)."""
    from long_vita_b200 import ops

    emb, norm_w, out_w, eps = head
    s = ids.shape[1]
    x = ops.embed_scatter(ids, emb).view(s, 1, -1)
    for layer in layers:
        x, _ = layer(hidden_states=x, attention_mask=None, rotary_pos_emb=table, inference_params=ip)
    h = ops.rmsnorm(x.view(s, -1), norm_w, eps)
    del x
    if ip is not None:
        ip.sequence_len_offset += s
    return ops.linear(h[-1:], out_w)


def _mirror(model, ids, ip, pos0):
    s = ids.shape[1]
    mask = torch.zeros(1, s, dtype=torch.bool, device="cuda")
    mask[0, -1] = True
    pos = torch.arange(pos0, pos0 + s, device="cuda").unsqueeze(0)
    return model(ids, pos, None, inference_params=ip, logit_mask=mask)[0]


def _mirror_params(capacity):
    import types

    return types.SimpleNamespace(key_value_memory_dict={}, max_sequence_length=capacity, use_kv_cache=True)


def _run(cfg, mirror, layers, head, ids, steps, forced=None):
    """The mirror's and the --spec loop's last-row logits for the prompt and `steps` decode steps, each fed the
    mirror's greedy token (or `forced`); returns (mirror logits, spec logits, the spec loop's cache)."""
    s = ids.shape[1]
    cap = s + steps
    mip, want, toks = _mirror_params(cap), [], []
    with torch.no_grad():
        want.append(_mirror(mirror, ids, mip, 0))
        for i in range(steps):
            toks.append(want[-1][-1].float().argmax().view(1, 1) if forced is None else forced[:, i : i + 1])
            want.append(_mirror(mirror, toks[-1], mip, s + i))
        del mip
        gc.collect()
        ip, got = inference_params(cap), []
        got.append(_spec(layers, head, ids, ip, rotary_table(cfg, cap, "cuda")))
        for i in range(steps):
            got.append(_spec(layers, head, toks[i], ip, rotary_table(cfg, cap, "cuda")))
    return want, got, ip.key_value_memory_dict["b200_kv_cache"]


@pytest.mark.parametrize("n_dev", [None, 1])
def test_tiny_spec_loop_equals_the_mirror(lib_built, monkeypatch, n_dev):
    from long_vita_b200.config import LongVITAConfig
    from long_vita_b200.kv_cache import KVCache, OffloadedKVCache

    cfg = LongVITAConfig.tiny(layers=2, vit_layers=1)
    mirror, layers, head = _setup(cfg, 17)
    ids = torch.randint(0, cfg.vocab_size, (1, 2000), device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    if n_dev is not None:
        _placed(monkeypatch, n_dev)
    want, got, cache = _run(cfg, mirror, layers, head, ids, 16)
    assert type(cache) is (KVCache if n_dev is None else OffloadedKVCache)
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape == (1, cfg.vocab_size) and torch.equal(a, b), i


def _geometry_14b(layers):
    from long_vita_b200.config import LongVITAConfig

    cfg = LongVITAConfig()
    return dataclasses.replace(cfg, num_hidden_layers=layers,
                               visual=dataclasses.replace(cfg.visual, num_hidden_layers=1))


def test_14b_geometry_at_18432_tokens_with_two_host_layers(lib_built, monkeypatch):
    from long_vita_b200.kv_cache import OffloadedKVCache

    s, steps = 18432, 16
    _need_host(2 * 2 * (s + steps) * ROW, "two 18 432-token caches")
    cfg = _geometry_14b(4)
    mirror, layers, head = _setup(cfg, 9)
    g = torch.Generator("cuda").manual_seed(4)
    ids = torch.randint(0, cfg.vocab_size, (1, s), device="cuda", generator=g)
    forced = torch.randint(0, cfg.vocab_size, (1, steps), device="cuda", generator=g)
    with torch.no_grad():
        plain = _spec(layers, head, ids, None, rotary_table(cfg, s, "cuda"))
    _placed(monkeypatch, 2)
    want, got, cache = _run(cfg, mirror, layers, head, ids, steps, forced)
    assert isinstance(cache, OffloadedKVCache) and cache.n_dev == 2 and len(cache.host) == 2
    assert torch.equal(got[0], plain) and torch.equal(got[0], want[0])
    for i in range(1, steps + 1):
        assert torch.equal(got[i], want[i]), i


def test_million_token_prompt_with_both_layers_on_the_host(lib_built, monkeypatch):
    from long_vita_b200.kv_cache import OffloadedKVCache

    T, steps = 1058816, 2
    _need_host(2 * (T + steps) * ROW, "the 1 058 816-token prompt")
    cfg = _geometry_14b(2)
    mirror, layers, head = _setup(cfg, 5)
    ids = torch.randint(0, cfg.vocab_size, (1, T), device="cuda", generator=torch.Generator("cuda").manual_seed(6))
    _placed(monkeypatch, 0)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    want, got, cache = _run(cfg, mirror, layers, head, ids, steps)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print(f"\n[spec layer 1M] peak device memory above the weights: {peak / 2**30:.2f} GiB; the cache pins "
          f"{cache.host_bytes() / 1e9:.2f} GB and holds {cache.bytes()} device bytes")
    assert isinstance(cache, OffloadedKVCache) and cache.n_dev == 0
    assert cache.host_bytes() == 2 * (T + steps) * 4096 and cache.bytes() == 0
    for i in range(steps + 1):
        assert torch.equal(got[i], want[i]), i
    assert peak <= 60 * 2**30
