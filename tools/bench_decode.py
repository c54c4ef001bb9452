"""Decode-step timing with the K/V cache (SURVEY.md 8f-2) next to the reference's re-prefill loop.

    python tools/bench_decode.py [--frames 64] [--tokens 16] [--layers 48]

Prefills the configured prompt once with use_cache=True, then times `--tokens` single-token forward passes
(CUDA events, after 3 warm-up tokens).  Reports ms / token, the HBM traffic a step must move (all decoder
weights + LM head once, the K/V cache once) and the fraction of the measured HBM peak that corresponds to,
plus the kernel-only time of `ops.attention_decode` at this context.  The reference's Megatron serving loop
feeds the whole sequence for every token (generation.py:127-135), so its per-token cost is the prefill time
`bench.py` reports.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from long_vita_b200 import ops  # noqa: E402
from long_vita_b200.config import LongVITAConfig  # noqa: E402
from long_vita_b200.hf.modeling import LongVITAForCausalLM  # noqa: E402
from long_vita_b200.synthetic import build_prompt, synthetic_frames  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--tokens", type=int, default=16)
    ap.add_argument("--layers", type=int, default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    cfg = LongVITAConfig.long_vita_14b()
    model = LongVITAForCausalLM.from_synthetic(cfg, seed=1234, device="cuda", num_layers=a.layers)
    n_layers = len(model.model.layers)
    ids, idx = build_prompt(cfg, a.frames, n_text=16, pad_multiple=2048)
    frames = synthetic_frames(cfg, a.frames)
    S = ids.shape[1]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = model(input_ids=ids.cuda(), images=frames.cuda(), image_indices=idx.cuda(), use_cache=True, num_logits_to_keep=1,
                max_cache_len=S + a.tokens + 8)
    e1.record()
    torch.cuda.synchronize()
    prefill_ms = e0.elapsed_time(e1)
    cache = out.past_key_values
    tok = out.logits[0, -1].float().argmax().view(1, 1)
    times = []
    n0 = ops.launch_count()
    for i in range(a.tokens + 3):
        e0.record()
        out = model(input_ids=tok, past_key_values=cache, use_cache=True, num_logits_to_keep=1)
        tok = out.logits[0, -1].float().argmax().view(1, 1)
        e1.record()
        torch.cuda.synchronize()
        if i >= 3:
            times.append(e0.elapsed_time(e1))
    launches = (ops.launch_count() - n0) / (a.tokens + 3)
    ms = sorted(times)[len(times) // 2]
    L = len(cache)
    per_layer_w = (cfg.q_size + 2 * cfg.kv_size) * cfg.hidden_size + cfg.q_size * cfg.hidden_size + 3 * cfg.intermediate_size * cfg.hidden_size
    w_bytes = 2 * (n_layers * per_layer_w + cfg.vocab_size * cfg.hidden_size)
    kv_bytes = 2 * 2 * n_layers * L * cfg.kv_size
    try:
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:  # noqa: BLE001
        peak = 3350.0       # H100 SXM data sheet (HBM3), the same fallback as bench.py
    # kernel-only: the decode attention of one layer at this context
    q = torch.randn(cfg.num_attention_heads, cfg.head_dim, device="cuda", dtype=torch.bfloat16)
    for _ in range(3):
        ops.attention_decode(q, cache.k[0], cache.v[0], L)
    e0.record()
    for _ in range(20):
        ops.attention_decode(q, cache.k[0], cache.v[0], L)
    e1.record()
    torch.cuda.synchronize()
    attn_ms = e0.elapsed_time(e1) / 20
    print(json.dumps({
        "what": "decode step with K/V cache", "context": L, "layers": n_layers, "ms_per_token": ms,
        "tokens_per_s": 1e3 / ms, "prefill_ms": prefill_ms, "speedup_vs_re_prefill": prefill_ms / ms,
        "bytes_per_token": w_bytes + kv_bytes, "hbm_gbs": (w_bytes + kv_bytes) / ms / 1e6,
        "hbm_frac": (w_bytes + kv_bytes) / ms / 1e6 / peak, "lv_launches_per_token": launches,
        "attn_decode_ms_per_layer": attn_ms, "attn_decode_gbs": 2 * 2 * L * cfg.kv_size / attn_ms / 1e6,
    }))


if __name__ == "__main__":
    main()
