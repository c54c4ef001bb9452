"""Decode under Megatron's `--use-kv-cache` protocol: the `--spec` decoder layer against B200GPTVLModel, on one GPU.

    python tools/bench_spec_decode.py [--context 18432] [--long 1058816] [--steps 16] [--rounds 3] [--out DIR]

Both paths run Megatron's loop (the prompt once, then one token per forward).  The `--spec` loop is the one a Megatron
job runs: every forward builds the rotary table of `max_sequence_length` positions (RotaryEmbedding.forward, as
megatron-core 0.7 does), calls each B200TransformerLayer with the shared `inference_params`, then the final norm and
the LM head of the last row, and advances `sequence_len_offset`.  The mirror is B200GPTVLModel with a last-row
`logit_mask`.  The mirror runs the `--spec` layers' own re-ordered weights (DecoderLayer objects), so the two differ
only in the per-layer protocol, and the weights exist once.

1. 48 layers of the 14B geometry over a `--context`-token device cache: ms per token over `--steps` decode steps
   (host clock around the steps and a device synchronise), the two paths alternated `--rounds` times.  Then the
   `--spec` forward without a cache over context + 1 tokens: what a token costs when Megatron generates without
   `--use-kv-cache` (the whole prefill again).
2. 2 layers at `--long` tokens with both layers on the host tier: the same alternated decode timing.

Prints one JSON object (and writes it to DIR/spec_decode.json with --out), with the card's name and power limit read
in the same run.  Random weights and tokens: the timings do not depend on their values.
"""
import argparse
import dataclasses
import gc
import json
import os
import statistics
import subprocess
import sys
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from long_vita_b200 import kv_cache, ops  # noqa: E402
from long_vita_b200.config import LongVITAConfig  # noqa: E402
from long_vita_b200.hf import modeling  # noqa: E402
from long_vita_b200.megatron import checkpoint as ck  # noqa: E402
from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel  # noqa: E402
from long_vita_b200.megatron.stub import build_module  # noqa: E402
from long_vita_b200.megatron.transformer_layer import get_b200_layer_spec  # noqa: E402
from long_vita_b200.weights import synthetic_state_dict  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return r.stdout.strip() or torch.cuda.get_device_name(0)


def models(layers):
    """(the --spec layers, the mirror on their DecoderLayers, the head) at the 14B geometry with `layers` layers."""
    base = LongVITAConfig()
    cfg = dataclasses.replace(base, num_hidden_layers=layers, visual=dataclasses.replace(base.visual,
                                                                                       num_hidden_layers=1))
    mcfg = types.SimpleNamespace(hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_attention_heads,
                                 num_query_groups=cfg.num_key_value_heads, kv_channels=cfg.head_dim,
                                 ffn_hidden_size=cfg.intermediate_size, layernorm_epsilon=cfg.rms_norm_eps,
                                 num_layers=layers, params_dtype=torch.bfloat16)
    spec = [build_module(get_b200_layer_spec(), config=mcfg, layer_number=i + 1) for i in range(layers)]
    mirror = B200GPTVLModel(cfg, ck.hf_to_mcore(synthetic_state_dict(cfg, seed=3, device="cuda", llm_layers=[]), cfg))
    mirror.layers = [layer._decoder_layer() for layer in spec]
    head = (mirror.word_embeddings, mirror.final_layernorm, mirror.output_weight, cfg.rms_norm_eps)
    return cfg, spec, mirror, head


def rotary_table(cfg, n):
    inv = modeling.rope_inv_freq(cfg, "cuda")
    freqs = torch.outer(torch.arange(n, device="cuda").float(), inv)
    return torch.cat((freqs, freqs), dim=-1).view(n, 1, 1, cfg.head_dim)


def spec_forward(cfg, layers, head, ids, ip, table_rows):
    emb, norm_w, out_w, eps = head
    s = ids.shape[1]
    table = rotary_table(cfg, table_rows)
    x = ops.embed_scatter(ids, emb).view(s, 1, -1)
    for layer in layers:
        x, _ = layer(hidden_states=x, attention_mask=None, rotary_pos_emb=table, inference_params=ip)
    h = ops.rmsnorm(x.view(s, -1), norm_w, eps)
    del x
    if ip is not None:
        ip.sequence_len_offset += s
    return ops.linear(h[-1:], out_w)


def mirror_forward(model, ids, ip, pos0):
    s = ids.shape[1]
    mask = torch.zeros(1, s, dtype=torch.bool, device="cuda")
    mask[0, -1] = True
    return model(ids, torch.arange(pos0, pos0 + s, device="cuda").unsqueeze(0), None, inference_params=ip,
                 logit_mask=mask)


def seconds(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def decode(cfg, spec, mirror, head, T, steps, rounds):
    """Prefill both paths on a T-token prompt, then alternate `steps`-token decode runs; ms per token per round."""
    cap = T + steps * (rounds + 1)
    ids = torch.randint(0, cfg.vocab_size, (1, T), device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    tok = torch.zeros((1, 1), dtype=torch.int64, device="cuda")
    mip = types.SimpleNamespace(key_value_memory_dict={}, max_sequence_length=cap, use_kv_cache=True)
    sip = types.SimpleNamespace(max_batch_size=1, max_sequence_length=cap, sequence_len_offset=0, batch_size_offset=0,
                                key_value_memory_dict={})
    pos = [T]
    with torch.no_grad():
        prefill = {"mirror_s": seconds(lambda: mirror_forward(mirror, ids, mip, 0)),
                   "spec_s": seconds(lambda: spec_forward(cfg, spec, head, ids, sip, cap))}
        del ids

        def run_mirror():
            for _ in range(steps):
                mirror_forward(mirror, tok, mip, pos[0])
                pos[0] += 1

        def run_spec():
            for _ in range(steps):
                spec_forward(cfg, spec, head, tok, sip, cap)

        run_mirror(), run_spec()                                    # warm-up
        t_m, t_s = [], []
        for _ in range(rounds):
            t_m.append(seconds(run_mirror) * 1e3 / steps)
            t_s.append(seconds(run_spec) * 1e3 / steps)
    caches = [mip.key_value_memory_dict["b200_kv_cache"], sip.key_value_memory_dict["b200_kv_cache"]]
    kinds = [type(c).__name__ + ("" if isinstance(c, kv_cache.KVCache) else f"(n_dev={c.n_dev})") for c in caches]
    return {"tokens": T, "layers": len(spec), "caches": kinds, "prefill": prefill,
            "mirror_ms_per_token": t_m, "spec_ms_per_token": t_s,
            "mirror_median": statistics.median(t_m), "spec_median": statistics.median(t_s),
            "spec_over_mirror": statistics.median(t_s) / statistics.median(t_m)}


def no_cache(cfg, spec, head, T, reps):
    """ms per generated token of the --spec path without a cache: the forward over the prompt and the new token."""
    ids = torch.randint(0, cfg.vocab_size, (1, T + 1), device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    with torch.no_grad():
        spec_forward(cfg, spec, head, ids, None, T + 1)
        return [seconds(lambda: spec_forward(cfg, spec, head, ids, None, T + 1)) * 1e3 for _ in range(reps)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--context", type=int, default=18432)
    ap.add_argument("--long", type=int, default=1058816)
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card()}
    cfg, spec, mirror, head = models(48)
    res["device_cache"] = decode(cfg, spec, mirror, head, a.context, a.steps, a.rounds)
    gc.collect()
    torch.cuda.empty_cache()
    t = no_cache(cfg, spec, head, a.context, 2)
    res["no_cache"] = {"tokens": a.context, "ms_per_token": t, "median": statistics.median(t),
                       "over_spec_decode": statistics.median(t) / res["device_cache"]["spec_median"]}
    del spec, mirror, head
    gc.collect()
    torch.cuda.empty_cache()
    if a.long:
        cfg, spec, mirror, head = models(2)
        kv_cache.device_layers = lambda *args, **kw: 0                  # both layers on the host tier
        res["host_cache"] = decode(cfg, spec, mirror, head, a.long, a.steps, a.rounds)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "spec_decode.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
