"""Questions about a prefilled context on one GPU: ops.attention_host_rows per host layer, and a question against a
re-prefill, alternated in one process.

    python tools/bench_context_questions.py [--rows 131072 1058816] [--m 16 128 1024] [--reps 3]
                                            [--context 1058816] [--question 128] [--model-reps 1] [--out DIR]

(a) attention_host_rows over `rows` host rows of the 14B geometry (40:8 x 128; 4096 bytes per row in bf16, 2112 in
    FP8) for M query rows, each timing alternated with a pinned host-to-device `copy_` of the same bytes: ms, GB/s of
    host rows and the fraction of the copy's rate.
(b) A 14B model of 2 decoder layers with a `--context`-token context whose layers are both on the host: a
    `--question`-token question asked of the context against a re-prefill of prompt + question (the forward without
    a cache, the cheapest way to answer without a context), alternated.  The 48-layer figures (46 host layers) are
    derived from the per-layer ones and labelled so.

Prints one JSON object (and writes DIR/context_questions.json with --out), with the card's name, power limit and SM
clock read in the same run.  Random weights, ids and cache rows: the timings do not depend on their values.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_offload_decode import card, timed  # noqa: E402
from bench_offload_fp8 import FORMATS, host_layer, name  # noqa: E402
from long_vita_b200 import kv_cache, ops  # noqa: E402
from long_vita_b200.config import LongVITAConfig  # noqa: E402
from long_vita_b200.hf.modeling import LongVITAForCausalLM  # noqa: E402


def sm_clock():
    """The SM clock now (MHz), read between measurements."""
    r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return r.stdout.strip()


def host_rows(rows_list, ms, reps, cfg):
    out = []
    g = torch.Generator(device="cuda").manual_seed(1)
    for rows in rows_list:
        for dt in FORMATS:
            host = host_layer(dt, rows, cfg, g)
            dev = torch.empty(host.shape, dtype=host.dtype, device="cuda")
            nbytes = host.numel() * host.element_size()
            for M in ms:
                q = torch.randn((M, cfg.num_attention_heads, cfg.head_dim), device="cuda",
                                generator=g).to(torch.bfloat16)
                fns = {"attention_host_rows": lambda: ops.attention_host_rows(q, host, rows),
                       "copy": lambda: dev.copy_(host, non_blocking=True)}
                for f in fns.values():
                    f()
                t = {k: [] for k in fns}
                for _ in range(reps):
                    for k, f in fns.items():
                        t[k].append(timed(f))
                ms_k, ms_c = statistics.median(t["attention_host_rows"]), statistics.median(t["copy"])
                out.append({"rows": rows, "format": name(dt), "M": M, "host_bytes": nbytes,
                            "ms": round(ms_k, 2), "GB_per_s": round(nbytes / ms_k / 1e6, 1),
                            "copy_ms": round(ms_c, 2), "copy_GB_per_s": round(nbytes / ms_c / 1e6, 1),
                            "fraction_of_copy": round(ms_c / ms_k, 3),
                            "ms_all": [round(x, 2) for x in t["attention_host_rows"]]})
                print(json.dumps(out[-1]), flush=True)
            del host, dev
            torch.cuda.empty_cache()
    return out


def model_run(T, n, reps, cfg):
    model = LongVITAForCausalLM.from_synthetic(cfg, seed=7, device="cuda", num_layers=2)
    g = torch.Generator(device="cuda").manual_seed(5)
    ids = torch.randint(0, cfg.vocab_size, (1, T), device="cuda", generator=g)
    qq = torch.randint(0, cfg.vocab_size, (1, n), device="cuda", generator=g)
    real = kv_cache.device_layers
    kv_cache.device_layers = lambda *a, **kw: 0                # both layers on the host
    try:
        with torch.no_grad():
            ctx = model.prefill_context(ids)
    finally:
        kv_cache.device_layers = real
    assert isinstance(ctx.cache, kv_cache.OffloadedKVCache) and ctx.cache.n_dev == 0
    both = torch.cat([ids, qq], 1)
    with torch.no_grad():
        fns = {"question": lambda: model(input_ids=qq, past_key_values=ctx.session(n), use_cache=True,
                                         num_logits_to_keep=1),
               "re_prefill": lambda: model(input_ids=both, num_logits_to_keep=1)}
        fns["question"]()
        t = {k: [] for k in fns}
        for _ in range(reps):
            for k, f in fns.items():
                t[k].append(timed(f))
            t["question"].extend(timed(fns["question"]) for _ in range(2))
    q_ms, p_ms = statistics.median(t["question"]), statistics.median(t["re_prefill"])
    return {"context": T, "question": n, "layers": 2, "host_layers": 2,
            "question_ms": round(q_ms, 1), "re_prefill_ms": round(p_ms, 1), "speedup": round(p_ms / q_ms, 1),
            "question_ms_all": [round(x, 1) for x in t["question"]],
            "derived_48_layers": {"note": "derived, not measured: 46 host layers at the per-layer question time and "
                                          "48 layers at the per-layer re-prefill time",
                                  "question_s": round(46 * q_ms / 2 / 1e3, 2),
                                  "re_prefill_s": round(48 * p_ms / 2 / 1e3, 1)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[131072, 1058816])
    ap.add_argument("--m", type=int, nargs="+", default=[16, 128, 1024])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--context", type=int, default=1058816)
    ap.add_argument("--question", type=int, default=128)
    ap.add_argument("--model-reps", type=int, default=1)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_context_questions needs a CUDA device")
    cfg = LongVITAConfig()
    res = {"card": card(), "sm_clock": sm_clock(), "host_rows": host_rows(args.rows, args.m, args.reps, cfg)}
    if args.context:
        res["model"] = model_run(args.context, args.question, args.model_reps, cfg)
        print(json.dumps(res["model"]), flush=True)
    res["card_after"] = card()
    res["sm_clock_after"] = sm_clock()
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "context_questions.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
