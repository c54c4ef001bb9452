"""The decoder's prefill attention in FP8 (e4m3) against bf16, on one GPU, alternated in one process.

    python tools/bench_fp8_attn.py [--lengths 16384,131072,1058816] [--rounds 2] [--prefill-tokens 1058816]
                                   [--layers 2] [--out DIR]

1. Kernel: causal 40:8 x 128 attention at each length, bf16 (lv_attn_fwd) against FP8: the whole
   ops.attention_fwd_fp8 call (K / V quantisation + lv_attn_fwd_fp8) and lv_attn_fwd_fp8 alone on K / V quantised
   once; modes alternated over `--rounds` rounds, each round timing every mode with CUDA events.  TFLOP/s are over the
   visible pairs: 4 hq d T (T + 1) / 2 over the time.  The quantisation pass alone is reported with its HBM rate
   (reads 2 T hkv d bf16, writes the e4m3 bytes and the scales).
2. Prefill: a `--layers`-layer model of the 14B geometry over `--prefill-tokens` random token ids (the 1M bench
   length runs the row-chunked layer; no frames, so the time is the decoder's), one forward per mode with
   num_logits_to_keep=1, alternated; reported per decoder layer (the forward's time over the layer count, embedding
   and LM head included).
The card's name, power limit and SM clock limit are read in the same run.  Prints one JSON object (and writes
DIR/fp8_attn.json with --out).  Random inputs: the timings do not depend on their values.
"""
import argparse
import dataclasses
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_offload_decode import card, timed  # noqa: E402
from long_vita_b200 import ops  # noqa: E402
from long_vita_b200.config import LongVITAConfig  # noqa: E402
from long_vita_b200.hf import modeling  # noqa: E402

FP8 = torch.float8_e4m3fn
HQ, HKV, D = 40, 8, 128


def kernel_section(T, rounds):
    g = torch.Generator(device="cuda").manual_seed(T)
    q = torch.randn((1, T, HQ, D), generator=g, device="cuda").to(torch.bfloat16)
    k = torch.randn((1, T, HKV, D), generator=g, device="cuda").to(torch.bfloat16)
    v = torch.randn((1, T, HKV, D), generator=g, device="cuda").to(torch.bfloat16)
    out = torch.empty_like(q)
    flops = 4.0 * HQ * D * T * (T + 1) / 2
    p = ops.attn_params(q, k, v, out, causal=True)
    bufs, f = ops._attn_fp8_kv(p, q.device)
    n = 20 if T <= 32768 else (3 if T <= 262144 else 1)
    modes = {
        "bf16": lambda: ops.attention_fwd(q, k, v, causal=True, out=out),
        "fp8_call": lambda: ops.attention_fwd_fp8(q, k, v, causal=True, out=out),
        "fp8_kernel": lambda: ops._call("lv_attn_fwd_fp8", ops.C.byref(p), ops.C.byref(f)),
        "quant_kv": lambda: ops._attn_fp8_kv(p, q.device),
    }
    for fn in modes.values():       # module load, tensor maps, allocator
        fn()
    torch.cuda.synchronize()
    ms = {m: [] for m in modes}
    for _ in range(rounds):
        for m, fn in modes.items():
            ms[m].append(timed(fn, n if m != "quant_kv" else 20))
    res = {"tokens": T, "ms": {m: min(v_) for m, v_ in ms.items()}, "ms_all": ms}
    res["tflops"] = {m: flops / (res["ms"][m] * 1e-3) / 1e12 for m in ("bf16", "fp8_call", "fp8_kernel")}
    qbytes = 2 * T * HKV * D * 2 + ops.attn_fp8_kv_bytes(T, HKV, D)
    res["quant_kv_GBps"] = qbytes / (res["ms"]["quant_kv"] * 1e-3) / 1e9
    res["speedup_call"] = res["ms"]["bf16"] / res["ms"]["fp8_call"]
    res["speedup_kernel"] = res["ms"]["bf16"] / res["ms"]["fp8_kernel"]
    del q, k, v, out, bufs
    torch.cuda.empty_cache()
    return res


def prefill_section(T, layers):
    cfg = dataclasses.replace(LongVITAConfig.long_vita_14b(), num_hidden_layers=layers)
    model = modeling.LongVITAForCausalLM.from_synthetic(cfg, seed=1234, device="cuda", num_layers=layers)
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(0, cfg.vocab_size, (1, T), generator=g).cuda()
    res = {"tokens": T, "layers": layers, "plan": "streamed" if T > modeling.STREAM_THRESHOLD else
           ("row-chunked" if len(modeling.row_chunks(T)) > 1 else "whole")}
    logits = {}
    for dt, name in ((torch.bfloat16, "bf16"), (FP8, "fp8")):
        model.model.attn_dtype = dt

        def step():
            with torch.no_grad():
                logits[name] = model(input_ids=ids, num_logits_to_keep=1).logits
        ms = timed(step)
        res[f"{name}_ms_per_layer"] = ms / layers
    res["speedup"] = res["bf16_ms_per_layer"] / res["fp8_ms_per_layer"]
    res["last_logit_rel_diff"] = float((logits["fp8"].float() - logits["bf16"].float()).norm()
                                       / logits["bf16"].float().norm())
    del model
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lengths", default="16384,131072,1058816")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--prefill-tokens", type=int, default=1058816)
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_attn.py measures on a CUDA device; none is visible")
    torch.cuda.set_device(0)
    res = {"card": card(), "kernel": []}
    for T in (int(x) for x in args.lengths.split(",") if x):
        r = kernel_section(T, args.rounds)
        print(json.dumps(r), flush=True)
        res["kernel"].append(r)
    if args.prefill_tokens > 0 and args.layers > 0:
        res["prefill"] = prefill_section(args.prefill_tokens, args.layers)
        print(json.dumps(res["prefill"]), flush=True)
    res["card_after"] = card()
    print(json.dumps(res))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "fp8_attn.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
