"""The decoder's linears in FP8 (e4m3) against bf16, on one GPU, alternated in one process.

    python tools/bench_fp8_linear.py [--reps 20] [--steps 3] [--decode-steps 32] [--layers 48] [--out DIR]

1. GEMM: each of the four decoder linears at T = 18 432 rows (the 16K bench prompt), bf16 (lv_gemm_bias_act) against
   FP8: the whole ops.linear call (per-row quantisation of x + lv_gemm_fp8) and lv_gemm_fp8 alone; TFLOP/s = 2 T N K
   over the time.
2. GEMV at M = 1: microseconds per call and weight GB/s (N K bytes of W: 2 per value in bf16, 1 in FP8).  Each mode
   rotates over enough copies of the weight (over 200 MB of FP8 bytes, four times the 50 MB L2) that every call
   streams its weight from HBM.
3. The 48-layer 14B prefill of the 64-frame bench prompt, built as bench.py builds it (synthetic.build_prompt,
   synthetic_frames, seed 1234): ms per step, both models resident, steps alternated.
4. Decode: ms per token over an 18 432-token cache (one prefill with use_cache=True per mode, then single-token
   steps), bf16 and FP8 alternated over `--decode-rounds` rounds; the cache class and device layer count of each mode
   are reported.  With `--profile`, a torch.profiler trace of 4 decode steps per mode, in a pass of its own after the
   timed rounds: DIR/decode_<mode>.txt (top kernels and host ops) and the GPU busy time per step.
5. Resident weight bytes of the decoder linears and of the whole model (torch.cuda.memory_allocated around the build).
Derived, not measured: the device K/V layers of a 1 058 816-token generation (kv_cache.device_layers with the free
memory left beside each model), and the largest streamed prompt from the 19 689 B per token of DESIGN §8.

Prints one JSON object (and writes DIR/fp8_linear.json with --out), with the card's name and power limit read in the
same run.  Random weights and inputs: the timings do not depend on their values.
"""
import argparse
import gc
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_offload_decode import card, timed  # noqa: E402
from long_vita_b200 import _lib, kv_cache, ops  # noqa: E402
from long_vita_b200.config import LongVITAConfig  # noqa: E402
from long_vita_b200.hf import modeling  # noqa: E402
from long_vita_b200.hf.modeling import LongVITAForCausalLM  # noqa: E402
from long_vita_b200.synthetic import build_prompt, synthetic_frames  # noqa: E402

FP8 = torch.float8_e4m3fn
T = 18432
STREAM_BYTES_PER_TOKEN = 19689          # DESIGN §8: the streamed bench workload, frames included
STREAM_LARGEST_BF16 = 2_459_648         # DESIGN §8: derived largest prompt with the bf16 48-layer weights


def linears(cfg):
    H, I = cfg.hidden_size, cfg.intermediate_size
    qkv = (cfg.num_attention_heads + 2 * cfg.num_key_value_heads) * cfg.head_dim
    return {"wqkv": (qkv, H, "bias"), "wo": (H, cfg.num_attention_heads * cfg.head_dim, None),
            "w_gate_up": (2 * I, H, "swiglu"), "w_down": (H, I, None)}


def gemm_section(cfg, reps):
    g = torch.Generator(device="cuda").manual_seed(0)
    out = {}
    for name, (N, K, kind) in linears(cfg).items():
        act = "swiglu" if kind == "swiglu" else None
        w = (torch.randn((N, K), device="cuda", generator=g) * 0.02).to(torch.bfloat16)
        b = torch.randn((N,), device="cuda", generator=g).to(torch.bfloat16) if kind == "bias" else None
        w8 = ops.Fp8Weight.quantize(w)
        res = {}
        for M in (T, 1):
            x = torch.randn((M, K), device="cuda", generator=g).to(torch.bfloat16)
            xq, xs = ops.quant_rows_fp8(x)
            y = torch.empty((M, N // 2 if act else N), dtype=torch.bfloat16, device="cuda")
            # M = 1: rotate over weight copies whose FP8 bytes exceed 4x L2, so that no call finds its weight in L2
            n_copies = 1 if M == T else -(-200_000_000 // (N * K)) + 1
            ws = [w] + [w.clone() for _ in range(n_copies - 1)]
            w8s = [w8] + [ops.Fp8Weight(w8.data.clone(), w8.scale.clone()) for _ in range(n_copies - 1)]
            turn = {"bf16": 0, "fp8": 0, "fp8_gemm_only": 0}

            def nxt(key, lst):
                turn[key] = (turn[key] + 1) % len(lst)
                return lst[turn[key]]

            def gemm8():
                v = nxt("fp8_gemm_only", w8s)
                _lib.check(_lib.lib().lv_gemm_fp8(xq.data_ptr(), xs.data_ptr(), v.data.data_ptr(),
                                                  v.scale.data_ptr(), None if b is None else b.data_ptr(),
                                                  y.data_ptr(), M, N, K, K, K, y.stride(0), 3 if act else 0,
                                                  torch.cuda.current_stream().cuda_stream), "lv_gemm_fp8")

            fns = {"bf16": lambda: ops.linear(x, nxt("bf16", ws), b, act=act, out=y),
                   "fp8": lambda: ops.linear(x, nxt("fp8", w8s), b, act=act, out=y), "fp8_gemm_only": gemm8}
            n = reps if M == T else 20 * reps
            for f in fns.values():
                timed(f, 3)
            ms = {k: [] for k in fns}
            for _ in range(3):                                   # alternated rounds
                for k, f in fns.items():
                    ms[k].append(timed(f, n))
            best = {k: min(v) for k, v in ms.items()}
            if M == T:
                res["gemm"] = {k: {"ms": round(v, 4), "tflops": round(2.0 * M * N * K / v / 1e9, 1)}
                               for k, v in best.items()}
            else:
                res["gemv_m1"] = {k: {"us": round(v * 1e3, 2),
                                      "weight_gbs": round(N * K * (2 if k == "bf16" else 1) / v / 1e6, 1)}
                                  for k, v in best.items()}
            del ws, w8s
        out[name] = {"N": N, "K": K, **res}
        del w, w8
    return out


def model_bytes(build):
    gc.collect()
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    model = build()
    torch.cuda.synchronize()
    return model, torch.cuda.memory_allocated() - m0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--decode-steps", type=int, default=32)
    ap.add_argument("--layers", type=int, default=48)
    ap.add_argument("--decode-rounds", type=int, default=5)
    ap.add_argument("--skip-gemm", action="store_true")
    ap.add_argument("--skip-prefill", action="store_true")
    ap.add_argument("--profile", action="store_true", help="trace decode steps (needs --out)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_fp8_linear.py needs a CUDA device"
    cfg = LongVITAConfig()
    res = {"card": card(), "T": T}
    if not args.skip_gemm:
        res["linears"] = gemm_section(cfg, args.reps)
        print(json.dumps(res["linears"]), flush=True)

    models, resident = {}, {}
    for dt in (torch.bfloat16, FP8):
        models[dt], resident[dt] = model_bytes(lambda: LongVITAForCausalLM.from_synthetic(
            cfg, seed=1234, device="cuda", num_layers=args.layers, linear_dtype=dt))
    names = {torch.bfloat16: "bf16", FP8: "fp8"}
    res["resident_bytes"] = {names[dt]: {"model": resident[dt],
                                         "decoder_linears": sum(L.linear_bytes() for L in models[dt].model.layers)}
                             for dt in models}

    ids, idx = build_prompt(cfg, 64, 16, pad_multiple=2048)
    ids, idx = ids.cuda(), idx.cuda()
    images = synthetic_frames(cfg, 64, device="cuda")
    S = ids.shape[1]
    with torch.no_grad():
        def prefill(dt):
            return models[dt](input_ids=ids, images=images, image_indices=idx, num_logits_to_keep=1).logits

        if not args.skip_prefill:
            for dt in models:
                prefill(dt)
            ms = {dt: [] for dt in models}
            for _ in range(args.steps):
                for dt in models:
                    ms[dt].append(timed(lambda: prefill(dt)))
            res["prefill_16k"] = {names[dt]: {"tokens": S, "ms_per_step": [round(v, 2) for v in ms[dt]],
                                              "tokens_per_s": round(S / (min(ms[dt]) / 1e3), 1)} for dt in models}
            print(json.dumps(res["prefill_16k"]), flush=True)

        steps = args.decode_steps
        capacity = T + 4 + args.decode_rounds * steps + (4 if args.profile else 0) + 8
        caches = {dt: models[dt](input_ids=ids[:, :T], use_cache=True, num_logits_to_keep=1,
                                 max_cache_len=capacity).past_key_values for dt in models}
        tok = ids[:, :1]

        def step(dt):
            models[dt](input_ids=tok, past_key_values=caches[dt], use_cache=True)

        for dt in models:
            timed(lambda: step(dt), 4)
        dec = {dt: [] for dt in models}
        for _ in range(args.decode_rounds):                      # alternated rounds
            for dt in models:
                dec[dt].append(timed(lambda: step(dt), steps))
        res["decode_18432"] = {names[dt]: {"ms_per_token": [round(v, 3) for v in dec[dt]],
                                           "cache": type(caches[dt]).__name__,
                                           "device_layers": len(getattr(caches[dt], "k", []))} for dt in models}
        print(json.dumps(res["decode_18432"]), flush=True)
        if args.profile and args.out:
            os.makedirs(args.out, exist_ok=True)
            prof_res = {}
            for dt in models:
                acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
                with torch.profiler.profile(activities=acts) as prof:
                    for _ in range(4):
                        step(dt)
                    torch.cuda.synchronize()
                ka = prof.key_averages()
                with open(os.path.join(args.out, f"decode_{names[dt]}.txt"), "w") as f:
                    f.write(ka.table(sort_by="self_device_time_total", row_limit=30) + "\n")
                    f.write(ka.table(sort_by="self_cpu_time_total", row_limit=30) + "\n")
                prof_res[names[dt]] = {"gpu_busy_ms_per_step": round(sum(e.self_device_time_total for e in ka) / 4e3, 3)}
            res["decode_profile"] = prof_res
            print(json.dumps(prof_res), flush=True)
        del caches
        gc.collect()
        torch.cuda.empty_cache()

    # derived: placement of a 1 058 816-token generation beside each model alone, and the largest streamed prompt
    total = torch.cuda.mem_get_info()[1]
    other = {torch.bfloat16: resident[FP8], FP8: resident[torch.bfloat16]}
    derived = {}
    rows, L = 1_058_816, args.layers
    row = 2 * cfg.num_key_value_heads * cfg.head_dim * 2
    span = max(r1 - r0 for r0, r1 in modeling.row_chunks(STREAM_LARGEST_BF16))
    for dt in models:
        free = torch.cuda.mem_get_info()[0] + other[dt]         # as if the other model were not resident
        n_dev = kv_cache.device_layers(
            free, rows + 1024, L, row, rows * modeling.prefill_bytes_per_token(cfg, rows, False, dt),
            rows * modeling.prefill_bytes_per_token(cfg, rows, False, dt))
        fp8_span = span * (cfg.intermediate_size + 4) if dt == FP8 else 0
        largest = (STREAM_LARGEST_BF16 * STREAM_BYTES_PER_TOKEN + resident[torch.bfloat16] - resident[dt]
                   - fp8_span) // STREAM_BYTES_PER_TOKEN
        derived[names[dt]] = {"device_kv_layers_at_1058816": n_dev, "largest_streamed_prompt": int(largest)}
    res["derived"] = derived
    res["hbm_total_bytes"] = total
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "fp8_linear.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
