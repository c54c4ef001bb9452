"""Time the weight gradient added to an fp32 main_grad two ways, in one process, alternating, with CUDA events:

  * "hook":  `ops.linear_wgrad` into a fresh bf16 [N, K] tensor, then `main_grad.add_(dw)` - what Megatron's DDP hook does
             when gradient_accumulation_fusion is off;
  * "fused": `ops.linear_wgrad_accumulate` - the same GEMM adding its fp32 accumulator to main_grad in the epilogue.

    python tools/bench_wgrad_accum.py [--iters 10] [--warmup 3] [--shapes decoder vit lm_head]

Shapes: the four weights of one 14B decoder layer at T = 18 432 tokens, the four of an InternViT-300M layer at 64 frames
x 1025 tokens, and one LM-head vocabulary chunk (16 384 rows of the 5120-wide head, M = 2048 selected rows).  One JSON
line per weight: ms of each variant, GB/s over its algorithmic bytes (both read dY and X once; "hook" then moves 12 B per
weight element - bf16 dW written and read, main_grad read and written - "fused" 8 B), the peak of memory allocated
during one call above what was allocated before it, and whether the results agree exactly: fused from zero rounds to the
bf16 dW, and fused from a prior P equals P + that zero-start accumulator.  The card's name and power limit come first.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from long_vita_b200 import ops  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                             f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001 - the number is informative only
        pl = f"unknown ({type(e).__name__})"
    return name, pl


def weights(which):
    """(name, T, N_out, K_in): dW [N_out, K_in] = dY^T [N_out, T] . X [T, K_in]."""
    out = []
    if "decoder" in which:
        T, H = 18432, 5120
        out += [(f"decoder.{n}", T, no, ki) for n, no, ki in
                (("qkv", 7168, H), ("proj", H, H), ("fc1", 27648, H), ("fc2", H, 13824))]
    if "vit" in which:
        T, C, Fh = 64 * 1025, 1024, 4096
        out += [(f"vit.{n}", T, no, ki) for n, no, ki in
                (("qkv", 3 * C, C), ("proj", C, C), ("fc1", Fh, C), ("fc2", C, Fh))]
    if "lm_head" in which:
        out.append(("lm_head.chunk", 2048, 16384, 5120))
    return out


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def peak_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shapes", nargs="+", default=["decoder", "vit", "lm_head"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_wgrad_accum: no CUDA device")
    name, pl = card()
    print(json.dumps({"card": name, "power_limit": pl, "torch": torch.__version__}), flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    for wname, T, N, K in weights(args.shapes):
        dy = torch.randn(T, N, generator=g, device="cuda").to(torch.bfloat16)
        x = (torch.randn(T, K, generator=g, device="cuda") * T ** -0.5).to(torch.bfloat16)
        main_grad = torch.zeros((N, K), dtype=torch.float32, device="cuda")
        hook = lambda: main_grad.add_(ops.linear_wgrad(dy, x))
        fused = lambda: ops.linear_wgrad_accumulate(dy, x, main_grad)
        fused()
        acc0 = main_grad.clone()
        agree = torch.equal(acc0.to(torch.bfloat16), ops.linear_wgrad(dy, x))
        prior = torch.randn((N, K), generator=g, device="cuda")
        main_grad.copy_(prior)
        fused()
        agree = agree and torch.equal(main_grad, prior + acc0)
        del acc0, prior
        for _ in range(args.warmup):
            hook(), fused()
        torch.cuda.synchronize()
        ms = {"hook": [], "fused": []}
        for _ in range(2):              # alternate the variants
            ms["hook"].append(timed(hook, args.iters))
            ms["fused"].append(timed(fused, args.iters))
        operands = 2 * T * (N + K)
        nbytes = {"hook": operands + 12 * N * K, "fused": operands + 8 * N * K}
        rec = {"weight": wname, "T": T, "N": N, "K": K, "exact_relations_hold": agree}
        for v, t in ms.items():
            best = min(t)
            rec[f"{v}_ms"] = round(best, 3)
            rec[f"{v}_gbps"] = round(nbytes[v] / best / 1e6, 1)
            rec[f"{v}_tflops"] = round(2.0 * T * N * K / best / 1e9, 1)
        rec["hook_peak_mb"] = round(peak_bytes(hook) / 2 ** 20, 1)
        rec["fused_peak_mb"] = round(peak_bytes(fused) / 2 ** 20, 1)
        rec["speedup"] = round(rec["hook_ms"] / rec["fused_ms"], 3)
        print(json.dumps(rec), flush=True)
        del dy, x, main_grad, hook, fused
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
