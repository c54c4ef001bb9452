"""Time the backward GEMMs with transposed operands two ways, in one process, with CUDA events:

  * "copy":  the transposed-copy composition - the operand that is contiguous along the wrong dimension is written out
             transposed (zero-padded to a multiple of 8 along the contraction), then the K-major GEMM runs;
  * "mn":    the same product with the transposed view handed to the GEMM as an MN-major operand (`lv_gemm_ex`).

    python tools/bench_gemm_layouts.py [--iters 10] [--warmup 3] [--shapes decoder vit lm_head]

Shapes: the four GEMMs of one 14B decoder layer at T = 18 432 tokens (dX = dY W and dW = dY^T X each), the four of an
InternViT-300M layer at 64 frames x 1025 tokens (C = 1024, MLP 4096), and one LM-head vocabulary chunk (16 384 rows
of the 5120-wide head, M = 2048 selected rows).  One JSON line per product: ms of each variant (the copy included in
"copy"), the GEMM's algorithmic TFLOP/s (2 M N K / time), and whether the two results are bit-identical.  The card's
name and power limit come first.
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


def kmajor_copy(t):
    """[T, X] -> contiguous [X, T'] (T' = T rounded up to a multiple of 8, zero columns): the transposed copy the
    K-major GEMM needs when the contraction runs over T."""
    rows, cols = t.shape
    if rows % 8 == 0:
        return t.t().contiguous()
    out = torch.zeros((cols, (rows + 7) // 8 * 8), dtype=t.dtype, device=t.device)
    out[:, :rows] = t.t()
    return out


def products(which):
    """(name, M, N, K, kind): kind "dx" = dY[M, K] . W[K, N] (W stored [K, N], nn.Linear layout), "dw" = dY^T . X with
    dY [K, M] and X [K, N] (K = tokens)."""
    out = []
    if "decoder" in which:
        T, H = 18432, 5120
        for name, n_out, k_in in (("qkv", 7168, H), ("o", H, H), ("gate_up", 27648, H), ("down", H, 13824)):
            out.append((f"decoder.{name}.dx", T, k_in, n_out, "dx"))
            out.append((f"decoder.{name}.dw", n_out, k_in, T, "dw"))
    if "vit" in which:
        T, C, Fh = 64 * 1025, 1024, 4096
        for name, n_out, k_in in (("qkv", 3 * C, C), ("proj", C, C), ("fc1", Fh, C), ("fc2", C, Fh)):
            out.append((f"vit.{name}.dx", T, k_in, n_out, "dx"))
            out.append((f"vit.{name}.dw", n_out, k_in, T, "dw"))
    if "lm_head" in which:
        M, c, chunk = 2048, 5120, 16384
        out.append(("lm_head.chunk.dsel", M, c, chunk, "dx"))
        out.append(("lm_head.chunk.dw", chunk, c, M, "dw"))
    return out


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shapes", nargs="+", default=["decoder", "vit", "lm_head"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm_layouts: no CUDA device")
    name, pl = card()
    print(json.dumps({"card": name, "power_limit": pl, "torch": torch.__version__}), flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    for pname, M, N, K, kind in products(args.shapes):
        if kind == "dx":
            dy = torch.randn(M, K, generator=g, device="cuda").to(torch.bfloat16)
            w = (torch.randn(K, N, generator=g, device="cuda") * K ** -0.5).to(torch.bfloat16)
            copy = lambda: ops.linear(dy, kmajor_copy(w))
            mn = lambda: ops.linear(dy, w.t())
        else:
            dy = torch.randn(K, M, generator=g, device="cuda").to(torch.bfloat16)
            x = (torch.randn(K, N, generator=g, device="cuda") * K ** -0.5).to(torch.bfloat16)
            copy = lambda: ops.linear(kmajor_copy(dy), kmajor_copy(x))
            mn = lambda: ops.linear(dy.t(), x.t())
        same = torch.equal(copy(), mn())
        for _ in range(args.warmup):
            copy(), mn()
        torch.cuda.synchronize()
        ms = {"copy": [], "mn": []}
        for _ in range(2):              # alternate the variants
            ms["copy"].append(timed(copy, args.iters))
            ms["mn"].append(timed(mn, args.iters))
        fl = 2.0 * M * N * K
        rec = {"product": pname, "M": M, "N": N, "K": K, "bit_identical": same}
        for v, t in ms.items():
            best = min(t)
            rec[f"{v}_ms"] = round(best, 3)
            rec[f"{v}_tflops"] = round(fl / best / 1e9, 1)
        rec["speedup"] = round(rec["copy_ms"] / rec["mn_ms"], 3)
        print(json.dumps(rec), flush=True)
        del dy, copy, mn
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
