"""Per-kernel timing on one H100 (CUDA events on the launching stream, warm-up, L2 flush between
timed launches) next to the same-box comparators the reference would run (flash-attn 2.8,
cuDNN SDPA, cuBLAS via torch.matmul).  Writes the JSON given by --out (default kernels.json).

  python tools/bench_kernels.py [--only attn|gemm|elem] [--quick]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from long_vita_b200 import ops  # noqa: E402

PEAKS = {}
try:
    PEAKS = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
except Exception:
    pass
# without MEASURED_PEAKS.json: the H100 SXM data sheet (dense bf16, HBM3), the same fallback as bench.py
HBM = PEAKS.get("hbm_gbs", 3350.0)
TF = PEAKS.get("bf16_tflops", 989.0)

_flush = None


def flush_l2():
    global _flush
    if _flush is None:
        _flush = torch.empty(512 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    _flush.zero_()


def timeit(fn, iters=10, warmup=3, flush=True):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush:
            flush_l2()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def bench_attn(results, quick):
    import flash_attn

    shapes = [
        ("llm16k", 1, 16384, 40, 8, 128, True),
        ("llm32k", 1, 32768, 40, 8, 128, True),
        ("vit64", 64, 1025, 16, 16, 64, False),
        ("llm4k_nc", 1, 4096, 40, 8, 128, False),
    ]
    if not quick:
        shapes.append(("llm128k", 1, 131072, 40, 8, 128, True))
    for name, b, s, hq, hkv, d, causal in shapes:
        q = torch.randn(b, s, hq, d, device="cuda", dtype=torch.bfloat16)
        k = torch.randn(b, s, hkv, d, device="cuda", dtype=torch.bfloat16)
        v = torch.randn(b, s, hkv, d, device="cuda", dtype=torch.bfloat16)
        flops = 4.0 * b * hq * d * (s * (s + 1) / 2 if causal else s * s)
        iters = 3 if s >= 100000 else 10
        med, best = timeit(lambda: ops.attention_fwd(q, k, v, causal=causal), iters=iters)
        r = {"kernel": "attn_fwd", "shape": name, "ms": med, "ms_best": best, "tflops": flops / med / 1e9,
             "frac_of_measured_peak": flops / med / 1e9 / TF}
        if s < 100000:
            fm, _ = timeit(lambda: flash_attn.flash_attn_func(q, k, v, causal=causal), iters=iters)
            r["flash_attn2_ms"] = fm
            r["flash_attn2_tflops"] = flops / fm / 1e9
            try:
                qt, kt, vt = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
                with torch.nn.attention.sdpa_kernel(torch.nn.attention.SDPBackend.CUDNN_ATTENTION):
                    cm, _ = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(
                        qt, kt, vt, is_causal=causal, enable_gqa=True), iters=iters)
                r["cudnn_sdpa_ms"] = cm
                r["cudnn_sdpa_tflops"] = flops / cm / 1e9
            except Exception as e:  # noqa: BLE001
                r["cudnn_sdpa_error"] = str(e)[:200]
        print(json.dumps(r), flush=True)
        results.append(r)
        del q, k, v


def bench_gemm(results, quick):
    shapes = [
        ("llm_qkv", 16384, 7168, 5120), ("llm_o", 16384, 5120, 5120), ("llm_gate_up", 16384, 27648, 5120),
        ("llm_down", 16384, 5120, 13824), ("vit_qkv", 65600, 3072, 1024), ("vit_proj", 65600, 1024, 1024),
        ("vit_fc1", 65600, 4096, 1024), ("vit_fc2", 65600, 1024, 4096), ("lm_head_m2", 2, 152064, 5120),
        ("square8k", 8192, 8192, 8192),
        # one context-parallel rank of 8 on the 18K prompt (2304 tokens): few M-blocks, wave quantisation matters
        ("cp8_qkv", 2304, 7168, 5120), ("cp8_o", 2304, 5120, 5120), ("cp8_gate_up", 2304, 27648, 5120), ("cp8_down", 2304, 5120, 13824),
    ]
    for name, M, N, K in shapes:
        x = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
        w = torch.randn(N, K, device="cuda", dtype=torch.bfloat16) * 0.02
        out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        flops = 2.0 * M * N * K
        med, best = timeit(lambda: ops.linear(x, w, out=out))
        cm, cb = timeit(lambda: torch.matmul(x, w.t(), out=out))
        byts = 2.0 * (M * K + N * K + M * N)
        r = {"kernel": "gemm", "shape": name, "M": M, "N": N, "K": K, "ms": med, "tflops": flops / med / 1e9,
             "frac_of_measured_peak": flops / med / 1e9 / TF, "gbs": byts / med / 1e6, "cublas_ms": cm,
             "cublas_tflops": flops / cm / 1e9}
        print(json.dumps(r), flush=True)
        results.append(r)
        del x, w, out


def bench_elem(results, quick):
    T, H, I = 16384, 5120, 13824
    x = torch.randn(T, H, device="cuda", dtype=torch.bfloat16)
    w = torch.ones(H, device="cuda", dtype=torch.bfloat16)
    gu = torch.randn(T, 2 * I, device="cuda", dtype=torch.bfloat16)
    qkv = torch.randn(T, 7168, device="cuda", dtype=torch.bfloat16)
    pos = torch.arange(T, device="cuda")
    inv = (1.0 / (1e6 ** (torch.arange(0, 128, 2, device="cuda").float() / 128)))
    cos, sin = ops.rope_table(pos, inv)
    q = qkv[:, :5120].view(T, 40, 128)
    vit = torch.randn(64, 1025, 1024, device="cuda", dtype=torch.bfloat16)
    cases = [
        ("rmsnorm", lambda: ops.rmsnorm(x, w), 2 * T * H * 2),
        ("rmsnorm_residual", lambda: ops.rmsnorm(x, w, residual=x), 4 * T * H * 2),
        ("swiglu", lambda: ops.swiglu(gu), 3 * T * I * 2),
        ("rope_q", lambda: ops.rope(q, cos, sin, out=q), 2 * T * 5120 * 2 + 2 * T * 128 * 2),
        ("layernorm_vit", lambda: ops.layernorm(vit, w[:1024], w[:1024]), 2 * vit.numel() * 2),
        ("pixel_shuffle", lambda: ops.pixel_shuffle(vit, 32, True), 2 * 64 * 1024 * 1024 * 2),
        ("ls_residual_vit", lambda: ops.ls_residual(vit, vit, w[:1024]), 3 * vit.numel() * 2),
    ]
    for name, fn, byts in cases:
        med, best = timeit(fn, iters=10)
        r = {"kernel": name, "ms": med, "gbs": byts / med / 1e6, "frac_of_measured_hbm": byts / med / 1e6 / HBM}
        print(json.dumps(r), flush=True)
        results.append(r)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=None)
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default="kernels.json")
    a = ap.parse_args()
    results = []
    if a.only in (None, "attn"):
        bench_attn(results, a.quick)
    if a.only in (None, "gemm"):
        bench_gemm(results, a.quick)
    if a.only in (None, "elem"):
        bench_elem(results, a.quick)
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    json.dump({"peaks": {"hbm_gbs": HBM, "bf16_tflops": TF}, "results": results}, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
