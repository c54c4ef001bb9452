"""Attention backward timing (dQ, dK, dV; algorithmic FLOPs = 2.5x forward) next to flash-attn 2.8, then packed rows
of documents (lv_attn_docs_fwd / lv_attn_docs_bwd, `--reset-attention-mask`) next to dense causal attention at the
same S and flash_attn_varlen_func.  Packed TFLOP/s count the visible pairs only: 4 hq d sum_i L_i (L_i + 1) / 2
(x 2.5 for the backward).  Every line carries the card name and its power limit."""
import json, os, subprocess, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from long_vita_b200 import ops
import flash_attn

def timeit(fn, iters=5, warmup=2):
    for _ in range(warmup): fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize(); ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]

def card():
    try:
        w = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        w = ""
    return {"card": torch.cuda.get_device_name(), "power_limit_w": float(w) if w else None}


CARD = card()

for name, s, hq, hkv, d, causal in [("llm8k", 8192, 40, 8, 128, True), ("llm16k", 16384, 40, 8, 128, True)]:
    q = torch.randn(1, s, hq, d, device="cuda", dtype=torch.bfloat16)
    k = torch.randn(1, s, hkv, d, device="cuda", dtype=torch.bfloat16)
    v = torch.randn(1, s, hkv, d, device="cuda", dtype=torch.bfloat16)
    do = torch.randn_like(q)
    out, lse = ops.attention_fwd(q, k, v, causal=causal, return_lse=True)
    flops = 2.5 * 4.0 * hq * d * (s * (s + 1) / 2)
    ms = timeit(lambda: ops.attention_bwd(do, q, k, v, out, lse, causal=causal))
    qf, kf, vf = (t.clone().requires_grad_(True) for t in (q, k, v))
    of = flash_attn.flash_attn_func(qf, kf, vf, causal=causal)
    fms = timeit(lambda: torch.autograd.grad(of, (qf, kf, vf), do, retain_graph=True))
    print(json.dumps({"kernel": "attn_bwd", "shape": name, "ms": ms, "tflops": flops / ms / 1e9, "flash_attn2_ms": fms,
                      "flash_attn2_tflops": flops / fms / 1e9, **CARD}), flush=True)


def doc_lengths(S, lo, hi, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    while sum(out) < S:
        out.append(int(torch.randint(lo, hi + 1, (1,), generator=g)))
    out[-1] -= sum(out) - S
    return [n for n in out if n > 0]


hq, hkv, d = 40, 8, 128
for S in (16384, 32768):
    q = torch.randn(1, S, hq, d, device="cuda", dtype=torch.bfloat16)
    k = torch.randn(1, S, hkv, d, device="cuda", dtype=torch.bfloat16)
    v = torch.randn(1, S, hkv, d, device="cuda", dtype=torch.bfloat16)
    do = torch.randn_like(q)
    dense = 4.0 * hq * d * (S * (S + 1) / 2)
    out, lse = ops.attention_fwd(q, k, v, causal=True, return_lse=True)
    dense_f = timeit(lambda: ops.attention_fwd(q, k, v, causal=True))
    dense_b = timeit(lambda: ops.attention_bwd(do, q, k, v, out, lse, causal=True))
    for mix, lo, hi in (("long", 1024, 8192), ("short", 64, 1024)):
        lengths = doc_lengths(S, lo, hi, seed=S + lo)
        cu_list = [0]
        for n in lengths:
            cu_list.append(cu_list[-1] + n)
        cu = ops.packed_cu_seqlens(actual_seq_len=cu_list[1:], device="cuda", seq_len=S)
        vis = 4.0 * hq * d * sum(n * (n + 1) / 2 for n in lengths)
        pout, plse = ops.attention_fwd(q, k, v, causal=True, return_lse=True, cu_seqlens=cu)
        f_ms = timeit(lambda: ops.attention_fwd(q, k, v, causal=True, cu_seqlens=cu))
        b_ms = timeit(lambda: ops.attention_bwd(do, q, k, v, pout, plse, causal=True, cu_seqlens=cu))
        rec = {"kernel": "attn_docs", "S": S, "mix": mix, "n_docs": len(lengths), "visible_fraction": vis / dense,
               "fwd_ms": f_ms, "fwd_tflops_visible": vis / f_ms / 1e9, "bwd_ms": b_ms,
               "bwd_tflops_visible": 2.5 * vis / b_ms / 1e9, "dense_causal_fwd_ms": dense_f,
               "dense_causal_fwd_tflops": dense / dense_f / 1e9, "dense_causal_bwd_ms": dense_b,
               "dense_causal_bwd_tflops": 2.5 * dense / dense_b / 1e9}
        try:
            q3, k3, v3 = (t[0].clone().requires_grad_(True) for t in (q, k, v))
            m = max(lengths)
            fa_f = timeit(lambda: flash_attn.flash_attn_varlen_func(q3, k3, v3, cu, cu, m, m, causal=True))
            of = flash_attn.flash_attn_varlen_func(q3, k3, v3, cu, cu, m, m, causal=True)
            fa_b = timeit(lambda: torch.autograd.grad(of, (q3, k3, v3), do[0], retain_graph=True))
            rec.update({"flash_varlen_fwd_ms": fa_f, "flash_varlen_fwd_tflops_visible": vis / fa_f / 1e9,
                        "flash_varlen_bwd_ms": fa_b, "flash_varlen_bwd_tflops_visible": 2.5 * vis / fa_b / 1e9})
        except AttributeError:
            pass
        print(json.dumps({**rec, **CARD}), flush=True)
