"""FP8 training of one `--spec` decoder layer (B2) at the 14B geometry against bf16.

Workload: one B200TransformerLayer, forward + backward at T = 18 432 tokens (the stage-2 length of the bench layout),
in bf16, fp8="e4m3" and fp8="hybrid", alternated in one process; best window after warm-up.  Reports:
  * step ms and peak device memory per mode (the FP8 weight copies are made inside every step: W in the forward, W^T
    in the backward, from the weights' current values, so their quantisation time and memory are in both figures);
  * per linear, TFLOP/s of dgrad and wgrad: the FP8 kernel alone (operands quantised beforehand), the FP8 call with its
    quantisation passes, and the bf16 call; wgrad both into a bf16 dW and fused into an fp32 main_grad;
  * the bytes per token the layer's forward keeps for its backward, measured: the distinct storages autograd saves
    (torch.autograd.graph.saved_tensors_hooks), parameters excluded;
  * the card name and power limit, read in the same run.
Weights are synthetic (normal(0, 0.02)); training quality on a real run is not measured.

    python tools/bench_fp8_train.py [--tokens 18432] [--steps 5] [--warmup 2] [--windows 3] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

H, HEADS, GROUPS, HN, INTER = 5120, 40, 8, 128, 13824
LINEARS = {"qkv": ((HEADS + 2 * GROUPS) * HN, H), "proj": (H, HEADS * HN), "fc1": (2 * INTER, H), "fc2": (H, INTER)}


def _card():
    name = torch.cuda.get_device_name(0)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        power = r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def _mcfg(fp8):
    return types.SimpleNamespace(hidden_size=H, num_attention_heads=HEADS, num_query_groups=GROUPS, kv_channels=HN,
                                 ffn_hidden_size=INTER, layernorm_epsilon=1e-6, hidden_dropout=0.0,
                                 attention_dropout=0.0, params_dtype=torch.bfloat16, num_layers=1, fp8=fp8)


def _time(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def step_times(T, steps, warmup, windows):
    from long_vita_b200.megatron.transformer_layer import B200TransformerLayer

    torch.manual_seed(0)
    modes = [None, "e4m3", "hybrid"]
    layers = {}
    state = None
    for m in modes:
        layer = B200TransformerLayer(_mcfg(m))
        if state is None:
            state = layer.state_dict()
        else:
            layer.load_state_dict(state)
        for p in layer.parameters():
            p.requires_grad_(True)
        layers[m] = layer
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn((T, 1, H), device="cuda", generator=g).to(torch.bfloat16).requires_grad_(True)
    dy = (torch.randn((T, 1, H), device="cuda", generator=g) * 1e-2).to(torch.bfloat16)
    inv = 1.0 / 1e6 ** (torch.arange(0, HN, 2, device="cuda", dtype=torch.float32) / HN)
    f = torch.outer(torch.arange(T, device="cuda", dtype=torch.float32), inv)
    freqs = torch.cat([f, f], -1).view(T, 1, 1, HN)

    def step(layer):
        for p in layer.parameters():
            p.grad = None
        x.grad = None
        out, _ = layer(hidden_states=x, attention_mask=None, rotary_pos_emb=freqs)
        out.backward(dy)

    best, peak, saved = {m: float("inf") for m in modes}, {}, {}
    for m in modes:
        saved[m] = saved_bytes(layers[m], x, freqs) / T
        for _ in range(warmup):
            step(layers[m])
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        step(layers[m])
        torch.cuda.synchronize()
        peak[m] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    for _ in range(windows):
        for m in modes:
            best[m] = min(best[m], _time(lambda: step(layers[m]), steps))
    del layers
    torch.cuda.empty_cache()
    return {str(m): {"step_ms": round(best[m], 2), "peak_extra_gib": round(peak[m], 2),
                     "saved_for_backward_bytes_per_token": round(saved[m])} for m in modes}


def gemm_rates(T, iters, windows):
    from long_vita_b200 import ops

    E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
    g = torch.Generator(device="cuda").manual_seed(2)
    out = {}
    for name, (N, K) in LINEARS.items():
        w = (torch.randn((N, K), device="cuda", generator=g) * 0.02).to(torch.bfloat16)
        x = torch.randn((T, K), device="cuda", generator=g).to(torch.bfloat16)
        dy = (torch.randn((T, N), device="cuda", generator=g) * 1e-2).to(torch.bfloat16)
        wt = ops.Fp8Weight(*ops.quant_cols_fp8_t(w))
        xt = ops.quant_cols_fp8_t(x)
        mg = torch.zeros((N, K), dtype=torch.float32, device="cuda")
        flops = 2.0 * T * N * K
        cases = {
            "dgrad_bf16": lambda: ops.linear(dy, w.t()),
            "wgrad_bf16": lambda: ops.linear_wgrad(dy, x),
            "wgrad_acc_bf16": lambda: ops.linear_wgrad_accumulate(dy, x, mg),
        }
        for dt, tag in ((E4M3, "e4m3"), (E5M2, "e5m2")):
            dq, ds = ops.quant_rows_fp8(dy, dt)
            dtq, dts = ops.quant_cols_fp8_t(dy, dt)
            dx = torch.empty((T, K), dtype=torch.bfloat16, device="cuda")
            dw = torch.empty((N, K), dtype=torch.bfloat16, device="cuda")
            cases.update({
                f"dgrad_{tag}_call": (lambda dt=dt: ops.linear_fp8_dgrad(dy, wt, dt)),
                f"dgrad_{tag}_kernel": (lambda dq=dq, ds=ds, dx=dx: ops._gemm_fp8_grad("b", dq, ds, wt.data, wt.scale,
                                                                                         dx, False)),
                f"wgrad_{tag}_call": (lambda dt=dt: ops.linear_fp8_wgrad(dy, xt, dt)),
                f"wgrad_{tag}_kernel": (lambda dtq=dtq, dts=dts, dw=dw: ops._gemm_fp8_grad("b", dtq, dts, xt[0], xt[1],
                                                                                            dw, False)),
                f"wgrad_acc_{tag}_call": (lambda dt=dt: ops.linear_fp8_wgrad_accumulate(dy, xt, mg, dt)),
                f"wgrad_acc_{tag}_kernel": (lambda dtq=dtq, dts=dts: ops._gemm_fp8_grad("b", dtq, dts, xt[0], xt[1],
                                                                                         mg, True)),
            })
        best = {k: float("inf") for k in cases}
        for fn in cases.values():
            fn()
        torch.cuda.synchronize()
        for _ in range(windows):
            for k, fn in cases.items():
                best[k] = min(best[k], _time(fn, iters))
        out[name] = {k: round(flops / (ms * 1e-3) / 1e12, 1) for k, ms in best.items()}
        del w, x, dy, wt, xt, mg, cases
        torch.cuda.empty_cache()
    return out


def saved_bytes(layer, x, freqs):
    """Bytes of the distinct storages one forward of `layer` saves for its backward (parameters excluded)."""
    params = {p.untyped_storage().data_ptr() for p in layer.parameters()}
    storages = {}

    def pack(t):
        st = t.untyped_storage()
        if st.data_ptr() not in params:
            storages[st.data_ptr()] = st.nbytes()
        return t

    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        out, _ = layer(hidden_states=x, attention_mask=None, rotary_pos_emb=freqs)
    del out
    return sum(storages.values())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=18432)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--gemm-iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_train needs a CUDA device")
    import long_vita_b200  # noqa: F401

    card, power = _card()
    res = {"card": card, "power_limit_and_max_sm_clock": power, "tokens": a.tokens,
           "step": step_times(a.tokens, a.steps, a.warmup, a.windows),
           "gemm_tflops": gemm_rates(a.tokens, a.gemm_iters, a.windows)}
    print(f"# {card}, power limit / max SM clock: {power}")
    for m, r in res["step"].items():
        print(f"step {m:>6}: {r['step_ms']:8.2f} ms, peak +{r['peak_extra_gib']:.2f} GiB, "
              f"saved for backward {r['saved_for_backward_bytes_per_token']} B / token")
    for name, r in res["gemm_tflops"].items():
        print(f"{name:>5}: " + ", ".join(f"{k} {v}" for k, v in r.items()))
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
