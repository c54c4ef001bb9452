"""The FP8 host tier of the K/V cache against the bf16 one, on one GPU, alternated in one process.

    python tools/bench_offload_fp8.py [--rows 131072 1058816 2115584] [--context 1058816] [--reps 5]
                                      [--prefill-reps 1] [--out DIR]

1. Bandwidth: lv_attn_decode_host and lv_attn_decode_host_fp8 (+ the merge) over `rows` host rows of the 14B geometry
   (40:8 x 128; 4096 and 2112 bytes per row), each against a pinned host-to-device `copy_` of its own bytes.
2. Decode step at `--context` tokens on a 14B model of 1 and 2 decoder layers with every layer on the host, bf16 and
   FP8: ms per host layer = step(2 layers) - step(1 layer).  The 48-layer figure with 46 host layers is derived.
3. One layer's rows to the host at `--context` rows (strided, out of a QKV buffer): lv_rows_to_host against
   lv_rows_to_host_fp8; the time to pin one layer's buffer in each format; and the prefill of a `--context`-token
   text prompt on the 2-layer model without a cache, with a bf16 and with an FP8 host tier, alternated.

Prints one JSON object (and writes DIR/offload_fp8.json with --out), with the card's name and power limit read in
the same run.  Random weights, ids and cache rows: the timings do not depend on their values.
"""
import argparse
import gc
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_offload_decode import card, fill_host, timed  # noqa: E402
from long_vita_b200 import kv_cache, ops  # noqa: E402
from long_vita_b200.config import LongVITAConfig  # noqa: E402
from long_vita_b200.hf.modeling import LongVITAForCausalLM  # noqa: E402

FP8 = torch.float8_e4m3fn
FORMATS = (torch.bfloat16, FP8)


def name(dt):
    return "fp8" if dt == FP8 else "bf16"


def fill_fp8(host, g):
    """Random rows quantised into host by lv_rows_to_host_fp8, 65 536 rows at a time."""
    hkv = host.shape[1] // (2 * 128 + 8)              # ops.kv_fp8_row_bytes(hkv, 128) is in [264 hkv, 264 hkv + 8)
    for r0 in range(0, host.shape[0], 65536):
        r1 = min(r0 + 65536, host.shape[0])
        kv = torch.randn((r1 - r0, 2, hkv, 128), device="cuda", generator=g).to(torch.bfloat16)
        ops.kv_rows_to_host_fp8(kv[:, 0], kv[:, 1], host[r0:r1])
    torch.cuda.synchronize()


def host_layer(dt, rows, cfg, g):
    hkv, d = cfg.num_key_value_heads, cfg.head_dim
    if dt == FP8:
        h = ops.pinned_fp8_rows(rows, hkv, d)
        fill_fp8(h, g)
    else:
        h = ops.pinned_rows(rows, 2 * hkv * d)
        fill_host(h, g)
    return h


def bandwidth(rows_list, reps, cfg):
    out = []
    g = torch.Generator(device="cuda").manual_seed(1)
    q = torch.randn((cfg.num_attention_heads, cfg.head_dim), device="cuda", generator=g).to(torch.bfloat16)
    for rows in rows_list:
        hosts = {dt: host_layer(dt, rows, cfg, g) for dt in FORMATS}
        devs = {dt: torch.empty(h.shape, dtype=h.dtype, device="cuda") for dt, h in hosts.items()}
        fns = {("kernel", torch.bfloat16): lambda: ops.attention_decode_host(q, hosts[torch.bfloat16], rows),
               ("kernel", FP8): lambda: ops.attention_decode_host_fp8(q, hosts[FP8], rows)}
        for dt in FORMATS:
            fns[("copy", dt)] = (lambda dt=dt: devs[dt].copy_(hosts[dt], non_blocking=True))
        for f in fns.values():
            f()
        t = {k: [] for k in fns}
        for _ in range(reps):
            for k, f in fns.items():
                t[k].append(timed(f))
        for dt in FORMATS:
            nbytes = hosts[dt].numel() * hosts[dt].element_size()
            mk, mc = statistics.median(t[("kernel", dt)]), statistics.median(t[("copy", dt)])
            out.append({"format": name(dt), "rows": rows, "bytes": nbytes, "kernel_ms": mk, "copy_ms": mc,
                        "kernel_gbs": nbytes / mk / 1e6, "copy_gbs": nbytes / mc / 1e6, "kernel_over_copy": mc / mk,
                        "kernel_ms_all": t[("kernel", dt)], "copy_ms_all": t[("copy", dt)]})
        del hosts, devs
        gc.collect()
        torch.cuda.empty_cache()
    return out


def host_cache(model, n_layers, T, dt, g):
    cfg = model.config
    c = kv_cache.OffloadedKVCache(n_layers, 0, T + 64, cfg.num_key_value_heads, cfg.head_dim, "cuda", host_dtype=dt)
    for h in c.host:
        (fill_fp8 if dt == FP8 else fill_host)(h, g)
    c._len = T
    return c


def decode_steps(model, T, reps):
    layers = model.model.layers
    g = torch.Generator(device="cuda").manual_seed(2)
    tok = torch.zeros((1, 1), dtype=torch.int64, device="cuda")
    caches = {dt: host_cache(model, 2, T, dt, g) for dt in FORMATS}   # the 1-layer model reads the first layer
    t = {(dt, n): [] for dt in FORMATS for n in (1, 2)}
    for _ in range(reps):
        for (dt, n) in t:
            cache = caches[dt]
            model.model.layers = layers[:n]

            def step():
                cache._len = T                   # every step decodes the token at position T
                model(input_ids=tok, past_key_values=cache, use_cache=True, num_logits_to_keep=1)
            step()
            t[(dt, n)].append(timed(step))
    model.model.layers = layers
    del caches
    gc.collect()
    torch.cuda.empty_cache()
    return {k: statistics.median(v) for k, v in t.items()}


def row_copies(cfg, T, reps):
    """Seconds of one layer's K|V rows out of a QKV buffer (pitch (hq + 2 hkv) d) to a bf16 and to an FP8 host layer,
    and seconds to pin each layer buffer."""
    hq, hkv, d = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    cols = (hq + 2 * hkv) * d
    buf = torch.randn((T, cols), device="cuda").to(torch.bfloat16)
    k, v = buf[:, hq * d : (hq + hkv) * d].view(T, hkv, d), buf[:, (hq + hkv) * d :].view(T, hkv, d)
    out = {"pin_s": {}, "copy_s": {}}
    hosts = {}
    for dt in FORMATS:
        t0 = time.perf_counter()
        hosts[dt] = ops.pinned_fp8_rows(T, hkv, d) if dt == FP8 else ops.pinned_rows(T, 2 * hkv * d)
        out["pin_s"][name(dt)] = time.perf_counter() - t0
    fns = {torch.bfloat16: lambda: ops.kv_rows_to_host(k, v, hosts[torch.bfloat16]),
           FP8: lambda: ops.kv_rows_to_host_fp8(k, v, hosts[FP8])}
    for f in fns.values():
        f()
    t = {dt: [] for dt in FORMATS}
    for _ in range(reps):
        for dt, f in fns.items():
            t[dt].append(timed(f) / 1e3)
    for dt in FORMATS:
        s = statistics.median(t[dt])
        out["copy_s"][name(dt)] = s
        out.setdefault("host_gbs", {})[name(dt)] = hosts[dt].numel() * hosts[dt].element_size() / s / 1e9
    del buf, k, v, hosts
    gc.collect()
    torch.cuda.empty_cache()
    return out


def prefill(model, T, reps):
    """Seconds of a prefill without a cache and with every layer on a bf16 / FP8 host tier (the cache, made
    beforehand, is passed empty: its pinned allocation is not in the time)."""
    g = torch.Generator(device="cuda").manual_seed(3)
    ids = torch.randint(0, model.config.vocab_size, (1, T), device="cuda", generator=g)
    cfg = model.config
    times = {"none": [], "bf16": [], "fp8": []}
    for _ in range(reps):
        for kind in times:
            cache = None
            if kind != "none":
                cache = kv_cache.OffloadedKVCache(len(model.model.layers), 0, T + 1, cfg.num_key_value_heads,
                                                  cfg.head_dim, "cuda", host_dtype=FP8 if kind == "fp8" else
                                                  torch.bfloat16)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with torch.no_grad():
                out = model(input_ids=ids, past_key_values=cache, use_cache=cache is not None, num_logits_to_keep=1)
            torch.cuda.synchronize()
            times[kind].append(time.perf_counter() - t0)
            del out, cache
            gc.collect()
            torch.cuda.empty_cache()
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[131072, 1058816, 2115584])
    ap.add_argument("--context", type=int, default=1058816)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--prefill-reps", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    cfg = LongVITAConfig()
    res = {"card": card(), "bandwidth": bandwidth(a.rows, a.reps, cfg)}
    for b in res["bandwidth"]:
        print(f"[bandwidth] {b['format']} {b['rows']} rows: kernel {b['kernel_ms']:.1f} ms, {b['kernel_gbs']:.1f} GB/s; "
              f"pinned copy {b['copy_gbs']:.1f} GB/s ({100 * b['kernel_over_copy']:.0f} %)", flush=True)

    model = LongVITAForCausalLM.from_synthetic(cfg, seed=1234, device="cuda", num_layers=2)
    T = a.context
    with torch.no_grad():
        st = decode_steps(model, T, a.reps)
    L = cfg.num_hidden_layers
    res["decode"] = {"context": T, "step_ms": {f"{name(dt)}_{n}_layers": v for (dt, n), v in st.items()}}
    for dt in FORMATS:
        host_ms = st[(dt, 2)] - st[(dt, 1)]
        res["decode"][f"{name(dt)}_host_layer_ms"] = host_ms
        res["decode"][f"{name(dt)}_derived_48_layers_46_on_host_s"] = 46 * host_ms / 1e3
        print(f"[decode] {name(dt)}, {T} tokens: {host_ms:.2f} ms per host layer; 46 host layers "
              f"~{46 * host_ms / 1e3:.2f} s per token (derived)", flush=True)

    res["row_copies"] = row_copies(cfg, T, a.reps)
    print(f"[row copies] one layer, {T} rows: {res['row_copies']}", flush=True)
    pf = prefill(model, T, a.prefill_reps)
    none = statistics.median(pf["none"])
    res["prefill"] = {"context": T, "layers": 2, "s": pf}
    for kind in ("bf16", "fp8"):
        t = statistics.median(pf[kind])
        res["prefill"][f"{kind}_added_fraction"] = (t - none) / none
        print(f"[prefill] {T} tokens, 2 layers: {none:.2f} s without a cache, {t:.2f} s with both layers on a {kind} "
              f"host tier ({100 * (t - none) / none:+.2f} %)", flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "offload_fp8.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
