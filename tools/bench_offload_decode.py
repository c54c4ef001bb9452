"""Decoding with the K/V cache partly in pinned host memory (kv_cache.OffloadedKVCache), on one GPU.

    python tools/bench_offload_decode.py [--rows 131072 1058816 2115584] [--context 1058816] [--reps 5]
                                         [--prefill-reps 2] [--out DIR]

1. Bandwidth: lv_attn_decode_host (+ the merge) over `rows` host rows of the 14B geometry (40:8 x 128, 4 KB per
   row), against a pinned host-to-device `copy_` of the same bytes in the same process, runs alternated: the copy is
   the PCIe roofline, and the obvious alternative design (stage the layer on the device, then attention_decode).
2. Decode step at `--context` tokens on a 14B model of 1 and of 2 decoder layers, every layer on the device or every
   layer on the host; ms per layer = step(2 layers) - step(1 layer).  Extrapolated to 48 layers with the placement
   kv_cache.device_layers picks for that prompt on this card (derived, not measured).
3. One layer's device-to-host row copy at `--context` rows, strided (row-chunked layer) and contiguous (streamed
   layer), and the time to pin its host buffer.  Then the prefill of a `--context`-token text prompt on a 2-layer 14B
   model without a cache and with both layers on the host tier, runs alternated: the time the row copies add.

Prints one JSON object (and writes it to DIR/offload_decode.json with --out), with the card's name and power limit
read in the same run.  Random weights, ids and cache rows: the timings do not depend on their values.
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from long_vita_b200 import kv_cache, ops  # noqa: E402
from long_vita_b200.config import LongVITAConfig  # noqa: E402
from long_vita_b200.hf import modeling  # noqa: E402
from long_vita_b200.hf.modeling import LongVITAForCausalLM  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return r.stdout.strip() or torch.cuda.get_device_name(0)


def timed(fn, n=1):
    """Device milliseconds of n calls of fn (CUDA events)."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def fill_host(host, g):
    """Random bf16 rows, written through a device buffer of 65 536 rows at a time."""
    for r0 in range(0, host.shape[0], 65536):
        r1 = min(r0 + 65536, host.shape[0])
        host[r0:r1].copy_(torch.randn((r1 - r0, host.shape[1]), device="cuda", generator=g).to(torch.bfloat16))


def bandwidth(rows_list, reps, cfg):
    hkv, d = cfg.num_key_value_heads, cfg.head_dim
    out = []
    g = torch.Generator(device="cuda").manual_seed(1)
    q = torch.randn((cfg.num_attention_heads, d), device="cuda", generator=g).to(torch.bfloat16)
    for rows in rows_list:
        host = ops.pinned_rows(rows, 2 * hkv * d)
        fill_host(host, g)
        dev = torch.empty(host.shape, dtype=host.dtype, device="cuda")
        kernel = lambda: ops.attention_decode_host(q, host, rows)           # noqa: E731
        copy = lambda: dev.copy_(host, non_blocking=True)                     # noqa: E731
        kernel(), copy()
        tk, tc = [], []
        for _ in range(reps):
            tk.append(timed(kernel))
            tc.append(timed(copy))
        nbytes = host.numel() * 2
        mk, mc = statistics.median(tk), statistics.median(tc)
        out.append({"rows": rows, "bytes": nbytes, "kernel_ms": mk, "copy_ms": mc, "kernel_gbs": nbytes / mk / 1e6,
                    "copy_gbs": nbytes / mc / 1e6, "kernel_over_copy": mc / mk,
                    "kernel_ms_all": tk, "copy_ms_all": tc})
        del host, dev
        gc.collect()
        torch.cuda.empty_cache()
    return out


def filled_cache(model, n_layers, T, on_host, g):
    cfg = model.config
    if on_host:
        c = kv_cache.OffloadedKVCache(n_layers, 0, T + 64, cfg.num_key_value_heads, cfg.head_dim, "cuda")
        for h in c.host:
            fill_host(h, g)
    else:
        c = kv_cache.KVCache(n_layers, T + 64, cfg.num_key_value_heads, cfg.head_dim, "cuda")
        for t in c.k + c.v:
            t.normal_(generator=g)
    c._len = T
    return c


def decode_steps(model, T, reps):
    layers = model.model.layers
    g = torch.Generator(device="cuda").manual_seed(2)
    tok = torch.zeros((1, 1), dtype=torch.int64, device="cuda")
    res = {}
    for on_host in (False, True):
        for n in (1, 2):
            model.model.layers = layers[:n]
            cache = filled_cache(model, n, T, on_host, g)

            def step():
                cache._len = T                   # every step decodes the token at position T
                model(input_ids=tok, past_key_values=cache, use_cache=True, num_logits_to_keep=1)
            step()
            res[(on_host, n)] = statistics.median(timed(step) for _ in range(reps))
            del cache
            gc.collect()
            torch.cuda.empty_cache()
    model.model.layers = layers
    return res


def row_copies(cfg, T, reps):
    """Seconds of one layer's K|V rows to the host tier: the row-chunked layer's strided copy out of a QKV buffer
    (pitch (hq + 2 hkv) d) and the streamed layer's contiguous copy out of its K|V buffer."""
    hq, hkv, d = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    host = ops.pinned_rows(T, 2 * hkv * d)
    out = {}
    for name, cols in (("strided_s", (hq + 2 * hkv) * d), ("contiguous_s", 2 * hkv * d)):
        buf = torch.zeros((T, cols), dtype=torch.bfloat16, device="cuda")
        k = buf[:, cols - 2 * hkv * d : cols - hkv * d].view(T, hkv, d)
        v = buf[:, cols - hkv * d :].view(T, hkv, d)
        ops.kv_rows_to_host(k, v, host)
        out[name] = statistics.median(timed(lambda: ops.kv_rows_to_host(k, v, host)) for _ in range(reps)) / 1e3
        del buf, k, v
        torch.cuda.empty_cache()
    t0 = time.perf_counter()
    extra = ops.pinned_rows(T, 2 * hkv * d)
    out["pinned_alloc_s"] = time.perf_counter() - t0
    out["gbs"] = {k: T * 4 * hkv * d / t / 1e9 for k, t in out.items() if k != "pinned_alloc_s"}
    del host, extra
    gc.collect()
    return out


def prefill(model, T, reps):
    """Seconds of a prefill without a cache and with every layer on the host tier (the cache, made beforehand, is
    passed empty: its pinned allocation is not in the time)."""
    g = torch.Generator(device="cuda").manual_seed(3)
    ids = torch.randint(0, model.config.vocab_size, (1, T), device="cuda", generator=g)
    cfg = model.config
    times = {"none": [], "host": []}
    for _ in range(reps):
        for kind in ("none", "host"):
            cache = None
            if kind == "host":
                cache = kv_cache.OffloadedKVCache(len(model.model.layers), 0, T + 1, cfg.num_key_value_heads,
                                                  cfg.head_dim, "cuda")
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            with torch.no_grad():
                out = model(input_ids=ids, past_key_values=cache, use_cache=kind == "host", num_logits_to_keep=1)
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
    ap.add_argument("--prefill-reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    cfg = LongVITAConfig()
    res = {"card": card(), "bandwidth": bandwidth(a.rows, a.reps, cfg)}
    for b in res["bandwidth"]:
        print(f"[bandwidth] {b['rows']} rows: kernel {b['kernel_gbs']:.1f} GB/s, pinned copy {b['copy_gbs']:.1f} GB/s "
              f"({100 * b['kernel_over_copy']:.0f} %)", flush=True)

    model = LongVITAForCausalLM.from_synthetic(cfg, seed=1234, device="cuda", num_layers=2)
    T = a.context
    with torch.no_grad():
        st = decode_steps(model, T, a.reps)
    dev_layer, host_layer = st[(False, 2)] - st[(False, 1)], st[(True, 2)] - st[(True, 1)]
    rest = st[(False, 1)] - dev_layer
    L = cfg.num_hidden_layers
    free = kv_cache.device_free_bytes("cuda")
    # the placement a 48-layer model would get for this prompt: free memory with the other 46 layers' weights resident
    layer_w = sum(t.numel() * t.element_size() for t in vars(model.model.layers[0]).values() if torch.is_tensor(t))
    free48 = free - (L - 2) * layer_w
    n_dev = kv_cache.device_layers(free48, T + 1024, L, 2 * 2 * cfg.num_key_value_heads * cfg.head_dim,
                                   T * modeling.prefill_bytes_per_token(cfg, T, False),
                                   T * modeling.prefill_bytes_per_token(cfg, T, T > modeling.STREAM_THRESHOLD))
    res["decode"] = {"context": T, "step_ms": {f"{'host' if h else 'device'}_{n}_layers": v for (h, n), v in st.items()},
                     "device_layer_ms": dev_layer, "host_layer_ms": host_layer, "rest_of_step_ms": rest,
                     "derived_48_layers": {"device_layers": n_dev,
                                           "ms_per_token": rest + n_dev * dev_layer + (L - n_dev) * host_layer,
                                           "ms_per_token_all_host": rest + L * host_layer}}
    print(f"[decode] {T} tokens: {dev_layer:.2f} ms per device layer, {host_layer:.2f} ms per host layer; "
          f"48 layers with {n_dev} on the device: {res['decode']['derived_48_layers']['ms_per_token']:.0f} ms per "
          f"token (derived)", flush=True)

    res["row_copies"] = row_copies(cfg, T, a.reps)
    print(f"[row copies] one layer, {T} rows: {res['row_copies']}", flush=True)
    pf = prefill(model, T, a.prefill_reps)
    none, host = statistics.median(pf["none"]), statistics.median(pf["host"])
    res["prefill"] = {"context": T, "layers": 2, "s_no_cache": pf["none"], "s_host_cache": pf["host"],
                      "added_s_per_host_layer": (host - none) / 2, "added_fraction": (host - none) / none}
    print(f"[prefill] {T} tokens, 2 layers: {none:.2f} s without a cache, {host:.2f} s with both layers on the host "
          f"({100 * (host - none) / none:+.2f} %); pinning the cache beforehand took "
          f"{2 * res['row_copies']['pinned_alloc_s']:.2f} s", flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "offload_decode.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
