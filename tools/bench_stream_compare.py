"""The row-chunked and the streamed decoder layer on the same prompt, alternately in one process.

    python tools/bench_stream_compare.py [--frames 4096] [--layers 2] [--rounds 2] [--out cmp.json]

Runs `LongVITAForCausalLM.forward` (num_logits_to_keep=1) on the bench prompt of `--frames` frames (4096 -> 1 058 816
tokens; synthetic frames on the device) with a model of `--layers` decoder layers of the 14B geometry, once per plan
and round, in the order row-chunked, streamed, row-chunked, ...  The streamed runs patch hf.modeling.STREAM_THRESHOLD
below the prompt length; the span plan (row_chunks) is the same for both.  Each decoder layer is timed on the host
around a device synchronise.  Prints one JSON line: the card's name and power limit, the seconds per layer of every
run, the mean per plan, and whether the kept logits of every run are torch.equal to the first run's.
"""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from long_vita_b200.config import LongVITAConfig  # noqa: E402
from long_vita_b200.hf import modeling  # noqa: E402
from long_vita_b200.synthetic import build_prompt, synthetic_frames  # noqa: E402
from tools.mem_row_chunks import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4096)
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    name, pl = card()
    cfg = dataclasses.replace(LongVITAConfig.long_vita_14b(), num_hidden_layers=args.layers)
    model = modeling.LongVITAForCausalLM.from_synthetic(cfg, seed=1234, device=dev)
    ids, idx = build_prompt(cfg, args.frames, 16, pad_multiple=2048)
    T = ids.shape[1]
    ids, idx = ids.to(dev), idx.to(dev)
    frames = synthetic_frames(cfg, args.frames, device=dev)

    times = []
    for layer in model.model.layers:
        def timed(*a, _fwd=layer.forward, **kw):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = _fwd(*a, **kw)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
            return out
        layer.forward = timed

    default = modeling.STREAM_THRESHOLD
    runs, first = [], None
    for _ in range(args.rounds):
        for plan in ("row-chunked", "streamed"):
            modeling.STREAM_THRESHOLD = default if plan == "row-chunked" else min(default, T - 1)
            assert modeling.streams(T, modeling.attention_step()) == (plan == "streamed")
            times.clear()
            with torch.no_grad():
                logits = model(input_ids=ids, images=frames, image_indices=idx, num_logits_to_keep=1).logits
            first = logits if first is None else first
            runs.append({"plan": plan, "layer_s": [round(t, 3) for t in times],
                         "logits_equal_first": torch.equal(logits, first)})
            print(json.dumps(runs[-1]), file=sys.stderr, flush=True)
    modeling.STREAM_THRESHOLD = default
    mean = {p: round(sum(sum(r["layer_s"]) for r in runs if r["plan"] == p)
                     / sum(len(r["layer_s"]) for r in runs if r["plan"] == p), 3) for p in ("row-chunked", "streamed")}
    line = {"gpu": name, "power_limit": pl, "tokens": T, "frames": args.frames, "layers": args.layers,
            "spans": len(modeling.row_chunks(T)), "runs": runs, "mean_s_per_layer": mean,
            "all_logits_equal": all(r["logits_equal_first"] for r in runs)}
    print(json.dumps(line), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(line, fh, indent=1)


if __name__ == "__main__":
    main()
