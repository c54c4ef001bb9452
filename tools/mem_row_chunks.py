"""Peak device memory of the long-prompt prefill, per phase, with the row-chunked or the streamed decoder layer.

    python tools/mem_row_chunks.py [--frames 2048 4096] [--layers 2] [--stream-threshold ROWS] [--out mem.json]

Runs `LongVITAForCausalLM.forward` (num_logits_to_keep=1) on the bench prompt of each frame count (2048 frames ->
530 432 tokens, 4096 -> 1 058 816; synthetic frames on the device, as `bench.py --long-run` draws them) with a model of
`--layers` decoder layers of the 14B geometry.  The decoder layers are identical, so the per-layer pattern is that of
the 48-layer model.  Above `--stream-threshold` rows (default: hf.modeling.STREAM_THRESHOLD) the layers stream
(every op, attention included, span by span).  Phases, each the peak of memory allocated above the resident model,
frames and ids:

  vision          the ViT tower + projector (encode_images, or scatter_images when streamed) and the embedding
                  scatter;
  pre-attention   norms, QKV GEMMs and RoPE of a layer (of a span, when streamed), up to its attention call;
  attention       the attention call, up to the O-projection (the row-chunked layer has released its QKV buffer);
  post-attention  O-projection, norm, MLP and residual add, up to the next layer (the next span's Q GEMM, when
                  streamed), or through the final norm and the LM head.

From the two lengths it fits peak = a + b T of the whole forward and gives the largest T the 48-layer model takes on
this card: the 48-layer weights and the frames (which grow with T at 4.67 KB per visual token) are added to the fit,
and the limit is the memory free at start-up plus what this process holds, less 1 GiB for allocator slack.  That
figure is derived from the fit, not run.  Prints one JSON line (the card's name and power limit first).
"""
from __future__ import annotations

import argparse
import dataclasses
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from long_vita_b200 import ops  # noqa: E402
from long_vita_b200.config import LongVITAConfig  # noqa: E402
from long_vita_b200.hf import modeling  # noqa: E402
from long_vita_b200.synthetic import build_prompt, synthetic_frames  # noqa: E402

GiB = 2 ** 30


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                             f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001 - the number is informative only
        pl = f"unknown ({type(e).__name__})"
    return name, pl


class PhasePeaks:
    """Splits max_memory_allocated into phases at the vision tower (LongVITAModel.encode_images or
    hf.modeling.scatter_images), the start of each decoder layer (DecoderLayer.forward), its attention call
    (ops.attention_fwd), the first GEMM after it and a streamed span's Q GEMM (ops.linear), each wrapped for the
    run."""

    def __init__(self, model, base):
        self.base, self.peaks, self.phase = base, {}, None
        self.model, self._attn, self._linear = model, ops.attention_fwd, ops.linear
        ops.attention_fwd, ops.linear = self.attention, self.linear
        self._enc = model.model.encode_images
        model.model.encode_images = self.encode
        self._scatter = modeling.scatter_images
        modeling.scatter_images = self.scatter
        self._wqkv = {layer.wqkv.data_ptr() for layer in model.model.layers}
        for layer in model.model.layers:
            layer.forward = self.layer_entry(layer.forward)

    def close(self):
        self.switch(None)
        ops.attention_fwd, ops.linear = self._attn, self._linear
        modeling.scatter_images = self._scatter
        del self.model.model.encode_images
        for layer in self.model.model.layers:
            del layer.forward

    def switch(self, phase):
        torch.cuda.synchronize()
        if self.phase is not None:
            p = torch.cuda.max_memory_allocated() - self.base
            self.peaks[self.phase] = max(self.peaks.get(self.phase, 0), p)
        torch.cuda.reset_peak_memory_stats()
        self.phase = phase

    def encode(self, images):
        self.switch("vision")          # until the first layer: the ViT, the projector and the embedding scatter
        return self._enc(images)

    def scatter(self, *a, **kw):
        self.switch("vision")          # the streamed form: the ViT chunks, each scattered into x as it is made
        return self._scatter(*a, **kw)

    def layer_entry(self, fwd):
        def run(*a, **kw):
            self.switch("pre-attention")
            return fwd(*a, **kw)
        return run

    def attention(self, *a, **kw):
        if self.phase == "vision":     # the ViT's own attention calls
            return self._attn(*a, **kw)
        self.switch("attention")
        return self._attn(*a, **kw)

    def linear(self, x, weight, *a, **kw):
        if self.phase == "attention":  # the O-projection: the layer has released its QKV buffer
            self.switch("post-attention")     # until the next layer, or through the final norm and the LM head
        elif self.phase == "post-attention" and weight.data_ptr() in self._wqkv:
            self.switch("pre-attention")      # a streamed layer's next span (its Q GEMM)
        return self._linear(x, weight, *a, **kw)


def run(model, cfg, frames_n, dev):
    ids, idx = build_prompt(cfg, frames_n, 16, pad_multiple=2048)
    T = ids.shape[1]
    ids, idx = ids.to(dev), idx.to(dev)
    frames = synthetic_frames(cfg, frames_n, device=dev)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    pp = PhasePeaks(model, base)
    with torch.no_grad():
        logits = model(input_ids=ids, images=frames, image_indices=idx, num_logits_to_keep=1).logits
    pp.close()
    peaks = {k: round(v / GiB, 3) for k, v in pp.peaks.items()}
    total = max(pp.peaks.values()) + base
    del frames, logits
    torch.cuda.empty_cache()
    return T, total, base, peaks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs=2, default=[2048, 4096])
    ap.add_argument("--layers", type=int, default=2)
    ap.add_argument("--stream-threshold", type=int, default=None,
                    help="rows above which the decoder layers stream (default: hf.modeling.STREAM_THRESHOLD)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.stream_threshold is not None:
        modeling.STREAM_THRESHOLD = args.stream_threshold
    dev = torch.device("cuda", 0)
    name, pl = card()
    free0, total_mem = torch.cuda.mem_get_info()
    full = LongVITAConfig.long_vita_14b()
    cfg = dataclasses.replace(full, num_hidden_layers=args.layers)
    model = modeling.LongVITAForCausalLM.from_synthetic(cfg, seed=1234, device=dev)
    layer_bytes = sum(t.numel() * t.element_size() for t in vars(model.model.layers[0]).values()
                      if isinstance(t, torch.Tensor))
    points, rows = [], []
    for f in args.frames:
        T, total, base, peaks = run(model, cfg, f, dev)
        points.append((T, total))
        rows.append({"frames": f, "tokens": T, "resident_gib": round(base / GiB, 3), "phase_peak_above_resident_gib": peaks,
                     "peak_total_gib": round(total / GiB, 3)})
        print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
    (t0, p0), (t1, p1) = points
    b = (p1 - p0) / (t1 - t0)                     # bytes per token, frames included
    a = p0 - b * t0
    missing = (full.num_hidden_layers - args.layers) * layer_bytes
    limit = free0 - GiB                           # what this process could allocate at start-up, less slack
    t_max = int((limit - a - missing) // b) // 2048 * 2048
    line = {"gpu": name, "power_limit": pl, "card_total_gib": round(total_mem / GiB, 2), "layers_run": args.layers,
            "stream_threshold": modeling.STREAM_THRESHOLD,
            "points": rows, "bytes_per_token_fit": round(b, 1), "decoder_layer_gib": round(layer_bytes / GiB, 3),
            "largest_tokens_48_layers_derived": t_max,
            "peak_48_layers_at_longest_derived_gib": round((a + missing + b * points[-1][0]) / GiB, 2)}
    print(json.dumps(line), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(line, fh, indent=1)


if __name__ == "__main__":
    main()
