"""Time forward + backward of the trainable vision side (`B200VisionModel`: InternViT-300M + projector) against the same
tower in eager bf16 PyTorch (nn.functional layers, SDPA attention), the stand-in for the stock Megatron modules the
reference trains with.

    python tools/bench_vit_train.py [--frames 64 256] [--iters 5] [--warmup 2]

Configurations (one JSON line each):
  * "train"        - the whole tower and the projector train (stage 2 of the 14B fine-tuning scripts; 64 frames is a
                     16K-token packed sample's worth of images);
  * "vit_frozen"   - `vision_model_freeze`: the tower runs under no_grad, only the projector trains (stages 1, 3, 4).
A configuration that does not fit in device memory is reported as such instead of timed.  FLOPs are algorithmic,
from the shapes: forward GEMMs + attention (4 S^2 C per frame and layer); a trained part counts 3x its forward.
Peak memory is torch.cuda.max_memory_allocated over one step, and `saved_bytes_per_frame` the memory the forward
leaves allocated for the backward, divided by the frame count.  The card name and its power limit are printed with the
numbers.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from long_vita_b200.config import LongVITAConfig  # noqa: E402
from long_vita_b200.megatron.vision_model import B200VisionModel  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                             f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001 - the number is informative only
        pl = f"unknown ({type(e).__name__})"
    return name, pl


def flops(cfg, frames):
    """(ViT forward, projector forward) FLOPs for `frames` frames."""
    v = cfg.visual
    C, Fh, S = v.hidden_size, v.intermediate_size, v.num_patches + 1
    per_layer = 2 * S * C * 3 * C + 2 * S * C * C + 4 * S * C * Fh + 4 * S * S * C
    vit = frames * (2 * v.num_patches * C * 3 * v.patch_size ** 2 + v.num_hidden_layers * per_layer)
    proj = frames * (2 * 256 * 4 * C * C + 2 * 256 * C * cfg.hidden_size)
    return vit, proj


class EagerVision(torch.nn.Module):
    """The same tower in plain bf16 PyTorch, sharing B200VisionModel's parameters (Megatron layouts)."""

    def __init__(self, m: B200VisionModel):
        super().__init__()
        self.m = m

    def forward(self, images):
        m, v = self.m, self.m.vcfg
        vit = m.vit
        H, D, C = v.num_attention_heads, v.head_dim, v.hidden_size
        freeze_ctx = torch.no_grad() if m.vision_model_freeze else torch.enable_grad()
        with freeze_ctx:
            x = F.conv2d(images, vit.conv1.weight, vit.conv1.bias, stride=v.patch_size).flatten(2).transpose(1, 2)
            x = torch.cat([vit.class_token.expand(x.shape[0], 1, C), x], dim=1) + vit.position_embeddings.weight
            n, S, _ = x.shape
            for L in vit.decoder.layers:
                a, mm = L.self_attention, L.mlp
                h = F.layer_norm(x, (C,), L.input_layernorm.weight, L.input_layernorm.bias, m.eps)
                qkv = F.linear(h, a.linear_qkv.weight, a.linear_qkv.bias).view(n, S, H, 3, D)
                q, k, vv = (qkv[:, :, :, i].transpose(1, 2) for i in range(3))
                o = F.scaled_dot_product_attention(q, k, vv).transpose(1, 2).reshape(n, S, C)
                x = x + F.linear(o, a.linear_proj.weight, a.linear_proj.bias) * L.ls1
                h = F.layer_norm(x, (C,), L.pre_mlp_layernorm.weight, L.pre_mlp_layernorm.bias, m.eps)
                f = F.linear(F.gelu(F.linear(h, mm.linear_fc1.weight, mm.linear_fc1.bias)), mm.linear_fc2.weight,
                             mm.linear_fc2.bias)
                x = x + f * L.ls2
            g = v.grid
            x = x[:, 1:].reshape(n, g // 2, 2, g // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(n, -1, 4 * C)
        enc = m.vision_projection.encoder
        y = F.layer_norm(x, (4 * C,), m.pre_proj_layernorm.weight, m.pre_proj_layernorm.bias, m.pre_proj_eps)
        return F.linear(F.gelu(F.linear(y, enc.linear_fc1.weight)), enc.linear_fc2.weight)


def step(fn, images, d_out):
    out = fn(images)
    out.backward(d_out)


def measure(fn, model, images, d_out, iters, warmup):
    for _ in range(warmup):
        step(fn, images, d_out)
        model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    # memory left allocated by the forward for the backward
    base = torch.cuda.memory_allocated()
    out = fn(images)
    torch.cuda.synchronize()
    saved = torch.cuda.memory_allocated() - base - out.numel() * out.element_size()
    out.backward(d_out)
    del out
    model.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        step(fn, images, d_out)
        model.zero_grad(set_to_none=True)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, torch.cuda.max_memory_allocated(), saved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--configs", nargs="+", default=["train", "vit_frozen"])
    args = ap.parse_args()
    name, pl = card()
    print(json.dumps({"card": name, "power_limit": pl, "torch": torch.__version__}), flush=True)
    cfg = LongVITAConfig()
    for conf in args.configs:
        m = B200VisionModel(cfg.hidden_size, cfg.visual, device="cuda", vision_model_freeze=(conf == "vit_frozen"))
        eager = EagerVision(m)
        for n in args.frames:
            g = torch.Generator(device="cuda").manual_seed(n)
            images = torch.randn(n, 3, 448, 448, generator=g, device="cuda").to(torch.bfloat16)
            d_out = torch.randn(n, 256, cfg.hidden_size, generator=g, device="cuda").to(torch.bfloat16)
            fv, fp = flops(cfg, n)
            work = (fv if conf == "vit_frozen" else 3 * fv) + 3 * fp
            rec = {"config": conf, "frames": n, "tokens": n * (cfg.visual.num_patches + 1), "algorithmic_tflop": work / 1e12}
            for impl, fn in (("b200", lambda x: m(images=x)), ("eager_sdpa", eager)):
                try:
                    ms, peak, saved = measure(fn, m, images, d_out, args.iters, args.warmup)
                    rec[impl] = {"ms": round(ms, 2), "tflops": round(work / ms / 1e9, 1), "peak_gb": round(peak / 2 ** 30, 2),
                                 "saved_bytes_per_frame": int(saved / n)}
                except torch.cuda.OutOfMemoryError:
                    rec[impl] = "out of memory"
                m.zero_grad(set_to_none=True)
                torch.cuda.empty_cache()
            if isinstance(rec["b200"], dict) and isinstance(rec["eager_sdpa"], dict):
                rec["speedup_vs_eager"] = round(rec["eager_sdpa"]["ms"] / rec["b200"]["ms"], 3)
            print(json.dumps(rec), flush=True)
            del images, d_out
        del m, eager
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
