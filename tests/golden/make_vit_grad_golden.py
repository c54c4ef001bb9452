"""Generate tests/golden/ref_vit_grads.pt from the reference's OWN modules (run where /root/reference is mounted):
    python tests/golden/make_vit_grad_golden.py

The reference's HF InternVisionModel + ResamplerProjector (modeling_intern_vit.py, resampler_projector.py), loaded as
oracle/ref_loader.py loads them for ref_vit_tiny.pt, run forward and backward in fp32 torch autograd on
LongVITAConfig.tiny(vit_layers=2): two seeded frames, the class token dropped before the projector
(modeling_long_vita.py:97) and a seeded upstream gradient on the projector output.  The file holds the projector
output and the gradient of every parameter (HF names), subsampled (`subsample`) so that it stays under 1 MB.
Machines without the reference only read the file; `golden_inputs` regenerates the inputs.
"""
import hashlib
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from long_vita_b200.config import LongVITAConfig  # noqa: E402
from long_vita_b200.weights import synthetic_state_dict  # noqa: E402

SEED = 5151
N_FRAMES = 2
STRIDE = 5            # flat stride of the stored gradients of tensors with more than KEEP_WHOLE elements
KEEP_WHOLE = 4096
TOKEN_STRIDE = 8      # every 8th projector output token is stored


def golden_config():
    return LongVITAConfig.tiny(layers=1, vit_layers=2)


def golden_inputs():
    """(cfg, vision weights fp32 with HF names, images fp32 [2, 3, 448, 448] (bf16-representable), upstream grad)."""
    cfg = golden_config()
    v = cfg.visual
    w = synthetic_state_dict(cfg, seed=SEED, dtype=torch.float32, perturb=True, llm_layers=[])
    w = {k: t for k, t in w.items() if k.startswith(("model.vision_model.", "model.vision_projection."))}
    g = torch.Generator().manual_seed(SEED)
    images = torch.randn(N_FRAMES, 3, v.image_size, v.image_size, generator=g).to(torch.bfloat16).float()
    d_out = torch.randn(N_FRAMES, v.tokens_per_image, cfg.hidden_size, generator=g)
    return cfg, w, images, d_out


def subsample(t: torch.Tensor) -> torch.Tensor:
    flat = t.reshape(-1)
    return flat.clone() if flat.numel() <= KEEP_WHOLE else flat[::STRIDE].clone()


def sha(t: torch.Tensor) -> str:
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def main():
    from oracle import ref_loader

    ref = ref_loader.load()
    cfg, w, images, d_out = golden_inputs()
    v = cfg.visual
    vcfg = ref.InternVisionConfig(
        num_channels=3, patch_size=v.patch_size, image_size=v.image_size, qkv_bias=True, hidden_size=v.hidden_size,
        num_attention_heads=v.num_attention_heads, intermediate_size=v.intermediate_size, qk_normalization=False,
        num_hidden_layers=v.num_hidden_layers, use_flash_attn=False, hidden_act="gelu", norm_type="layer_norm",
        layer_norm_eps=v.layer_norm_eps, dropout=0.0, drop_path_rate=0.0, attention_dropout=0.0,
        initializer_range=0.02, initializer_factor=1.0,
    )
    model = ref.InternVisionModel(vcfg).train()
    model.load_state_dict({k[len("model.vision_model."):]: t for k, t in w.items() if k.startswith("model.vision_model.")},
                          strict=True)
    proj = ref.ResamplerProjector(types.SimpleNamespace(hidden_size=cfg.hidden_size), vcfg).train()
    proj.load_state_dict({k[len("model.vision_projection."):]: t for k, t in w.items()
                          if k.startswith("model.vision_projection.")}, strict=True)
    vit_out = model(images).last_hidden_state
    out = proj(vit_out[:, 1:, :])
    out.backward(d_out)
    grads = {}
    for prefix, mod in (("model.vision_model.", model), ("model.vision_projection.", proj)):
        for name, p in mod.named_parameters():
            assert p.grad is not None, name
            grads[prefix + name] = subsample(p.grad)
    assert set(grads) == set(w), set(grads) ^ set(w)
    path = os.path.join(HERE, "ref_vit_grads.pt")
    torch.save({"seed": SEED, "stride": STRIDE, "keep_whole": KEEP_WHOLE, "token_stride": TOKEN_STRIDE,
                "images_sha256": sha(images), "d_out_sha256": sha(d_out),
                "out_sub": out.detach()[:, ::TOKEN_STRIDE].clone(), "grads_sub": grads}, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
