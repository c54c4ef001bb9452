"""Trainable InternViT-300M tower + projector on the fused kernels: a drop-in for `MegatronVisionModel`.

The reference builds its vision side in `long_vita_megatron/pretrain_long_vita.py:310-596` (`MegatronVisionModel`,
reached through the module-level `vision_model_provider`, :599-601, which `model_provider` passes to GPTVLModel as
`external_feature_model_provider`, :641-655).  `B200VisionModel` is that module for `--vision-model-type intern_300m`
with every forward and backward operator in liblvb200.so:

    images [N, 3, 448, 448] -> chunks of 256 frames (forward_chunk, :522-533)
      -> conv1 + class token + position embedding          (InternViTModel.forward, intern_vit_model.py:203-216)
      -> 24 x [LN -> QKV -> attention -> proj -> *ls1 + res -> LN -> fc1 -> GELU -> fc2 -> *ls2 + res]
                                                            (InternViTTransformerLayer.forward, intern_vit_model.py:40-85)
      -> drop cls + pixel-shuffle x0.5                      (forward_downsample, :467-483, 572-582)
      -> pre_proj_layernorm -> linear_fc1 -> GELU -> linear_fc2   (forward_projection, :455-465)
      -> [N, 256, hidden]

Parameters carry Megatron's names and layouts (`vit.conv1.*`, `vit.class_token`, `vit.position_embeddings.weight`,
`vit.decoder.layers.{i}.…`, `pre_proj_layernorm.*`, `vision_projection.encoder.linear_fc{1,2}.weight`): the keys
`megatron/checkpoint.py` maps under `external_feature_model.`, and the names the reference's layer-wise learning-rate
decay keys on.  `linear_qkv` keeps the per-head [H, (q, k, v), D] row interleave; attention reads q / k / v as strided
views of the GEMM output and writes dQ / dK / dV through the same strides into one buffer (`ops.vit_attention`).

One forward body serves training and inference: every operator is a `torch.autograd.Function`, which records nothing
under `no_grad`.  In that body fc1 runs without its activation and GELU follows as its own kernel, so the backward has
the bf16 pre-activation (Megatron's MLP applies the activation after the linear in the same way).

`vision_model_freeze` / `vision_projector_freeze` run the tower / the projector under `no_grad`, as the reference does
(:485-520).  Recompute and vision context parallelism are refused (NotImplementedError); no shipped 14B script sets
them.  `gradient_accumulation_fusion` (`--no-gradient-accumulation-fusion` unset) adds every weight gradient of the
tower and the projector, the patch-embedding conv weight included, to the weight's fp32 `main_grad` inside the GEMM.
The flags are read once, at construction.
"""
from __future__ import annotations

from contextlib import nullcontext
from typing import Optional

import torch

from .. import ops
from ..config import VisionConfig


class _Params(torch.nn.Module):
    """Empty container so parameters get Megatron's dotted names."""


class B200VisionModel(torch.nn.Module):
    chunk_size = 256           # frames per ViT call (MegatronVisionModel.forward_chunk, pretrain_long_vita.py:522-533)

    def __init__(self, hidden_size: int, vision: Optional[VisionConfig] = None, *, vision_model_freeze: bool = False,
                 vision_projector_freeze: bool = False, vision_model_recompute: bool = False,
                 vision_projector_recompute: bool = False, vision_context_parallel: bool = False,
                 layernorm_epsilon: Optional[float] = None, params_dtype=torch.bfloat16, device=None,
                 gradient_accumulation_fusion: bool = False):
        super().__init__()
        if vision_model_recompute or vision_projector_recompute:
            raise NotImplementedError("B200VisionModel: --vision-model-recompute / --vision-projector-recompute are not "
                                      "supported (activations are kept for the backward)")
        if vision_context_parallel:
            raise NotImplementedError("B200VisionModel: --vision-context-parallel is not supported")
        v = vision or VisionConfig()
        self.vcfg = v
        self.vision_model_freeze = bool(vision_model_freeze)
        self.vision_projector_freeze = bool(vision_projector_freeze)
        self.gradient_accumulation_fusion = bool(gradient_accumulation_fusion)
        self.eps = v.layer_norm_eps if layernorm_epsilon is None else float(layernorm_epsilon)
        self.pre_proj_eps = v.pre_proj_ln_eps
        C, F, ps = v.hidden_size, v.intermediate_size, v.patch_size
        if device is None:
            device = torch.cuda.current_device() if torch.cuda.is_available() else "cpu"
        dt = params_dtype

        def P(*shape, fill=None, std=0.02):
            t = torch.empty(*shape, dtype=dt, device=device)
            t = t.fill_(fill) if fill is not None else t.normal_(0, std)
            return torch.nn.Parameter(t)

        self.vit = _Params()
        vit = self.vit
        vit.conv1 = _Params()
        vit.conv1.weight = P(C, 3, ps, ps)
        vit.conv1.bias = P(C, fill=0.0)
        vit.class_token = P(1, 1, C, std=1.0)
        vit.position_embeddings = _Params()
        vit.position_embeddings.weight = P(v.num_patches + 1, C)
        vit.decoder = _Params()
        layers = []
        for _ in range(v.num_hidden_layers):
            L = _Params()
            L.input_layernorm = _Params()
            L.input_layernorm.weight, L.input_layernorm.bias = P(C, fill=1.0), P(C, fill=0.0)
            L.self_attention = _Params()
            L.self_attention.linear_qkv = _Params()
            L.self_attention.linear_qkv.weight, L.self_attention.linear_qkv.bias = P(3 * C, C), P(3 * C, fill=0.0)
            L.self_attention.linear_proj = _Params()
            L.self_attention.linear_proj.weight, L.self_attention.linear_proj.bias = P(C, C), P(C, fill=0.0)
            L.pre_mlp_layernorm = _Params()
            L.pre_mlp_layernorm.weight, L.pre_mlp_layernorm.bias = P(C, fill=1.0), P(C, fill=0.0)
            L.mlp = _Params()
            L.mlp.linear_fc1 = _Params()
            L.mlp.linear_fc1.weight, L.mlp.linear_fc1.bias = P(F, C), P(F, fill=0.0)
            L.mlp.linear_fc2 = _Params()
            L.mlp.linear_fc2.weight, L.mlp.linear_fc2.bias = P(C, F), P(C, fill=0.0)
            L.ls1, L.ls2 = P(C, fill=0.01), P(C, fill=0.01)           # InternViTTransformerLayer, intern_vit_model.py:30-31
            layers.append(L)
        vit.decoder.layers = torch.nn.ModuleList(layers)
        c4 = 4 * C                                                     # pixel-shuffle x0.5 folds 2 x 2 tokens
        self.pre_proj_layernorm = _Params()
        self.pre_proj_layernorm.weight, self.pre_proj_layernorm.bias = P(c4, fill=1.0), P(c4, fill=0.0)
        self.vision_projection = _Params()
        self.vision_projection.encoder = _Params()
        enc = self.vision_projection.encoder
        enc.linear_fc1 = _Params()
        enc.linear_fc1.weight = P(C, c4)                               # ffn_hidden_size = ViT hidden (:423)
        enc.linear_fc2 = _Params()
        enc.linear_fc2.weight = P(hidden_size, C)

    # -- the tower ---------------------------------------------------------------------------------------------
    def _vit(self, images: torch.Tensor) -> torch.Tensor:
        v, vit = self.vcfg, self.vit
        H, D = v.num_attention_heads, v.head_dim
        fuse = self.gradient_accumulation_fusion
        x = ops.patch_embed_autograd(images, vit.conv1.weight, vit.conv1.bias, vit.class_token,
                                     vit.position_embeddings.weight, v.patch_size, fuse)       # [n, S, C]
        n, S, C = x.shape
        x = x.view(n * S, C)
        for L in vit.decoder.layers:
            a, m = L.self_attention, L.mlp
            h, x = ops.layernorm_autograd(x, L.input_layernorm.weight, L.input_layernorm.bias, self.eps, passthrough=True)
            qkv = ops.linear_autograd(h, a.linear_qkv.weight, a.linear_qkv.bias, fuse)      # [n*S, H*3*D]
            att = ops.vit_attention(qkv.view(n, S, 3 * C), H, D ** -0.5)
            o = ops.linear_autograd(att.view(n * S, C), a.linear_proj.weight, a.linear_proj.bias, fuse)
            x = ops.ls_residual_autograd(x, o, L.ls1)
            h, x = ops.layernorm_autograd(x, L.pre_mlp_layernorm.weight, L.pre_mlp_layernorm.bias, self.eps,
                                          passthrough=True)
            f = ops.gelu_autograd(ops.linear_autograd(h, m.linear_fc1.weight, m.linear_fc1.bias, fuse))
            f = ops.linear_autograd(f, m.linear_fc2.weight, m.linear_fc2.bias, fuse)
            x = ops.ls_residual_autograd(x, f, L.ls2)
        return x.view(n, S, C)

    def _project(self, x: torch.Tensor) -> torch.Tensor:
        n, t, c4 = x.shape
        enc = self.vision_projection.encoder
        y = ops.layernorm_autograd(x.reshape(n * t, c4), self.pre_proj_layernorm.weight, self.pre_proj_layernorm.bias,
                                   self.pre_proj_eps)
        fuse = self.gradient_accumulation_fusion
        y = ops.gelu_autograd(ops.linear_autograd(y, enc.linear_fc1.weight, None, fuse))
        y = ops.linear_autograd(y, enc.linear_fc2.weight, None, fuse)
        return y.view(n, t, -1)

    def forward_once(self, images: torch.Tensor) -> torch.Tensor:
        with torch.no_grad() if self.vision_model_freeze else nullcontext():
            x = ops.pixel_shuffle_autograd(self._vit(images), self.vcfg.grid, has_cls=True)   # drop cls + shuffle
        with torch.no_grad() if self.vision_projector_freeze else nullcontext():
            return self._project(x)

    def forward(self, **kw_args) -> torch.Tensor:
        """`images` [N, 3, S, S] -> [N, 256, hidden] (MegatronVisionModel.forward, pretrain_long_vita.py:535-563)."""
        images = kw_args["images"]
        if images.dtype != self.vit.conv1.weight.dtype:
            images = images.to(self.vit.conv1.weight.dtype)
        outs = [self.forward_once(images[i : i + self.chunk_size]) for i in range(0, images.shape[0], self.chunk_size)]
        return outs[0] if len(outs) == 1 else torch.cat(outs, dim=0)


def _arg(args, name, default):
    v = getattr(args, name, default)
    return default if v is None else v


def _vit_args(args, v: VisionConfig):
    """A copy of Megatron's args with the InternViT-300M geometry, what the reference hands to the ViT's checkpoint load
    (get_vision_model_args_intern_300m, pretrain_long_vita.py:183-223, applied to a deepcopy at :329-330)."""
    from copy import deepcopy

    a = deepcopy(args)
    for name, value in (("num_layers", v.num_hidden_layers), ("hidden_size", v.hidden_size),
                        ("ffn_hidden_size", v.intermediate_size), ("num_attention_heads", v.num_attention_heads),
                        ("kv_channels", v.head_dim), ("num_query_groups", v.num_attention_heads),
                        ("group_query_attention", False), ("add_bias_linear", True), ("add_qkv_bias", True),
                        ("gated_linear_unit", False), ("swiglu", False), ("normalization", "LayerNorm"),
                        ("hidden_dropout", 0.0), ("attention_dropout", 0.0), ("patch_dim", v.patch_size),
                        ("recompute_method", None), ("recompute_granularity", None), ("recompute_num_layers", None)):
        setattr(a, name, value)
    return a


def b200_vision_model_provider(config, *external_args, args=None, load_checkpoint=None):
    """Same call as the reference's `vision_model_provider(config)` (pretrain_long_vita.py:599-601; GPTVLModel calls it
    as `provider(config, *external_args)`): builds the vision side from Megatron's global args (read here, once).
    `args` may be passed instead (tests, Megatron-free callers).  Geometries other than the shipped InternViT-300M one
    are refused.

    `--vit-load DIR` is honoured as in MegatronVisionModel.__init__ (pretrain_long_vita.py:392-393): the tower's
    weights are loaded with the reference's `load_checkpoint([vit], None, None, load_arg="vit_load", args=vit_args)`
    (`load_checkpoint` may be passed in; by default long_vita_megatron.training.checkpointing.load_checkpoint).  If that
    loader cannot be imported the provider raises instead of leaving the tower at its random initialisation."""
    if args is None:
        from megatron.training import get_args      # only reached inside a Megatron job

        args = get_args()
    if _arg(args, "vision_model_type", "intern_300m") != "intern_300m":
        raise NotImplementedError(f"B200VisionModel implements --vision-model-type intern_300m, not {args.vision_model_type}")
    if not _arg(args, "add_class_token", True) or not _arg(args, "vision_projector_pre_norm", True):
        raise NotImplementedError("B200VisionModel needs --add-class-token and --vision-projector-pre-norm")
    if float(_arg(args, "vision_downsample_ratio", 0.5)) != 0.5 or int(_arg(args, "vision_downsample_stride", 1)) != 1:
        raise NotImplementedError("B200VisionModel implements --vision-downsample-ratio 0.5 (pixel shuffle) only")
    if int(_arg(args, "tensor_model_parallel_size", 1)) > 1:
        raise NotImplementedError("B200VisionModel holds whole weights: tensor_model_parallel_size must be 1")
    v = VisionConfig()
    image_size = int(_arg(args, "image_size", v.image_size))
    if image_size != v.image_size:
        v = VisionConfig(image_size=image_size)
    vit_load = getattr(args, "vit_load", None)
    if vit_load is not None and load_checkpoint is None:
        try:
            from long_vita_megatron.training.checkpointing import load_checkpoint
        except ImportError as e:
            raise NotImplementedError(f"--vit-load {vit_load}: the reference's checkpoint loader "
                                      "(long_vita_megatron.training.checkpointing.load_checkpoint) is not importable, "
                                      "so the ViT weights cannot be loaded") from e
    model = B200VisionModel(
        int(args.hidden_size), v,
        vision_model_freeze=bool(_arg(args, "vision_model_freeze", False)),
        vision_projector_freeze=bool(_arg(args, "vision_projector_freeze", False)),
        vision_model_recompute=bool(_arg(args, "vision_model_recompute", False)),
        vision_projector_recompute=bool(_arg(args, "vision_projector_recompute", False)),
        vision_context_parallel=bool(_arg(args, "vision_context_parallel", False)),
        layernorm_epsilon=float(_arg(args, "norm_epsilon", v.layer_norm_eps)),
        params_dtype=getattr(config, "params_dtype", None) or torch.bfloat16,
        gradient_accumulation_fusion=bool(_arg(args, "gradient_accumulation_fusion", False)),
    )
    if vit_load is not None:
        load_checkpoint([model.vit], None, None, load_arg="vit_load", args=_vit_args(args, v))
    return model
