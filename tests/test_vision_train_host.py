"""Training the vision side (InternViT tower + projector) on a box without a GPU: fixture pinning of the fp32 oracle
gradients, the composition of `B200VisionModel` under CPU oracle forms of its operators, its Megatron state-dict
surface, flags and provider registration, the stage-1 composition with a frozen decoder layer, and the argument
checks of the new C entry points."""
from __future__ import annotations

import ctypes as C
import os
import sys
import types

import pytest
import torch

from long_vita_b200.config import LongVITAConfig
from long_vita_b200.megatron import checkpoint as CK
from long_vita_b200.megatron.vision_model import B200VisionModel, b200_vision_model_provider
from oracle import model as OM
from tests import vision_oracle as VO

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
sys.path.insert(0, GOLD)

from make_vit_grad_golden import golden_inputs, sha, subsample  # noqa: E402


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.fixture(scope="module")
def gold():
    g = torch.load(os.path.join(GOLD, "ref_vit_grads.pt"))
    cfg, w, images, d_out = golden_inputs()
    assert sha(images) == g["images_sha256"] and sha(d_out) == g["d_out_sha256"]
    return g, cfg, w, images, d_out


def test_fixture_is_small():
    assert os.path.getsize(os.path.join(GOLD, "ref_vit_grads.pt")) < 1 << 20


def test_oracle_autograd_reproduces_reference_gradients(gold):
    g, cfg, w, images, d_out = gold
    leaves = {k: t.clone().requires_grad_(True) for k, t in w.items()}
    vit = OM.vit_forward(cfg, leaves, images)
    out = OM.projector_forward(cfg, leaves, vit[:, 1:, :])
    out.backward(d_out)
    assert rel(out.detach()[:, :: g["token_stride"]], g["out_sub"]) <= 1e-5
    assert set(g["grads_sub"]) == set(leaves)
    for k, t in leaves.items():
        assert rel(subsample(t.grad), g["grads_sub"][k]) <= 1e-5, k


def _vision_model(cfg, w, dtype=torch.float32, **flags):
    m = B200VisionModel(cfg.hidden_size, cfg.visual, params_dtype=dtype, device="cpu", **flags)
    sd = {k[len(CK.EFM):]: t.to(dtype) for k, t in CK.hf_to_mcore(w, cfg).items()}
    m.load_state_dict(sd, strict=True)
    return m


def _grads_hf(m, cfg):
    return CK.mcore_to_hf({CK.EFM + k: p.grad for k, p in m.named_parameters() if p.grad is not None}, cfg)


def test_b200_vision_model_reproduces_reference_gradients(gold):
    """The whole composition (layouts, QKV interleave, strided dQKV, residual-stream gradient routing through the
    LayerNorm backward, patch-embedding gradients, pixel-shuffle inverse) under fp32 oracle forms of every operator."""
    g, cfg, w, images, d_out = gold
    m = _vision_model(cfg, w)
    with VO.vision_oracle_ops():
        out = m(images=images)
        out.backward(d_out)
    assert out.shape == (2, 256, cfg.hidden_size)
    assert rel(out.detach()[:, :: g["token_stride"]], g["out_sub"]) <= 1e-5
    grads = _grads_hf(m, cfg)
    assert set(grads) == set(g["grads_sub"])
    for k, t in grads.items():
        assert rel(subsample(t), g["grads_sub"][k]) <= 1e-5, k


def test_bf16_composition_runs_and_keeps_dtype(gold):
    _, cfg, w, images, d_out = gold
    m = _vision_model(cfg, w, dtype=torch.bfloat16)
    with VO.vision_oracle_ops():
        out = m(images=images)                      # fp32 images are cast to the parameters' dtype
        out.backward(d_out.to(torch.bfloat16))
    assert out.dtype == torch.bfloat16
    assert all(p.grad is not None and p.grad.dtype == torch.bfloat16 for p in m.parameters())


def test_state_dict_keys_are_the_vision_part_of_hf_to_mcore_and_round_trip(gold):
    _, cfg, w, _, _ = gold
    m = _vision_model(cfg, w)
    expect = {k[len(CK.EFM):] for k in CK.hf_to_mcore(w, cfg)}
    sd = m.state_dict()
    assert set(sd) == expect
    back = CK.mcore_to_hf({CK.EFM + k: t for k, t in sd.items()}, cfg)
    assert set(back) == set(w)
    for k in w:
        assert torch.equal(back[k], w[k]), k
    m2 = B200VisionModel(cfg.hidden_size, cfg.visual, params_dtype=torch.float32, device="cpu")
    m2.load_state_dict(sd, strict=True)
    assert all(torch.equal(a, b) for a, b in zip(m2.state_dict().values(), sd.values()))


def test_default_geometry_is_internvit_300m():
    m = B200VisionModel(5120, device="meta")                       # shapes only, no memory
    vit = sum(p.numel() for k, p in m.named_parameters() if k.startswith("vit."))
    assert 300e6 < vit < 310e6 and len(m.vit.decoder.layers) == 24
    assert m.vision_projection.encoder.linear_fc1.weight.shape == (1024, 4096)
    assert m.vision_projection.encoder.linear_fc2.weight.shape == (5120, 1024)


@pytest.mark.parametrize("vit_freeze,proj_freeze", [(True, False), (False, True), (True, True)])
def test_freeze_flags_give_no_gradients_and_no_backward_calls(gold, vit_freeze, proj_freeze):
    _, cfg, w, images, d_out = gold
    m = _vision_model(cfg, w, vision_model_freeze=vit_freeze, vision_projector_freeze=proj_freeze)
    with VO.vision_oracle_ops():
        out = m(images=images[:1])
        if out.requires_grad:
            out.backward(d_out[:1])
    calls = dict(VO.calls)
    vit_params = [p for k, p in m.named_parameters() if k.startswith("vit.")]
    proj_params = [p for k, p in m.named_parameters() if not k.startswith("vit.")]
    if vit_freeze:
        assert all(p.grad is None for p in vit_params)
        for op in ("attention_bwd", "ls_residual_bwd", "patch_im2col", "pixel_shuffle_bwd"):
            assert calls.get(op, 0) == 0, (op, calls)
    if proj_freeze:
        assert all(p.grad is None for p in proj_params)
    if proj_freeze:
        # the projector runs under no_grad, as in the reference (pretrain_long_vita.py:508-520): its output carries
        # no graph, so nothing upstream of it (the tower included) receives a gradient either
        assert not out.requires_grad and sum(calls.get(op, 0) for op in VO.BACKWARD_OPS) == 0
        assert all(p.grad is None for p in vit_params)
    else:
        assert all(p.grad is not None for p in proj_params)
        # the pre-projection LayerNorm's input comes from the no_grad tower: weight / bias gradients only, no dx
        expect = {"layernorm_bwd": 1, "gelu_bwd": 1, "layernorm_bwd_no_dx": 1 if vit_freeze else 0}
        assert {k: calls.get(k, 0) for k in expect} == expect and sum(calls.values()) == sum(expect.values()), calls


@pytest.mark.parametrize("flag", ["vision_model_recompute", "vision_projector_recompute", "vision_context_parallel"])
def test_refused_flags_raise(flag):
    cfg = LongVITAConfig.tiny()
    with pytest.raises(NotImplementedError):
        B200VisionModel(cfg.hidden_size, cfg.visual, device="cpu", **{flag: True})
    args = types.SimpleNamespace(hidden_size=cfg.hidden_size, **{flag: True})
    with pytest.raises(NotImplementedError):
        b200_vision_model_provider(types.SimpleNamespace(params_dtype=torch.bfloat16), args=args)


def test_provider_reads_args_once_and_refuses_other_towers():
    args = types.SimpleNamespace(hidden_size=640, vision_model_type="intern_300m", add_class_token=True,
                                 vision_projector_pre_norm=True, vision_downsample_ratio=0.5, vision_model_freeze=True,
                                 vision_projector_freeze=False, norm_epsilon=1e-6, image_size=448)
    m = b200_vision_model_provider(types.SimpleNamespace(params_dtype=torch.bfloat16), args=args)
    assert m.vision_model_freeze and not m.vision_projector_freeze
    assert m.vision_projection.encoder.linear_fc2.weight.shape == (640, 1024)
    args.vision_model_freeze = False                                   # later changes to args are not seen by forward
    assert m.vision_model_freeze
    for bad in ({"vision_model_type": "siglip_400m"}, {"add_class_token": False}, {"vision_projector_pre_norm": False},
                {"vision_downsample_ratio": 0.25}, {"tensor_model_parallel_size": 8}):
        a = types.SimpleNamespace(**{**vars(args), **bad})
        with pytest.raises(NotImplementedError):
            b200_vision_model_provider(None, args=a)


class _Manager:
    """The reference registry's semantics (patch_utils.py:45-72 with parse_path): *wrapper functions decorate the
    original attribute, others replace it; "pkg.module.Class.attr" patches a class attribute."""

    def __init__(self):
        self.patches = {}

    def register_patch(self, name, fn):
        self.patches.setdefault(name, []).append(fn)

    def apply_patches(self):
        for name, fns in self.patches.items():
            mod_name, attr = name.rsplit(".", 1)
            owner = sys.modules.get(mod_name)
            if owner is None:
                owner_mod, cls_name = mod_name.rsplit(".", 1)
                owner = getattr(sys.modules.get(owner_mod), cls_name, None)
                if owner is None:
                    continue                               # Megatron itself is not installed here
            for fn in fns:
                new = fn(getattr(owner, attr)) if fn.__name__.endswith(("wrapper", "decorator")) else fn
                setattr(owner, attr, new)


def _stand_in_gpt_vl_module(monkeypatch):
    """A stand-in `long_vita_megatron.core.models.multimodal.gpt_vl_model` whose GPTVLModel calls the provider the way
    the reference's does (gpt_vl_model.py:111-114)."""
    mod = types.ModuleType("long_vita_megatron.core.models.multimodal.gpt_vl_model")

    class GPTVLModel:
        def __init__(self, config, transformer_layer_spec=None, external_feature_model_provider=None, external_args=(),
                     **kw):
            self.external_feature_model = external_feature_model_provider(config, *external_args)

    mod.GPTVLModel = GPTVLModel
    monkeypatch.setitem(sys.modules, mod.__name__, mod)
    return mod


def test_vision_registration_is_opt_in_and_replaces_the_stock_provider_at_model_build(monkeypatch):
    """The training script runs as `__main__` (torchrun pretrain_long_vita.py), so its `model_provider` passes its own
    module-level `vision_model_provider`; the patch acts where GPTVLModel receives it, whatever module it came from."""
    from long_vita_b200.megatron import core_attention as CA

    mod = _stand_in_gpt_vl_module(monkeypatch)
    main = types.ModuleType("__main__stand_in")                  # the entry script's namespace

    def vision_model_provider(config):
        return "stock"

    main.vision_model_provider = vision_model_provider

    def model_provider():                                        # pretrain_long_vita.py:641-655, looked up at call time
        return mod.GPTVLModel(types.SimpleNamespace(params_dtype=torch.float32),
                              external_feature_model_provider=main.vision_model_provider).external_feature_model

    orig_init = mod.GPTVLModel.__init__
    m = _Manager()
    CA.register_b200_patches(m)                                  # default: attention only, the vision side untouched
    assert mod.GPTVLModel.__init__ is orig_init and model_provider() == "stock"
    assert list(m.patches) == ["megatron.core.transformer.dot_product_attention.DotProductAttention.forward"]

    calls = []
    monkeypatch.setattr("long_vita_b200.megatron.vision_model.b200_vision_model_provider",
                        lambda config, *a, **k: calls.append((config, a)) or "b200")
    m = _Manager()
    CA.register_b200_patches(m, vision_model=True)
    assert model_provider() == "b200" and len(calls) == 1
    own = lambda config: "own"                                   # noqa: E731 - any other provider passes through
    assert mod.GPTVLModel(None, external_feature_model_provider=own).external_feature_model == "own"


def _provider_args(**kw):
    base = dict(hidden_size=640, vision_model_type="intern_300m", add_class_token=True, vision_projector_pre_norm=True,
                vision_downsample_ratio=0.5, vision_model_freeze=True, vision_projector_freeze=False, norm_epsilon=1e-6,
                image_size=448, num_layers=48, vit_load=None)
    base.update(kw)
    return types.SimpleNamespace(**base)


def test_provider_honours_vit_load():
    """--vit-load: the tower's weights come from the reference's load_checkpoint, called as MegatronVisionModel does
    (pretrain_long_vita.py:392-393: the tower alone, no optimizer, load_arg "vit_load", the ViT geometry in the args);
    the projector keeps its own initialisation and the caller's args are not modified."""
    seen = []

    def load_checkpoint(model, optimizer, opt_param_scheduler, load_arg="load", strict=True, args=None):
        seen.append((len(model), optimizer, opt_param_scheduler, load_arg, getattr(args, load_arg), args.num_layers,
                     args.hidden_size, args.num_attention_heads, args.kv_channels))
        with torch.no_grad():
            for p in model[0].parameters():
                p.fill_(0.5)
        return 0

    args = _provider_args(vit_load="/ckpt/InternViT-300M-448px")
    m = b200_vision_model_provider(types.SimpleNamespace(params_dtype=torch.bfloat16), args=args,
                                   load_checkpoint=load_checkpoint)
    assert seen == [(1, None, None, "vit_load", "/ckpt/InternViT-300M-448px", 24, 1024, 16, 64)]
    for k, p in m.named_parameters():
        assert bool((p == 0.5).all()) == k.startswith("vit."), k
    assert args.num_layers == 48 and args.hidden_size == 640


def test_provider_refuses_vit_load_without_the_reference_loader(monkeypatch):
    monkeypatch.setitem(sys.modules, "long_vita_megatron.training.checkpointing", None)     # import fails
    with pytest.raises(NotImplementedError, match="vit-load"):
        b200_vision_model_provider(types.SimpleNamespace(params_dtype=torch.bfloat16),
                                   args=_provider_args(vit_load="/ckpt/vit"))


def test_provider_called_as_gpt_vl_model_calls_it(monkeypatch):
    """GPTVLModel calls `provider(config, *external_args)`: positional extras never take the place of Megatron's args,
    which come from get_args()."""
    meg, training = types.ModuleType("megatron"), types.ModuleType("megatron.training")
    training.get_args = lambda: _provider_args(hidden_size=320)
    monkeypatch.setitem(sys.modules, "megatron", meg)
    monkeypatch.setitem(sys.modules, "megatron.training", training)
    m = b200_vision_model_provider(types.SimpleNamespace(params_dtype=torch.bfloat16), "extra", "args")
    assert isinstance(m, B200VisionModel) and m.vision_projection.encoder.linear_fc2.weight.shape == (320, 1024)


def test_stage1_frozen_decoder_layer_passes_gradient_to_projector(gold):
    """Stage 1: ViT and LLM frozen, projector trained.  Projector features scattered into the embeddings go through a
    frozen B200TransformerLayer; the gradient reaches the projector and no LLM or ViT weight gets one."""
    from long_vita_b200.megatron import stub
    from long_vita_b200.megatron.transformer_layer import B200TransformerLayer

    _, cfg, w, images, _ = gold
    m = _vision_model(cfg, w, dtype=torch.bfloat16, vision_model_freeze=True)
    tc = stub.TransformerConfig(hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_attention_heads,
                                num_query_groups=cfg.num_key_value_heads, kv_channels=cfg.head_dim)
    tc.ffn_hidden_size, tc.layernorm_epsilon, tc.params_dtype = 256, 1e-6, torch.bfloat16
    layer = B200TransformerLayer(tc)
    assert all(not p.requires_grad for p in layer.parameters())
    s = 300
    g = torch.Generator().manual_seed(3)
    with VO.vision_oracle_ops():
        feat = m(images=images[:1])                                         # [1, 256, H]
        emb = (torch.randn(s, 1, cfg.hidden_size, generator=g) * 0.5).to(torch.bfloat16)
        idx = torch.arange(20, 276)
        emb = emb.index_put((idx, torch.zeros_like(idx)), feat[0])         # feature rows of one image
        freqs = torch.randn(s, 1, 1, cfg.head_dim, generator=g)
        out, _ = layer(emb, None, rotary_pos_emb=freqs)
        out.float().square().mean().backward()
    assert all(p.grad is None for p in layer.parameters())
    assert all(p.grad is None for k, p in m.named_parameters() if k.startswith("vit."))
    for k, p in m.named_parameters():
        if not k.startswith("vit."):
            assert p.grad is not None and float(p.grad.float().abs().sum()) > 0, k


# ------------------------------------------------------------------------------------------------
# argument errors of the new C entry points: LV_EINVAL + lv_last_error text, before any device is touched
# ------------------------------------------------------------------------------------------------
def _lib_or_skip():
    from long_vita_b200 import _lib

    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("liblvb200.so not built")
    return _lib.lib()


A = 1 << 20        # a 16-byte-aligned fake device address: every call below is rejected before it is dereferenced
MIS = A + 2        # misaligned


@pytest.mark.parametrize("name,args,needle", [
    ("lv_layernorm_bwd", (None, A, A, None, A, A, A, 4, 1024, 1e-6, None), "null pointer"),
    ("lv_layernorm_bwd", (A, A, A, None, A, A, A, 4, 1020, 1e-6, None), "multiple of 8"),
    ("lv_layernorm_bwd", (A, A, A, None, A, A, A, 4, 16384, 1e-6, None), "<= 8192"),
    ("lv_layernorm_bwd", (A, A, MIS, None, A, A, A, 4, 1024, 1e-6, None), "16-byte aligned"),
    ("lv_layernorm_bwd", (A, A, A, MIS, A, A, A, 4, 1024, 1e-6, None), "16-byte aligned"),
    ("lv_layernorm_bwd", (A, A, A, A, None, A, A, 4, 1024, 1e-6, None), "add_in needs dx"),
    ("lv_layernorm_bwd", (A, A, A, None, A, None, A, 4, 1024, 1e-6, None), "null pointer"),
    ("lv_gelu_bwd", (A, None, A, 4, 1024, 0, None), "null pointer"),
    ("lv_gelu_bwd", (A, A, A, 4, 1001, 0, None), "multiple of 8"),
    ("lv_gelu_bwd", (A, A, MIS, 4, 1024, 0, None), "16-byte aligned"),
    ("lv_gelu_bwd", (A, A, A, 4, 1024, 2, None), "approx"),
    ("lv_ls_residual_bwd", (A, A, None, A, A, 4, 1024, None), "null pointer"),
    ("lv_ls_residual_bwd", (A, A, A, A, A, 4, 12, None), "multiple of 8"),
    ("lv_ls_residual_bwd", (A, MIS, A, A, A, 4, 1024, None), "16-byte aligned"),
    ("lv_pixel_shuffle_bwd", (None, A, 2, 32, 128, 1, None), "null pointer"),
    ("lv_pixel_shuffle_bwd", (A, A, 2, 31, 128, 1, None), "even"),
    ("lv_pixel_shuffle_bwd", (A, A, 2, 32, 100, 1, None), "multiple of 8"),
    ("lv_pixel_shuffle_bwd", (A, MIS, 2, 32, 128, 1, None), "16-byte aligned"),
    ("lv_patch_im2col", (A, None, 2, 448, 14, 640, None), "null pointer"),
    ("lv_patch_im2col", (A, A, 2, 448, 14, 588 - 8, None), "kpad"),
    ("lv_patch_im2col", (A, A, 2, 448, 14, 596 + 2, None), "kpad"),
    ("lv_patch_im2col", (A, A, 2, 450, 14, 640, None), "geometry"),
    ("lv_patch_im2col", (MIS, A, 2, 448, 14, 640, None), "16-byte aligned"),
])
def test_new_entry_points_reject_bad_arguments(name, args, needle):
    import threading

    lib = _lib_or_skip()
    res = {}

    def call():                       # the error text is thread-local: a worker thread leaves the caller's untouched
        res["rc"] = getattr(lib, name)(*args)
        res["err"] = lib.lv_last_error().decode()

    t = threading.Thread(target=call)
    t.start()
    t.join()
    assert res["rc"] == -1                               # LV_EINVAL
    assert needle in res["err"], res["err"]
