"""GPU parity of the composed path: InternViT tower, projector, Qwen2 decoder layer (teacher-forced),
and the whole LongVITAForCausalLM.forward on a tiny geometry that keeps the 14B head structure
(GQA 5:1, head_dim 128 / 64, 448/14 patches) - against the CPU oracle on identical bf16 weights."""
from functools import partial

import pytest
import torch

from long_vita_b200.config import LongVITAConfig
from long_vita_b200.weights import synthetic_state_dict
from oracle import model as OM
from oracle import ops as O
from tests.util import max_rel, rel_fro

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def setup(lib_built):
    from long_vita_b200.hf import modeling

    cfg = LongVITAConfig.tiny(layers=2, vit_layers=2)
    w = synthetic_state_dict(cfg, seed=2024, dtype=torch.bfloat16, perturb=True)
    wg = {k: v.cuda() for k, v in w.items()}
    return cfg, w, wg, modeling


def make_inputs(cfg, s=700, n_img=2, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, cfg.vocab_size, (1, s), generator=g)
    images = torch.randn(n_img, 3, 448, 448, generator=g).to(torch.bfloat16)
    starts = [5 + i * 300 for i in range(n_img)]
    idx_s = torch.stack([torch.arange(st, st + 256) for st in starts])
    idx = torch.stack([torch.zeros_like(idx_s), idx_s])
    return ids, images, idx


def test_vit_tower_and_projector(setup):
    cfg, w, wg, M = setup
    _, images, _ = make_inputs(cfg)
    vit = M.InternVisionModel(cfg, wg)(images.cuda())
    w32 = OM.cast_weights(w, torch.float32)
    ref = OM.vit_forward(cfg, w32, images.float())
    assert rel_fro(vit, ref) < 6e-3, rel_fro(vit, ref)            # 2 layers of bf16 activations vs fp32
    refb = OM.vit_forward(cfg, w, images)                            # the eager bf16 sequence on CPU
    assert rel_fro(vit, refb) < 6e-3
    proj = M.ResamplerProjector(cfg, wg)(vit, has_cls=True)
    pref = OM.projector_forward(cfg, w32, vit.float().cpu()[:, 1:, :])   # teacher-forced on our ViT output
    assert rel_fro(proj, pref) < 5e-3, rel_fro(proj, pref)   # LN + 2 bf16 GEMMs + GELU vs the fp32 oracle


def test_decoder_layer_teacher_forced(setup):
    cfg, w, wg, M = setup
    s = 640
    g = torch.Generator().manual_seed(3)
    x = torch.randn(s, cfg.hidden_size, generator=g).to(torch.bfloat16)
    pos = torch.arange(s)
    inv = O.rope_inv_freq(cfg.head_dim, cfg.rope_theta)
    cos, sin = O.rope_tables(pos, inv, torch.bfloat16)
    w32 = OM.cast_weights(w, torch.float32)
    ref = OM.decoder_layer(cfg, w32, 0, x.float(), cos.float(), sin.float())
    layer = M.DecoderLayer(cfg, wg, 0)
    xg, delta = layer.forward(x.cuda(), None, cos.cuda(), sin.cuda(), partial(M.attention_step(), 0))
    out = xg.float() + delta.float()
    assert rel_fro(out, ref) < 4e-3, (rel_fro(out, ref), max_rel(out, ref))


def test_whole_forward_matches_oracle(setup):
    cfg, w, wg, M = setup
    ids, images, idx = make_inputs(cfg)
    model = M.LongVITAForCausalLM(cfg, wg)
    out = model(input_ids=ids.cuda(), images=images.cuda(), image_indices=idx.cuda(), num_logits_to_keep=4,
                output_hidden_states=True)
    assert out.logits.shape == (1, 4, cfg.vocab_size)
    w32 = OM.cast_weights(w, torch.float32)
    logits, hidden, h_final = OM.long_vita_forward(cfg, w32, ids, images.float(), idx, num_logits_to_keep=4,
                                                   return_hidden=True)
    # embedding + scatter is an index op: bit-exact against the bf16 oracle embedding
    emb_ref = OM.long_vita_forward(cfg, w, ids, images, idx, num_layers=0, return_hidden=True)[1][0]
    text_rows = torch.ones(ids.shape[1], dtype=torch.bool)
    text_rows[idx[1].reshape(-1)] = False
    assert torch.equal(out.hidden_states[0][0].cpu()[text_rows], emb_ref[text_rows])
    for li, (hg, hr) in enumerate(zip(out.hidden_states[:-1], hidden)):
        assert rel_fro(hg[0], hr) < 8e-3, (li, rel_fro(hg[0], hr))
    assert rel_fro(out.logits[0], logits[0]) < 1e-2, rel_fro(out.logits[0], logits[0])
    # same argmax tokens as the fp32 oracle
    assert torch.equal(out.logits[0].float().argmax(-1).cpu(), logits[0].argmax(-1))


def test_forward_without_images_and_full_logits(setup):
    cfg, w, wg, M = setup
    ids, _, _ = make_inputs(cfg, s=130)
    model = M.LongVITAForCausalLM(cfg, wg)
    out = model(input_ids=ids.cuda())
    assert out.logits.shape == (1, 130, cfg.vocab_size)
    ref = OM.long_vita_forward(cfg, OM.cast_weights(w, torch.float32), ids)
    assert rel_fro(out.logits[0], ref[0]) < 1e-2


def test_signature_guards(setup):
    cfg, w, wg, M = setup
    model = M.LongVITAForCausalLM(cfg, wg)
    ids = torch.zeros(1, 8, dtype=torch.long).cuda()
    with pytest.raises(NotImplementedError):
        model(input_ids=ids, output_attentions=True)
    with pytest.raises(ValueError):
        model(input_ids=None)


def test_siglip_tower_matches_oracle(lib_built):
    """a9: SigLIP geometry (head_dim 72, no class token, tanh-GELU) on a 2-layer, 2-head slice."""
    from long_vita_b200.hf.siglip import SigLIPConfig, SigLIPViTModel

    cfg = SigLIPConfig(hidden_size=144, ffn_hidden_size=304, num_layers=2, num_attention_heads=2, kv_channels=72)
    g = torch.Generator().manual_seed(21)

    def rn(*shape, std=0.05):
        return (torch.randn(*shape, generator=g) * std).to(torch.bfloat16)

    C, I = cfg.hidden_size, cfg.ffn_hidden_size
    w = {"conv1.weight": rn(C, 3, 14, 14), "conv1.bias": rn(C), "position_embeddings.weight": rn(cfg.num_patches, C, std=1.0)}
    for i in range(cfg.num_layers):
        p = f"decoder.layers.{i}."
        w.update({
            p + "input_layernorm.weight": (1 + rn(C)).to(torch.bfloat16), p + "input_layernorm.bias": rn(C),
            p + "self_attention.linear_qkv.weight": rn(3 * C, C), p + "self_attention.linear_qkv.bias": rn(3 * C),
            p + "self_attention.linear_proj.weight": rn(C, C), p + "self_attention.linear_proj.bias": rn(C),
            p + "pre_mlp_layernorm.weight": (1 + rn(C)).to(torch.bfloat16), p + "pre_mlp_layernorm.bias": rn(C),
            p + "mlp.linear_fc1.weight": rn(I, C), p + "mlp.linear_fc1.bias": rn(I),
            p + "mlp.linear_fc2.weight": rn(C, I), p + "mlp.linear_fc2.bias": rn(C),
        })
    images = torch.randn(2, 3, 448, 448, generator=g).to(torch.bfloat16)
    out = SigLIPViTModel(cfg, {k: v.cuda() for k, v in w.items()})(images.cuda())
    ref = OM.siglip_forward(cfg, OM.cast_weights(w, torch.float32), images.float())
    assert out.shape == (2, 1024, C)
    assert rel_fro(out, ref) < 6e-3, rel_fro(out, ref)


def test_whole_forward_matches_the_references_own_forward(lib_built):
    """GPU model against the committed outputs of the reference's own LongVITAForCausalLM.forward run on CPU in
    fp32 (tests/golden/ref_long_vita_tiny.pt, generated by tests/golden/make_golden.py from /root/reference)."""
    import os
    import sys

    from long_vita_b200.hf import modeling

    gold_dir = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    sys.path.insert(0, gold_dir)
    from make_golden import long_vita_inputs

    gold = torch.load(os.path.join(gold_dir, "ref_long_vita_tiny.pt"))
    cfg = LongVITAConfig.tiny(layers=2, vit_layers=1)
    w = synthetic_state_dict(cfg, seed=gold["seed"], dtype=torch.float32, perturb=True)
    ids, images, idx = long_vita_inputs(cfg, gold["seed"])
    model = modeling.LongVITAForCausalLM(cfg, {k: v.to(torch.bfloat16).cuda() for k, v in w.items()})
    out = model(input_ids=ids.cuda(), images=images.to(torch.bfloat16).cuda(), image_indices=idx.cuda(),
                num_logits_to_keep=8, output_hidden_states=True)
    # the fixture is fp32 with fp32 weights; bf16 weights + activations alone give ~6.6e-3 (CPU emulation)
    assert rel_fro(out.logits[0], gold["logits_last8"]) < 2e-2, rel_fro(out.logits[0], gold["logits_last8"])
    assert torch.equal(out.logits[0].float().argmax(-1).cpu(), gold["logits_last8"].argmax(-1))
    rows = gold["rows"]
    for li in range(cfg.num_hidden_layers + 1):
        assert rel_fro(out.hidden_states[li][0].cpu()[rows], gold["hidden_rows"][li]) < 1.5e-2, li


def test_kv_cache_decode_matches_full_forward(setup):
    """8f-2 on the kernels: prefill with use_cache, single-token decode steps (flash-decoding composition over
    lv_attn_fwd) and a 3-token chunk against the full forward over the extended sequence."""
    cfg, w, wg, M = setup
    ids, images, idx = make_inputs(cfg, s=700)
    extra = torch.randint(0, cfg.vocab_size, (1, 6), generator=torch.Generator().manual_seed(8))
    model = M.LongVITAForCausalLM(cfg, wg)
    full = model(input_ids=torch.cat([ids, extra], dim=1).cuda(), images=images.cuda(), image_indices=idx.cuda()).logits
    out = model(input_ids=ids.cuda(), images=images.cuda(), image_indices=idx.cuda(), use_cache=True,
                num_logits_to_keep=1, max_cache_len=1024)
    cache = out.past_key_values
    assert len(cache) == 700
    assert rel_fro(out.logits[0, -1], full[0, 699]) < 1e-2
    for i in range(3):
        out = model(input_ids=extra[:, i : i + 1].cuda(), past_key_values=cache, use_cache=True)
        assert len(cache) == 701 + i
        assert rel_fro(out.logits[0, 0], full[0, 700 + i]) < 1.5e-2, (i, rel_fro(out.logits[0, 0], full[0, 700 + i]))
        assert int(out.logits[0, 0].float().argmax()) == int(full[0, 700 + i].float().argmax())
    out = model(input_ids=extra[:, 3:].cuda(), past_key_values=cache, use_cache=True)
    assert len(cache) == 706 and rel_fro(out.logits[0], full[0, 703:]) < 1.5e-2
    gen = model.generate_greedy(ids.cuda(), images.cuda(), idx.cuda(), max_new_tokens=4)
    assert gen.shape == (1, 4)
