"""GPU: weight gradients accumulated into an fp32 `main_grad` inside the wgmma GEMM (`lv_gemm_wgrad_acc_f32`,
`ops.linear_wgrad_accumulate`), and Megatron's gradient_accumulation_fusion on the three training surfaces.

The accumulate epilogue shares the mainloop, ring, rasterisation and k-order of the bf16 GEMM, and adds with one IEEE
fp32 round-to-nearest add that keeps subnormals, so these relations are exact (torch.equal), not tolerances:
  zero start:    main_grad.to(bf16) == linear_wgrad(dy, x)           (the accumulator the bf16 path rounds)
  seeded start:  main_grad == prior + acc0                            acc0 = the zero-start result, + = torch's fp32 add
  repeat:        a second call from the same prior gives the same bits
  T = 0:         main_grad unchanged
  outside:       the columns of a wider parent tensor, the rows around a row slice and the patch weight's padding
                 columns keep their sentinel values
acc0 is also held against float64 (tests/gemm_ref.py): elementwise |acc0 - r| <= K 2^-23 (|A| |W|^T), which has no bf16
term; the worst ratio and the worst 64 x 64 chunk's relative error are printed.
"""
import math

import pytest
import torch

from long_vita_b200.config import LongVITAConfig
from tests.gemm_ref import _chunk_sums, gemm_ref
from tests.util import randn_bf16, seeded

pytestmark = pytest.mark.gpu

SENTINEL = -7.25
f32, bf16 = torch.float32, torch.bfloat16

DECODER = {"qkv": (7168, 5120), "proj": (5120, 5120), "fc1": (27648, 5120), "fc2": (5120, 13824)}   # [N_out, K_in]
VIT = {"qkv": (3072, 1024), "proj": (1024, 1024), "fc1": (4096, 1024), "fc2": (1024, 4096)}
FUSED_SUFFIXES = ("conv1.weight", "linear_qkv.weight", "linear_proj.weight", "linear_fc1.weight", "linear_fc2.weight")


@pytest.fixture(scope="module")
def L(lib_built):
    from long_vita_b200 import ops

    return ops


def _randn(shape, seed, dtype=bf16, scale=1.0):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return (torch.randn(shape, generator=g, device="cuda") * scale).to(dtype)


def _check_against_float64(acc0, a, w, name):
    """acc0 [M, N] fp32 = a [M, K] . w [N, K]^T (any strides): elementwise K 2^-23 (|a| |w|^T) bound."""
    K = a.shape[1]
    r = gemm_ref(a, w)
    absd = gemm_ref(a.abs(), w.abs())
    d = acc0.double() - r
    bound = K * 2.0 ** -23 * absd
    ratio = torch.where(bound > 0, d.abs() / bound, torch.where(d == 0, torch.zeros_like(d), torch.full_like(d, math.inf)))
    worst = float(ratio.max())
    chunk = float((_chunk_sums(d) / _chunk_sums(r).clamp_min(1e-300)).sqrt().max())
    print(f"{name}: worst |acc - r| / (K 2^-23 |A||W|^T) = {worst:.3e}, worst 64x64 chunk relative error {chunk:.3e}")
    assert worst <= 1.0, (name, worst)
    del r, absd, d, bound, ratio


def _exact_relations(L, dy, x, name, col_pad=8, row_pad=3, dw_bf16=None):
    """Every exact relation of the module docstring for main_grad [N, K] += dy^T x, main_grad being the [N, K] window of
    a parent with `row_pad` sentinel rows above and below and `col_pad` sentinel columns to the right.  Returns acc0."""
    N, K = dy.shape[1], x.shape[1]
    parent = torch.full((N + 2 * row_pad, K + col_pad), SENTINEL, dtype=f32, device="cuda")
    mg = parent[row_pad : row_pad + N, :K]

    def outside_untouched():
        inner = torch.zeros_like(parent, dtype=torch.bool)
        inner[row_pad : row_pad + N, :K] = True
        assert bool((parent[~inner] == SENTINEL).all()), f"{name}: wrote outside main_grad"

    mg.zero_()
    L.linear_wgrad_accumulate(dy, x, mg)
    acc0 = mg.clone()
    want = L.linear_wgrad(dy, x) if dw_bf16 is None else dw_bf16
    assert torch.equal(acc0.to(bf16), want), f"{name}: zero start != linear_wgrad"
    del want
    outside_untouched()
    prior = _randn((N, K), N + K, f32, scale=math.sqrt(dy.shape[0]))
    mg.copy_(prior)
    L.linear_wgrad_accumulate(dy, x, mg)
    first = mg.clone()
    assert torch.equal(first, prior + acc0), f"{name}: seeded start != prior + acc0"
    mg.copy_(prior)
    L.linear_wgrad_accumulate(dy, x, mg)
    assert torch.equal(mg, first), f"{name}: two calls differ"
    L.linear_wgrad_accumulate(dy[:0], x[:0], mg)
    assert torch.equal(mg, first), f"{name}: T = 0 changed main_grad"
    outside_untouched()
    return acc0


@pytest.mark.parametrize("T", [18432, 16897])
@pytest.mark.parametrize("layer", list(DECODER))
def test_decoder_weights(L, layer, T):
    N, K = DECODER[layer]
    dy, x = _randn((T, N), 1 + T), _randn((T, K), 2 + T)
    acc0 = _exact_relations(L, dy, x, f"decoder {layer} T={T}")
    _check_against_float64(acc0, dy.t(), x.t(), f"decoder {layer} T={T}")


@pytest.mark.parametrize("layer", list(VIT))
def test_vit_weights_at_64_frames(L, layer):
    N, K = VIT[layer]
    T = 64 * 1025
    dy, x = _randn((T, N), 3), _randn((T, K), 4)
    acc0 = _exact_relations(L, dy, x, f"vit {layer}")
    _check_against_float64(acc0, dy.t(), x.t(), f"vit {layer}")


def test_patch_embedding_weight_at_64_frames(L):
    """dW = dP^T col over the 588 real im2col columns of the 640-wide matrix: main_grad is the first 588 columns of a
    [1024, 640] parent whose 52 padding columns must keep their sentinels."""
    images = _randn((64, 3, 448, 448), 5)
    col = L.patch_im2col(images, 14, 640)                                  # [65536, 640]
    dp = _randn((col.shape[0], 1024), 6)
    dw_bf16 = L.linear_wgrad(dp, col)[:, :588]
    acc0 = _exact_relations(L, dp, col[:, :588], "patch embedding", col_pad=52, row_pad=0, dw_bf16=dw_bf16)
    _check_against_float64(acc0, dp.t(), col[:, :588].t(), "patch embedding")


@pytest.mark.parametrize("T", [1, 17, 63, 64, 65])
def test_short_token_counts(L, T):
    dy, x = _randn((T, 5120), 7 + T), _randn((T, 5120), 8 + T)
    acc0 = _exact_relations(L, dy, x, f"proj T={T}")
    _check_against_float64(acc0, dy.t(), x.t(), f"proj T={T}")


def test_m_and_n_tails(L):
    """N_out = 520 (a 128-row tile with 8 rows), K_in = 1000 (the last 256-column tile holds 232 columns)."""
    dy, x = _randn((777, 520), 9), _randn((777, 1000), 10)
    acc0 = _exact_relations(L, dy, x, "tails", col_pad=24, row_pad=5)
    _check_against_float64(acc0, dy.t(), x.t(), "tails")


def test_lm_head_vocabulary_chunk(L):
    """One vocabulary chunk of the LM head: d_logits [M, 16384] is a row-strided view of the chunk buffer."""
    M = 4096
    buf = _randn((M, 16384 + 64), 11)
    dy, x = buf[:, :16384], _randn((M, 5120), 12)
    acc0 = _exact_relations(L, dy, x, "lm head chunk")
    _check_against_float64(acc0, dy.t(), x.t(), "lm head chunk")


def test_subnormal_prior_is_kept(L):
    """Rows of dW that are exactly zero leave a subnormal prior as it is (add.rn.f32 without .ftz)."""
    dy, x = _randn((100, 64), 13), _randn((100, 128), 14)
    dy[:, :8] = 0
    tiny = torch.full((64, 128), 3e-42, dtype=f32, device="cuda")
    assert float(tiny[0, 0]) != 0.0 and float(tiny[0, 0]) < torch.finfo(f32).tiny
    L.linear_wgrad_accumulate(dy, x, tiny)
    assert bool((tiny[:8] == 3e-42).all())


def test_rejected_main_grads(L):
    dy, x = _randn((16, 64), 15), _randn((16, 128), 16)
    with pytest.raises(RuntimeError, match="float32"):
        L.linear_wgrad_accumulate(dy, x, torch.zeros((64, 128), dtype=bf16, device="cuda"))
    with pytest.raises(RuntimeError, match="main_grad is"):
        L.linear_wgrad_accumulate(dy, x, torch.zeros((128, 64), dtype=f32, device="cuda"))
    with pytest.raises(RuntimeError, match="unit column"):
        L.linear_wgrad_accumulate(dy, x, torch.zeros((128, 64), dtype=f32, device="cuda").t())


def test_masked_lm_head_ce_accumulates_chunk_row_slices(L):
    """Three vocabulary chunks (the last 1000 rows): each accumulates into its row slice of main_grad; the result is the
    un-fused dW before its rounding, and the second micro-batch adds in fp32."""
    s, c, V, M = 900, 640, 2 * 16384 + 1000, 700
    g = seeded(17)
    h = randn_bf16((s, 1, c), g).cuda()
    w = randn_bf16((V, c), g, c ** -0.5).cuda()
    mask = torch.zeros(1, s, dtype=torch.bool)
    mask[0, torch.randperm(s, generator=g)[:M]] = True
    labels = torch.randint(0, V, (1, M), generator=g).cuda()
    ups = [torch.randn(1, M, generator=g).cuda() for _ in range(2)]

    def run(fuse, i, weight):
        hd = h.clone().requires_grad_(True)
        loss = L.masked_lm_head_ce(hd, weight, mask.cuda(), labels, accumulate_wgrad=fuse)
        loss.backward(ups[i])
        return loss.detach(), hd.grad, weight.grad

    def fused_weight():
        wf = w.clone().requires_grad_(True)
        wf.main_grad = torch.zeros((V, c), dtype=f32, device="cuda")
        return wf

    acc0 = []
    for i in range(2):
        loss, dh, dw = run(False, i, w.clone().requires_grad_(True))
        wf = fused_weight()
        loss_f, dh_f, dw_f = run(True, i, wf)
        assert torch.equal(loss_f, loss) and torch.equal(dh_f, dh)
        assert dw_f is None                                      # no grad_added_to_main_grad attribute: no gradient
        assert torch.equal(wf.main_grad.to(bf16), dw)
        acc0.append(wf.main_grad)
    wf = fused_weight()
    run(True, 0, wf)
    run(True, 1, wf)
    assert torch.equal(wf.main_grad, acc0[0] + acc0[1])


# ------------------------------------------------------------------------------------------------
# surfaces: fusion on against fusion off on the same inputs, two micro-batches
# ------------------------------------------------------------------------------------------------
def _attach_main_grads(params):
    """What Megatron's DistributedDataParallel does: an fp32 main_grad per parameter, grad_added_to_main_grad = False."""
    for p in params:
        p.main_grad = torch.zeros(p.shape, dtype=f32, device=p.device)
        p.grad_added_to_main_grad = False


def _same(a, b):
    return a is b if a is None or b is None else torch.equal(a, b)


def _compare_surface(run_off, run_on, fused_names, n_mb=2):
    """run_off(i) / run_on(i, zero_first) -> (outputs dict, grads dict of the un-fused parameters, main_grads dict).
    Outputs and un-fused gradients are bit-identical between the runs, each micro-batch's acc0 rounds to the un-fused
    weight gradient, and the micro-batches accumulated into one main_grad give the fp32 sum of their acc0."""
    off = [run_off(i) for i in range(n_mb)]
    off = [(o, {k: None if t is None else t.clone() for k, t in g.items()}, m) for o, g, m in off]
    acc0 = []
    for i in range(n_mb):                       # each micro-batch from a zeroed main_grad
        outs, grads, mgs = run_on(i, True)
        for k in outs:
            assert torch.equal(outs[k], off[i][0][k]), (i, k)
        for k in grads:
            assert _same(grads[k], off[i][1][k]), (i, k)
        for k in fused_names:
            assert torch.equal(mgs[k].to(bf16), off[i][1][k]), (i, k)
        acc0.append({k: mgs[k].clone() for k in fused_names})
    for i in range(n_mb):                       # the micro-batches accumulated into one main_grad
        _, _, mgs = run_on(i, i == 0)
    for k in fused_names:
        total = acc0[0][k]
        for a in acc0[1:]:
            total = total + a[k]
        assert torch.equal(mgs[k], total), k


def test_transformer_layer(lib_built):
    from types import SimpleNamespace

    from long_vita_b200.megatron import checkpoint as ck
    from long_vita_b200.megatron.transformer_layer import B200TransformerLayer
    from long_vita_b200.weights import llm_layer_weights
    from oracle import ops as O

    cfg = LongVITAConfig.tiny(layers=1)
    mc = ck.hf_to_mcore(llm_layer_weights(cfg, 0, seed=21, dtype=bf16, perturb=True), cfg)

    def layer(fuse):
        mcfg = SimpleNamespace(hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_attention_heads,
                               num_query_groups=cfg.num_key_value_heads, kv_channels=cfg.head_dim,
                               ffn_hidden_size=cfg.intermediate_size, layernorm_epsilon=cfg.rms_norm_eps,
                               hidden_dropout=0.0, attention_dropout=0.0, params_dtype=bf16)
        if fuse is not None:
            mcfg.gradient_accumulation_fusion = fuse
        m = B200TransformerLayer(mcfg, layer_number=1)
        m.load_state_dict({k[len("decoder.layers.0."):]: v.cuda() for k, v in mc.items()}, strict=True)
        for p in m.parameters():
            p.requires_grad_(True)
        return m

    s = 384
    inv = O.rope_inv_freq(cfg.head_dim, cfg.rope_theta)
    freqs = torch.outer(torch.arange(s).float(), inv)
    emb = torch.cat((freqs, freqs), dim=-1)[:, None, None, :].cuda()
    g = seeded(22)
    data = [(randn_bf16((s, 1, cfg.hidden_size), g).cuda(), randn_bf16((s, 1, cfg.hidden_size), g, 0.1).cuda())
            for _ in range(2)]
    off_layer, on_layer = layer(None), layer(True)
    fused = [n for n, _ in on_layer.named_parameters() if n.endswith(FUSED_SUFFIXES)]
    assert len(fused) == 4
    _attach_main_grads([p for n, p in on_layer.named_parameters() if n in fused])

    def run(m, i):
        m.zero_grad(set_to_none=True)
        x = data[i][0].clone().requires_grad_(True)
        out, _ = m(hidden_states=x, attention_mask=None, rotary_pos_emb=emb)
        out.backward(data[i][1])
        return {"out": out.detach(), "dx": x.grad}

    def run_off(i):
        outs = run(off_layer, i)
        return outs, {n: p.grad for n, p in off_layer.named_parameters()}, None

    def run_on(i, zero_first):
        params = dict(on_layer.named_parameters())
        if zero_first:
            for n in fused:
                params[n].main_grad.zero_()
        outs = run(on_layer, i)
        for n in fused:
            assert params[n].grad_added_to_main_grad is True
        return outs, {n: p.grad for n, p in params.items() if n not in fused}, {n: params[n].main_grad for n in fused}

    _compare_surface(run_off, run_on, fused)


def _vision_models(cfg, freeze):
    from long_vita_b200.megatron import checkpoint as CK
    from long_vita_b200.megatron.vision_model import B200VisionModel
    from long_vita_b200.weights import global_weights, vit_layer_weights

    w = global_weights(cfg, 31, "cpu", f32, perturb=True, with_lm=False)
    for i in range(cfg.visual.num_hidden_layers):
        w.update(vit_layer_weights(cfg, i, 31, "cpu", f32, perturb=True))
    sd = {k[len(CK.EFM):]: t.to(bf16) for k, t in CK.hf_to_mcore(w, cfg).items()}
    models = []
    for fuse in (False, True):
        m = B200VisionModel(cfg.hidden_size, cfg.visual, device="cuda", vision_model_freeze=freeze,
                            gradient_accumulation_fusion=fuse)
        m.load_state_dict(sd, strict=True)
        models.append(m)
    return models


@pytest.mark.parametrize("freeze", [False, True])
def test_vision_model(lib_built, freeze):
    cfg = LongVITAConfig.tiny(layers=1, vit_layers=2)
    off_m, on_m = _vision_models(cfg, freeze)
    fused_all = [n for n, _ in on_m.named_parameters() if n.endswith(FUSED_SUFFIXES)]
    assert "vit.conv1.weight" in fused_all and len(fused_all) == 1 + 4 * cfg.visual.num_hidden_layers + 2
    fused = [n for n in fused_all if not (freeze and n.startswith("vit."))]
    params = dict(on_m.named_parameters())
    _attach_main_grads([params[n] for n in fused_all])
    g = seeded(32)
    data = [(randn_bf16((2, 3, 448, 448), g).cuda(), randn_bf16((2, 256, cfg.hidden_size), g).cuda()) for _ in range(2)]

    def run(m, i):
        m.zero_grad(set_to_none=True)
        out = m(images=data[i][0])
        out.backward(data[i][1])
        return {"out": out.detach()}

    def run_off(i):
        outs = run(off_m, i)
        return outs, {n: p.grad for n, p in off_m.named_parameters()}, None

    def run_on(i, zero_first):
        if zero_first:
            for n in fused:
                params[n].main_grad.zero_()
        outs = run(on_m, i)
        return outs, {n: p.grad for n, p in params.items() if n not in fused_all}, {n: params[n].main_grad for n in fused}

    _compare_surface(run_off, run_on, fused)
    for n in fused_all:
        if n in fused:
            assert params[n].grad_added_to_main_grad is True, n
        else:                                   # frozen tower: never touched
            assert params[n].grad is None and params[n].grad_added_to_main_grad is False, n
            assert bool((params[n].main_grad == 0).all()), n


def test_gptvl_lm_head_and_cross_entropy(lib_built):
    from long_vita_b200.megatron import checkpoint as ck
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel
    from long_vita_b200.weights import synthetic_state_dict

    cfg = LongVITAConfig.tiny(layers=2, vit_layers=1)
    mc = {k: v.cuda() for k, v in ck.hf_to_mcore(synthetic_state_dict(cfg, seed=41, dtype=bf16, perturb=True),
                                                    cfg).items()}
    off_m, on_m = B200GPTVLModel(cfg, mc), B200GPTVLModel(cfg, mc, gradient_accumulation_fusion=True)
    for m in (off_m, on_m):
        m.output_weight = m.output_weight.detach().clone().requires_grad_(True)
    _attach_main_grads([on_m.output_weight])
    s = 300
    g = torch.Generator().manual_seed(42)
    data = []
    for _ in range(2):
        ids = torch.randint(0, cfg.vocab_size, (1, s), generator=g).cuda()
        mask = torch.zeros(1, s, dtype=torch.bool)
        mask[0, torch.randperm(s, generator=g)[:120]] = True
        labels = torch.randint(0, cfg.vocab_size, (1, s), generator=g).cuda()
        data.append((ids, mask.cuda(), labels, torch.randn(1, 120, generator=g).cuda()))
    pos = torch.arange(s).unsqueeze(0).cuda()

    def run(m, i):
        m.output_weight.grad = None
        ids, mask, labels, up = data[i]
        loss = m(ids, pos, None, labels=labels, logit_mask=mask)
        loss.backward(up)
        return {"loss": loss.detach()}

    def run_off(i):
        return run(off_m, i), {"output_weight": off_m.output_weight.grad}, None

    def run_on(i, zero_first):
        if zero_first:
            on_m.output_weight.main_grad.zero_()
        outs = run(on_m, i)
        assert on_m.output_weight.grad_added_to_main_grad is True
        return outs, {}, {"output_weight": on_m.output_weight.main_grad}

    _compare_surface(run_off, run_on, ["output_weight"])
