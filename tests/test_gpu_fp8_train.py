"""FP8 training of the `--spec` decoder layer on the H100 (lv_quant_rows_fp8_fmt, lv_quant_cols_fp8_t,
lv_gemm_fp8_grad; ops.linear_fp8_autograd; B200TransformerLayer with config.fp8).

* Quantisers: the bytes and scales of quant_rows_fp8 (e5m2) and quant_cols_fp8_t (e4m3, e5m2) equal the CPU
  restatement of tests/fp8_ref.py, with zero columns, columns too small to scale, magnitudes from 1e-30 to 1e30,
  padded token counts and a strided input.
* dgrad and wgrad against float64 over the dequantised operands (tests/gemm_ref.py), per 64 x 64 output chunk and
  elementwise, with e4m3 and e5m2 A operands, for the four 14B decoder linears at T = 18 432, 16 897 (wgrad's
  contraction padded to 16 912 with zeros) and 2304.  The bound is that of tests/test_gpu_fp8_linear.py: products of
  FP8 values are exact (e5m2 x e4m3 too), the accumulation is promoted out of the tensor cores every 128 k-values
  (`partial_rounding` = 2^-11), CHUNK_BOUND sits below the error of an unpromoted accumulation.  Measured on an H100
  80GB HBM3: worst chunk excess 3.9e-4 (dgrad) and 1.7e-4 (wgrad); a build without promotion
  (LV_EXTRA_DEFINES=-DLV_FP8_NO_PROMOTION) gives 1.5-2.1e-3 and fails all 16 dgrad / wgrad cases at T = 18 432.
* The fused fp32 main_grad holds the relations of the bf16 fusion: from zero, its bf16 rounding is the plain wgrad
  product; from a prior P it is P + the from-zero value, exactly.
* One 14B-geometry layer, forward and backward at 18 432 tokens: the FP8 gradients ("e4m3", "hybrid") against the bf16
  gradients per parameter (relative Frobenius deviation and cosine, limits from the measured values with margin), and
  fp8=None gradients torch.equal to the layer without the field.
* A tiny two-layer model trained with Adam on seeded synthetic data, with fp32 master weights copied back into the
  bf16 parameters through `.data.copy_` as Megatron's bf16 optimizers do (no `_version` bump, same `data_ptr`): the
  FP8 loss tracks the bf16 loss, so every step trains on the updated weights.
The weights are synthetic, so training quality on a real run is not measured here.
"""
import pytest
import torch

from tests.fp8_ref import E4M3, E5M2, dequant, quant_cols_t_ref, quant_rows_ref
from tests.gemm_ref import check_gemm, gemm_ref

pytestmark = pytest.mark.gpu

H, QKV, INTER = 5120, 7168, 13824
LINEARS = {"qkv": (QKV, H), "proj": (H, H), "fc1": (2 * INTER, H), "fc2": (H, INTER)}   # (N out, K in)
PARTIAL = 2.0 ** -11
CHUNK_BOUND = 5e-4
WORST = {}
# FP8 against bf16 gradients of one 14B-geometry layer at 18 432 tokens, worst parameter, measured on an H100 80GB
# HBM3 (700 W): relative Frobenius 0.140 / cosine 0.9902 for e4m3, 0.166 / 0.9862 for hybrid; limits with ~1.4x margin
# on the deviation
GRAD_REL_LIMIT = {"e4m3": 0.2, "hybrid": 0.23}
GRAD_COS_MIN = {"e4m3": 0.98, "hybrid": 0.972}
# tiny model, Adam: largest gap of the FP8 loss to the bf16 loss over the steps, relative to the initial bf16 loss
# (the loss falls ~300x, so a gap relative to the current loss would measure the FP8 noise floor, not the tracking);
# measured on an H100 80GB HBM3 (700 W): 0.0028 for e4m3, 0.0038 for hybrid
LOSS_REL_LIMIT = 0.02


@pytest.fixture(scope="module")
def L(lib_built):
    from long_vita_b200 import ops

    yield ops
    print(f"\n[fp8_train] worst figures { {k: (round(v, 6) if isinstance(v, float) else v) for k, v in WORST.items()} }")


def _note(key, value, worst=max):
    WORST[key] = value if key not in WORST else worst(WORST[key], value)


def _wild(R, C, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    mag = torch.logspace(-30, 30, 13, device="cuda")[torch.randint(0, 13, (1, C), device="cuda", generator=g)]
    x = (torch.randn((R, C), device="cuda", generator=g) * mag).to(torch.bfloat16)
    x[:, ::7] = 0
    x[:, 3] = 0
    x[min(5, R - 1), 3] = torch.tensor([1], dtype=torch.int16).view(torch.bfloat16)   # a bf16-subnormal amax
    return x


# ------------------------------------------------------------------------------------------------
# quantisers
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R,C", [(16897, 5120), (37, 13824), (2304, 7168), (1, 8)])
def test_quantisers_are_the_restatement(L, R, C):
    x = _wild(R, C, R + C)
    wide = torch.zeros((R, C + 24), dtype=torch.bfloat16, device="cuda")
    wide[:, 8 : 8 + C] = x
    xc = x.cpu()
    for dtype in (E4M3, E5M2):
        qc_ref, sc_ref = quant_cols_t_ref(xc, dtype)
        qr_ref, sr_ref = quant_rows_ref(xc, dtype) if C % 16 == 0 else (None, None)
        for src in (x, wide[:, 8 : 8 + C]):
            q, s = L.quant_cols_fp8_t(src, dtype)
            torch.cuda.synchronize()
            assert q.dtype == dtype and q.shape == qc_ref.shape
            assert torch.equal(q.view(torch.uint8).cpu(), qc_ref), f"cast-transpose {dtype} {R}x{C}"
            assert torch.equal(s.cpu().view(torch.int32), sc_ref.view(torch.int32))
            if qr_ref is not None:
                q, s = L.quant_rows_fp8(src, dtype)
                assert q.dtype == dtype
                assert torch.equal(q.view(torch.uint8).cpu(), qr_ref), f"rows {dtype} {R}x{C}"
                assert torch.equal(s.cpu().view(torch.int32), sr_ref.view(torch.int32))


# ------------------------------------------------------------------------------------------------
# dgrad / wgrad against float64
# ------------------------------------------------------------------------------------------------
def _dy(T, N, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn((T, N), device="cuda", generator=g) * 1e-3).to(torch.bfloat16)


@pytest.mark.parametrize("dtype", [E4M3, E5M2], ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("T", [18432, 16897, 2304])
@pytest.mark.parametrize("lin", list(LINEARS))
def test_dgrad(L, lin, T, dtype):
    N, K = LINEARS[lin]
    g = torch.Generator(device="cuda").manual_seed(N + K)
    w = (torch.randn((N, K), device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    wt = L.Fp8Weight(*L.quant_cols_fp8_t(w))
    dy = _dy(T, N, T + N)
    dx = L.linear_fp8_dgrad(dy, wt, dtype)
    dq, ds = L.quant_rows_fp8(dy, dtype)
    a = dequant(dq, ds)
    b = dequant(wt.data, wt.scale)                                   # W^T [K, N]
    r = check_gemm(dx, gemm_ref(a, b), a, b, chunk_bound=CHUNK_BOUND, partial_rounding=PARTIAL,
                   name=f"dgrad {lin} T={T} {dtype}")
    _note("dgrad_chunk_excess", r["chunk_excess"])
    _note("dgrad_elem_ratio", r["elem_ratio"])


@pytest.mark.parametrize("dtype", [E4M3, E5M2], ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("T", [18432, 16897, 2304])
@pytest.mark.parametrize("lin", list(LINEARS))
def test_wgrad(L, lin, T, dtype):
    N, K = LINEARS[lin]
    g = torch.Generator(device="cuda").manual_seed(T + K)
    x = torch.randn((T, K), device="cuda", generator=g).to(torch.bfloat16)
    dy = _dy(T, N, T + N + 1)
    xt = L.quant_cols_fp8_t(x)
    dw = L.linear_fp8_wgrad(dy, xt, dtype)
    dq, ds = L.quant_cols_fp8_t(dy, dtype)
    a, b = dequant(dq, ds), dequant(*xt)                              # dY^T [N, T16], X^T [K, T16]
    r = check_gemm(dw, gemm_ref(a, b), a, b, chunk_bound=CHUNK_BOUND, partial_rounding=PARTIAL,
                   name=f"wgrad {lin} T={T} {dtype}")
    _note("wgrad_chunk_excess", r["chunk_excess"])
    _note("wgrad_elem_ratio", r["elem_ratio"])
    if lin in ("proj", "fc2") and T != 2304:
        # fused main_grad: from zero, its bf16 rounding is the plain product; from P, exactly P + that accumulator
        mg0 = torch.zeros((N, K), dtype=torch.float32, device="cuda")
        L.linear_fp8_wgrad_accumulate(dy, xt, mg0, dtype)
        assert torch.equal(mg0.to(torch.bfloat16), dw)
        p = torch.randn((N, K), device="cuda", generator=g)
        mgp = p.clone()
        L.linear_fp8_wgrad_accumulate(dy, xt, mgp, dtype)
        assert torch.equal(mgp, p + mg0)


# ------------------------------------------------------------------------------------------------
# one 14B-geometry layer, forward + backward at 18 432 tokens
# ------------------------------------------------------------------------------------------------
def _mcfg(h, heads, groups, ffn, **extra):
    import types

    m = types.SimpleNamespace(hidden_size=h, num_attention_heads=heads, num_query_groups=groups, kv_channels=128,
                              ffn_hidden_size=ffn, layernorm_epsilon=1e-6, hidden_dropout=0.0, attention_dropout=0.0,
                              params_dtype=torch.bfloat16, num_layers=1)
    for k, v in extra.items():
        setattr(m, k, v)
    return m


def _freqs(s, hn=128, base=1e6):
    inv = 1.0 / base ** (torch.arange(0, hn, 2, device="cuda", dtype=torch.float32) / hn)
    f = torch.outer(torch.arange(s, device="cuda", dtype=torch.float32), inv)
    return torch.cat([f, f], dim=-1).view(s, 1, 1, hn)


def _layer_grads(layer, x, dy, freqs):
    x = x.clone().requires_grad_(True)
    for p in layer.parameters():
        p.grad = None
    out, _ = layer(hidden_states=x, attention_mask=None, rotary_pos_emb=freqs)
    out.backward(dy)
    torch.cuda.synchronize()
    return {"x": x.grad, **{n: p.grad for n, p in layer.named_parameters()}}


def test_14b_layer_gradients(L):
    from long_vita_b200.megatron.transformer_layer import B200TransformerLayer

    torch.manual_seed(0)
    s = 18432
    dims = (H, 40, 8, INTER)
    base = B200TransformerLayer(_mcfg(*dims))
    for p in base.parameters():
        p.requires_grad_(True)
    state = base.state_dict()
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn((s, 1, H), device="cuda", generator=g).to(torch.bfloat16)
    dy = (torch.randn((s, 1, H), device="cuda", generator=g) * 1e-2).to(torch.bfloat16)
    freqs = _freqs(s)
    ref = _layer_grads(base, x, dy, freqs)
    none = B200TransformerLayer(_mcfg(*dims, fp8=None))
    none.load_state_dict(state)
    for p in none.parameters():
        p.requires_grad_(True)
    got = _layer_grads(none, x, dy, freqs)
    assert all(torch.equal(got[n], ref[n]) for n in ref), "fp8=None changed a gradient"
    del none, got
    for fp8 in ("e4m3", "hybrid"):
        layer = B200TransformerLayer(_mcfg(*dims, fp8=fp8))
        layer.load_state_dict(state)
        for p in layer.parameters():
            p.requires_grad_(True)
        got = _layer_grads(layer, x, dy, freqs)
        for n, r in ref.items():
            a, r = got[n].double().flatten(), r.double().flatten()
            rel = float((a - r).norm() / r.norm())
            cos = float(a @ r / (a.norm() * r.norm()))
            _note(f"{fp8}_grad_rel", rel)
            _note(f"{fp8}_grad_cos", cos, min)
            print(f"[fp8_train] {fp8} {n}: rel {rel:.4f} cos {cos:.5f}")
            assert rel <= GRAD_REL_LIMIT[fp8] and cos >= GRAD_COS_MIN[fp8], (fp8, n, rel, cos)
        del layer, got
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------
# a tiny model trained with Adam on fp32 master weights (Megatron's Float16OptimizerWithFloat16Params)
# ------------------------------------------------------------------------------------------------
def _train(fp8, steps=40, s=256):
    from long_vita_b200.megatron.transformer_layer import B200TransformerLayer

    torch.manual_seed(5)
    layers = [B200TransformerLayer(_mcfg(640, 5, 1, 1024, fp8=fp8, num_layers=2), layer_number=i + 1)
              for i in range(2)]
    params = [p for layer in layers for p in layer.parameters()]
    for p in params:
        p.requires_grad_(True)
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn((s, 1, 640), device="cuda", generator=g).to(torch.bfloat16)
    target = torch.randn((s, 1, 640), device="cuda", generator=g).to(torch.bfloat16)
    freqs = _freqs(s)
    masters = [p.detach().float().clone().requires_grad_(True) for p in params]
    opt = torch.optim.Adam(masters, lr=1e-3)
    losses = []
    for _ in range(steps):
        for p in params:
            p.grad = None
        h = x
        for layer in layers:
            h, _ = layer(hidden_states=h, attention_mask=None, rotary_pos_emb=freqs)
        loss = (h.float() - target.float()).pow(2).mean()
        loss.backward()
        for p, m in zip(params, masters):
            m.grad = p.grad.float()
        opt.step()
        for p, m in zip(params, masters):
            p.data.copy_(m)                          # the write-back of Megatron's bf16 optimizers
        losses.append(float(loss))
    return losses


def test_tiny_model_trains_like_bf16(L):
    ref = _train(None)
    for fp8 in ("e4m3", "hybrid"):
        got = _train(fp8)
        gap = max(abs(a - b) for a, b in zip(got, ref)) / ref[0]
        _note(f"{fp8}_loss_rel_gap", gap)
        print(f"[fp8_train] {fp8} loss {got[0]:.4f} -> {got[-1]:.4f} (bf16 {ref[0]:.4f} -> {ref[-1]:.4f}), gap {gap:.5f}")
        assert got[-1] < 0.1 * got[0] and gap <= LOSS_REL_LIMIT, (fp8, gap)
