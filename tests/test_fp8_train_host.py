"""CPU tests of FP8 training of the `--spec` decoder layer (config.fp8 = "e4m3" / "hybrid").

* The restatements of tests/fp8_ref.py, whose bytes the GPU quantisers must reproduce: the e5m2 row quantiser
  and the cast-transpose in both formats, with padding columns, all-zero columns, saturation at both formats' largest
  values and strided inputs.
* ops.linear_fp8_autograd on the CPU oracle forms of the FP8 operators: the output and every gradient (dX, dW, the
  bias, the fused fp32 main_grad) equal fp32 autograd of the same product over the dequantised operands to 1e-5.
* B200TransformerLayer with fp8 = "e4m3" and "hybrid" on a tiny geometry: each of the four linears runs its forward,
  dgrad and wgrad in FP8 with the configured gradient format; every gradient, main_grad included, equals fp32 autograd
  of the same composition with each linear's operands dequantised; fp8_wgrad=False reaches the bf16 wgrad; fp8=None
  makes the same operator calls as the layer without the field; the refusals raise with nothing launched.
"""
from __future__ import annotations

import types

import pytest
import torch

from long_vita_b200 import ops
from long_vita_b200.config import LongVITAConfig
from long_vita_b200.megatron import checkpoint as CK
from tests.fp8_ref import E4M3, E5M2, FP8_MAX, dequant, quant_cols_t_ref, quant_rows_ref
from tests.fp8_train_ref import oracle_fp8_ops

bf16, f32 = torch.bfloat16, torch.float32


# ------------------------------------------------------------------------------------------------
# restatements
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [E4M3, E5M2])
def test_rows_rule(dtype):
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(6, 64, generator=g) * torch.logspace(-20, 20, 6)[:, None]).to(bf16)
    x[2] = 0
    x[3, :] = 0
    x[3, 7] = torch.tensor([1], dtype=torch.int16).view(bf16)       # a bf16-subnormal amax: too small to scale
    q, s = quant_rows_ref(x, dtype)
    mx = FP8_MAX[dtype]
    assert float(s[2]) == 0 and float(s[3]) == 0 and not bool(q[2:4].any())
    for r in (0, 1, 4, 5):
        amax = x[r].float().abs().max()
        assert float(s[r]) == float(amax / mx)
        j = int(x[r].float().abs().argmax())
        assert abs(float(q[r].view(dtype)[j].float())) == mx          # the row's amax maps to the format's max
    d = dequant(q, s, dtype)
    rel = {E4M3: 2.0 ** -4, E5M2: 2.0 ** -3}[dtype]                    # half an ulp of 3 / 2 mantissa bits
    normal = (d.abs() >= s.double()[:, None] * {E4M3: 2.0 ** -6, E5M2: 2.0 ** -14}[dtype]) & (s[:, None] > 0)
    err = (d - x.double()).abs()
    bad = err[normal] > rel * (1 + 2.0 ** -20) * x.double().abs()[normal]     # + the scale's own fp32 rounding
    assert not bool(bad.any()), (err[normal][bad][:4], x.double()[normal][bad][:4])


@pytest.mark.parametrize("dtype", [E4M3, E5M2])
def test_saturation_at_the_format_maximum(dtype):
    """x * inv can round above the largest finite value (amax * (M / amax) > M in fp32); it saturates to M, never to
    NaN / inf."""
    mx = FP8_MAX[dtype]
    found = 0
    for bits in range(0x3F80, 0x4000):                               # every bf16 amax in [1, 2)
        a = torch.tensor([bits], dtype=torch.int16).view(bf16)
        x = torch.cat([a, -a, torch.zeros(14, dtype=bf16)]).view(1, 16)
        q, s = quant_rows_ref(x, dtype)
        v = q.view(dtype).float()
        assert float(v[0, 0]) == mx and float(v[0, 1]) == -mx
        found += int(float(a) * float(torch.tensor(mx, dtype=f32) / float(a)) > mx)
    assert found > 0                                                  # the rounding does overshoot for some amax


@pytest.mark.parametrize("dtype", [E4M3, E5M2])
@pytest.mark.parametrize("R", [1, 16, 37, 130])
def test_cast_transpose_rule(dtype, R):
    g = torch.Generator().manual_seed(R)
    C = 48
    x = (torch.randn(R, C, generator=g) * torch.logspace(-8, 8, C)[None, :]).to(bf16)
    x[:, 5] = 0                                                       # an all-zero column
    q, s = quant_cols_t_ref(x, dtype)
    R16 = -(-R // 16) * 16
    assert q.shape == (C, R16) and s.shape == (C,)
    assert not bool(q[:, R:].any())                                   # padding columns are zero
    assert float(s[5]) == 0 and not bool(q[5].any())
    qr, sr = quant_rows_ref(x.t().contiguous(), dtype)                # per column = the row rule on x^T
    assert torch.equal(q[:, :R], qr) and torch.equal(s, sr)
    # a strided view of the same values quantises the same
    wide = torch.zeros((R, C + 24), dtype=bf16)
    wide[:, 8 : 8 + C] = x
    q2, s2 = quant_cols_t_ref(wide[:, 8 : 8 + C], dtype)
    assert torch.equal(q, q2) and torch.equal(s, s2)


# ------------------------------------------------------------------------------------------------
# the differentiable FP8 linear
# ------------------------------------------------------------------------------------------------
def _ref_linear_grads(x, w, b, dy, grad_dtype):
    """fp32 autograd of y = X' W'^T + b over the dequantised operands of each product: X per token, W per output
    channel (forward); dY per token and W^T per input channel (dgrad); dY^T per output channel and X^T per input
    channel (wgrad)."""
    T = x.shape[0]
    xr = dequant(*quant_rows_ref(x), E4M3).float()
    wr = dequant(*quant_rows_ref(w), E4M3).float()
    y = xr @ wr.t() + (0 if b is None else b.float())
    dyr = dequant(*quant_rows_ref(dy, grad_dtype), grad_dtype).float()
    wt = dequant(*quant_cols_t_ref(w), E4M3).float()                  # [K, N]
    dyt = dequant(*quant_cols_t_ref(dy, grad_dtype), grad_dtype).float()[:, :T]
    xt = dequant(*quant_cols_t_ref(x), E4M3).float()[:, :T]
    wv = wt.t().clone().requires_grad_(True)                          # dgrad: dX = dY' . (W^T)'^T
    xv = torch.zeros_like(xr, requires_grad=True)
    (xv @ wv.t()).backward(dyr)
    dx = xv.grad
    xv2 = xt.t().clone()                                              # wgrad: dW = (dY^T)' . (X^T)'^T
    wv2 = torch.zeros_like(wr, requires_grad=True)
    (xv2 @ wv2.t()).backward(dyt.t())
    return y, dx, wv2.grad, dy.float().sum(0)


@pytest.mark.parametrize("grad_dtype", [E4M3, E5M2])
@pytest.mark.parametrize("fuse", [False, True])
def test_linear_fp8_autograd_against_dequantised_fp32(grad_dtype, fuse):
    g = torch.Generator().manual_seed(3)
    T, K, N = 37, 64, 48
    x = torch.randn(T, K, generator=g).to(bf16).requires_grad_(True)
    w = torch.nn.Parameter((torch.randn(N, K, generator=g) * 0.05).to(bf16))
    b = torch.nn.Parameter((torch.randn(N, generator=g) * 0.1).to(bf16))
    dy = (torch.randn(T, N, generator=g) * 1e-3).to(bf16)
    if fuse:
        w.main_grad = torch.full((N, K), 0.25, dtype=f32)
        w.grad_added_to_main_grad = False
    with oracle_fp8_ops():
        y = ops.linear_fp8_autograd(x, w, b, grad_dtype, True, fuse)
        y.backward(dy)
    y_ref, dx_ref, dw_ref, db_ref = _ref_linear_grads(x.detach(), w.detach(), b.detach(), dy, grad_dtype)

    def close(a, r, name):
        assert (a.float() - r).abs().max() <= 1e-5 * r.abs().max() + 2.0 ** -8 * r.abs().max() * (a.dtype == bf16), name

    close(y, y_ref, "y")
    close(x.grad, dx_ref, "dx")
    close(b.grad, db_ref, "db")
    if fuse:
        assert w.grad_added_to_main_grad is True
        assert (w.main_grad - 0.25 - dw_ref).abs().max() <= 1e-5 * dw_ref.abs().max()
    else:
        close(w.grad, dw_ref, "dw")


# ------------------------------------------------------------------------------------------------
# the layer
# ------------------------------------------------------------------------------------------------
def _mcfg(cfg, **extra):
    m = types.SimpleNamespace(hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_attention_heads,
                              num_query_groups=cfg.num_key_value_heads, kv_channels=cfg.head_dim,
                              ffn_hidden_size=cfg.intermediate_size, layernorm_epsilon=cfg.rms_norm_eps,
                              hidden_dropout=0.0, attention_dropout=0.0, params_dtype=bf16)
    for k, v in extra.items():
        setattr(m, k, v)
    return m


def _layer(**extra):
    from long_vita_b200.megatron.transformer_layer import B200TransformerLayer
    from long_vita_b200.weights import llm_layer_weights

    cfg = LongVITAConfig.tiny(layers=1)
    mc = CK.hf_to_mcore(llm_layer_weights(cfg, 0, seed=5, dtype=bf16, perturb=True), cfg)
    layer = B200TransformerLayer(_mcfg(cfg, **extra), layer_number=1)
    layer.load_state_dict({k[len("decoder.layers.0."):]: v for k, v in mc.items()}, strict=True)
    for p in layer.parameters():
        p.requires_grad_(True)
    return cfg, layer


LINEAR_WEIGHTS = ["mlp.linear_fc1.weight", "mlp.linear_fc2.weight", "self_attention.linear_proj.weight",
                  "self_attention.linear_qkv.weight"]


def _run(cfg, layer, s=32):
    g = torch.Generator().manual_seed(6)
    x = torch.randn(s, 1, cfg.hidden_size, generator=g).to(bf16).requires_grad_(True)
    dy = torch.randn(s, 1, cfg.hidden_size, generator=g).to(bf16)
    with oracle_fp8_ops():
        out, _ = layer(hidden_states=x, attention_mask=None, rotary_pos_emb=None)
        out.backward(dy)
    return out.detach(), x.grad


class _Recorder:
    """Wraps ops functions (looked up at call time by the layer) and records (name, arguments' shapes / dtypes)."""

    def __init__(self, monkeypatch, names):
        self.calls = []
        for n in names:
            fn = getattr(ops, n)
            monkeypatch.setattr(ops, n, self._wrap(n, fn))

    def _wrap(self, name, fn):
        def f(*a, **k):
            self.calls.append((name, tuple((tuple(t.shape), t.dtype) if isinstance(t, torch.Tensor) else
                                           (t if isinstance(t, torch.dtype) else type(t).__name__) for t in a)))
            return fn(*a, **k)
        return f


# (the quantisers and linear_fp8 are replaced by their oracle forms inside _run, so they are seen through these)
FP8_CALLS = ["linear_fp8_autograd", "linear_fp8_dgrad", "linear_fp8_wgrad", "linear_fp8_wgrad_accumulate",
             "linear_wgrad", "linear_wgrad_accumulate"]


@pytest.mark.parametrize("fp8", ["e4m3", "hybrid"])
@pytest.mark.parametrize("fuse", [False, True])
def test_layer_routes_its_four_linears_through_fp8(monkeypatch, fp8, fuse):
    cfg, layer = _layer(fp8=fp8, gradient_accumulation_fusion=fuse)
    params = dict(layer.named_parameters())
    if fuse:
        for n in LINEAR_WEIGHTS:
            params[n].main_grad = torch.zeros(params[n].shape, dtype=f32)
            params[n].grad_added_to_main_grad = False
    rec = _Recorder(monkeypatch, FP8_CALLS)
    _run(cfg, layer)
    names = [c[0] for c in rec.calls]
    wgrad = "linear_fp8_wgrad_accumulate" if fuse else "linear_fp8_wgrad"
    assert names.count("linear_fp8_autograd") == 4 and names.count("linear_fp8_dgrad") == 4
    assert names.count(wgrad) == 4 and len(names) == 12
    weights = sorted(tuple(params[n].shape) for n in LINEAR_WEIGHTS)
    assert sorted(a[1][0] for n, a in rec.calls if n == "linear_fp8_autograd") == weights
    gd = E4M3 if fp8 == "e4m3" else E5M2
    assert all(a[-1] == gd for n, a in rec.calls if n in ("linear_fp8_dgrad", wgrad))
    assert all(p.grad is not None for n, p in params.items() if not (fuse and n in LINEAR_WEIGHTS))
    if fuse:
        assert all(params[n].grad_added_to_main_grad is True and bool(params[n].main_grad.any()) for n in LINEAR_WEIGHTS)


def _dequantised_reference(cfg, layer, fp8, s=32):
    """fp32 autograd of the layer's composition with every linear replaced by its FP8 products over dequantised
    operands (the same recipe as _ref_linear_grads), the other operators being the CPU oracle's; returns the output,
    dX and the parameter gradients."""
    gd = E4M3 if fp8 == "e4m3" else E5M2

    class RefLinear(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, w, b):
            ctx.save_for_backward(x, w)
            ctx.has_bias = b is not None
            return _ref_linear_fwd(x, w, b)

        @staticmethod
        def backward(ctx, dy):
            x, w = ctx.saved_tensors
            dy2 = dy.reshape(-1, w.shape[0]).contiguous()
            x2 = x.reshape(-1, w.shape[1])
            with torch.enable_grad():
                _, dx, dw, db = _ref_linear_grads(x2, w, None, dy2, gd)
            return dx.to(bf16).view(x.shape), dw.to(bf16), (db.to(bf16) if ctx.has_bias else None)

    def lin(x, w, b=None, accumulate_wgrad=False):
        return RefLinear.apply(x, w, b)

    layer.fp8 = None                                                  # the bf16 composition, with RefLinear linears
    saved = ops.linear_autograd
    try:
        ops.linear_autograd = lin
        return _run(cfg, layer, s)
    finally:
        ops.linear_autograd = saved
        layer.fp8 = fp8


def _ref_linear_fwd(x, w, b):
    K = x.shape[-1]
    xr = dequant(*quant_rows_ref(x.reshape(-1, K)), E4M3).float()
    wr = dequant(*quant_rows_ref(w), E4M3).float()
    y = xr @ wr.t() + (0 if b is None else b.float())
    return y.to(bf16).view(*x.shape[:-1], -1)


@pytest.mark.parametrize("fp8", ["e4m3", "hybrid"])
@pytest.mark.parametrize("fuse", [False, True])
def test_layer_gradients_equal_the_dequantised_composition(fp8, fuse):
    cfg, layer = _layer(fp8=fp8, gradient_accumulation_fusion=fuse)
    params = dict(layer.named_parameters())
    if fuse:
        for n in LINEAR_WEIGHTS:
            params[n].main_grad = torch.zeros(params[n].shape, dtype=f32)
    out, dx = _run(cfg, layer)
    got = {n: (p.main_grad if fuse and n in LINEAR_WEIGHTS else p.grad).float() for n, p in params.items()}
    _, ref = _layer(fp8=fp8)
    out_r, dx_r = _dequantised_reference(cfg, ref, fp8)
    _close(out, out_r, "out")
    _close(dx, dx_r, "dx")
    for n, p in ref.named_parameters():
        _close(got[n], p.grad, n)


def _close(a, r, name):
    """|a - r| <= 1e-5 max|r| beside the bf16 rounding of the stored result (one bf16 ulp of the element)."""
    a, r = a.double(), r.double()
    ulp = 2.0 ** (torch.floor(torch.log2(r.abs().clamp_min(1e-30))) - 7)
    assert bool(((a - r).abs() <= 1e-5 * r.abs().max() + ulp).all()), (name, float((a - r).abs().max()))


def test_fp8_wgrad_false_reaches_the_bf16_wgrad(monkeypatch):
    cfg, layer = _layer(fp8="hybrid", fp8_wgrad=False)
    rec = _Recorder(monkeypatch, FP8_CALLS)
    _run(cfg, layer)
    names = [c[0] for c in rec.calls]
    assert names.count("linear_wgrad") == 4 and names.count("linear_fp8_dgrad") == 4
    assert "linear_fp8_wgrad" not in names and "linear_fp8_wgrad_accumulate" not in names


@pytest.mark.parametrize("field", ["absent", None])
def test_fp8_none_makes_the_bf16_calls(monkeypatch, field):
    names = ["linear_autograd", "rmsnorm_autograd", "swiglu_autograd", "rope_autograd", "attention"] + FP8_CALLS
    seqs, outs = [], []
    for extra in ({}, {} if field == "absent" else {"fp8": None}):
        cfg, layer = _layer(**extra)
        with monkeypatch.context() as m:
            rec = _Recorder(m, names)
            outs.append(_run(cfg, layer) + tuple(p.grad for p in layer.parameters()))
        seqs.append(rec.calls)
    assert seqs[0] == seqs[1] and not any(n.startswith("linear_fp8") for n, _ in seqs[0])
    assert all(torch.equal(a, b) for a, b in zip(outs[0], outs[1]))


def test_fp8_inference_uses_the_fp8_decoder_layer():
    cfg, layer = _layer(fp8="e4m3")
    with oracle_fp8_ops():
        dec = layer._decoder_layer()
    assert all(isinstance(w, ops.Fp8Weight) for w in (dec.wqkv, dec.wo, dec.w_gate_up, dec.w_down))
    _, plain = _layer()
    with oracle_fp8_ops():
        assert not isinstance(plain._decoder_layer().wo, ops.Fp8Weight)


@pytest.mark.parametrize("fp8", ["e4m3", "hybrid"])
def test_weights_written_through_data_are_used_by_the_next_step(fp8):
    """Megatron's bf16 optimizers write the updated weights with `param.data.copy_(...)` (the distributed optimizer
    into the same buffer), which moves neither `_version` nor `data_ptr`.  The next training step must use the new
    values: its output and gradients equal those of a fresh layer built with them."""
    cfg, layer = _layer(fp8=fp8)
    _run(cfg, layer)
    g = torch.Generator().manual_seed(11)
    new = {}
    for n, p in layer.named_parameters():
        stamp = (p._version, p.data_ptr())
        new[n] = (p.detach().float() * (1 + 0.5 * torch.rand(p.shape, generator=g))).to(bf16)
        p.data.copy_(new[n])
        assert (p._version, p.data_ptr()) == stamp                      # the update is invisible to a stamp
        p.grad = None
    out, dx = _run(cfg, layer)
    _, fresh = _layer(fp8=fp8)
    fresh.load_state_dict(new, strict=False)
    out_f, dx_f = _run(cfg, fresh)
    assert torch.equal(out, out_f) and torch.equal(dx, dx_f)
    fresh_params = dict(fresh.named_parameters())
    assert all(torch.equal(p.grad, fresh_params[n].grad) for n, p in layer.named_parameters())


@pytest.mark.parametrize("extra,exc", [({"fp8": "e5m2"}, ValueError), ({"fp8": True}, ValueError),
                                       ({"fp8": "hybrid", "fp8_dot_product_attention": True}, NotImplementedError),
                                       ({"fp8": "e4m3", "fp8_multi_head_attention": True}, NotImplementedError)])
def test_refusals_before_anything_runs(monkeypatch, extra, exc):
    from long_vita_b200 import _lib
    from long_vita_b200.megatron.transformer_layer import B200TransformerLayer

    def no_launch(*a, **k):
        raise AssertionError("nothing may be launched")

    monkeypatch.setattr(_lib, "lib", no_launch)
    with pytest.raises(exc):
        B200TransformerLayer(_mcfg(LongVITAConfig.tiny(layers=1), **extra), layer_number=1)


def test_delayed_scaling_fields_are_ignored():
    cfg, plain = _layer(fp8="e4m3")
    _, delayed = _layer(fp8="e4m3", fp8_margin=2, fp8_interval=4, fp8_amax_history_len=16,
                        fp8_amax_compute_algo="max")
    a, b = _run(cfg, plain), _run(cfg, delayed)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
