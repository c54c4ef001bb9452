"""CPU tests of the FP8 (e4m3) decoder linears (ops.Fp8Weight, ops.linear_fp8, DecoderLayer(linear_dtype=...)).

* The row quantiser of csrc/fp8_core.h (lv_fp8_quant_row, the text quant_rows_fp8_kernel compiles), built with gcc:
  byte for byte the torch restatement (tests/fp8_ref.quant_rows_ref) for every finite bf16 value under several amax,
  zero rows and rows with a bf16-subnormal amax, at row lengths 5120 and 13 824.
* The wrappers with the recording stub library of tests/test_ops_args_host.py: the C calls of quant_rows_fp8 and of
  linear with an Fp8Weight (a row slice included), and every refusal with nothing recorded.
* Host logic on the CPU oracle, with the FP8 twins below: a tiny FP8 model gives torch.equal logits across the
  whole-tensor, row-chunked and streamed plans (per-row scales keep every row's product independent of the span it
  is computed in), generate() runs, .to() moves the FP8 weights, state_dict() refuses, bad linear_dtype values raise,
  and the prefill memory accounting adds the quantised A operand in FP8 only.

The GPU twin is tests/test_gpu_fp8_linear.py.
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F

from long_vita_b200 import ops
from long_vita_b200.config import LongVITAConfig
from long_vita_b200.hf import modeling
from long_vita_b200.weights import synthetic_state_dict
from tests.fp8_ref import build_rows_shim, check_rows, finite_bf16, quant_rows_ref
from tests.test_ops_args_host import P, _bf16, lib  # noqa: F401  (lib is the recording-stub fixture)
from tests.test_row_chunks_host import _inputs
from tests.test_stream_layer_host import _equal, _three_plans

FP8 = torch.float8_e4m3fn


# ------------------------------------------------------------------------------------------------
# the shared quantiser built with gcc, against the restatement
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return build_rows_shim(tmp_path_factory.mktemp("fp8_rows_host"))


@pytest.mark.parametrize("n", [5120, 13824])
def test_every_finite_bf16_value_against_several_amax(core, n):
    """The finite bf16 values sorted by magnitude fill rows of n - 1; the last element of each row is its amax: the
    row's largest |x| times 1 (x = +-amax, q = +-M), 3 and 2^8, 2^16, 2^24 (e4m3 subnormals and underflow)."""
    x = finite_bf16()
    x = x[x.float().abs().argsort()]
    x = torch.cat([x, x[-1:].expand(-len(x) % (n - 1))]).view(-1, n - 1)
    top = x.float().abs().amax(1, keepdim=True)
    for f in (1.0, 3.0, 2.0 ** 8, 2.0 ** 16, 2.0 ** 24):
        amax = (top * f).to(torch.bfloat16)
        keep = (torch.isfinite(amax.float()) & (amax.float() >= top))[:, 0]
        q, _ = check_rows(core, torch.cat([x, amax], 1)[keep])
        if f == 1.0:
            assert bool((q[top[keep, 0] >= 1e-30, -1] == 0x7E).all())


@pytest.mark.parametrize("n", [5120, 13824])
def test_zero_rows_and_subnormal_amax(core, n):
    g = torch.Generator().manual_seed(n)
    x = torch.zeros(6, n, dtype=torch.bfloat16)
    x[1] = -0.0
    x[2, 5] = torch.tensor([1], dtype=torch.int16).view(torch.bfloat16)           # amax 9.2e-41: M / amax overflows
    x[3, :4] = torch.tensor([0, 1, 0x8001, 0x7F], dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    x[4] = (torch.randn(n, generator=g) * 1e-36).to(torch.bfloat16)               # inv finite
    x[5] = (torch.randn(n, generator=g) * 30).to(torch.bfloat16)
    q, scale = check_rows(core, x)
    assert bool((q[:4] == 0).all()) and bool((scale[:4] == 0).all()) and scale[4] > 0 and scale[5] > 0


# ------------------------------------------------------------------------------------------------
# the wrappers' C calls and refusals (recording stub)
# ------------------------------------------------------------------------------------------------
def _fp8(*shape):
    return torch.zeros(*shape, dtype=FP8)


def _w8(N, K):
    return ops.Fp8Weight(_fp8(N, K), torch.zeros(N, dtype=torch.float32))


def test_quant_rows_calls(lib):  # noqa: F811
    x = _bf16(5, 48)
    q, s = ops.quant_rows_fp8(x)
    wide = _bf16(5, 72)
    q2, s2 = ops.quant_rows_fp8(wide[:, 8:56])                                # a strided view is read in place
    assert q.dtype == FP8 and s.dtype == torch.float32 and q.shape == (5, 48) and s.shape == (5,)
    assert lib.calls == [("lv_quant_rows_fp8_fmt", P(x), P(q), P(s), 5, 48, 48, 0),
                         ("lv_quant_rows_fp8_fmt", P(wide) + 16, P(q2), P(s2), 5, 48, 72, 0)]


def test_linear_fp8_calls(lib):  # noqa: F811
    w = _w8(96, 64)
    x, b = _bf16(2, 3, 64), _bf16(96)
    y = ops.linear(x, w, b)
    assert y.shape == (2, 3, 96)
    (n0, xp, xq, xs, M, K, ldx, fmt), g = lib.calls
    assert (n0, xp, M, K, ldx, fmt) == ("lv_quant_rows_fp8_fmt", P(x), 6, 64, 64, 0)
    assert g == ("lv_gemm_fp8", xq, xs, P(w.data), P(w.scale), P(b), P(y), 6, 96, 64, 64, 64, 96, 0)
    # a row slice of the weight (the streamed plan's Q and K|V launches) into rows of a wider buffer, and SwiGLU
    lib.calls.clear()
    kv = _bf16(10, 64)
    ws = w[32:96]
    assert isinstance(ws, ops.Fp8Weight) and ws.shape == (64, 64)
    ops.linear(x.view(6, 64)[:4], ws, b[32:96], out=kv[3:7])
    assert lib.calls[1][3:8] == (P(w.data) + 32 * 64, P(w.scale) + 32 * 4, P(b) + 32 * 2, P(kv) + 3 * 128, 4)
    assert lib.calls[1][8:] == (64, 64, 64, 64, 64, 0)
    lib.calls.clear()
    h = ops.linear(x, w, act="swiglu")
    assert h.shape == (2, 3, 48) and lib.calls[1][5:] == (None, P(h), 6, 96, 64, 64, 64, 48, 3)


def _refusals():
    w = _w8(96, 64)
    return [
        ("x dtype", lambda: ops.linear(torch.zeros(4, 64), w)),
        ("bias dtype", lambda: ops.linear(_bf16(4, 64), w, torch.zeros(96))),
        ("out dtype", lambda: ops.linear(_bf16(4, 64), w, out=torch.zeros(4, 96))),
        ("weight dtype", lambda: ops.Fp8Weight(torch.zeros(96, 64, dtype=torch.uint8), torch.zeros(96))),
        ("scale shape", lambda: ops.Fp8Weight(_fp8(96, 64), torch.zeros(95))),
        ("K mismatch", lambda: ops.linear(_bf16(4, 48), w)),
        ("K not a multiple of 16", lambda: ops.linear(_bf16(4, 40), _w8(96, 40))),
        ("N not a multiple of 8", lambda: ops.linear(_bf16(4, 64), _w8(92, 64))),
        ("misaligned weight rows", lambda: ops.linear(_bf16(4, 64), ops.Fp8Weight(_fp8(96, 72)[:, :64],
                                                                                   torch.zeros(96)))),
        ("short out", lambda: ops.linear(_bf16(4, 64), w, out=_bf16(3, 96))),
        ("narrow out", lambda: ops.linear(_bf16(4, 64), w, out=_bf16(4, 88))),
        ("out row stride", lambda: ops.linear(_bf16(4, 64), w, out=_bf16(4, 100)[:, :96])),
        ("misaligned out", lambda: ops.linear(_bf16(4, 64), w, out=_bf16(4 * 96 + 4)[4:].view(4, 96))),
        ("activation", lambda: ops.linear(_bf16(4, 64), w, act="gelu")),
        ("SwiGLU with bias", lambda: ops.linear(_bf16(4, 64), w, _bf16(96), act="swiglu")),
        ("bias length", lambda: ops.linear(_bf16(4, 64), w, _bf16(95))),
        ("quant K", lambda: ops.quant_rows_fp8(_bf16(4, 24))),
        ("quant rank", lambda: ops.quant_rows_fp8(_bf16(2, 4, 64))),
    ]


@pytest.mark.parametrize("case", range(len(_refusals())), ids=[r[0] for r in _refusals()])
def test_refusals_launch_nothing(lib, case):  # noqa: F811
    _, fn = _refusals()[case]
    with pytest.raises(ValueError):
        fn()
    assert lib.calls == []


def test_only_contiguous_row_slices():
    w = _w8(96, 64)
    for bad in (slice(0, 96, 2), 3, (slice(None), slice(0, 32))):
        with pytest.raises(TypeError):
            w[bad]


# ------------------------------------------------------------------------------------------------
# host logic on the CPU oracle, with FP8 twins
# ------------------------------------------------------------------------------------------------
def _quant_rows_twin(x):
    """quant_rows_fp8 restated (tests/fp8_ref.quant_rows_ref)."""
    q, s = quant_rows_ref(x.reshape(-1, x.shape[-1]).cpu())
    return q.view(FP8), s


def _fp8_product(x, w, bias, act, out):
    """lv_gemm_fp8 restated in float64 over the dequantised operands; a row's result depends only on that row."""
    xq, xs = _quant_rows_twin(x)
    y = (xq.double() * xs.double()[:, None]) @ (w.data.double() * w.scale.double()[:, None]).t()
    if bias is not None:
        y = y + bias.double()
    if act == "swiglu":
        y = F.silu(y[:, 0::2].to(torch.bfloat16).float()) * y[:, 1::2].to(torch.bfloat16).float()
    y = y.to(torch.bfloat16)
    if out is not None:
        out.view(y.shape).copy_(y)
        y = out
    return y.view(*x.shape[:-1], y.shape[-1])


@contextlib.contextmanager
def fp8_twins():
    """ops.quant_rows_fp8 and the FP8 branch of ops.linear on the CPU (inside or outside the oracle contexts)."""
    saved = ops.linear, ops.quant_rows_fp8
    bf16_linear = ops.linear

    def linear(x, weight, bias=None, act=None, out=None):
        if isinstance(weight, ops.Fp8Weight):
            return _fp8_product(x, weight, bias, act, out)
        return bf16_linear(x, weight, bias, act, out)

    ops.linear, ops.quant_rows_fp8 = linear, _quant_rows_twin
    try:
        yield
    finally:
        ops.linear, ops.quant_rows_fp8 = saved


@pytest.fixture(scope="module")
def tiny():
    cfg = LongVITAConfig.tiny(layers=2, vit_layers=1)
    return cfg, synthetic_state_dict(cfg, seed=31, dtype=torch.bfloat16, perturb=True)


def _fp8_model(cfg, w):
    with fp8_twins():
        return modeling.LongVITAForCausalLM(cfg, w, linear_dtype=FP8)


def test_fp8_layers_hold_fp8_weights(tiny):
    cfg, w = tiny
    model = _fp8_model(cfg, w)
    H, I, q = cfg.hidden_size, cfg.intermediate_size, cfg.q_size + 2 * cfg.kv_size
    for L in model.model.layers:
        for name, shape in (("wqkv", (q, H)), ("wo", (H, cfg.q_size)), ("w_gate_up", (2 * I, H)), ("w_down", (H, I))):
            t = getattr(L, name)
            assert isinstance(t, ops.Fp8Weight) and t.data.dtype == FP8 and t.shape == shape
        assert L.bqkv.dtype == L.ln1.dtype == torch.bfloat16
        assert L.linear_bytes() == sum(n * k + 4 * n for n, k in ((q, H), (H, cfg.q_size), (2 * I, H), (H, I)))
    assert model.lm_head.dtype == torch.bfloat16 and model.model.vision_model.layers[0]["attn.qkv.weight"].dtype == \
        torch.bfloat16
    # the FP8 weight is the quantised fused bf16 weight
    ref = modeling.DecoderLayer(cfg, w, 0)
    q8, s8 = _quant_rows_twin(ref.w_gate_up)
    assert torch.equal(model.model.layers[0].w_gate_up.data.view(torch.uint8), q8.view(torch.uint8))
    assert torch.equal(model.model.layers[0].w_gate_up.scale, s8)


def test_three_plans_give_equal_logits(tiny):
    cfg, w = tiny
    model = _fp8_model(cfg, w)
    model.model.vision_chunk = 1
    ids, images, idx = _inputs(cfg)

    def run():
        with fp8_twins():
            a = model(input_ids=ids, images=images, image_indices=idx, num_logits_to_keep=100)
            b = model(input_ids=ids, images=images, image_indices=idx, output_hidden_states=True)
        return a.logits, b.logits, b.hidden_states

    whole, chunked, streamed = _three_plans(run, ids.shape[1], scatters=2 * 2)
    assert _equal(chunked, whole) and _equal(streamed, whole)
    # FP8 is a different product: the logits are not the bf16 model's
    with fp8_twins():
        from tests.test_stream_layer_host import stream_oracle_ops

        with stream_oracle_ops():
            bf = modeling.LongVITAForCausalLM(cfg, w)(input_ids=ids, images=images, image_indices=idx,
                                                       num_logits_to_keep=100).logits
    assert not torch.equal(bf, whole[0])
    assert float((bf.float() - whole[0].float()).norm() / bf.float().norm()) < 0.1


def test_generate_runs(tiny):
    cfg, w = tiny
    model = _fp8_model(cfg, w)
    ids, images, idx = _inputs(cfg, s=300, n_img=1)
    from tests.test_stream_layer_host import stream_oracle_ops

    with stream_oracle_ops(), fp8_twins():
        out = model.generate(inputs=ids, images=images, image_indices=idx, max_new_tokens=3)
        first = model(input_ids=ids, images=images, image_indices=idx, num_logits_to_keep=1).logits
    assert out.shape == (1, 303) and torch.equal(out[:, :300], ids)
    assert int(out[0, 300]) == int(first[0, -1].float().argmax())


def test_to_moves_and_never_casts_fp8_weights(tiny):
    cfg, w = tiny
    model = _fp8_model(cfg, w)
    before = model.model.layers[1].wo
    model.to(torch.float32)
    after = model.model.layers[1].wo
    assert isinstance(after, ops.Fp8Weight) and after.data.dtype == FP8 and after.scale.dtype == torch.float32
    assert torch.equal(after.data.view(torch.uint8), before.data.view(torch.uint8))
    assert model.model.layers[1].ln1.dtype == torch.float32          # the bf16 tensors are cast as before


def test_state_dict_of_an_fp8_model_refuses(tiny):
    cfg, w = tiny
    with pytest.raises(NotImplementedError):
        _fp8_model(cfg, w).state_dict()
    assert "model.layers.0.self_attn.q_proj.weight" in modeling.LongVITAForCausalLM(cfg, w).state_dict()


@pytest.mark.parametrize("bad", [torch.float16, torch.float32, torch.float8_e5m2, "fp8", None])
def test_bad_linear_dtype_raises(tiny, bad):
    cfg, w = tiny
    with pytest.raises(ValueError, match="linear_dtype"):
        modeling.LongVITAForCausalLM(cfg, w, linear_dtype=bad)
    with pytest.raises(ValueError, match="linear_dtype"):
        modeling.LongVITAForCausalLM.from_synthetic(cfg, device="cpu", linear_dtype=bad)
    with pytest.raises(ValueError, match="linear_dtype"):
        modeling.LongVITAForCausalLM.from_pretrained("/nonexistent", linear_dtype=bad)
    with pytest.raises(ValueError, match="linear_dtype"):
        modeling.DecoderLayer(cfg, w, 0, linear_dtype=bad)


def test_layers_must_match_linear_dtype(tiny):
    cfg, w = tiny
    bf16_layers = [modeling.DecoderLayer(cfg, w, i) for i in range(cfg.num_hidden_layers)]
    with fp8_twins():
        fp8_layers = [modeling.DecoderLayer(cfg, w, i, FP8) for i in range(cfg.num_hidden_layers)]
    with pytest.raises(ValueError, match="linear_dtype"):
        modeling.LongVITAForCausalLM(cfg, w, bf16_layers, linear_dtype=FP8)
    with pytest.raises(ValueError, match="linear_dtype"):
        modeling.LongVITAForCausalLM(cfg, w, fp8_layers)
    assert modeling.LongVITAForCausalLM(cfg, w, fp8_layers, linear_dtype=FP8).model.layers[0].wqkv is \
        fp8_layers[0].wqkv


@pytest.mark.parametrize("T", [18432, 1058816, 2115584])
def test_prefill_bytes_add_the_fp8_operand(T):
    """bf16 is unchanged; FP8 adds the e4m3 rows and scales of the widest linear input (the down projection's 13 824)
    over the longest span of the plan."""
    cfg = LongVITAConfig()
    for streamed in (False, True):
        bf = modeling.prefill_bytes_per_token(cfg, T, streamed)
        assert modeling.prefill_bytes_per_token(cfg, T, streamed, torch.bfloat16) == bf
        span = max(r1 - r0 for r0, r1 in modeling.row_chunks(T))
        extra = modeling.prefill_bytes_per_token(cfg, T, streamed, FP8) - bf
        assert extra == -(-span * (13824 + 4) // T) and extra * T >= span * 13828
