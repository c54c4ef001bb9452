"""The FP8 (e4m3) linears on the H100 (lv_quant_rows_fp8_fmt, lv_gemm_fp8, ops.linear with an ops.Fp8Weight).

* Quantiser: the rows lv_quant_rows_fp8_fmt writes are byte for byte the CPU restatement of the rule
  (tests/fp8_ref.quant_rows_ref), at K = 5120 and 13 824, with zero rows, rows too small
  to scale, magnitudes from 1e-30 to 1e30 and a strided input.
* GEMM and GEMV against float64 over the dequantised operands (tests/gemm_ref.py: r = (A_q s_a) (W_q s_w)^T + bias,
  in float64), per 64 x 64 output chunk and elementwise:
  - the four decoder linears at T = 18 432, 16 897 (a one-row last M-block) and 2304; N tails; tile counts 1, SM - 1,
    SM and SM + 1; the plain / bias and the fused SwiGLU epilogues; the GEMV at M = 1 .. 4.
  - The fused SwiGLU is checked bit for bit against ops.swiglu of the plain product, whose elements are its gate and
    up values: the float64 check applies to the product, and SwiGLU keeps the bf16 rounding sequence of the bf16 GEMM.
  - Bound.  The products of e4m3 values are exact, and the scales multiply the fp32 sum once each (2 roundings of
    2^-24, inside the ulp term of gemm_ref).  What is left is the accumulation.  Hopper's FP8 wgmma adds into its
    accumulator with ~14 bits kept (DeepSeek-V3 §3.3.2), truncating; the kernel restarts that accumulator at every
    128-deep k-block (four k32 instructions) and adds it to an fp32 sum.  Within a k-block the partial sum never
    exceeds S_b = sum_b |a_k w_k|, so four truncating adds lose at most 4 2^-13 S_b, and over all blocks at most
    4 2^-13 sum_k |a_k w_k|: `partial_rounding` = 2^-11 in gemm_ref's elementwise bound (plus K 2^-23 for the fp32
    adds).  An accumulation left in the tensor cores for all K / 32 = 432 instructions at K = 13 824 may lose 2^-13
    of the running sum at each of them, up to 432 2^-13 ~ 5 % of sum |a_k w_k| - 100x the bound.  For the per-chunk
    RMS the same argument with random-signed errors gives ~sqrt(4) 2^-14 ~ 1.2e-4 relative for the promoted sum and
    ~sqrt(432 / 2) 2^-14 ~ 9e-4 without promotion, so CHUNK_BOUND sits below the latter.  Measured on an H100
    80GB HBM3: the worst chunk excess is 3.9e-4 with promotion; a build without it (LV_EXTRA_DEFINES=
    -DLV_FP8_NO_PROMOTION) gives 1.0e-3 at K = 1 040, 1.5-2.8e-3 at K = 5 120 and 3.1-3.6e-3 at K = 13 824, and fails
    every case of this file's GEMM tests but the K = 16 one.
* Model: a 4-layer 14B-geometry model at 18 432 tokens, FP8 against bf16: relative Frobenius deviation of the prefill
  logits and greedy-token agreement over 16 teacher-forced decode steps (limits from the measured values with
  margin); FP8 prefill logits torch.equal between the whole-tensor and row-chunked plans; resident linear weight bytes
  equal to the shapes' N K + 4 N per linear.  The weights are synthetic: quality on a trained checkpoint is NOT
  measured here.
"""
import pytest
import torch

from tests.gemm_ref import check_gemm, gemm_ref
from tests.fp8_ref import quant_rows_ref

pytestmark = pytest.mark.gpu

H, QKV, INTER = 5120, 7168, 13824
LINEARS = {"wqkv": (QKV, H, "bias"), "wo": (H, H, None), "w_gate_up": (2 * INTER, H, "swiglu"),
           "w_down": (H, INTER, None)}
PARTIAL = 2.0 ** -11
CHUNK_BOUND = 5e-4
WORST = {}
# measured on an H100 80GB HBM3 (700 W): prefill logits 0.294 and decode 0.303 relative, greedy 10/16;
# limits with margin
LOGIT_REL_LIMIT = 0.4
AGREE_MIN = 8


@pytest.fixture(scope="module")
def L(lib_built):
    from long_vita_b200 import ops

    yield ops
    print(f"\n[fp8_linear] worst figures { {k: (round(v, 6) if isinstance(v, float) else v) for k, v in WORST.items()} }")


def _note(key, value, worst=max):
    WORST[key] = value if key not in WORST else worst(WORST[key], value)


# ------------------------------------------------------------------------------------------------
# quantiser
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [5120, 13824, 16])
def test_quant_rows_is_the_restatement(L, K):
    g = torch.Generator(device="cuda").manual_seed(K)
    M = 1000
    mag = torch.logspace(-30, 30, 13, device="cuda")[torch.randint(0, 13, (M, 1), device="cuda", generator=g)]
    x = (torch.randn((M, K), device="cuda", generator=g) * mag).to(torch.bfloat16)
    x[::7] = 0
    x[3, :] = 0
    x[3, 5] = torch.tensor([1], dtype=torch.int16).view(torch.bfloat16)          # a bf16 subnormal amax
    wide = torch.zeros((M, K + 24), dtype=torch.bfloat16, device="cuda")
    wide[:, 8 : 8 + K] = x
    for src in (x, wide[:, 8 : 8 + K]):                                           # contiguous, and a strided view
        q, s = L.quant_rows_fp8(src)
        torch.cuda.synchronize()
        q_ref, s_ref = quant_rows_ref(x.cpu())
        assert q.dtype == torch.float8_e4m3fn and s.dtype == torch.float32
        assert torch.equal(q.view(torch.uint8).cpu(), q_ref) and torch.equal(s.cpu().view(torch.int32),
                                                                           s_ref.view(torch.int32))
    assert float(s_ref[3]) == 0 and bool((q_ref[3] == 0).all())


# ------------------------------------------------------------------------------------------------
# GEMM / GEMV against float64
# ------------------------------------------------------------------------------------------------
def _operands(L, M, N, K, bias, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn((M, K), device="cuda", generator=g).to(torch.bfloat16)
    w = (torch.randn((N, K), device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    b = (torch.randn((N,), device="cuda", generator=g) * 0.5).to(torch.bfloat16) if bias else None
    return x, L.Fp8Weight.quantize(w), b


def _check(L, x, w8, b, act, name):
    """The plain product against float64; the fused SwiGLU bit for bit against ops.swiglu of the plain product (its
    gate and up are the plain epilogue's values: same mainloop, same k-order, same scaling and bf16 rounding)."""
    y = L.linear(x, w8, b, act=act)
    plain = L.linear(x, w8, b) if act == "swiglu" else y
    xq, xs = L.quant_rows_fp8(x)
    a = xq.float().double() * xs.double()[:, None]
    w = w8.data.float().double() * w8.scale.double()[:, None]
    ref = gemm_ref(a, w, b)
    r = check_gemm(plain, ref, a, w, b, chunk_bound=CHUNK_BOUND, partial_rounding=PARTIAL, name=name)
    _note("chunk_excess", r["chunk_excess"])
    _note("elem_ratio", r["elem_ratio"])
    if act == "swiglu":
        gate_up = torch.cat([plain[:, 0::2], plain[:, 1::2]], dim=1)         # lv_swiglu reads [gate | up]
        assert torch.equal(y, L.swiglu(gate_up)), f"{name}: fused SwiGLU differs from swiglu(plain product)"
    return y


@pytest.mark.parametrize("T", [18432, 16897, 2304])
@pytest.mark.parametrize("lin", list(LINEARS))
def test_decoder_linears(L, T, lin):
    N, K, kind = LINEARS[lin]
    x, w8, b = _operands(L, T, N, K, kind == "bias", T + N + K)
    _check(L, x, w8, b, "swiglu" if kind == "swiglu" else None, f"{lin} T={T}")


@pytest.mark.parametrize("M,N,K", [(300, 200, 5120), (129, 1000, 1040), (5, 8, 16), (640, 5128, 13824)])
def test_tails(L, M, N, K):
    x, w8, b = _operands(L, M, N, K, True, M * N)
    _check(L, x, w8, b, None, f"tails {M}x{N}x{K}")
    x, w8, _ = _operands(L, M, 2 * N if N % 16 else N, K, False, M * N + 1)
    _check(L, x, w8, None, "swiglu", f"tails swiglu {M}x{N}x{K}")


@pytest.mark.parametrize("extra", [-1, 0, 1, None])
def test_tile_counts(L, extra):
    """1, SM - 1, SM and SM + 1 output tiles of 128 x 128 (one M-block of 128 rows)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = 1 if extra is None else sms + extra
    x, w8, b = _operands(L, 128, 128 * tiles, 5120, True, tiles)
    _check(L, x, w8, b, None, f"tiles {tiles}")


@pytest.mark.parametrize("M", [1, 2, 3, 4])
@pytest.mark.parametrize("lin", list(LINEARS))
def test_gemv(L, M, lin):
    N, K, kind = LINEARS[lin]
    x, w8, b = _operands(L, M, N, K, kind == "bias", 7 * M + N)
    _check(L, x, w8, b, "swiglu" if kind == "swiglu" else None, f"gemv {lin} M={M}")


def test_out_rows_of_a_wider_buffer(L):
    """The row-chunked plan writes rows of the QKV buffer, the streamed plan its K|V buffer: out is a row slice."""
    x, w8, b = _operands(L, 300, 2048, 5120, True, 11)
    buf = torch.full((400, 2048), 7.0, dtype=torch.bfloat16, device="cuda")
    L.linear(x, w8, b, out=buf[50:350])
    assert torch.equal(buf[50:350], L.linear(x, w8, b))
    assert bool((buf[:50] == 7).all()) and bool((buf[350:] == 7).all())


# ------------------------------------------------------------------------------------------------
# a 4-layer 14B-geometry model
# ------------------------------------------------------------------------------------------------
def _model(layers, linear_dtype):
    from long_vita_b200.config import LongVITAConfig
    from long_vita_b200.hf.modeling import LongVITAForCausalLM

    return LongVITAForCausalLM.from_synthetic(LongVITAConfig(), seed=7, device="cuda", num_layers=layers,
                                              linear_dtype=linear_dtype)


def test_model_fp8_against_bf16(L, monkeypatch):
    from long_vita_b200.hf import modeling

    s, steps = 18432, 16
    g = torch.Generator(device="cuda").manual_seed(3)
    bf = _model(4, torch.bfloat16)
    ids = torch.randint(0, bf.config.vocab_size, (1, s), device="cuda", generator=g)
    with torch.no_grad():
        ref = bf(input_ids=ids, use_cache=True, num_logits_to_keep=64, max_cache_len=s + steps)
        bf_logits, bf_cache = ref.logits, ref.past_key_values
        fp = _model(4, torch.float8_e4m3fn)
        out = fp(input_ids=ids, use_cache=True, num_logits_to_keep=64, max_cache_len=s + steps)
        rel = float((out.logits.float() - bf_logits.float()).norm() / bf_logits.float().norm())
        fp_cache = out.past_key_values
        agree, worst = 0, 0.0
        tok = bf_logits[0, -1].float().argmax().view(1, 1)
        for _ in range(steps):
            a = bf(input_ids=tok, past_key_values=bf_cache, use_cache=True).logits[0, -1].float()
            b = fp(input_ids=tok, past_key_values=fp_cache, use_cache=True).logits[0, -1].float()
            worst = max(worst, float((b - a).norm() / a.norm()))
            agree += int(a.argmax()) == int(b.argmax())
            tok = a.argmax().view(1, 1)                 # teacher forcing: both take the bf16 run's token
        # whole-tensor against row-chunked, FP8
        whole = fp(input_ids=ids, num_logits_to_keep=64).logits
        monkeypatch.setattr(modeling, "ROW_CHUNK_THRESHOLD", 8192)
        monkeypatch.setattr(modeling, "ROW_CHUNK", 4096)
        assert len(modeling.row_chunks(s)) > 1
        chunked = fp(input_ids=ids, num_logits_to_keep=64).logits
    _note("prefill_logit_rel", rel)
    _note("decode_logit_rel", worst)
    WORST["greedy_agree"] = f"{agree}/{steps}"
    print(f"\n[fp8 model] prefill logits rel {rel:.4e}, decode worst rel {worst:.4e}, greedy {agree}/{steps}")
    assert rel < LOGIT_REL_LIMIT and worst < LOGIT_REL_LIMIT and agree >= AGREE_MIN
    assert torch.equal(whole, chunked)
    # resident bytes of the linears: N K e4m3 + 4 N scale bytes per linear
    want = 4 * sum(N * K + 4 * N for N, K, _ in LINEARS.values())
    assert sum(layer.linear_bytes() for layer in fp.model.layers) == want
    assert sum(layer.linear_bytes() for layer in bf.model.layers) == 4 * sum(2 * N * K for N, K, _ in LINEARS.values())
