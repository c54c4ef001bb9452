"""GPU: the wgmma GEMM against the float64 reference of tests/gemm_ref.py, per 64 x 64 output chunk and elementwise, at
the shapes the product runs: the 14B decoder's linears at the bench prompt (T = 18 432) and at ragged token counts,
the InternViT tower and projector at 64 frames, the scheduler's edges (tile counts around the SM count, part-empty
tiles, N tails), the backward products at training shapes, decode-sized M (the GEMV and the LM head), and the LM head
fused with the cross-entropy, layer by layer.  cuBLAS (bf16 in, fp32 accumulation) is the yardstick at the prefill
shapes.

Inputs are generated on the device from seeds; weights have the model's scale K^-0.5.  Each case prints one
`GEMM-REF {...}` line with its worst figures (run with -s to see them)."""
import contextlib
import json
import math

import pytest
import torch

from tests.gemm_ref import check_gemm, check_untouched, gemm_ref, ulp_bf16

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
DECODER = {"qkv": (7168, 5120, True, None), "o": (5120, 5120, False, None), "gate_up": (27648, 5120, False, "swiglu"),
           "down": (5120, 13824, False, None)}
VIT = {"qkv": (3072, 1024, True, None), "proj": (1024, 1024, True, None), "fc1": (4096, 1024, True, "gelu"),
       "fc2": (1024, 4096, True, None)}
PROJECTOR = {"proj_fc1": (5120, 4096, True, "gelu"), "proj_fc2": (5120, 5120, True, None)}
VIT_ROWS = 64 * 1025            # 64 frames x (1 + 32 x 32) tokens


@pytest.fixture(scope="module")
def L(lib_built):
    from long_vita_b200 import ops

    return ops


@pytest.fixture(autouse=True)
def _memory():
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    _memory.base = torch.cuda.memory_allocated()
    yield
    torch.cuda.empty_cache()


def _report(res, **extra):
    res = dict(res, **extra)
    res["peak_extra_gb"] = round((torch.cuda.max_memory_allocated() - _memory.base) / 2 ** 30, 2)
    print("GEMM-REF " + json.dumps(res))


def _randn(shape, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.randn(shape, generator=g, device="cuda", dtype=BF)
    return t.mul_(scale) if scale != 1.0 else t


def _weights(L, N, K, bias, act, seed):
    if act == "swiglu":      # rows interleaved (gate_i, up_i), as the decoder loads them
        w = L.interleave_gate_up(_randn((N // 2, K), seed, K ** -0.5), _randn((N // 2, K), seed + 1, K ** -0.5))
    else:
        w = _randn((N, K), seed, K ** -0.5)
    return w, (_randn((N,), seed + 2, 0.5) if bias else None)


@contextlib.contextmanager
def _cublas_fp32_reduction():
    m = torch.backends.cuda.matmul
    old = m.allow_bf16_reduced_precision_reduction
    m.allow_bf16_reduced_precision_reduction = False
    try:
        yield
    finally:
        m.allow_bf16_reduced_precision_reduction = old


def _cublas(a, w, b):
    with _cublas_fp32_reduction():
        return torch.nn.functional.linear(a, w, b)


def _forward(L, name, M, N, K, bias, act, seed, pad=0, cublas=False):
    """An epilogue with an inner bf16 rounding (GELU, SwiGLU) turns an fp32 accumulation difference that flips that
    rounding into a whole ulp of the output, which weighs on a 64 x 64 chunk far more than on the product (measured
    up to 3e-3 for SwiGLU at T = 18 432, 7e-4 for GELU).  So the 1e-3 per-chunk bound is asserted on the product the
    same kernel computes without the epilogue (act = None); the fused output is held to the elementwise bound, its
    per-chunk excess is reported, and the fused SwiGLU must equal the unfused GEMM + lv_swiglu bit for bit."""
    a = _randn((M, K), seed)
    w, b = _weights(L, N, K, bias, act, seed + 10)
    n_out = N // 2 if act == "swiglu" else N
    buf = None
    if pad:
        buf = torch.full((M, n_out + pad), 7.0, dtype=BF, device="cuda")
        y = L.linear(a, w, b, act, out=buf[:, :n_out])
        check_untouched(buf, n_out, 7.0, name)
    else:
        y = L.linear(a, w, b, act)
    extra = {"M": M, "N": N, "K": K}
    if act is not None:
        ref = gemm_ref(a, w, b, act)
        fused = check_gemm(y, ref, a, w, b, act, chunk_bound=math.inf, name=name + " fused")
        extra.update(fused_chunk_excess=fused["chunk_excess"], fused_elem_ratio=fused["elem_ratio"])
        del ref
        plain = L.linear(a, w, b)
        if act == "swiglu":
            assert torch.equal(y, L.swiglu(torch.cat([plain[:, 0::2], plain[:, 1::2]], 1))), name
        y = plain
    ref = gemm_ref(a, w, b)
    res = check_gemm(y, ref, a, w, b, name=name)
    if cublas:
        cub = check_gemm(_cublas(a, w, b), ref, a, w, b, chunk_bound=math.inf, elementwise=False)
        extra.update(cublas_chunk_excess=cub["chunk_excess"], cublas_total_excess=cub["total_excess"])
        assert res["chunk_excess"] <= 2 * cub["chunk_excess"] + 1e-5, (res, cub)
    _report(res, **extra)


# ------------------------------------------------------------------------------------------------
# forward: prefill, ragged rasterisation, the vision tower and projector
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layer", list(DECODER))
@pytest.mark.parametrize("T", [18432, 16897, 2304])
def test_decoder_forward(L, T, layer):
    """T = 18 432 is the bench prompt (cuBLAS yardstick there).  T = 16 897 gives 133 M-blocks, the last holding one
    row: 11 raster groups of 12 + 1 at K = 5120, 16 groups of 8 + 5 at K = 13 824.  T = 2304 is a context-parallel
    rank's share."""
    N, K, bias, act = DECODER[layer]
    _forward(L, f"decoder {layer} T={T}", T, N, K, bias, act, seed=T + N, cublas=T == 18432)


@pytest.mark.parametrize("layer", list(VIT) + list(PROJECTOR))
def test_vision_forward(L, layer):
    """The tower at 64 frames (65 600 rows: 513 M-blocks = 8 raster groups of 64 + 1 at K = 1024), the projector at
    16 384 rows."""
    N, K, bias, act = {**VIT, **PROJECTOR}[layer]
    M = VIT_ROWS if layer in VIT else 16384
    _forward(L, f"vision {layer}", M, N, K, bias, act, seed=M + N + K)


def test_patch_embed_64_frames(L):
    """65 536 patch rows, K = 640 (588 real): the conv as im2col + GEMM + bias, then bf16(. + pos)."""
    n, size, ps, C = 64, 448, 14, 1024
    images = _randn((n, 3, size, size), 1)
    conv_w, conv_b = _randn((C, 3, ps, ps), 2, 588 ** -0.5), _randn((C,), 3, 0.5)
    cls, pos = _randn((1, 1, C), 4), _randn((1, 1 + (size // ps) ** 2, C), 5)
    w_pad = L.pad_patch_weight(conv_w)
    out = L.patch_embed(images, w_pad, conv_b, cls, pos, ps)
    col = L.patch_im2col(images, ps, w_pad.shape[1])
    want_col = images.unfold(2, ps, ps).unfold(3, ps, ps).permute(0, 2, 3, 1, 4, 5).reshape(-1, 3 * ps * ps)
    assert torch.equal(col[:, :588], want_col) and not bool(col[:, 588:].any())
    P = (size // ps) ** 2
    post = pos[0, 1:].repeat(n, 1)
    ref = gemm_ref(col, w_pad, conv_b, post=post)
    fused = check_gemm(out[:, 1:].reshape(n * P, C), ref, col, w_pad, conv_b, "post", chunk_bound=math.inf,
                       name="patch_embed")
    assert torch.equal(out[:, 0], (cls[0, 0].float() + pos[0, 0].float()).to(BF).expand(n, C))
    del ref
    res = check_gemm(L.linear(col, w_pad, conv_b), gemm_ref(col, w_pad, conv_b), col, w_pad, conv_b,
                     name="patch_embed product")
    _report(res, M=n * P, N=C, K=w_pad.shape[1], fused_chunk_excess=fused["chunk_excess"])


# ------------------------------------------------------------------------------------------------
# the persistent scheduler's edges
# ------------------------------------------------------------------------------------------------
def _edge_cases():
    cases = []
    for ti, tiles in enumerate(["1", "sm-1", "sm", "sm+1", "2sm+1"]):
        for mi, M in enumerate([5, 64, 65, 127, 129]):
            cases.append((tiles, M, [8, 248][(ti + mi) % 2], [None, "gelu_tanh"][mi % 2]))
    return cases


@pytest.mark.parametrize("tiles,M,n_tail,act", _edge_cases())
def test_scheduler_edges(L, tiles, M, n_tail, act):
    """Tile counts 1, SM - 1, SM, SM + 1 and 2 SM + 1 (one CTA per SM, so zero, one and two tiles per CTA and every
    CTA but one idle); M rows whose last tile leaves the second consumer warpgroup's half empty (5, 64, 129), partly
    valid (65, 127); N % 256 = 8 or 248; a strided output."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    target = {"1": 1, "sm-1": sm - 1, "sm": sm, "sm+1": sm + 1, "2sm+1": 2 * sm + 1}[tiles]
    num_m = (M + 127) // 128
    num_n = max(1, target // num_m)
    N = 256 * (num_n - 1) + n_tail
    _forward(L, f"edge tiles={num_m * num_n} M={M} N={N}", M, N, 1024, True, act, seed=M * 1000 + N, pad=24)


# ------------------------------------------------------------------------------------------------
# backward products at training shapes
# ------------------------------------------------------------------------------------------------
BWD = [(f"decoder {k} T={T}", T, *v[:3]) for T in (18432, 16897) for k, v in DECODER.items()] + \
      [(f"vit {k}", VIT_ROWS, *v[:3]) for k, v in VIT.items()]


@pytest.mark.parametrize("name,T,N,K,bias", BWD, ids=[c[0].replace(" ", "-") for c in BWD])
def test_linear_backward(L, name, T, N, K, bias):
    """dX = dY W (W read MN-major), dW = dY^T X (both MN-major, the contraction over T, T % 8 != 0 at 16 897) and
    db = column sums of dY, each against float64."""
    x = _randn((T, K), T + K).requires_grad_(True)
    w = _randn((N, K), N + K, K ** -0.5).requires_grad_(True)
    b = _randn((N,), N, 0.5).requires_grad_(True) if bias else None
    dy = _randn((T, N), T + N)
    L.linear_autograd(x, w, b).backward(dy)
    xd, wd = x.detach(), w.detach()
    dx = check_gemm(x.grad, gemm_ref(dy, wd.t()), dy, wd.t(), name=name + " dX")
    x.grad = None
    dw = check_gemm(w.grad, gemm_ref(dy.t(), xd.t()), dy.t(), xd.t(), name=name + " dW")
    extra = {"T": T, "N": N, "K": K, "dX": dx, "dW": dw}
    if bias:
        ones = torch.ones((1, T), dtype=BF, device="cuda")
        extra["db"] = check_gemm(b.grad.view(1, N), gemm_ref(ones, dy.t()), ones, dy.t(), name=name + " db")
    _report({"name": name}, **extra)


def test_gate_up_forward_and_weight_gradient_are_deterministic(L):
    T, (N, K, _, _) = 18432, DECODER["gate_up"]
    x = _randn((T, K), 1)
    w, _ = _weights(L, N, K, False, "swiglu", 2)
    dy = _randn((T, N), 3)
    y0, y1 = L.linear(x, w, act="swiglu"), L.linear(x, w, act="swiglu")
    assert torch.equal(y0, y1)
    del y0, y1
    assert torch.equal(L.linear_wgrad(dy, x), L.linear_wgrad(dy, x))


# ------------------------------------------------------------------------------------------------
# decode: M = 1 .. 4 (the weight-stream GEMV; the LM head's 594 N-tiles take the tensor-core kernel)
# ------------------------------------------------------------------------------------------------
DECODE = {**DECODER, **PROJECTOR, "lm_head": (152064, 5120, False, None)}


@pytest.mark.parametrize("M,layer", [(M, k) for k in DECODE for M in (1, 2, 3, 4) if k != "lm_head" or M <= 2])
def test_decode(L, M, layer):
    N, K, bias, act = DECODE[layer]
    _forward(L, f"decode {layer} M={M}", M, N, K, bias, act, seed=M * 7 + N)


# ------------------------------------------------------------------------------------------------
# LM head fused with the cross-entropy, training
# ------------------------------------------------------------------------------------------------
def test_lm_head_ce_training(L):
    """c = 5120, V = 152 064 in 10 chunks of 16 384 (the last 4608 wide), M = 4099 rows selected from s = 18 432.
    (a) each chunk's logits per chunk against float64, into a strided buffer; (b) loss and lse against an fp64
    cross-entropy of those same bf16 logits; (c) lv_ce_grad elementwise against the fp64 formula on the same logits and
    lse; (d) dW per chunk; (e) d_sel against fp64 sum_c dlogits_c W_c.  Ignored rows: loss 0, zero gradient."""
    c, V, chunk, s, M = 5120, 152064, 16384, 18432, 4099
    chunks = L._ce_chunks(V, chunk)
    assert len(chunks) == 10 and chunks[-1][1] - chunks[-1][0] == 4608
    g = torch.Generator().manual_seed(7)
    idx = torch.randperm(s, generator=g)[:M].sort().values.cuda()
    labels = torch.randint(0, V, (M,), generator=g)
    special = [-100, 0, 16383, 16384, 147455, 147456, 152063]
    labels[: len(special)] = torch.tensor(special)
    labels[M // 2] = -100
    labels = labels.cuda()
    h = _randn((s, 1, c), 8)
    w = _randn((V, c), 9, c ** -0.5)
    peaked = 11                                       # a row whose softmax is nearly one-hot, labelled at its argmax
    h[int(idx[peaked])] *= 32
    labels[peaked] = int(L.linear(h[int(idx[peaked])], w).float().argmax())
    mask = torch.zeros((1, s), dtype=torch.bool, device="cuda")
    mask[0, idx] = True
    dloss = _randn((1, M), 10).float()
    hg, wg = h.clone().requires_grad_(True), w.clone().requires_grad_(True)
    loss = L.masked_lm_head_ce(hg, wg, mask, labels.view(1, M), vocab_chunk=chunk)
    loss.backward(dloss)
    sel = h[idx, 0]
    ign = labels < 0
    worst = {}

    def keep(key, res):
        if key not in worst or res["chunk_excess"] > worst[key]["chunk_excess"] or res["elem_ratio"] > worst[key]["elem_ratio"]:
            worst[key] = {k: res[k] for k in ("name", "chunk_excess", "elem_ratio", "total_excess", "mismatch")}

    # (a) logits per chunk, (b) fp64 cross-entropy of those bf16 logits
    logits = torch.empty((M, V), dtype=BF, device="cuda")
    lse64 = torch.full((M,), -math.inf, dtype=torch.float64, device="cuda")
    buf = torch.empty((M, chunk), dtype=BF, device="cuda")
    for v0, v1 in chunks:
        buf.fill_(7.0)
        lg = L.linear(sel, w[v0:v1], out=buf[:, : v1 - v0])
        keep("logits", check_gemm(lg, gemm_ref(sel, w[v0:v1]), sel, w[v0:v1], name=f"logits [{v0}, {v1})"))
        check_untouched(buf, v1 - v0, 7.0, "logits")
        logits[:, v0:v1] = lg
        lse64 = torch.logaddexp(lse64, torch.logsumexp(lg.double(), 1))
    tgt = logits.gather(1, labels.clamp_min(0).view(-1, 1)).view(-1).double()
    loss_ref = torch.where(ign, torch.zeros_like(lse64), lse64 - tgt)
    loss = loss.detach().view(-1)
    assert bool((loss[ign] == 0).all())
    loss_err = float(((loss.double() - loss_ref).abs() / (1 + loss_ref.abs())).max())
    assert loss_err < 2e-5, loss_err
    _, lse = L.lm_head_ce_fwd(sel, w, labels, chunk)
    lse_err = float(((lse.double() - lse64).abs() / (1 + lse64.abs())).max())
    assert lse_err < 2e-5, lse_err
    assert float(loss_ref[peaked]) < 1e-2                         # the nearly one-hot row

    # (c) lv_ce_grad: d = (exp(x) - onehot) dloss, x = logit - lse; __expf is within (2 + 1.2 |x|) fp32 ulps, the fp32
    # subtraction and product add one each
    dlogits = torch.empty_like(logits)
    dl = dloss.view(-1).double()
    ce_ratio = 0.0
    for v0, v1 in chunks:
        got = L.ce_grad(logits[:, v0:v1].clone(), labels, lse, dloss.view(-1), v0)
        x = logits[:, v0:v1].double() - lse.double().view(-1, 1)
        onehot = (labels.view(-1, 1) == torch.arange(v0, v1, device="cuda").view(1, -1)).double()
        gsc = torch.where(ign, torch.zeros_like(dl), dl).view(-1, 1)
        want = (x.exp() - onehot) * gsc
        bound = ulp_bf16(want) + gsc.abs() * x.exp() * (4 + 2 * x.abs()) * 2.0 ** -23 + 1e-37
        q = float(((got.double() - want).abs() / bound).max())
        assert q <= 1.0, (v0, q)
        ce_ratio = max(ce_ratio, q)
        assert not bool(got[ign].any())
        dlogits[:, v0:v1] = got
        del x, onehot, want, bound
    worst["ce_grad"] = {"elem_ratio": ce_ratio}

    # (d) dW per chunk: dlogits_c^T sel, the M = 4099 selected rows are the contraction
    for v0, v1 in chunks:
        keep("dW", check_gemm(wg.grad[v0:v1], gemm_ref(dlogits[:, v0:v1].t(), sel.t()), dlogits[:, v0:v1].t(), sel.t(),
                              name=f"dW [{v0}, {v1})"))
    # (e) d_sel = bf16(sum_c bf16(dlogits_c W_c) in fp32).  Each chunk's product (W_c read MN-major) per 64 x 64 chunk;
    # d_sel equal to that sum bit for bit; d_sel against fp64 sum_c dlogits_c W_c elementwise, each chunk's product
    # off by up to half a bf16 ulp of its |dlogits_c| |W_c| sum.  Its per-chunk excess over sqrt(2) roundings is
    # reported: a flipped rounding of one chunk's product is a whole ulp, measured up to 2.5e-3 in the 3-row chunks.
    ref = torch.zeros((M, c), dtype=torch.float64, device="cuda")
    acc = torch.zeros((M, c), dtype=torch.float32, device="cuda")
    for v0, v1 in chunks:
        rc = gemm_ref(dlogits[:, v0:v1], w[v0:v1].t())
        pc = L.linear(dlogits[:, v0:v1], w[v0:v1].t())
        keep("d_sel chunk products", check_gemm(pc, rc, dlogits[:, v0:v1], w[v0:v1].t(), name=f"d_sel [{v0}, {v1})"))
        ref += rc
        acc += pc.float()
        del rc, pc
    dsel = hg.grad[idx, 0]
    assert torch.equal(dsel, acc.to(BF))
    keep("d_sel", check_gemm(dsel, ref, dlogits, w.t(), floor_factor=2.0, partial_rounding=2.0 ** -8,
                             chunk_bound=math.inf, name="d_sel"))
    assert not bool(dsel[ign].any())
    rest = torch.ones(s, dtype=torch.bool, device="cuda")
    rest[idx] = False
    assert not bool(hg.grad[rest].any())
    _report({"name": "lm_head_ce"}, loss_err=loss_err, lse_err=lse_err, **worst)
