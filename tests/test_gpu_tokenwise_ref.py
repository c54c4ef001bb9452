"""GPU: the token-wise kernels of csrc/elementwise.cu against the float64 references of tests/tokenwise_ref.py,
elementwise and by rounding flips per tensor and per row, through long_vita_b200.ops:

- every entry of the norm row-tiling tables and both sides of their boundaries, with row counts around the rows per
  CTA and, for the backward, around the partial-buffer rows (one grid pass) and at 20 passes (the grid-stride
  accumulation of dw / db);
- the training shapes of the decoder (RMSNorm, RoPE on the fused QKV views, SwiGLU), the InternViT tower and
  projector (LayerNorm, GELU, layer scale) and the SigLIP width;
- numerical edges: zero rows, rows where eps dominates, an outlier channel, mean-offset LayerNorm rows, activations
  across the __expf overflow range;
- RoPE at every heads-per-thread grouping, in place and through strided outputs; the RoPE table at long and zig-zag
  positions; the flash-decoding merge on its own with empty splits;
- bit-reproducible norm backward, and 64-bit offsets beyond 2^31 elements.

Inputs are generated on the device from seeds.  Each case prints `TOKENWISE-REF {...}` lines with its worst figures
(run with -s to see them)."""
import json
import math

import pytest
import torch

from oracle import ops as O
from tests.tokenwise_ref import (bias_gelu_ref, check_tokenwise, check_untouched, decode_merge_ref, edge_groups, edge_op,
                                 edge_rows, flip_limits, gelu_bwd_ref, layernorm_bwd_ref, layernorm_dwdb_ref,
                                 layernorm_ref, ls_residual_bwd_ref, ls_residual_ref, merge, residual_sum,
                                 rmsnorm_bwd_ref, rmsnorm_dw_ref, rmsnorm_ref, rope_bwd_ref, rope_ref, rope_table_ref,
                                 swiglu_bwd_ref, swiglu_ref)

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
NORM_COLS = [8, 248, 1024, 1032, 1152, 4096, 4104, 5120, 5128, 8192, 16384]
LN_BWD_COLS = [8, 1024, 1032, 4096, 4104, 8192]
EPS = [1e-6, 1e-5]                 # the decoder and InternViT; the projector's LayerNorm
VIT_ROWS = 64 * 1025
SLAB = 4096                        # rows per reference slab of the large elementwise checks


@pytest.fixture(scope="module")
def L(lib_built):
    from long_vita_b200 import ops

    return ops


@pytest.fixture(autouse=True)
def _memory():
    torch.cuda.empty_cache()
    yield
    torch.cuda.empty_cache()


def _lib():
    from long_vita_b200 import _lib

    return _lib.lib()


def _randn(shape, seed, scale=1.0, mean=0.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    t = torch.randn(shape, generator=g, device="cuda", dtype=torch.float32 if mean else BF)
    if mean:
        return (t * scale + mean).to(BF)
    return t.mul_(scale) if scale != 1.0 else t


def _norm_w(cols, seed):
    return (1 + 0.1 * torch.randn(cols, generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda")).to(BF)


def _check(op, y, ref, name):
    return dict(check_tokenwise(y, *ref, name=name, **flip_limits(op, y.shape[-1] if y.dim() else 1)), op=op)


def _report(name, **figs):
    print("TOKENWISE-REF " + json.dumps({"name": name, **figs}))


def _by_rows(op, y, ref_fn, name, *inputs, rows=SLAB):
    """check_tokenwise over row slabs of y against ref_fn(*row slabs of inputs)."""
    worst = None
    for r0 in range(0, y.shape[0], rows):
        sl = slice(r0, r0 + rows)
        ref = ref_fn(*[t[sl] if t is not None and t.dim() > 1 else t for t in inputs])
        worst = merge(worst, _check(op, y[sl], ref, name))
        del ref
    return worst


def _parts(kind, rows, cols):
    return int(getattr(_lib(), f"lv_{kind}_bwd_partials")(rows, cols))


def _bwd_rows(kind, cols):
    """1, rows per CTA +- 1, the rows of one full grid pass +- 1 and 20 passes (read from the partial-buffer size)."""
    rpc = _parts(kind, 1, cols)
    full = _parts(kind, 1 << 40, cols)
    assert full == 2 * torch.cuda.get_device_properties(0).multi_processor_count * rpc
    return sorted({1, rpc - 1, rpc + 1, full - 1, full, full + 1, 20 * full} - {0}), rpc, full


# ------------------------------------------------------------------------------------------------
# norm row tiling
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cols", NORM_COLS)
def test_norm_forward_tiling(L, cols):
    rpc = _parts("rmsnorm", 1, cols)
    w, b = _norm_w(cols, cols), _randn((cols,), cols + 1, 0.1)
    for i, rows in enumerate(sorted({1, rpc - 1, rpc + 1} - {0})):
        eps = EPS[i % 2]
        x, res = _randn((rows, cols), 10 * rows + cols), _randn((rows, cols), 10 * rows + cols + 1)
        y, s = L.rmsnorm(x, w, eps, residual=res)
        assert torch.equal(s, residual_sum(x, res))
        a = _check("rmsnorm", y, rmsnorm_ref(x, w, eps, res), f"rmsnorm {rows}x{cols} residual")
        a = merge(a, _check("rmsnorm", L.rmsnorm(x, w, eps), rmsnorm_ref(x, w, eps), f"rmsnorm {rows}x{cols}"))
        c = _check("layernorm", L.layernorm(x, w, b, eps), layernorm_ref(x, w, b, eps), f"layernorm {rows}x{cols}")
        c = merge(c, _check("layernorm", L.layernorm(x, w, None, eps), layernorm_ref(x, w, None, eps),
                            f"layernorm {rows}x{cols} no bias"))
        _report(f"norm fwd {rows}x{cols}", rmsnorm=a, layernorm=c)


@pytest.mark.parametrize("cols", NORM_COLS)
def test_rmsnorm_backward_tiling(L, cols):
    rows_list, rpc, full = _bwd_rows("rmsnorm", cols)
    w = _norm_w(cols, cols)
    for i, rows in enumerate(rows_list):
        eps, add = EPS[i % 2], (i // 2) % 2 == 1
        x, dy = _randn((rows, cols), 3 * rows + cols, 2.0), _randn((rows, cols), 3 * rows + cols + 1)
        a = _randn((rows, cols), 3 * rows + cols + 2) if add else None
        dx, dw = L.rmsnorm_bwd(x, w, dy, eps, add_in=a)
        fx = _by_rows("rmsnorm_bwd", dx, lambda p, q, r: rmsnorm_bwd_ref(p, w, q, eps, r), f"rmsnorm_bwd dx {rows}x{cols}",
                      x, dy, a)
        fw = _check("norm_dw", dw, rmsnorm_dw_ref(x, w, dy, eps), f"rmsnorm_bwd dw {rows}x{cols}")
        _report(f"rmsnorm bwd {rows}x{cols} rpc={rpc} parts={full} add_in={add}", dx=fx, dw=fw)


@pytest.mark.parametrize("cols", LN_BWD_COLS)
def test_layernorm_backward_tiling(L, cols):
    rows_list, rpc, full = _bwd_rows("layernorm", cols)
    w = _norm_w(cols, cols)
    for i, rows in enumerate(rows_list):
        eps, add = EPS[i % 2], (i // 2) % 2 == 1
        x, dy = _randn((rows, cols), 5 * rows + cols, 2.0), _randn((rows, cols), 5 * rows + cols + 1)
        a = _randn((rows, cols), 5 * rows + cols + 2) if add else None
        dx, dw, db = L.layernorm_bwd(x, w, dy, eps, add_in=a)
        fx = _by_rows("layernorm_bwd", dx, lambda p, q, r: layernorm_bwd_ref(p, w, q, eps, r),
                      f"layernorm_bwd dx {rows}x{cols}", x, dy, a)
        rdw, rdb = layernorm_dwdb_ref(x, w, dy, eps)
        fw = _check("norm_dw", dw, rdw, f"layernorm_bwd dw {rows}x{cols}")
        fb = _check("norm_dw", db, rdb, f"layernorm_bwd db {rows}x{cols}")
        _, dw2, db2 = L.layernorm_bwd(x, w, dy, eps, need_dx=False)
        assert torch.equal(dw2, dw) and torch.equal(db2, db)
        _report(f"layernorm bwd {rows}x{cols} rpc={rpc} parts={full} add_in={add}", dx=fx, dw=fw, db=fb)


def test_zero_rows(L):
    """An empty batch: every token-wise entry point returns empty outputs (an empty tensor may have no storage, so its
    data pointer is null) and the parameter gradients come back as zeros."""
    for cols in (8, 1024, 5120):
        x = torch.empty((0, cols), dtype=BF, device="cuda")
        w = _norm_w(cols, 1)
        dx, dw = L.rmsnorm_bwd(x, w, x)
        assert dx.shape == (0, cols) and dw.shape == (cols,) and not bool(dw.any())
        assert L.rmsnorm(x, w).shape == (0, cols)
        dx, dw, db = L.layernorm_bwd(x, w, x)
        assert dx.shape == (0, cols) and not bool(dw.any()) and not bool(db.any())
        assert L.layernorm(x, w, w).shape == (0, cols)
        dy, dls = L.ls_residual_bwd(x, x, w)
        assert dy.shape == (0, cols) and not bool(dls.any())
        assert L.ls_residual(x, x, w, w).shape == (0, cols)
        assert L.bias_gelu(x, w).shape == (0, cols) and L.gelu_bwd(x, x).shape == (0, cols)
        gu = torch.empty((0, 2 * cols), dtype=BF, device="cuda")
        assert L.swiglu(gu).shape == (0, cols) and L.swiglu_bwd(gu, x).shape == (0, 2 * cols)
    cos, sin = L.rope_table(torch.empty(0, dtype=torch.int64, device="cuda"), O.rope_inv_freq(128, 1e6).cuda())
    assert cos.shape == (0, 128)
    assert L.rope(torch.empty((0, 8, 128), dtype=BF, device="cuda"), cos, sin).shape == (0, 8, 128)


# ------------------------------------------------------------------------------------------------
# training shapes
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [18432, 16897])
def test_decoder_rmsnorm_training(L, rows):
    cols, eps = 5120, 1e-6
    x, res, dy = _randn((rows, cols), rows), _randn((rows, cols), rows + 1), _randn((rows, cols), rows + 2)
    w = _norm_w(cols, 3)
    y, s = L.rmsnorm(x, w, eps, residual=res)
    assert torch.equal(s, residual_sum(x, res))
    fy = _by_rows("rmsnorm", y, lambda a, b: rmsnorm_ref(a, w, eps, b), "rmsnorm fwd", x, res)
    dx, dw = L.rmsnorm_bwd(s, w, dy, eps, add_in=res)
    fx = _by_rows("rmsnorm_bwd", dx, lambda p, q, r: rmsnorm_bwd_ref(p, w, q, eps, r), "rmsnorm dx", s, dy, res)
    fw = _check("norm_dw", dw, rmsnorm_dw_ref(s, w, dy, eps), "rmsnorm dw")
    _report(f"decoder rmsnorm {rows}x{cols}", fwd=fy, dx=fx, dw=fw)


@pytest.mark.parametrize("name,rows,cols,eps", [("vit", VIT_ROWS, 1024, 1e-6), ("projector", 16384, 4096, 1e-5),
                                                ("siglip", 16 * 729, 1152, 1e-6)])
def test_vision_layernorm_training(L, name, rows, cols, eps):
    x, dy, a = _randn((rows, cols), rows, 2.0), _randn((rows, cols), rows + 1), _randn((rows, cols), rows + 2)
    w, b = _norm_w(cols, 4), _randn((cols,), 5, 0.1)
    fy = _by_rows("layernorm", L.layernorm(x, w, b, eps), lambda t: layernorm_ref(t, w, b, eps), "layernorm fwd", x)
    dx, dw, db = L.layernorm_bwd(x, w, dy, eps, add_in=a)
    fx = _by_rows("layernorm_bwd", dx, lambda p, q, r: layernorm_bwd_ref(p, w, q, eps, r), "layernorm dx", x, dy, a)
    rdw, rdb = layernorm_dwdb_ref(x, w, dy, eps)
    fw, fb = _check("norm_dw", dw, rdw, "layernorm dw"), _check("norm_dw", db, rdb, "layernorm db")
    _report(f"{name} layernorm {rows}x{cols}", fwd=fy, dx=fx, dw=fw, db=fb)


def test_swiglu_training(L):
    rows, inter = 18432, 13824
    gu, dh = _randn((rows, 2 * inter), 1, 2.0), _randn((rows, inter), 2)
    fy = _by_rows("swiglu", L.swiglu(gu), swiglu_ref, "swiglu fwd", gu)
    fb = _by_rows("swiglu_bwd", L.swiglu_bwd(gu, dh), swiglu_bwd_ref, "swiglu bwd", gu, dh)
    _report(f"swiglu {rows}x{inter}", fwd=fy, bwd=fb)


@pytest.mark.parametrize("approx", ["none", "tanh"])
def test_gelu_training(L, approx):
    rows, cols = VIT_ROWS, 4096
    x, b, dy = _randn((rows, cols), 3, 2.0), _randn((cols,), 4, 0.5), _randn((rows, cols), 5)
    fy = _by_rows("gelu", L.bias_gelu(x, b, approx), lambda t: bias_gelu_ref(t, b, approx), f"gelu {approx}", x)
    fb = _by_rows("gelu_bwd", L.gelu_bwd(x, dy, approx), lambda p, d: gelu_bwd_ref(p, d, approx), f"gelu_bwd {approx}",
                  x, dy)
    _report(f"gelu {approx} {rows}x{cols}", fwd=fy, bwd=fb)


def test_layer_scale_residual_training(L):
    rows, cols = VIT_ROWS, 1024
    x, y, dout = _randn((rows, cols), 6), _randn((rows, cols), 7), _randn((rows, cols), 8)
    ls, b = _randn((cols,), 9, 0.1), _randn((cols,), 10, 0.5)
    fy = _by_rows("exact", L.ls_residual(x, y, ls, b), lambda p, q: ls_residual_ref(p, q, ls, b), "ls_residual", x, y)
    fy = merge(fy, _by_rows("exact", L.ls_residual(x, y, ls), lambda p, q: ls_residual_ref(p, q, ls), "ls_residual",
                            x, y))
    dy, dls = L.ls_residual_bwd(dout, y, ls)
    rdy, rdls = ls_residual_bwd_ref(dout, y, ls)
    fd = _check("exact", dy, rdy, "ls_residual_bwd dy")
    fl = _check("norm_dw", dls, rdls, "ls_residual_bwd dls")
    _report(f"ls_residual {rows}x{cols}", fwd=fy, dy=fd, dls=fl)


def test_rope_on_fused_qkv_views(L):
    """The decoder's prefill: q [T, 40, 128] and k [T, 8, 128] are views of the QKV GEMM output [T, 56 x 128],
    rotated in place; v stays untouched."""
    T, hq, hkv, d = 18432, 40, 8, 128
    qkv = _randn((T, (hq + 2 * hkv) * d), 11)
    before = qkv.clone()
    pos = torch.arange(T, device="cuda")
    cos, sin = L.rope_table(pos, O.rope_inv_freq(d, 1e6).cuda())
    q, k = qkv[:, : hq * d].view(T, hq, d), qkv[:, hq * d : (hq + hkv) * d].view(T, hkv, d)
    L.rope(q, cos, sin, out=q)
    L.rope(k, cos, sin, out=k)
    fq = _check("exact", q, rope_ref(before[:, : hq * d].view(T, hq, d), cos, sin), "rope q")
    fk = _check("exact", k, rope_ref(before[:, hq * d : (hq + hkv) * d].view(T, hkv, d), cos, sin), "rope k")
    assert torch.equal(qkv[:, (hq + hkv) * d :], before[:, (hq + hkv) * d :])
    _report(f"rope fused qkv T={T}", q=fq, k=fk)


# ------------------------------------------------------------------------------------------------
# numerical edges
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cols", [1024, 5120])
def test_norm_numerical_edges(L, cols):
    """The rows of tokenwise_ref.edge_rows, each group checked as a tensor of its own: zero rows (RMSNorm gives 0,
    LayerNorm b), rows of magnitude 1e-3 where eps dominates, an outlier channel at 1e4 among ones, ordinary rows and
    rows of 40 +- 0.5 (a one-pass E[x^2] - E[x]^2 variance flips several per cent of their roundings)."""
    w, b = _norm_w(cols, 1), _randn((cols,), 2, 0.1)
    for eps in EPS:
        seed = [3 * cols]

        def randn(shape, scale, mean):
            seed[0] += 1
            return _randn(shape, seed[0], scale, mean)

        x = edge_rows(cols, randn, "cuda")
        dy, a = _randn(x.shape, 4), _randn(x.shape, 5)
        y, yl = L.rmsnorm(x, w, eps), L.layernorm(x, w, b, eps)
        assert not bool(y[:8].any()) and torch.equal(yl[:8], b.expand(8, cols))
        dx, dw = L.rmsnorm_bwd(x, w, dy, eps, add_in=a)
        dxl, dwl, dbl = L.layernorm_bwd(x, w, dy, eps, add_in=a)
        figs = {}
        for group, sl in edge_groups():
            xs, dys, As = x[sl], dy[sl], a[sl]
            figs[group] = {
                "rmsnorm": _check("rmsnorm", y[sl], rmsnorm_ref(xs, w, eps), f"rmsnorm {group} rows"),
                "layernorm": _check(edge_op("layernorm", group), yl[sl], layernorm_ref(xs, w, b, eps),
                                    f"layernorm {group} rows"),
                "rms_dx": _check("rmsnorm_bwd", dx[sl], rmsnorm_bwd_ref(xs, w, dys, eps, As), f"rmsnorm_bwd {group} rows"),
                "ln_dx": _check(edge_op("layernorm_bwd", group), dxl[sl], layernorm_bwd_ref(xs, w, dys, eps, As),
                                f"layernorm_bwd {group} rows")}
        rdw, rdb = layernorm_dwdb_ref(x, w, dy, eps)
        figs.update(rms_dw=_check("norm_dw", dw, rmsnorm_dw_ref(x, w, dy, eps), "rmsnorm_bwd edges dw"),
                    ln_dw=_check("norm_dw", dwl, rdw, "layernorm_bwd edges dw"),
                    ln_db=_check("norm_dw", dbl, rdb, "layernorm_bwd edges db"))
        _report(f"norm edges {cols} eps={eps}", **figs)


def test_activations_across_the_expf_overflow_range(L):
    """Gate / pre-activation values on a grid over [-120, 120] (e^-g overflows fp32 below -88.7, __fdividef's
    denominator passes 2^126 below -87.3): every output finite and within its bound."""
    rows, cols = 48, 1024
    grid = torch.linspace(-120, 120, rows * cols, device="cuda").view(rows, cols)
    g = grid.to(BF)
    u, dy = _randn((rows, cols), 1), _randn((rows, cols), 2)
    gu = torch.cat([g, u], 1)
    fs = _check("swiglu", L.swiglu(gu), swiglu_ref(gu), "swiglu sweep")
    fsb = _check("swiglu_bwd", L.swiglu_bwd(gu, dy), swiglu_bwd_ref(gu, dy), "swiglu_bwd sweep")
    figs = {"swiglu": fs, "swiglu_bwd": fsb}
    for approx in ("none", "tanh"):
        figs[f"gelu {approx}"] = _check("gelu", L.bias_gelu(g, None, approx), bias_gelu_ref(g, None, approx),
                                        f"gelu {approx} sweep")
        figs[f"gelu_bwd {approx}"] = _check("gelu_bwd", L.gelu_bwd(g, dy, approx), gelu_bwd_ref(g, dy, approx),
                                            f"gelu_bwd {approx} sweep")
    _report("activation sweep [-120, 120]", **figs)


# ------------------------------------------------------------------------------------------------
# RoPE
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("heads", [40, 8, 5, 6, 3, 1])
def test_rope_head_groupings(L, heads, d):
    """heads % 8 == 0 -> 8 heads per thread, % 5 -> 5, % 2 -> 2, else 1.  In place in a view of a wider buffer, and
    through a strided output; nothing outside the views is written."""
    n, fill = 777, 3.0
    buf = torch.full((n, heads + 2, d + 16), fill, dtype=BF, device="cuda")
    x = buf[:, 1 : heads + 1, 8 : d + 8]
    x.copy_(_randn((n, heads, d), heads * d))
    x0 = x.clone()
    pos = torch.randint(0, 1 << 17, (n,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(d))
    cos, sin = L.rope_table(pos, O.rope_inv_freq(d, 1e6).cuda())
    ref = rope_ref(x0, cos, sin)
    obuf = torch.full((n, heads + 3, d + 8), fill, dtype=BF, device="cuda")
    out = obuf[:, 2 : heads + 2, :d]
    L.rope(x, cos, sin, out=out)
    fo = _check("exact", out, ref, f"rope strided out heads={heads} d={d}")
    check_untouched(obuf, out, fill, "rope out")
    assert torch.equal(x, x0)
    L.rope(x, cos, sin, out=x)
    fi = _check("exact", x, ref, f"rope in place heads={heads} d={d}")
    check_untouched(buf, x, fill, "rope in place")
    # autograd: the backward is the same kernel with -sin
    xg = x0.clone().requires_grad_(True)
    dy = _randn((n, heads, d), heads * d + 1)
    L.rope_autograd(xg, cos, sin).backward(dy)
    assert torch.equal(xg.grad, L.rope(dy, cos, -sin))
    fb = _check("rope_bwd", xg.grad, rope_bwd_ref(dy, cos, sin), f"rope bwd heads={heads} d={d}")
    _report(f"rope heads={heads} d={d}", out=fo, in_place=fi, bwd=fb)


def test_rope_table_positions(L):
    """Positions 0 .. 131 071 and the zig-zag positions of rank 5 of cp = 8 at a 1M-token context (angles up to 1e6
    radians in fp32)."""
    d = 128
    inv = O.rope_inv_freq(d, 1e6).cuda()
    figs = {}
    for name, pos in (("0..131071", torch.arange(1 << 17)), ("zigzag cp=8 rank 5", O.zigzag_positions(1 << 20, 8, 5))):
        pos = pos.cuda()
        cos, sin = L.rope_table(pos, inv)
        assert torch.equal(cos[:, : d // 2], cos[:, d // 2 :]) and torch.equal(sin[:, : d // 2], sin[:, d // 2 :])
        rc, rs = rope_table_ref(pos, inv)
        figs[name] = {"cos": _check("rope_table", cos[:, : d // 2], rc, f"cos {name}"),
                      "sin": _check("rope_table", sin[:, : d // 2], rs, f"sin {name}")}
    _report("rope_table", **figs)


# ------------------------------------------------------------------------------------------------
# flash-decoding merge
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("G,hkv", [(5, 8), (1, 1)])
@pytest.mark.parametrize("n", [1, 2, 150, 1000])
def test_decode_merge(L, n, G, hkv, d):
    """lse uniform over [-80, 80]; one split at -inf (n > 1), and for G hkv > 1 one head with every split at -inf."""
    gen = torch.Generator(device="cuda").manual_seed(n * 100 + G * 10 + d)
    o = _randn((n, G, hkv, d), n + d, 2.0)
    lse = torch.rand((n, hkv, G), generator=gen, device="cuda") * 160 - 80
    if n > 1:
        lse[n // 2] = -math.inf
    if G * hkv > 1:
        lse[:, hkv - 1, G - 1] = -math.inf
    out, lse_out = L.decode_merge(o, lse, return_lse=True)
    ref, Lr, bound = decode_merge_ref(o, lse)
    f = _check("decode_merge", out, ref, f"decode_merge n={n} G={G} hkv={hkv} d={d}")
    empty = torch.isneginf(Lr)
    assert bool(torch.isneginf(lse_out[empty]).all()) and not bool(out[empty].any())
    err = (lse_out.double() - Lr).abs()[~empty]
    ratio = float((err / bound[~empty]).max()) if err.numel() else 0.0
    assert ratio <= 1.0, ratio
    _report(f"decode_merge n={n} G={G} hkv={hkv} d={d}", out=f, lse_ratio=ratio, lse_err=float(err.max()))


# ------------------------------------------------------------------------------------------------
# determinism, 64-bit offsets
# ------------------------------------------------------------------------------------------------
def test_norm_backward_is_bit_reproducible(L):
    for rows, cols in ((18432, 5120), (VIT_ROWS, 1024)):
        x, dy, a = _randn((rows, cols), 1), _randn((rows, cols), 2), _randn((rows, cols), 3)
        w = _norm_w(cols, 4)
        r0, r1 = L.rmsnorm_bwd(x, w, dy, add_in=a), L.rmsnorm_bwd(x, w, dy, add_in=a)
        assert all(torch.equal(p, q) for p, q in zip(r0, r1))
        l0, l1 = L.layernorm_bwd(x, w, dy, add_in=a), L.layernorm_bwd(x, w, dy, add_in=a)
        assert all(torch.equal(p, q) for p, q in zip(l0, l1))


def _sampled_rows(rows, k=64):
    return [(0, k), (rows // 2 - k // 2, rows // 2 + k // 2), (rows - k, rows)]


def test_beyond_2_31_elements(L):
    """SwiGLU on gate_up [80 000, 27 648] (2.2e9 elements) and RMSNorm on [425 984, 5120] (2.18e9): rows at the start,
    middle and end against the reference."""
    rows, inter = 80000, 13824
    gu = _randn((rows, 2 * inter), 1, 2.0)
    assert gu.numel() > 2 ** 31
    y = L.swiglu(gu)
    figs = {}
    for r0, r1 in _sampled_rows(rows):
        figs[f"swiglu rows {r0}"] = _check("swiglu", y[r0:r1], swiglu_ref(gu[r0:r1]), f"swiglu rows {r0}..{r1}")
    del gu, y
    torch.cuda.empty_cache()
    rows, cols = 425984, 5120
    x = _randn((rows, cols), 2)
    assert x.numel() > 2 ** 31
    w = _norm_w(cols, 3)
    y = L.rmsnorm(x, w)
    for r0, r1 in _sampled_rows(rows):
        figs[f"rmsnorm rows {r0}"] = _check("rmsnorm", y[r0:r1], rmsnorm_ref(x[r0:r1], w, 1e-6), f"rmsnorm rows {r0}..{r1}")
    _report("beyond 2^31", **figs)
