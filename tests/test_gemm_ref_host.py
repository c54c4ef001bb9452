"""Pins the float64 GEMM reference and its checker (tests/gemm_ref.py) on the CPU, before any GPU test relies on them:
the reference equals a plain fp64 product with each epilogue's rounding order, slabbing does not change it, the checker
accepts bf16(ref) and an fp32-accumulated product, and it rejects each kind of wrong result a kernel could produce,
built here from correct data."""
import pytest
import torch
import torch.nn.functional as F

from tests.gemm_ref import bf16r, check_gemm, check_untouched, gemm_ref, ulp_bf16
from tests.util import randn_bf16, seeded

ACTS = [None, "gelu", "gelu_tanh", "swiglu"]


def _inputs(M, N, K, seed, with_bias):
    g = seeded(seed)
    a = randn_bf16((M, K), g)
    w = randn_bf16((N, K), g, K ** -0.5)
    b = randn_bf16((N,), g, 0.5) if with_bias else None
    return a, w, b


def _plain_fp64(a, w, b, act):
    y = a.double() @ w.double().t()
    if b is not None:
        y = y + b.double()
    if act == "swiglu":
        g = y[:, 0::2].to(torch.bfloat16).double()
        u = y[:, 1::2].to(torch.bfloat16).double()
        return F.silu(g).to(torch.bfloat16).double() * u
    if act:
        return F.gelu(y.to(torch.bfloat16).double(), approximate="tanh" if act == "gelu_tanh" else "none")
    return y


@pytest.mark.parametrize("act,with_bias", [(act, wb) for act in ACTS for wb in (False, True)
                                            if not (act == "swiglu" and wb)])     # the fused SwiGLU takes no bias
def test_reference_is_the_fp64_product_with_the_epilogue_rounding_order(act, with_bias):
    a, w, b = _inputs(70, 200, 136, seed=1, with_bias=with_bias)
    r = gemm_ref(a, w, b, act)
    assert r.dtype == torch.float64 and r.shape == (70, 100 if act == "swiglu" else 200)
    torch.testing.assert_close(r, _plain_fp64(a, w, b, act), rtol=1e-14, atol=1e-14)


def test_reference_post_add_rounds_the_product_first():
    a, w, b = _inputs(40, 64, 72, seed=2, with_bias=True)
    pos = randn_bf16((40, 64), seeded(3))
    want = (a.double() @ w.double().t() + b.double()).to(torch.bfloat16).double() + pos.double()
    torch.testing.assert_close(gemm_ref(a, w, b, post=pos), want, rtol=0, atol=0)


@pytest.mark.parametrize("act", [None, "swiglu"])
def test_slabbing_does_not_change_the_result(act):
    a, w, b = _inputs(300, 512, 200, seed=4, with_bias=act is None)
    whole = gemm_ref(a, w, b, act)
    # slabs of 128 columns x a few rows
    slabbed = gemm_ref(a, w, b, act, slab_bytes=8 * (2 * 128 * 200 + 5 * (200 + 128)))
    torch.testing.assert_close(slabbed, whole, rtol=1e-14, atol=1e-14)
    # transposed (MN-major) views in, as the backward checks pass them
    torch.testing.assert_close(gemm_ref(a.t().contiguous().t(), w.t().contiguous().t(), b, act), whole, rtol=1e-14,
                               atol=1e-14)


def test_ulp_bf16():
    x = torch.tensor([1.0, 1.5, -2.0, 0.75, 3.0e-3, 0.0], dtype=torch.float64)
    want = torch.tensor([2.0 ** -7, 2.0 ** -7, 2.0 ** -6, 2.0 ** -8, 2.0 ** -16, 2.0 ** -133], dtype=torch.float64)
    assert torch.equal(ulp_bf16(x), want)


@pytest.mark.parametrize("act", ACTS)
def test_checker_accepts_rounded_reference_and_fp32_accumulation(act):
    a, w, b = _inputs(200, 640, 1024, seed=5, with_bias=act != "swiglu")
    r = gemm_ref(a, w, b, act)
    res = check_gemm(r.to(torch.bfloat16), r, a, w, b, act)
    assert res["chunk_excess"] == 0.0 and res["mismatch"] == 0.0 and res["max_ulps"] <= 1.0
    # an fp32-accumulated product with the kernel's epilogue arithmetic in fp32
    y = a.float() @ w.float().t() + (0 if b is None else b.float())
    if act == "swiglu":
        gt, ut = y[:, 0::2].bfloat16().float(), y[:, 1::2].bfloat16().float()
        y = F.silu(gt).bfloat16().float() * ut
    elif act:
        y = F.gelu(y.bfloat16().float(), approximate="tanh" if act == "gelu_tanh" else "none")
    res = check_gemm(y.bfloat16(), r, a, w, b, act)
    assert res["chunk_excess"] < 2e-4, res


# ------------------------------------------------------------------------------------------------
# rejections: each corruption is built on the CPU from correct data
# ------------------------------------------------------------------------------------------------
def test_rejects_a_zeroed_chunk():
    a, w, b = _inputs(192, 320, 256, seed=6, with_bias=True)
    r = gemm_ref(a, w, b)
    y = r.to(torch.bfloat16)
    y[64:128, 128:192] = 0
    with pytest.raises(AssertionError, match="chunk excess"):
        check_gemm(y, r, a, w, b)


def test_rejects_one_k_block_left_out_of_one_tile():
    """K = 18 432: one 64-wide k-block of the 128 x 256 tile (1, 1) is missing, about sqrt(64 / K) = 6e-2 of each
    of the tile's chunks."""
    M, N, K = 256, 512, 18432
    a, w, _ = _inputs(M, N, K, seed=7, with_bias=False)
    r = gemm_ref(a, w)
    rows, cols, kb = slice(128, 256), slice(256, 512), slice(64 * 100, 64 * 101)
    y = r.clone()
    y[rows, cols] -= a[rows, kb].double() @ w[cols, kb].double().t()
    # the worst chunk named is one of the tile's eight
    with pytest.raises(AssertionError, match=r"chunk excess .* at output rows/cols \((128|192), (256|320|384|448)\)"):
        check_gemm(y.to(torch.bfloat16), r, a, w)


def test_rejects_columns_shifted_inside_one_tile():
    a, w, b = _inputs(128, 512, 512, seed=8, with_bias=True)
    r = gemm_ref(a, w, b)
    y = r.to(torch.bfloat16)
    y[:, 256:512] = torch.roll(y[:, 256:512], 8, dims=1)
    with pytest.raises(AssertionError, match="chunk excess"):
        check_gemm(y, r, a, w, b)


def test_rejects_one_element_three_ulps_off_where_the_bound_is_one():
    """At K = 64 the accumulation term K 2^-23 |a||w| is far below one ulp, so the bound is about one ulp.  A single
    element is invisible to the per-chunk norm; the elementwise check names it."""
    a, w, b = _inputs(128, 256, 64, seed=9, with_bias=False)
    r = gemm_ref(a, w, b)
    y = r.to(torch.bfloat16)
    i, j = 77, 131
    assert float(64 * 2.0 ** -23 * (a[i].double().abs() @ w[j].double().abs())) < 0.01 * float(ulp_bf16(r[i, j]))
    y[i, j] = (r[i, j] + 3 * ulp_bf16(r[i, j])).to(torch.bfloat16)
    with pytest.raises(AssertionError, match=r"elementwise .* at \(77, 131\)"):
        check_gemm(y, r, a, w, b)


def test_rejects_one_nan():
    a, w, b = _inputs(100, 264, 128, seed=10, with_bias=True)
    r = gemm_ref(a, w, b, "gelu")
    y = r.to(torch.bfloat16)
    y[99, 263] = float("nan")
    with pytest.raises(AssertionError, match="finite"):
        check_gemm(y, r, a, w, b, "gelu")


def test_rejects_a_wrong_bias_column():
    a, w, b = _inputs(130, 264, 128, seed=11, with_bias=True)
    r = gemm_ref(a, w, b)
    wrong = b.clone()
    wrong[200] += 0.25
    y = gemm_ref(a, w, wrong).to(torch.bfloat16)
    with pytest.raises(AssertionError, match="chunk excess|elementwise"):
        check_gemm(y, r, a, w, b)


def test_floor_factor_and_partial_rounding_are_what_widen_a_sum_of_rounded_partials():
    """d_sel of the LM head is an fp32 sum of bf16-rounded per-chunk products; the checker accepts it with the floor
    and the elementwise term that account for those roundings."""
    a, w, _ = _inputs(128, 256, 2048, seed=12, with_bias=False)
    r = gemm_ref(a, w)
    y = sum(bf16r(a[:, k0 : k0 + 512].double() @ w[:, k0 : k0 + 512].double().t()) for k0 in range(0, 2048, 512))
    y = y.float().bfloat16()
    res = check_gemm(y, r, a, w, floor_factor=2.0, partial_rounding=2.0 ** -8)
    assert res["chunk_excess"] < 1e-3


def test_check_untouched():
    buf = torch.full((4, 24), 7.0, dtype=torch.bfloat16)
    buf[:, :16] = 1
    check_untouched(buf, 16, 7.0)
    buf[3, 16] = 0
    with pytest.raises(AssertionError, match="wrote past"):
        check_untouched(buf, 16, 7.0)


@pytest.mark.parametrize("act", ACTS + ["post"])
def test_elementwise_bound_is_the_same_gathered_or_recomputed_by_rows(act):
    """check_gemm computes the bound of few flagged elements from gathered rows and columns, of many from whole output
    rows recomputed as products: both give the same numbers."""
    from tests.gemm_ref import _elem_bound

    a, w, b = _inputs(150, 384, 200, seed=13, with_bias=act != "swiglu")
    pos = randn_bf16((150, 384), seeded(14)) if act == "post" else None
    r = gemm_ref(a, w, b, None if act == "post" else act, post=pos)
    g = seeded(15)
    ii = torch.randint(0, 150, (500,), generator=g).sort().values
    jj = torch.randint(0, r.shape[1], (500,), generator=g)
    gathered = _elem_bound(ii, jj, r, a, w, b, act, 0.0, dense=False)
    by_rows = _elem_bound(ii, jj, r, a, w, b, act, 0.0, dense=True, dense_bytes=8 * (4 * 128 * 200 + 2 * 400 + 7 * 656))
    torch.testing.assert_close(by_rows, gathered, rtol=1e-12, atol=0)
