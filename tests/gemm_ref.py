"""Float64 reference and per-chunk checker for the wgmma GEMM (`lv_gemm_bias_act` / `lv_gemm_ex`, `ops.linear`).

`gemm_ref(a, w, bias, act, post)` computes, on the device of its inputs, in float64,

    pre = a w^T (+ bias)                                    a [M, K], w [N, K], any float dtype and any strides
    plain:       r = pre
    gelu / tanh: r = gelu(bf16(pre))                        nn.Linear rounds its output before the activation
    swiglu:      r = bf16(silu(bf16(g))) * bf16(u)          (g, u) = columns (2i, 2i + 1) of pre, N / 2 outputs
    post:        r = bf16(pre) + post                       the patch embedding: bf16(bf16(conv + b) + pos)

and returns r, the value before the final rounding to bf16 (so a caller can compute the rounding floor).  The product
runs in slabs of rows and columns so that one slab's float64 operands and output stay within `slab_bytes`.

`check_gemm(y, ref, a, w, ...)` asserts, for a bf16 result y of that GEMM,
  1. every element of y is finite;
  2. per 64 x 64 output chunk (the epilogue's TMA store unit, aligned to the output; for SwiGLU the N / 2 output
     columns), the error in excess of the bf16 rounding floor
         excess = sqrt(max(0, |y - r|^2 - floor_factor * |bf16(r) - r|^2)) / |r|
     is below `chunk_bound` (1e-3).  With iid operands one 64-wide k-block left out of a tile costs about
     sqrt(64 / K) of a chunk (3e-2 at K = 65 600), a zeroed or shifted chunk about 1;
  3. elementwise |y - r| <= ulp_bf16(r) + D, where, with E = (K 2^-23 + partial_rounding) (|a| |w|^T)_ij the worst
     case of the fp32 accumulation (truncating adds included) and of any bf16 rounding of partial products:
         plain:       D = E
         gelu / tanh: D = 1.13 (ulp_bf16(pre) + E)          max |gelu'| < 1.13: bf16(pre) may round the other way
         post:        D = ulp_bf16(pre) + E
         swiglu:      D = 1.01 (|bf16 u| (ulp_bf16(s) + 1.1 (ulp_bf16(g) + E_g)) + |s| (ulp_bf16(u) + E_u)),
                      s = silu(bf16 g), max |silu'| < 1.1.
     This catches NaN, misplaced columns and garbage in clipped tails, not subtle errors (at K = 5120, E is several
     ulps).  |a| |w|^T is computed only for the elements that exceed one ulp, from their gathered rows and columns.
It returns the worst figures: chunk excess and where, the worst elementwise |y - r| / bound, the whole-tensor excess
and the fraction of elements where y != bf16(r).

`check_untouched(buf, n_valid, fill)` asserts that a strided output (ldc > N) kept `fill` past its valid columns.
"""
import math
from typing import Optional

import torch
import torch.nn.functional as F

f64 = torch.float64
CHUNK = 64
GELU_LIP = 1.13      # max |d/dx gelu(x)| = 1.1289 (erf), 1.1295 (tanh form)
SILU_LIP = 1.1       # max |d/dx silu(x)| = 1.0998


def bf16r(x: torch.Tensor) -> torch.Tensor:
    """x rounded to bf16 (round to nearest even), back in float64."""
    return x.to(torch.bfloat16).to(f64)


def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """The bf16 unit in the last place at |x| (8 significant bits), float64; 2^-133 (the smallest subnormal) at 0."""
    _, e = torch.frexp(x.to(f64))
    u = torch.ldexp(torch.ones_like(x, dtype=f64), (e - 8).clamp_min(-133))
    return torch.where(x == 0, torch.full_like(u, 2.0 ** -133), u)


def _epilogue(pre: torch.Tensor, act: Optional[str], post: Optional[torch.Tensor]) -> torch.Tensor:
    if act == "swiglu":
        return bf16r(F.silu(bf16r(pre[:, 0::2]))) * bf16r(pre[:, 1::2])
    if act in ("gelu", "gelu_tanh"):
        return F.gelu(bf16r(pre), approximate="tanh" if act == "gelu_tanh" else "none")
    assert act is None, act
    if post is not None:
        return bf16r(pre) + post.to(f64)
    return pre


def gemm_ref(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, act: Optional[str] = None,
             post: Optional[torch.Tensor] = None, *, slab_bytes: int = 2 << 30) -> torch.Tensor:
    """float64 r [M, N] (N / 2 for swiglu) of the module docstring.  `post` [M, N] is added after a bf16 rounding."""
    M, K = a.shape
    N = w.shape[0]
    assert w.shape[1] == K and (act != "swiglu" or (N % 2 == 0 and bias is None and post is None))
    assert post is None or act is None
    budget = max(1, slab_bytes // 8)
    nc = N if N * K <= budget // 2 else max(128, budget // 2 // K // 128 * 128)
    mr = max(1, (budget - nc * K) // (K + nc))
    n_out = N // 2 if act == "swiglu" else N
    out = torch.empty((M, n_out), dtype=f64, device=a.device)
    b64 = None if bias is None else bias.to(f64)
    for n0 in range(0, N, nc):
        n1 = min(N, n0 + nc)
        wt = w[n0:n1].to(f64).t()
        o0, o1 = (n0 // 2, n1 // 2) if act == "swiglu" else (n0, n1)
        for m0 in range(0, M, mr):
            m1 = min(M, m0 + mr)
            pre = a[m0:m1].to(f64) @ wt
            if b64 is not None:
                pre += b64[n0:n1]
            out[m0:m1, o0:o1] = _epilogue(pre, act, None if post is None else post[m0:m1, n0:n1])
            del pre
        del wt
    return out


def _chunk_sums(x: torch.Tensor) -> torch.Tensor:
    """x [m, n] -> sums of x^2 over the 64 x 64 chunks [ceil(m / 64), ceil(n / 64)]."""
    m, n = x.shape
    x = F.pad(x * x, (0, -n % CHUNK, 0, -m % CHUNK))
    return x.view(x.shape[0] // CHUNK, CHUNK, x.shape[1] // CHUNK, CHUNK).sum((1, 3))


def _bound(rij, pre, absd, act):
    """ulp_bf16(r) + D of check 3, given the fp64 pre-activation(s) and accumulation term(s) of the elements."""
    if act == "swiglu":
        (g, u), (eg, eu) = pre, absd
        s = bf16r(F.silu(bf16r(g)))
        d = 1.01 * (bf16r(u).abs() * (ulp_bf16(s) + SILU_LIP * (ulp_bf16(g) + eg)) + s.abs() * (ulp_bf16(u) + eu))
    elif act in ("gelu", "gelu_tanh"):
        d = GELU_LIP * (ulp_bf16(pre[0]) + absd[0])
    elif act == "post":
        d = ulp_bf16(pre[0]) + absd[0]
    else:
        d = absd[0]
    return ulp_bf16(rij) + d


def _elem_bound(ii, jj, r, a, w, bias, act, partial_rounding, batch_bytes=1 << 28, dense_bytes=2 << 30, dense=None):
    """Elementwise bounds (module docstring, check 3) at the output elements (ii, jj), float64.  Few elements: their
    rows of a and columns of w are gathered.  Many: the flagged rows' whole output rows are recomputed as fp64 products
    (a [R, K] . w^T and |a| . |w|^T), which costs less than gathering K-long vectors per element."""
    K, N = a.shape[1], w.shape[0]
    eps = K * 2.0 ** -23 + partial_rounding
    out = torch.empty(ii.numel(), dtype=f64, device=r.device)
    b64 = None if bias is None else bias.to(f64)
    pair = act == "swiglu"
    rows_u = torch.unique(ii)
    if not (dense if dense is not None else 64 * ii.numel() >= rows_u.numel() * N):
        step = max(1, batch_bytes // (8 * K * (2 if pair else 1)))
        for s0 in range(0, ii.numel(), step):
            i, j = ii[s0 : s0 + step], jj[s0 : s0 + step]
            ai = a[i].to(f64)
            pre, absd = [], []
            for c in ([2 * j, 2 * j + 1] if pair else [j]):
                wc = w[c].to(f64)
                pre.append((ai * wc).sum(1) + (0 if b64 is None else b64[c]))
                absd.append(eps * (ai.abs() * wc.abs()).sum(1))
                del wc
            out[s0 : s0 + step] = _bound(r[i, j], pre, absd, act)
            del ai
        return out
    # ii is sorted (row-major scan); slabs of w rows outside, slabs of the flagged rows of a inside
    budget = dense_bytes // 8
    nc = N if N * K <= budget // 4 else max(128, budget // 4 // K // 128 * 128)
    rs = max(1, (budget - 2 * nc * K) // (2 * K + 2 * nc))
    cols = torch.stack([2 * jj, 2 * jj + 1] if pair else [jj])             # [1 or 2, n_flag] rows of w
    pre_v = torch.empty(cols.shape, dtype=f64, device=r.device)
    abs_v = torch.empty_like(pre_v)
    for n0 in range(0, N, nc):
        wt = w[n0 : n0 + nc].to(f64).t()
        wta = wt.abs()
        for u0 in range(0, rows_u.numel(), rs):
            R = rows_u[u0 : u0 + rs]
            lo, hi = int(torch.searchsorted(ii, R[0])), int(torch.searchsorted(ii, R[-1], right=True))
            loc = torch.searchsorted(R, ii[lo:hi])
            ar = a[R].to(f64)
            P, A = ar @ wt, ar.abs() @ wta
            for t in range(cols.shape[0]):
                c = cols[t, lo:hi]
                m = (c >= n0) & (c < n0 + nc)
                e = lo + torch.nonzero(m).view(-1)
                pre_v[t, e] = P[loc[m], c[m] - n0]
                abs_v[t, e] = A[loc[m], c[m] - n0]
            del ar, P, A
        del wt, wta
    if b64 is not None:
        pre_v += b64[cols]
    return _bound(r[ii, jj], list(pre_v), list(eps * abs_v), act)


def check_gemm(y: torch.Tensor, ref: torch.Tensor, a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None,
               act: Optional[str] = None, *, chunk_bound: float = 1e-3, floor_factor: float = 1.0,
               partial_rounding: float = 0.0, name: str = "", rows_per_slab: int = 0, elementwise: bool = True) -> dict:
    """Checks 1-3 of the module docstring for y [M, N_out] (a view; only its valid columns) against r = `ref` of
    gemm_ref(a, w, bias, act).  act "post" marks the patch-embedding epilogue (gemm_ref with `post`).  Returns the
    worst figures.  With chunk_bound=inf and elementwise=False it only measures (a yardstick such as cuBLAS)."""
    M, n = y.shape
    assert ref.shape == (M, n), (ref.shape, y.shape)
    assert bool(torch.isfinite(y).all()), f"{name}: finite: {int((~torch.isfinite(y)).sum())} non-finite elements"
    rows = rows_per_slab or max(CHUNK, (1 << 25) // max(1, n) // CHUNK * CHUNK)
    nm, nn = -(-M // CHUNK), -(-n // CHUNK)
    dd = torch.zeros((nm, nn), dtype=f64, device=y.device)
    ee, rr = torch.zeros_like(dd), torch.zeros_like(dd)
    flag_i, flag_j, worst_ulps = [], [], torch.zeros((), dtype=f64, device=y.device)
    mismatched = 0
    for r0 in range(0, M, rows):
        r1 = min(M, r0 + rows)
        rs = ref[r0:r1]
        d = y[r0:r1].to(f64) - rs
        e = bf16r(rs) - rs
        c0 = r0 // CHUNK
        dd[c0 : c0 + -(-(r1 - r0) // CHUNK)] += _chunk_sums(d)
        ee[c0 : c0 + -(-(r1 - r0) // CHUNK)] += _chunk_sums(e)
        rr[c0 : c0 + -(-(r1 - r0) // CHUNK)] += _chunk_sums(rs)
        mismatched += int((e != d).sum())
        ulps = d.abs() / ulp_bf16(rs)
        worst_ulps = torch.maximum(worst_ulps, ulps.max())
        fi, fj = torch.nonzero(ulps > 1.0, as_tuple=True)
        flag_i.append(fi + r0)
        flag_j.append(fj)
        del d, e, ulps
    excess = (dd - floor_factor * ee).clamp_min(0).sqrt() / rr.sqrt()
    excess = torch.where(rr > 0, excess, torch.where(dd > 0, torch.full_like(dd, math.inf), torch.zeros_like(dd)))
    k = int(excess.argmax())
    worst = float(excess.view(-1)[k])
    at = (k // nn * CHUNK, k % nn * CHUNK)
    total = math.sqrt(max(0.0, float(dd.sum() - floor_factor * ee.sum()))) / math.sqrt(max(float(rr.sum()), 1e-300))
    assert worst < chunk_bound, (f"{name}: chunk excess {worst:.3e} >= {chunk_bound:.1e} at output rows/cols {at} "
                                 f"(whole tensor {total:.3e})")
    ii, jj = torch.cat(flag_i), torch.cat(flag_j)
    ratio = min(1.0, float(worst_ulps))          # elements within one ulp are within every bound
    if ii.numel() and elementwise:
        bound = _elem_bound(ii, jj, ref, a, w, bias, act, partial_rounding)
        q = (y[ii, jj].to(f64) - ref[ii, jj]).abs() / bound
        kq = int(q.argmax())
        ratio = max(ratio, float(q[kq]))
        assert float(q[kq]) <= 1.0, (f"{name}: elementwise |y - r| = {float(q[kq] * bound[kq]):.3e} > bound "
                                     f"{float(bound[kq]):.3e} at ({int(ii[kq])}, {int(jj[kq])}), "
                                     f"y = {float(y[ii[kq], jj[kq]]):.6g}, r = {float(ref[ii[kq], jj[kq]]):.6g}")
    return {"name": name, "chunk_excess": worst, "chunk_at": at, "total_excess": total, "elem_ratio": ratio,
            "max_ulps": float(worst_ulps), "over_1ulp": int(ii.numel()), "mismatch": mismatched / max(1, M * n)}


def check_untouched(buf: torch.Tensor, n_valid: int, fill: float, name: str = "") -> None:
    """The columns of a strided output buffer past the valid N still hold `fill`."""
    assert bool((buf[:, n_valid:] == fill).all()), f"{name}: wrote past column {n_valid}"
