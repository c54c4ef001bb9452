"""Float64 references and an elementwise / rounding-flip checker for the token-wise kernels of csrc/elementwise.cu
(norms, RoPE, SwiGLU, GELU, layer-scale residual, the flash-decoding merge), forward and backward.

Every reference runs in float64 on the device of its inputs and reproduces the bf16 rounding points that the kernels
take from the reference model (cited in the kernel comments).  It returns `Ref(r, d, skip)`: r is the value before the
final rounding to bf16, d the propagated term D of check 2 below, skip the elements whose fp32 evaluation cancels
(excluded from check 3), or None.  Every reference of a per-row output (including the norms' dx) is row-independent and
returns float64 tensors the size of its input, so a large tensor is checked slab by slab of rows; the reductions over
rows (rmsnorm_dw_ref, layernorm_dwdb_ref, ls_residual_bwd_ref's dls) walk the rows themselves, in slabs of
`slab_bytes` of float64 intermediates.

`check_tokenwise(y, r, d, skip, ...)` asserts, for a bf16 kernel output y,
  1. finite: y is finite wherever r is;
  2. elementwise: |y - r| <= ulp_bf16(r) + D.  ulp_bf16(r) covers the final rounding.  With u = 2^-24 (the fp32 unit
     roundoff), n = cols of the row and the bf16 / fp32 inputs exact in float64:
       rmsnorm      z = s rstd, r = bf16(z) w:  D = |w| (ulp_bf16(z) + e_r |z|),  e_r = (n / 2 + 8) u
                    (an fp32 sum of n squares is within (n - 1) u, halved by the square root; the division, eps,
                    rsqrtf's 2 ulps and the product add 8 u; bf16(z) may round the other way);
       layernorm    D = |w| rstd (dm + |x - m| (e_v + 3 u)) + 2 u (|w xh| + |b|),  dm = n u mean|x| + u |m| the
                    error of the fp32 mean, e_v = ((n + 3) u + dm^2 / var) / 2 + 5 u that of rstd;
       rmsnorm_bwd  dx = rstd t [+ add_in], t = g w - xh m, m = mean(g w xh):
                    D = rstd (|xh| dmm + e_r |xh m| + 2 u (|g w| + |xh m|)) + (e_r + u) |rstd t| + u |r|,
                    dmm = (n + 2) u S + e_r S, S = mean|g w xh|;
       layernorm_bwd the same with mean(g w) and the error dxh = rstd dm + |xh| (e_v + 2 u) of xh;
       dw / db / dls (fp32 sums over rows, then one bf16 rounding):  D = rows 2^-23 sum|terms| (+ the xh error
                    summed over the rows for dw);
       swiglu       D = |u| (ulp_bf16(silu g) + e_s |silu g| + A),  e_s = (4 + 1.2 |g|) 2^-23 (__expf is within
                    2 + 1.173 |x| ulps, __fdividef 2), A = 2^-100: __fdividef returns 0 once 1 + e^-g > 2^126
                    (g < -87.3), where |silu g| < 1e-36;
       swiglu_bwd   dg = dh u sig h, h = 1 + g (1 - sig), du = dh g sig:
                    D_dg = |dh u| (sig e_s |h| + sig (|g| (sig e_s + 2 u |1 - sig|) + 4 u |h|) + A),
                    D_du = |dh g| sig (e_s + 2 u) + |dh| A;
       bias_gelu    pre = bf16(x + b) is exact, r = gelu(pre):  D = 2^-21 (|pre| + |r|).  1 + erf(x / sqrt 2) and
                    1 + tanh(.) cancel for x << 0: their few-ulp absolute error times x / 2 is the |pre| term;
       gelu_bwd     erf:  D = |dy| (2^-22 + |x phi(x)| (4 + x^2) 2^-23 + 2^-21 |gelu'|);
                    tanh: D = |dy| (e + |x| k (1 + 3 c x^2) (e + u) + 2^-21 |gelu'|), e = 2^-21 the error of tanhf
                    and its argument (1 - th^2 cancels, hence the second term);
       rope_table   r = cos / sin of the fp32 angle: D = 2^-22 |r| (sincosf is within 2 ulps);
       rope bwd     the float64 transpose rotation, two inner bf16 roundings: D = (ulp_bf16(a) + ulp_bf16(b)) / 2;
       decode_merge D = sum_s p_s e_s (|o_s| + |r|) + (n + 2) 2^-23 sum_s p_s |o_s| + 2^-100, p_s = e^(lse_s - L),
                    e_s = (4 + 1.7 |lse_s - max lse|) 2^-23; the merged lse within
                    2^-22 (|L| + |max lse|) + 2^-21 + 3 2^-23 log(n) + sum_s p_s e_s + n 2^-24 absolute;
       rmsnorm's fused residual sum, rope, rope_table's duplicate halves, ls_residual, ls_residual_bwd's dy: D = 0
                    and no flip: bit-exact;
  3. rounding flips: the fraction of elements with y != bf16(r) is at most `flip_frac`, and no row (last
     dimension) holds more than `flip_row` of them.  Not counted: `skip`, and the elements whose final (or, for
     RMSNorm, inner) rounding has its argument within TIE_BAND = 2^-19 relative of a bf16 tie.  Such ties are not
     rare: a row whose rstd is within 1e-7 of a number with a 5-bit mantissa puts 1 in 32 of its s rstd on a tie, and
     a row of equal values flips all at once.  A few ulps of fp32 error flip a rounding only near a tie;
     a norm statistic off by one 8-column vector (cols - 8, a dropped vector) flips 4 % (16 384 columns) to 66 %
     (1024) of that row's roundings, and a one-pass variance 2 to 4 % of a row of 40 +- 0.5, which check 2 cannot
     see.
The worst figures per op measured on an H100 80GB HBM3 (700 W) are listed in DESIGN.md ("Tolerances"); FLIPS keeps at
least twice each.

It returns the worst figures: elementwise ratio |y - r| / bound, largest |y - r| in ulps, flip fraction and the most
flips in one row.  `merge` combines the figures of row slabs.

`check_untouched(buf, view, fill)`: a kernel writing through a strided view left the rest of `buf` at `fill`.
"""
import math
from typing import NamedTuple, Optional

import torch
import torch.nn.functional as F

from tests.gemm_ref import bf16r, ulp_bf16

f64 = torch.float64
U = 2.0 ** -24                 # fp32 unit roundoff
A_TINY = 2.0 ** -100           # absolute floor of the __expf / __fdividef underflow range
TANH_K, TANH_C = math.sqrt(2.0 / math.pi), 0.044715


# Check 3's limits per op: (fraction of a tensor's elements, fraction of one row's) whose rounding may flip.  Each is
# at least twice the worst measured on an H100 (DESIGN.md, "Tolerances"); one flip per row, and per tensor, is
# always allowed.
# The mean-offset rows of the LayerNorm edges have their own: the fp32 mean of a row of 40 +- 0.5 is off by ~1e-5,
# which flips about 0.4 % of those outputs in a correct kernel; a one-pass variance flips 2 to 4 %.  The RoPE backward
# is held to check 2 and to bit-exactness with the forward kernel: its two inner roundings flip about a third of the
# results against the unrounded transpose.
FLIPS = {
    "exact": (0.0, 0.0),
    "rmsnorm": (1e-4, 0.005), "layernorm": (1e-4, 0.005), "layernorm_offset": (8e-3, 0.03),
    "rmsnorm_bwd": (3e-4, 0.01), "layernorm_bwd": (6e-4, 0.01), "norm_dw": (5e-3, 5e-3),
    "swiglu": (1e-4, 0.005), "swiglu_bwd": (1e-4, 0.005), "gelu": (2e-3, 0.008), "gelu_bwd": (2e-4, 0.005),
    "rope_table": (1e-4, 0.02), "decode_merge": (1e-3, 0.02), "rope_bwd": (1.0, 1.0),
}
TIE_BAND = 2.0 ** -19          # a rounding whose argument lies this close (relative) to a bf16 tie may go either way


def flip_limits(op: str, cols: int) -> dict:
    """check_tokenwise's flip_frac / flip_row for an output of `op` with rows of `cols` elements."""
    frac, row = FLIPS[op]
    return {"flip_frac": frac, "flip_row": 0 if row == 0 else math.ceil(row * cols) + 1}


class Ref(NamedTuple):
    r: torch.Tensor                       # float64 value before the final bf16 rounding
    d: object = 0.0                       # float64 propagated term D (tensor or scalar)
    skip: Optional[torch.Tensor] = None   # elements excluded from the flip count (cancelling fp32 evaluation)


def _d(t):
    return t.to(f64)


def near_tie(v: torch.Tensor, band: float = TIE_BAND) -> torch.Tensor:
    """v (float64) lies within band |v| of a midpoint between two bf16 values."""
    u = ulp_bf16(v)
    return (torch.remainder(v.abs() / u, 1.0) - 0.5).abs() * u <= band * v.abs()


def _slab_rows(cols: int, per_row: int, slab_bytes: int) -> int:
    return max(1, slab_bytes // (8 * per_row * max(1, cols)))


# ------------------------------------------------------------------------------------------------
# norms
# ------------------------------------------------------------------------------------------------
def residual_sum(x: torch.Tensor, residual: Optional[torch.Tensor]) -> torch.Tensor:
    """bf16(x + residual), the new residual stream (bit-exact: fp32 has more than 2 * 8 + 2 bits)."""
    return x if residual is None else bf16r(_d(x) + _d(residual)).to(torch.bfloat16)


def rmsnorm_ref(x, w, eps, residual=None) -> Ref:
    """r = bf16(s rstd) w, s = bf16(x + residual), rstd = (mean s^2 + eps)^-1/2 (oracle.ops.rmsnorm)."""
    s = _d(residual_sum(x, residual))
    n = s.shape[-1]
    rstd = torch.rsqrt(s.square().mean(-1, keepdim=True) + eps)
    z = s * rstd
    wd = _d(w)
    return Ref(bf16r(z) * wd, wd.abs() * (ulp_bf16(z) + (n / 2 + 8) * U * z.abs()), near_tie(z))


def _ln_stats(xd, eps):
    n = xd.shape[-1]
    m = xd.mean(-1, keepdim=True)
    var = (xd - m).square().mean(-1, keepdim=True)
    rstd = torch.rsqrt(var + eps)
    dm = n * U * xd.abs().mean(-1, keepdim=True) + U * m.abs()
    e_v = ((n + 3) * U + dm.square() / (var + eps)) / 2 + 5 * U
    return m, rstd, dm, e_v


def layernorm_ref(x, w, b, eps) -> Ref:
    """r = (x - mean) rstd w + b with two-pass float64 statistics (torch.nn.LayerNorm in fp32, one rounding)."""
    xd = _d(x)
    m, rstd, dm, e_v = _ln_stats(xd, eps)
    xh = (xd - m) * rstd
    wd = _d(w)
    bd = torch.zeros_like(wd) if b is None else _d(b)
    r = xh * wd + bd
    d = wd.abs() * rstd * (dm + (xd - m).abs() * (e_v + 3 * U)) + 2 * U * ((wd * xh).abs() + bd.abs())
    return Ref(r, d)


def _sum_ref(terms_fn, rows, cols, per_row, slab_bytes, device):
    """float64 sums over rows of terms_fn(r0, r1) -> (terms, |terms| bound), in row slabs; D = rows 2^-23 sum|terms|
    + the sum of the second output."""
    tot = torch.zeros(cols, dtype=f64, device=device)
    mag = torch.zeros_like(tot)
    extra = torch.zeros_like(tot)
    step = _slab_rows(cols, per_row, slab_bytes)
    for r0 in range(0, rows, step):
        t, e = terms_fn(r0, min(rows, r0 + step))
        tot += t.sum(0)
        mag += t.abs().sum(0)
        extra += e.sum(0)
    return Ref(tot, rows * 2.0 ** -23 * mag + extra)


def _rms_stats(xd, eps):
    rstd = torch.rsqrt(xd.square().mean(-1, keepdim=True) + eps)
    return xd * rstd, rstd


def rmsnorm_bwd_ref(x, w, dy, eps, add_in=None) -> Ref:
    """dx of y = bf16(x rstd) w with the inner rounding treated as the identity (as the kernel comment states):
    dx = rstd (dy w - xh mean(dy w xh)) [+ add_in].  Row-independent: the caller passes row slabs of a large tensor."""
    cols = x.shape[-1]
    e_r = (cols / 2 + 8) * U
    xh, rstd = _rms_stats(_d(x), eps)
    gw = _d(dy) * _d(w)
    m = (gw * xh).mean(-1, keepdim=True)
    S = (gw * xh).abs().mean(-1, keepdim=True)
    dmm = (cols + 2) * U * S + e_r * S
    dx0 = rstd * (gw - xh * m)
    r = dx0 if add_in is None else dx0 + _d(add_in)
    d = (rstd * (xh.abs() * dmm + e_r * (xh * m).abs() + 2 * U * (gw.abs() + (xh * m).abs()))
         + (e_r + U) * dx0.abs() + U * r.abs())
    return Ref(r, d)


def rmsnorm_dw_ref(x, w, dy, eps, *, slab_bytes=1 << 30) -> Ref:
    """dw = sum_rows dy xh of rmsnorm(x, w), over row slabs of `slab_bytes` float64 intermediates."""
    cols = x.shape[-1]
    x2, dy2 = x.reshape(-1, cols), dy.reshape(-1, cols)
    e_r = (cols / 2 + 8) * U

    def terms(r0, r1):
        t = _d(dy2[r0:r1]) * _rms_stats(_d(x2[r0:r1]), eps)[0]
        return t, (e_r + U) * t.abs()

    return _sum_ref(terms, x2.shape[0], cols, 4, slab_bytes, x.device)


def _ln_bwd_stats(xd, eps):
    m, rstd, dm, e_v = _ln_stats(xd, eps)
    xh = (xd - m) * rstd
    return xh, rstd, rstd * dm + xh.abs() * (e_v + 2 * U), e_v


def layernorm_bwd_ref(x, w, dy, eps, add_in=None) -> Ref:
    """dx of y = (x - mean) rstd w + b: g = dy w, dx = rstd (g - mean g - xh mean(g xh)) [+ add_in].
    Row-independent: the caller passes row slabs of a large tensor."""
    cols = x.shape[-1]
    xh, rstd, dxh, e_v = _ln_bwd_stats(_d(x), eps)
    gw = _d(dy) * _d(w)
    mg = gw.mean(-1, keepdim=True)
    mgx = (gw * xh).mean(-1, keepdim=True)
    dmg = (cols + 1) * U * gw.abs().mean(-1, keepdim=True)
    dmgx = (cols + 1) * U * (gw * xh).abs().mean(-1, keepdim=True) + (gw.abs() * dxh).mean(-1, keepdim=True)
    dx0 = rstd * (gw - mg - xh * mgx)
    r = dx0 if add_in is None else dx0 + _d(add_in)
    d = (rstd * (dmg + xh.abs() * dmgx + dxh * mgx.abs() + 3 * U * (gw.abs() + mg.abs() + (xh * mgx).abs()))
         + (e_v + U) * dx0.abs() + U * r.abs())
    return Ref(r, d)


def layernorm_dwdb_ref(x, w, dy, eps, *, slab_bytes=1 << 30):
    """(dw, db) = (sum_rows dy xh, sum_rows dy) of layernorm(x, w, b), over row slabs."""
    cols = x.shape[-1]
    x2, dy2 = x.reshape(-1, cols), dy.reshape(-1, cols)

    def dw_terms(r0, r1):
        xh, _, dxh, _ = _ln_bwd_stats(_d(x2[r0:r1]), eps)
        g = _d(dy2[r0:r1])
        return g * xh, g.abs() * dxh

    def db_terms(r0, r1):
        g = _d(dy2[r0:r1])
        return g, torch.zeros_like(g)

    rows = x2.shape[0]
    return _sum_ref(dw_terms, rows, cols, 6, slab_bytes, x.device), _sum_ref(db_terms, rows, cols, 2, slab_bytes, x.device)


# ------------------------------------------------------------------------------------------------
# RoPE
# ------------------------------------------------------------------------------------------------
def rope_angles(pos, inv_freq) -> torch.Tensor:
    """fp32(fp32(pos) inv_freq), the angle torch.outer computes in fp32 (rotary_pos_embedding.py), as float64."""
    return (pos.to(torch.float32).view(-1, 1) * inv_freq.to(torch.float32).view(1, -1)).to(f64)


def rope_table_ref(pos, inv_freq):
    """(cos, sin) Refs [n, dim / 2] of the fp32 angle (the kernel writes each twice: columns j and dim / 2 + j)."""
    ang = rope_angles(pos, inv_freq)
    c, s = ang.cos(), ang.sin()
    return Ref(c, 2.0 ** -22 * c.abs() + 2.0 ** -149), Ref(s, 2.0 ** -22 * s.abs() + 2.0 ** -149)


def rope_ref(x, cos, sin) -> Ref:
    """x [n, heads, dim]: bf16(x1 c) + bf16(-x2 s) | bf16(x2 c) + bf16(x1 s), the reference's bf16 sequence
    (bit-exact: each product of two bf16 values is exact in fp32)."""
    half = x.shape[-1] // 2
    xd, c, s = _d(x), _d(cos)[:, None, :], _d(sin)[:, None, :]
    x1, x2 = xd[..., :half], xd[..., half:]
    o1 = bf16r(x1 * c[..., :half]) + bf16r(-x2 * s[..., :half])
    o2 = bf16r(x2 * c[..., half:]) + bf16r(x1 * s[..., half:])
    return Ref(torch.cat([o1, o2], -1))


def rope_bwd_ref(dy, cos, sin) -> Ref:
    """Gradient of rope(x) as the float64 transpose of the rotation: dx1 = c1 dy1 + s2 dy2, dx2 = c2 dy2 - s1 dy1."""
    half = dy.shape[-1] // 2
    dd, c, s = _d(dy), _d(cos)[:, None, :], _d(sin)[:, None, :]
    d1, d2 = dd[..., :half], dd[..., half:]
    a1, b1 = c[..., :half] * d1, s[..., half:] * d2
    a2, b2 = c[..., half:] * d2, -s[..., :half] * d1
    r = torch.cat([a1 + b1, a2 + b2], -1)
    d = torch.cat([ulp_bf16(a1) + ulp_bf16(b1), ulp_bf16(a2) + ulp_bf16(b2)], -1) / 2
    return Ref(r, d)


# ------------------------------------------------------------------------------------------------
# activations, layer scale
# ------------------------------------------------------------------------------------------------
def _silu_err(g):
    return (4 + 1.2 * g.abs()) * 2.0 ** -23


def swiglu_ref(gate_up) -> Ref:
    """r = bf16(silu(g)) u, (g, u) = the two halves of gate_up (oracle.ops.swiglu)."""
    inter = gate_up.shape[-1] // 2
    g, u = _d(gate_up[..., :inter]), _d(gate_up[..., inter:])
    sl = F.silu(g)
    r = bf16r(sl) * u
    d = u.abs() * (ulp_bf16(sl) + _silu_err(g) * sl.abs() + A_TINY)
    return Ref(r, d, u.abs() * A_TINY > ulp_bf16(r) / 8)


def swiglu_bwd_ref(gate_up, dh) -> Ref:
    """[dg | du] of h = silu(g) u: dg = dh u sig (1 + g (1 - sig)), du = dh silu(g)."""
    inter = gate_up.shape[-1] // 2
    g, u, dd = _d(gate_up[..., :inter]), _d(gate_up[..., inter:]), _d(dh)
    sig = torch.sigmoid(g)
    h = 1 + g * (1 - sig)
    e_s = _silu_err(g)
    dg = dd * u * sig * h
    du = dd * g * sig
    d_dg = (dd * u).abs() * (sig * e_s * h.abs() + sig * (g.abs() * (sig * e_s + 2 * U * (1 - sig)) + 4 * U * h.abs()) + A_TINY)
    d_du = (dd * g).abs() * sig * (e_s + 2 * U) + dd.abs() * A_TINY
    r, d = torch.cat([dg, du], -1), torch.cat([d_dg, d_du], -1)
    return Ref(r, d, torch.cat([(dd * u).abs(), dd.abs()], -1) * A_TINY > ulp_bf16(r) / 8)


def gelu_pre(x, bias=None) -> torch.Tensor:
    """bf16(x + bias) in float64: the rounding nn.Linear's output takes before the activation."""
    return _d(x) if bias is None else bf16r(_d(x) + _d(bias))


def bias_gelu_ref(x, bias=None, approximate="none") -> Ref:
    pre = gelu_pre(x, bias)
    r = F.gelu(pre, approximate=approximate)
    absd = 2.0 ** -21 * pre.abs()
    return Ref(r, absd + 2.0 ** -21 * r.abs(), absd > ulp_bf16(r) / 8)


def gelu_grad64(x, approximate="none"):
    if approximate == "tanh":
        th = torch.tanh(TANH_K * (x + TANH_C * x ** 3))
        return 0.5 * (1 + th) + 0.5 * x * (1 - th * th) * TANH_K * (1 + 3 * TANH_C * x * x)
    return 0.5 * (1 + torch.erf(x / math.sqrt(2))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)


def gelu_bwd_ref(pre, dy, approximate="none") -> Ref:
    """dx = dy gelu'(pre)."""
    x, dd = _d(pre), _d(dy)
    gp = gelu_grad64(x, approximate)
    if approximate == "tanh":
        e = 2.0 ** -21
        absd = dd.abs() * (e + x.abs() * TANH_K * (1 + 3 * TANH_C * x * x) * (e + U))
    else:
        xphi = x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
        absd = dd.abs() * (2.0 ** -22 + xphi.abs() * (4 + x * x) * 2.0 ** -23)
    r = dd * gp
    return Ref(r, absd + 2.0 ** -21 * r.abs(), absd > ulp_bf16(r) / 8)


def ls_residual_ref(x, y, ls=None, bias=None) -> Ref:
    """x + bf16(bf16(y + bias) ls) (bit-exact: modeling_intern_vit.py's order)."""
    yd = _d(y)
    if bias is not None:
        yd = bf16r(yd + _d(bias))
    if ls is not None:
        yd = bf16r(yd * _d(ls))
    return Ref(_d(x) + yd)


def ls_residual_bwd_ref(dout, y, ls, *, slab_bytes=1 << 30):
    """(dy, dls): dy = dout ls (exact, one bf16 rounding), dls = sum_rows dout y."""
    cols = y.shape[-1]
    d2, y2 = dout.reshape(-1, cols), y.reshape(-1, cols)
    dls = _sum_ref(lambda r0, r1: (_d(d2[r0:r1]) * _d(y2[r0:r1]), torch.zeros((1, cols), dtype=f64, device=y.device)),
                   d2.shape[0], cols, 2, slab_bytes, y.device)
    return Ref(_d(dout) * _d(ls)), dls


# ------------------------------------------------------------------------------------------------
# flash-decoding merge
# ------------------------------------------------------------------------------------------------
def decode_merge_ref(o_part, lse_part):
    """o_part [n, G, hkv, d], lse_part [n, hkv, G] -> (Ref of out [hkv G, d], merged lse L [hkv G], its bound).
    out = sum_s e^(lse_s - L) o_s, L = log sum_s e^(lse_s); all splits at -inf give out = 0 and L = -inf."""
    n, G, hkv, d = o_part.shape
    lse = _d(lse_part).permute(1, 2, 0).reshape(hkv * G, n)             # head h = kvh G + g
    o = _d(o_part).permute(2, 1, 0, 3).reshape(hkv * G, n, d)
    L = torch.logsumexp(lse, -1)
    empty = torch.isneginf(L)
    p = torch.where(empty[:, None], torch.zeros_like(lse), torch.exp(lse - L[:, None]))
    m = lse.max(-1).values
    e = (4 + 1.7 * torch.where(torch.isneginf(lse), torch.zeros_like(lse), (lse - m[:, None]).abs())) * 2.0 ** -23
    r = (p[..., None] * o).sum(1)
    pe = p * e
    dd = (pe[..., None] * (o.abs() + r.abs()[:, None, :])).sum(1) + (n + 2) * 2.0 ** -23 * (p[..., None] * o.abs()).sum(1)
    lse_bound = (2.0 ** -22 * (L.abs() + m.abs()) + 2.0 ** -21 + 3 * 2.0 ** -23 * math.log(n) + pe.sum(-1)
                 + n * 2.0 ** -24)
    lse_bound = torch.where(empty, torch.zeros_like(lse_bound), lse_bound)
    return Ref(r, dd + A_TINY), L, lse_bound


# ------------------------------------------------------------------------------------------------
# checks
# ------------------------------------------------------------------------------------------------
def check_tokenwise(y: torch.Tensor, r: torch.Tensor, d=0.0, skip: Optional[torch.Tensor] = None, *, name: str = "",
                    flip_frac: float = 0.0, flip_row: int = 0) -> dict:
    """Checks 1-3 of the module docstring for y (bf16, any shape; rows along the last dimension) against Ref (r, d,
    skip).  flip_frac = flip_row = 0 and d = 0 demand y == bf16(r) everywhere."""
    assert y.shape == r.shape, (name, tuple(y.shape), tuple(r.shape))
    cols = y.shape[-1] if y.dim() else 1
    yd = y.to(f64).reshape(-1, cols)
    rd = r.reshape(-1, cols)
    fin = torch.isfinite(rd)
    bad = fin & ~torch.isfinite(yd)
    assert not bool(bad.any()), f"{name}: finite: {int(bad.sum())} non-finite elements where r is finite"
    err = (yd - rd).abs()
    err = torch.where(fin, err, torch.zeros_like(err))
    bound = ulp_bf16(rd) + (d.reshape(-1, cols) if torch.is_tensor(d) else d)
    q = err / bound
    k = int(q.argmax())
    ratio = float(q.view(-1)[k])
    max_ulps = float((err / ulp_bf16(rd)).max())
    at = (k // cols, k % cols)
    assert ratio <= 1.0, (f"{name}: elementwise |y - r| = {float(err.view(-1)[k]):.4e} > bound {float(bound.view(-1)[k]):.4e}"
                          f" at {at}, y = {float(yd.view(-1)[k]):.8g}, r = {float(rd.view(-1)[k]):.8g}")
    flips = (yd != bf16r(rd)) & fin & ~near_tie(rd)
    if skip is not None:
        flips &= ~skip.reshape(-1, cols)
    per_row = flips.sum(-1)
    n_flip, row_max = int(per_row.sum()), int(per_row.max()) if per_row.numel() else 0
    frac = n_flip / max(1, yd.numel())
    assert frac <= flip_frac or (flip_frac > 0 and n_flip <= 1), \
        f"{name}: flip fraction {frac:.3e} > {flip_frac:.1e} ({n_flip} of {yd.numel()})"
    assert row_max <= flip_row, (f"{name}: {row_max} flipped roundings in row {int(per_row.argmax())} "
                                 f"(at most {flip_row} of {cols})")
    return {"name": name, "elem_ratio": ratio, "max_ulps": max_ulps, "flip_frac": frac, "flip_row": row_max,
            "row_frac": row_max / cols, "n": yd.numel()}


def merge(a: Optional[dict], b: dict) -> dict:
    """Worst figures of two row slabs of one output."""
    if a is None:
        return dict(b)
    n = a["n"] + b["n"]
    return {"name": a["name"], "elem_ratio": max(a["elem_ratio"], b["elem_ratio"]),
            "max_ulps": max(a["max_ulps"], b["max_ulps"]),
            "flip_frac": (a["flip_frac"] * a["n"] + b["flip_frac"] * b["n"]) / n,
            "flip_row": max(a["flip_row"], b["flip_row"]), "row_frac": max(a["row_frac"], b["row_frac"]), "n": n,
            **({"op": a["op"]} if "op" in a else {})}


# ------------------------------------------------------------------------------------------------
# numerical-edge rows of the norms
# ------------------------------------------------------------------------------------------------
# (group, rows) in order.  Each group is checked as a tensor of its own, so that the flip fraction of the mean-offset
# rows is not diluted by the others.
EDGE_GROUPS = (("zero", 8), ("small", 8), ("outlier", 8), ("ordinary", 8), ("offset", 32))


def edge_rows(cols: int, randn, device) -> torch.Tensor:
    """The EDGE_GROUPS rows: zeros; magnitude 1e-3 (eps dominates); ones with one channel at 1e4; N(0, 1); 40 +- 0.5
    (a mean large against the spread).  randn(shape, scale, mean) returns a bf16 tensor on `device`."""
    o = torch.ones((8, cols), dtype=torch.bfloat16, device=device)
    o[torch.arange(8), torch.arange(8) * 7 % cols] = 1e4
    return torch.cat([torch.zeros((8, cols), dtype=torch.bfloat16, device=device), randn((8, cols), 1e-3, 0.0), o,
                      randn((8, cols), 1.0, 0.0), randn((32, cols), 0.5, 40.0)])


def edge_groups():
    """(group, row slice) of edge_rows."""
    r0 = 0
    for name, n in EDGE_GROUPS:
        yield name, slice(r0, r0 + n)
        r0 += n


def edge_op(op: str, group: str) -> str:
    """The FLIPS entry of `op` on an edge-row group: the mean-offset rows have their own where the op has one."""
    return op + "_offset" if group == "offset" and op + "_offset" in FLIPS else op


def check_untouched(buf: torch.Tensor, view: torch.Tensor, fill: float, name: str = "") -> None:
    """Every element of `buf` outside the strided `view` of it still holds `fill`."""
    mask = torch.ones(buf.numel(), dtype=torch.bool, device=buf.device)
    idx = torch.as_strided(torch.arange(buf.numel(), device=buf.device), view.shape, view.stride(),
                           view.storage_offset() - buf.storage_offset())
    mask[idx.reshape(-1)] = False
    outside = buf.reshape(-1)[mask]
    assert bool((outside == fill).all()), f"{name}: {int((outside != fill).sum())} elements outside the view written"
