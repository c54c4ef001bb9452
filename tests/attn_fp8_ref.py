"""The FP8 attention forward (`lv_attn_fwd_fp8`, ops.attention_fwd_fp8): the torch restatement of its operand rule
(csrc/attn_fp8_core.h), a float64 reference, and the checker its GPU tests use.

Rule (`quant_kv`, `quant_q`): K and V in 128-row blocks per (batch, kv head) aligned to key row 0, Q in 64-row groups
per (batch, query head) aligned to query row 0; each block is one e4m3 row of the rule of csrc/fp8_core.h
(tests/fp8_ref.quant_rows_ref).  V blocks are stored transposed with the key permutation `key_of`.

Reference: `attention_fwd_ref` of tests/attn_fwd_ref.py over the DEQUANTISED operands (q8 s_q, k8 s_k, v8 s_v), so the
quantisation of Q, K and V is part of the function being checked, not of its error.  What the kernel does beyond that
exact function, per query row (x = s * scale_log2, log2 domain), and what it costs:

  * s = q8 . k8 on the FP8 tensor cores.  The products are exact; the sum of 128 of them is kept to fewer bits than
    fp32 (about 14 on Hopper).  Bound: |ds| <= ACC D, D = scale |q| max_j |k_j| >= scale sum_i |q_i k_ij| (Cauchy-
    Schwarz), ACC = 2^-11 (four k32 steps, each within 2^-13 of the running sum).  A relative error ACC D of every p
    moves O by at most ACC D (A + |r|) (numerator and normaliser) and lse by ACC D.
  * p = ex2(x - m) in fp32 feeds l; P V takes e4m3(p 2^8) 2^-8: a relative rounding of at most 2^-4 for p >= 2^-14,
    and at most 2^-18 absolute below (subnormals, flush to zero).  In units of the row's final max the absolute part
    stays below 2^-18 (the running max only grows), and 1 / l <= min(1, exp(M - lse)) (M >= the largest logit), so the
    rounding moves O by at most 2^-4 A + 2^-18 SV min(1, exp(M - lse)), SV = sum over the visible keys of |v|.
  * acc = P8 V8 per 128-key tile in the tensor cores (within ACC of the tile's sum of |terms|, <= ACC (1 + 2^-4) A in
    all), then O = alpha O + s_v acc in fp32, the fp32 terms of tests/attn_fwd_ref.py, and out = bf16(O / l).

Bounds (u = 2^-24):
  lse:  |lse - lse_ref| <= LSE_RATIO (u (2 M + 2 |lse_ref| + 8 + sqrt(n)) + ACC D).
  elementwise (hard):  |o - r| <= ulp_bf16(r) + 2^-4 A + 2^-18 SV min(1, e^(M - lse)) + ACC D (A + |r|)
        + 1.07 ACC A + 2^-22 (n / 16 + 32) A + u (n / 4 + 32) |r|.  Any O(1) error (a key wrongly shown or hidden
        whose weight is O(1), as with planted keys) fails it.
  per row:  Z = rms over the columns of (o - r) / sqrt(2^-8 / 3 sigma^2 + ulp_bf16(r)^2 / 12 + (B / 2)^2 / 3) <= Z_ROW,
        where sigma^2 = sum P^2 v^2: an e4m3 rounding of p is uniform within half an ulp of at most 2^-3 p, variance
        <= 2^-8 / 3 p^2 per key; B the non-random terms of the elementwise bound other than the P rounding.
  exact edges:  every value finite; where A = 0 (zero V columns) the output is exactly 0.
  aggregate:  the relative Frobenius error against the reference is reported (`rel`), not bounded here: it is the
        quality figure of the FP8 rounding of P, about 2^-4 / sqrt(3) of a row's spread.

LSE_RATIO and Z_ROW are at least twice the worst figure measured on an H100 (DESIGN.md, "Tolerances").
"""
import math

import torch

from tests.attn_fwd_ref import _worst, attention_fwd_ref, ulp_bf16
from tests.fp8_ref import quant_rows_ref

FP8 = torch.float8_e4m3fn
BLOCK = 128          # key rows per K / V scale
QROWS = 64           # query rows per Q scale
ACC = 2.0 ** -11
LSE_RATIO = 8.0
Z_ROW = 3.0


def key_of(kappa):
    """Key (within its 128-key block) held by byte kappa of a transposed V row: kappa = 32 c + 16 h + 4 t + i holds key
    32 c + 16 h + 8 (i // 2) + 2 t + i % 2."""
    kappa = torch.as_tensor(kappa)
    return (kappa & ~15) | (((kappa >> 1) & 1) << 3) | (((kappa >> 2) & 3) << 1) | (kappa & 1)


def _blocks(x, rows):
    """x [b, s, h, d] -> [b, h, nb, rows * d] zero-padded blocks of `rows` rows, and nb."""
    b, s, h, d = x.shape
    nb = -(-s // rows)
    xp = torch.zeros((b, nb * rows, h, d), dtype=x.dtype, device=x.device)
    xp[:, :s] = x
    return xp.view(b, nb, rows, h, d).permute(0, 3, 1, 2, 4).reshape(b, h, nb, rows * d), nb


def quant_kv(k, v):
    """bf16 K / V [b, sk, hkv, d] -> (k8 uint8 [b, hkv, nt * 128, d], vt8 uint8 [b, hkv, nt, d, 128], k_scale,
    v_scale [b, hkv, nt]): the bytes lv_attn_fp8_quant_kv writes."""
    b, sk, hkv, d = k.shape
    kb, nt = _blocks(k, BLOCK)
    vb, _ = _blocks(v, BLOCK)
    kq, ks = quant_rows_ref(kb)                # zero padding rows never raise amax and quantise to zero bytes
    vq, vs = quant_rows_ref(vb)
    k8 = kq.view(b, hkv, nt * BLOCK, d)
    vq = vq.view(b, hkv, nt, BLOCK, d)
    perm = key_of(torch.arange(BLOCK)).to(vq.device)
    vt8 = vq[:, :, :, perm, :].transpose(-1, -2).contiguous()      # [b, hkv, nt, d, kappa] = v[key_of(kappa)]
    return k8, vt8, ks, vs


def dequant_kv(k8, vt8, ks, vs, sk):
    """The K / V [b, sk, hkv, d] float32 the FP8 kernel computes with: float(q) * scale."""
    b, hkv, rows, d = k8.shape
    nt = rows // BLOCK
    kf = (k8.view(FP8).float().view(b, hkv, nt, BLOCK, d) * ks[..., None, None]).view(b, hkv, rows, d)
    inv = torch.argsort(key_of(torch.arange(BLOCK)).to(vt8.device))
    vf = vt8.view(FP8).float()[..., inv].transpose(-1, -2) * vs[..., None, None]   # [b, hkv, nt, 128, d]
    vf = vf.reshape(b, hkv, rows, d)
    return kf.permute(0, 2, 1, 3)[:, :sk], vf.permute(0, 2, 1, 3)[:, :sk]


def quant_q(q, rows=None):
    """The kernel's Q rule on the query rows `rows` (None = all): q [b, sq, hq, d] bf16 -> the dequantised q8 s_q
    [b, n, hq, d] float32 of those rows (64-row groups per (batch, head) aligned to query row 0).  Only the groups
    holding a wanted row are quantised."""
    b, sq, hq, d = q.shape
    rows = torch.arange(sq, device=q.device) if rows is None else torch.as_tensor(rows).to(q.device)
    groups = torch.unique(rows // QROWS)
    src = (groups[:, None] * QROWS + torch.arange(QROWS, device=q.device)).reshape(-1)
    qg = torch.zeros((b, src.numel(), hq, d), dtype=q.dtype, device=q.device)
    ok = src < sq
    qg[:, ok] = q[:, src[ok]]
    qb, ng = _blocks(qg, QROWS)
    qq, qs = quant_rows_ref(qb)
    qf = (qq.view(FP8).float() * qs[..., None]).view(b, hq, ng * QROWS, d).permute(0, 2, 1, 3)
    at = torch.searchsorted(groups, rows // QROWS) * QROWS + rows % QROWS
    return qf[:, at]


def reference(q, k, v, *, q_rows=None, scale=None):
    """Float64 reference of the FP8 kernel on the rows `q_rows` (None = all) of a causal call (queries bottom-right
    aligned): attention_fwd_ref over the dequantised operands, plus the terms of the bounds (D, SV).  Inputs bf16 on
    one device."""
    d = q.shape[-1]
    sq, sk = q.shape[1], k.shape[1]
    scale = 1.0 / math.sqrt(d) if scale is None else float(scale)
    k8, vt8, ks, vs = quant_kv(k, v)
    kf, vf = dequant_kv(k8, vt8, ks, vs, sk)
    rows = torch.arange(sq, device=q.device) if q_rows is None else torch.as_tensor(q_rows).to(q.device)
    qf = quant_q(q, rows)
    ref = attention_fwd_ref(qf, kf, vf, causal=True, scale=scale, q_pos=rows + (sk - sq))
    G = q.shape[2] // k.shape[2]
    qn = qf.double().norm(dim=-1)                                                     # [b, n, hq]
    kmax = kf.double().norm(dim=-1).amax(1).repeat_interleave(G, dim=-1)              # [b, hq]
    ref["D"] = (scale * qn * kmax[:, None, :]).permute(0, 2, 1)                       # [b, hq, n]
    last = rows + (sk - sq)                                                            # last visible key of each row
    csum = vf.abs().cumsum(1)                                                          # [b, sk, hkv, d]
    ref["SV"] = csum[:, last].double().repeat_interleave(G, dim=2)                     # [b, n, hq, d]
    return ref


def check(out, lse, ref, label=""):
    """`out` [b, n, hq, d] and `lse` [b, hq, n] (or None) of the kernel on the reference's rows against `ref`
    (`reference`); asserts the bounds of the module docstring and returns the figures."""
    r, A, sig = ref["out"], ref["A"], ref["sigma"]
    dev = r.device
    o = out.to(dev, torch.float64)
    n = ref["n_keys"].to(torch.float64)
    u = 2.0 ** -24
    D = ref["D"]                                                                       # [b, hq, n]
    Dr = D.permute(0, 2, 1)[..., None]                                                 # [b, n, hq, 1]
    assert o.shape == r.shape, (label, o.shape, r.shape)
    assert bool(torch.isfinite(o).all()), (label, "non-finite output")
    zero = A == 0
    assert not bool(o[zero].any()), (label, "output not exactly 0 where no visible key has a nonzero value")
    stats = {}
    if lse is not None:
        g = lse.to(dev, torch.float64)
        assert bool(torch.isfinite(g).all()), (label, "non-finite lse")
        unit = u * (2 * ref["M"] + 2 * ref["lse"].abs() + 8 + n.sqrt()[None, None, :]) + ACC * D
        ratio = (g - ref["lse"]).abs() / unit
        stats["lse_ratio"] = float(ratio.max())
        assert stats["lse_ratio"] <= LSE_RATIO, (label, "lse", stats["lse_ratio"], _worst(ratio))
    nb = n[None, :, None, None]
    inv_l = torch.exp(ref["M"] - ref["lse"]).clamp(max=1.0).permute(0, 2, 1)[..., None]
    ulp = ulp_bf16(r)
    fixed = (2.0 ** -18 * ref["SV"] * inv_l + ACC * Dr * (A + r.abs()) + 1.07 * ACC * A
             + 2.0 ** -22 * (nb / 16 + 32) * A + u * (nb / 4 + 32) * r.abs())
    bound = ulp + 2.0 ** -4 * A + fixed
    err = (o - r).abs()
    elem = torch.where(zero, torch.zeros_like(err), err / bound)
    stats["elem_ratio"] = float(elem.max())
    assert stats["elem_ratio"] <= 1.0, (label, "elementwise", stats["elem_ratio"], _worst(elem.amax(-1)))
    var = 2.0 ** -8 / 3 * sig.square() + ulp.square() / 12 + (fixed / 2).square() / 3
    z2 = torch.where(zero, torch.zeros_like(err), err.square() / torch.where(zero, torch.ones_like(var), var))
    cols = (~zero).sum(-1).clamp_min(1)
    z_row = (z2.sum(-1) / cols).sqrt()
    stats["z_row"] = float(z_row.max())
    assert stats["z_row"] <= Z_ROW, (label, "per-row Z", stats["z_row"], _worst(z_row))
    rn = float(r.norm())
    stats["rel"] = float((o - r).norm()) / rn if rn > 0 else 0.0
    return stats
