"""Float64 reference for the fused attention forward, and the checker its GPU tests use.

`attention_fwd_ref` computes, on a set of query rows, the exact function `lv_attn_fwd` / `lv_attn_docs_fwd` define:

    out = softmax(scale * q k^T + mask) v,   lse = log sum_j exp(scale * q k_j),
    key j hidden from query row i iff kv_pos[j] > q_pos[i] (causal) or j < kv_lo[i] (documents: kv_lo = doc_start),

with the conventions of tests/attn_grad_ref.py: global positions (zig-zag segments and `kv_pos0` are just other
q_pos / kv_pos), query head h reads kv head h // G, any device, score blocks bounded by `block_bytes`, and a causal
chunk stops at its last visible key (a document chunk starts at its first).  Besides out and lse it returns, per
(row, head, column), A = P |V| and sigma = sqrt(P^2 V^2), which set the scale of the kernel's roundings, and per row
the number of visible keys n and the largest visible |logit| M.  A row that sees no key has out = 0 and lse = -inf.

`check_attn_fwd` holds a kernel result to bounds against that exact function - not against an emulation of this
kernel's 128-key tiling, so a restructured forward (other pipelining, lazy rescale) is judged by the same suite.
What the kernel does in fp32 / bf16, per query row (x = s * scale_log2, log2 domain):

  * s = q . k in fp32 (wgmma; bf16 products are exact, the sum of d of them is rounded);
  * x_j - m rounded once (fmaf), p_j = ex2.approx(x_j - m): relative error ~2^-22 per p;
  * l = sum of p in fp32, sequential per thread over n / 4 keys, rescaled by alpha once per key tile;
  * O = sum of bf16(p_j) v_j in the fp32 tensor-core accumulator, rescaled by alpha per tile; out = bf16(O / l);
  * lse = (m + log2 l) ln 2.

Bounds, u = 2^-24 (half an fp32 ulp):

  lse:  |lse - lse_ref| <= LSE_RATIO * u (2 M + 2 |lse_ref| + 8 + sqrt(n)).  2 M: the rounding of s and of
        s * scale_log2 (relative u each, on logits up to M); 2 |lse|: the final add and ln 2 multiply; 8: ex2.approx
        and log2f; sqrt(n): the random walk of n / 4 sequential fp32 additions into l.  One key wrongly hidden or
        shown moves lse by about p_j ~ 1/n, which this sees up to n of a few 10^4 keys; beyond that planted keys
        (below) turn the same error into an O(1) one.
  elementwise (hard):  |o - r| <= ulp_bf16(r) + 2^-8 A + 2^-22 (n / 16 + 32) A + u (n / 4 + 32) |r|.
        Rounding p to bf16 (relative <= 2^-8) moves O by at most 2^-8 sum p |v| = 2^-8 A; the output rounding is
        at most half an ulp of o (<= one ulp of r); the last two terms bound the fp32 accumulator (one rounding per
        16-key MMA step and per tile rescale, ex2's error) and the error of l.  Any O(1) error fails it.
  per row:  Z = rms over the columns of (o - r) / sqrt(2^-16 / 3 sigma^2 + ulp_bf16(r)^2 / 12) <= Z_ROW.
        The P rounding has variance about 2^-16 / 3 p^2 per key, so 2^-16 / 3 sigma^2 per output; the output rounding
        ulp^2 / 12.  A correct kernel gives Z about 1 per row; a missing key tile, a wrong V block or a wrong
        normalisation in one row gives many units.  A single key of weight 1/n adds only ~300 / sqrt(n).
  exact edges:  every value finite; where A = 0 (rows that see no key, zero V columns as in SigLIP's 72 -> 128
        padding) the output is exactly 0, and a row that sees no key has lse = -inf exactly.
  aggregate:  relative Frobenius error in excess of the bf16 floor, sqrt(e^2 - e_floor^2) < 2e-3, as in
        tests/test_gpu_attention.py.

`merged=True` is for flash-decoding (`ops.attention_decode`): the partial outputs are rounded to bf16 before their
log-sum-exp merge, one more rounding of at most 2^-8 A (variance at most (2^-8 A)^2 / 12).

LSE_RATIO and Z_ROW are at least twice the worst figure measured on an H100 (DESIGN.md, "Tolerances").

Planted keys (`plant_keys`) make one-key mask errors O(1) at any length: query row i becomes c k_t with key t
rescaled to norm 2 sqrt(d), c chosen so that key t's logit exceeds every other logit of the row by >= 20 (another
key's projection on k_t is below 7 for Gaussian keys, even among 425 984 of them).  If t is visible the row's output is
v_t; if the mask must hide t, a kernel that shows it returns ~v_t instead of the reference.
"""
import math
from typing import Optional

import torch

from tests.attn_grad_ref import _sample_rows  # noqa: F401  (the row sampler of every long attention test)

LSE_RATIO = 4.0
Z_ROW = 2.5
EXCESS = 2e-3
PLANT_GAP = 20.0


def attention_fwd_ref(q, k, v, *, causal: bool, scale: Optional[float] = None, q_pos=None, kv_pos=None, kv_lo=None,
                      q_rows=None, block_bytes: int = 1 << 30):
    """q [b, sq, hq, d], k / v [b, sk, hkv, d], any float dtype, one device.  `q_pos` [sq] / `kv_pos` [sk]: global
    positions (defaults: bottom-right aligned, q_pos = i + sk - sq, kv_pos = j).  `kv_lo` [sq]: first key row each
    query row may see (documents), None = 0.  `q_rows`: sorted int64 indices of the rows wanted (None = all).
    Returns a dict of float64 tensors: out, A, sigma [b, n, hq, d]; lse, M [b, hq, n]; n_keys [n] (int64)."""
    dev = q.device
    b, sq, hq, d = q.shape
    sk, hkv = k.shape[1], k.shape[2]
    G = hq // hkv
    f64 = torch.float64
    scale = 1.0 / math.sqrt(d) if scale is None else float(scale)
    q_pos = (torch.arange(sq) + (sk - sq) if q_pos is None else torch.as_tensor(q_pos)).to(dev, torch.int64)
    kv_pos = (torch.arange(sk) if kv_pos is None else torch.as_tensor(kv_pos)).to(dev, torch.int64)
    if causal and sk > 1:
        assert bool((kv_pos[1:] >= kv_pos[:-1]).all()), "kv_pos must be non-decreasing"
    lo_all = None if kv_lo is None else torch.as_tensor(kv_lo).to(dev, torch.int64)
    R = torch.arange(sq, device=dev) if q_rows is None else torch.as_tensor(q_rows).to(dev, torch.int64)
    n = R.numel()
    out = torch.zeros((b, n, hq, d), dtype=f64, device=dev)
    A = torch.zeros_like(out)
    sig = torch.zeros_like(out)
    lse = torch.full((b, hq, n), float("-inf"), dtype=f64, device=dev)
    M = torch.zeros((b, hq, n), dtype=f64, device=dev)
    n_keys = torch.zeros(n, dtype=torch.int64, device=dev)
    qc = max(1, block_bytes // (8 * b * G * sk))
    for r0 in range(0, n, qc):
        idx = R[r0 : r0 + qc]
        sl = slice(r0, r0 + idx.numel())
        pos = q_pos[idx]
        k1 = int(torch.searchsorted(kv_pos, pos.max(), right=True)) if causal else sk
        lo = None if lo_all is None else lo_all[idx]
        k0 = 0 if lo is None else min(int(lo.min()), k1)
        hidden = torch.zeros((idx.numel(), k1 - k0), dtype=torch.bool, device=dev)
        if causal:
            hidden |= kv_pos[None, k0:k1] > pos[:, None]
        if lo is not None:
            hidden |= torch.arange(k0, k1, device=dev)[None, :] < lo[:, None]
        n_keys[sl] = (~hidden).sum(-1)
        if k1 == k0:
            continue
        for h in range(hkv):
            heads = slice(h * G, (h + 1) * G)
            kc, vc = k[:, k0:k1, h].to(f64), v[:, k0:k1, h].to(f64)            # [b, nk, d]
            qf = q[:, idx, heads].to(f64).permute(0, 2, 1, 3)                   # [b, G, n, d]
            s = torch.matmul(qf * scale, kc.unsqueeze(1).transpose(-1, -2))    # [b, G, n, nk]
            s.masked_fill_(hidden, float("nan"))
            M[:, heads, sl] = torch.nan_to_num(s.abs(), nan=0.0).amax(-1)
            s.nan_to_num_(nan=float("-inf"))
            l = torch.logsumexp(s, dim=-1, keepdim=True)
            s.sub_(torch.where(torch.isinf(l), torch.zeros_like(l), l)).exp_()   # P; a row seeing nothing: 0
            lse[:, heads, sl] = l[..., 0]
            out[:, sl, heads] = torch.matmul(s, vc.unsqueeze(1)).permute(0, 2, 1, 3)
            A[:, sl, heads] = torch.matmul(s, vc.abs().unsqueeze(1)).permute(0, 2, 1, 3)
            sig[:, sl, heads] = torch.matmul(s.square_(), vc.square().unsqueeze(1)).sqrt_().permute(0, 2, 1, 3)
            del s
    return {"out": out, "lse": lse, "A": A, "sigma": sig, "M": M, "n_keys": n_keys}


def doc_lo(cu_seqlens, sq: int, device=None):
    """kv_lo of a packed row: the start of each row's document, from the boundaries 0 = c0 < ... < c_n = sq."""
    cu = torch.as_tensor(cu_seqlens, dtype=torch.int64).reshape(-1).to(device)
    rows = torch.arange(sq, device=device)
    return cu[torch.searchsorted(cu, rows, right=True) - 1]


def ulp_bf16(r):
    """Spacing of bf16 numbers at |r| (0 at r = 0)."""
    _, e = torch.frexp(r)
    return torch.where(r == 0, torch.zeros_like(r), torch.ldexp(torch.ones_like(r), (e - 8).to(torch.int32)))


def check_attn_fwd(out, lse, ref, *, merged: bool = False, excess_limit: float = EXCESS, label: str = ""):
    """`out` [b, n, hq, d] (the kernel's output on the reference's rows) and `lse` [b, hq, n] or None, against `ref`
    of attention_fwd_ref; any device.  Asserts the bounds of the module docstring and returns the measured figures
    (lse_ratio, elem_ratio, z_row, excess)."""
    r, A, sig = ref["out"], ref["A"], ref["sigma"]
    dev = r.device
    o = out.to(dev, torch.float64)
    n = ref["n_keys"].to(torch.float64)
    assert o.shape == r.shape, (label, o.shape, r.shape)
    assert bool(torch.isfinite(o).all()), (label, "non-finite output")
    zero = A == 0
    assert not bool(o[zero].any()), (label, "output not exactly 0 where no visible key has a nonzero value")
    stats = {}
    u = 2.0 ** -24
    if lse is not None:
        g = lse.to(dev, torch.float64)
        blind = ref["lse"] == float("-inf")
        assert bool((g[blind] == float("-inf")).all()), (label, "lse of a row that sees no key is not -inf")
        assert bool(torch.isfinite(g[~blind]).all()), (label, "non-finite lse on a row that sees keys")
        unit = u * (2 * ref["M"] + 2 * ref["lse"].abs() + 8 + n.sqrt()[None, None, :])
        ratio = torch.where(blind, torch.zeros_like(g), (g - ref["lse"]).abs() / unit)
        stats["lse_ratio"] = float(ratio.max()) if ratio.numel() else 0.0
        assert stats["lse_ratio"] <= LSE_RATIO, (label, "lse", stats["lse_ratio"], _worst(ratio))
    nb = n[None, :, None, None]
    ulp = ulp_bf16(r)
    bound = ulp + 2.0 ** -8 * A + 2.0 ** -22 * (nb / 16 + 32) * A + u * (nb / 4 + 32) * r.abs()
    var = 2.0 ** -16 / 3 * sig.square() + ulp.square() / 12
    if merged:
        bound = bound + 2.0 ** -8 * A
        var = var + (2.0 ** -8 * A).square() / 12
    err = (o - r).abs()
    elem = torch.where(zero, torch.zeros_like(err), err / bound)
    stats["elem_ratio"] = float(elem.max()) if elem.numel() else 0.0
    assert stats["elem_ratio"] <= 1.0, (label, "elementwise", stats["elem_ratio"], _worst(elem.amax(-1)))
    z2 = torch.where(zero, torch.zeros_like(err), err.square() / torch.where(zero, torch.ones_like(var), var))
    cols = (~zero).sum(-1).clamp_min(1)
    z_row = (z2.sum(-1) / cols).sqrt()                                           # [b, n, hq]
    stats["z_row"] = float(z_row.max()) if z_row.numel() else 0.0
    assert stats["z_row"] <= Z_ROW, (label, "per-row Z", stats["z_row"], _worst(z_row))
    rn = float(r.norm())
    if rn > 0:
        e_tot = float((o - r).norm()) / rn
        e_floor = float((r.to(torch.bfloat16).to(torch.float64) - r).norm()) / rn
        stats["excess"] = math.sqrt(max(e_tot * e_tot - e_floor * e_floor, 0.0))
        assert stats["excess"] < excess_limit, (label, "excess", stats["excess"], e_tot, e_floor)
    return stats


def _worst(t):
    """Index and value of the largest entry of t (for assertion messages)."""
    i = int(t.argmax())
    return tuple(int(x) for x in torch.unravel_index(torch.tensor(i), t.shape)), float(t.reshape(-1)[i])


def plant_keys(q, k, rows, targets, *, scale: Optional[float] = None):
    """In place, for every batch entry and head: key row targets[m] is rescaled to norm 2 sqrt(d) and query row rows[m]
    becomes c k_t (kv head h // G for query head h), c = PLANT_GAP / (scale |k_t| (|k_t| - 7)), so that key t's logit
    beats every other logit of the row by at least PLANT_GAP (module docstring).  Rows must be distinct."""
    d = q.shape[-1]
    G = q.shape[2] // k.shape[2]
    scale = 1.0 / math.sqrt(d) if scale is None else float(scale)
    rows = torch.as_tensor(rows, dtype=torch.int64).to(q.device)
    targets = torch.as_tensor(targets, dtype=torch.int64).to(q.device)
    assert rows.unique().numel() == rows.numel(), "planted rows must be distinct"
    kt = k[:, targets].float()
    kt = (kt * (2 * math.sqrt(d) / kt.norm(dim=-1, keepdim=True))).to(k.dtype)
    k[:, targets] = kt
    ktf = kt.float()
    nrm = ktf.norm(dim=-1, keepdim=True)
    c = PLANT_GAP / (scale * nrm * (nrm - 7.0))
    q[:, rows] = (c * ktf).repeat_interleave(G, dim=2).to(q.dtype)


def check_planted(ref, v, rows_sel, targets, visible: bool, label: str = ""):
    """Sanity of a plant, on the reference alone: a visible target's row output is v_t; a hidden target's row output is
    far from v_t, so a kernel that shows the key fails check_attn_fwd by O(1).  `rows_sel` index the reference's rows."""
    G = ref["out"].shape[2] // v.shape[2]
    vt = v[:, torch.as_tensor(targets, dtype=torch.int64).to(v.device)].to(torch.float64).repeat_interleave(G, dim=2)
    vt = vt.to(ref["out"].device)
    r = ref["out"][:, torch.as_tensor(rows_sel, dtype=torch.int64).to(ref["out"].device)]
    dist = (r - vt).norm(dim=-1) / vt.norm(dim=-1)
    if visible:
        assert float(dist.max()) < 1e-2, (label, "visible plant does not dominate its row", float(dist.max()))
    else:
        assert float(dist.min()) > 0.3, (label, "hidden plant: the reference row is already near v_t", float(dist.min()))
