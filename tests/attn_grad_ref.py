"""Float64 reference for the gradients of the fused attention, at training lengths, and the checker its GPU tests use.

`attention_grads` computes dQ on a set of query rows and dK / dV on a set of key rows of

    out = softmax(scale * q k^T + mask) v,
    key j hidden from query row i iff kv_pos[j] > q_pos[i] (causal) or j < kv_lo[i] (documents: kv_lo = doc_start),

the attention `lv_attn_fwd` / `lv_attn_bwd` / `lv_attn_docs_bwd` define (query head h reads kv head h // G, G = hq /
hkv; positions are global, so zig-zag context-parallel segments and `kv_pos0` are just other `q_pos` / `kv_pos`).  It
runs on the device of its inputs, CPU or CUDA, in float64, with the textbook formulas per query row i:

    s = scale q_i K^T (masked), lse, P = exp(s - lse), O_i = P V, delta_i = rowsum(dO_i * O_i),
    dQ_i = scale (P * (dO_i V^T - delta_i)) K,   dV_j = sum_i P_ij dO_i,   dK_j = scale sum_i dS_ij q_i.

Rows are independent, so work goes in (query chunk x query heads of one kv group) blocks sized to keep the score
block near `block_bytes`.  For dK / dV only the query chunks that can see some requested key are visited, each with
its own lse and delta.  With a causal mask a chunk's scores stop at the last key it can see (kv_pos must be
non-decreasing), and a document chunk starts at its first.  A query row that sees no key has P = 0 and gets dQ = 0,
never NaN.

Why `out=`: the backward reads the forward's bf16 output, and delta = rowsum(dO * O) taken from it differs from the
exact delta by the output rounding.  In dS = P (dP - delta) that difference is not damped where dP - delta is small
against dP (rows that see few keys, a peaked softmax), so at bf16 precision the gradient of the exact function is the
wrong target for those rows; flash-attn 2's backward shows the same difference.  With `out` the reference computes the
gradient the backward is asked for, given its inputs.

`check_attn_bwd` holds a kernel result to bounds against that function, derived from what `attn_bwd.cu` does per
visible (i, j) in fp32 / bf16 (not from its tiling, so a restructured backward is judged by the same suite):

  * x = q . k and dP = dO . v by wgmma in fp32 (bf16 products exact, a sum of d of them rounded);
  * P = ex2(fmaf(x, scale log2e, -lse log2e)) with the forward's fp32 lse;
  * delta = fp32 rowsum(dO * O) over the forward's bf16 O;
  * dS = P (dP - delta) scale in fp32, rounded to bf16;
  * dV += bf16(P) dO, dK += bf16(dS) q, dQ += bf16(dS) k in fp32 accumulators (one rounding per 16-deep MMA step),
    then one bf16 rounding of each output.

`terms=True` also returns, per output element, the magnitudes that set the scale of those roundings:

    A_q = scale (P * |dP - delta|) |K|,            A_k = scale (P * |dP - delta|)^T |Q|,     A_v = P^T |dO|,
    E_q = scale (P * (|dO| |V|^T + rowsum|dO * O|)) |K|,   E_k = the same with ^T and |Q|,
    sig_q = scale sqrt(dS^2 K^2),   sig_k = scale sqrt((dS^2)^T Q^2),   sig_v = sqrt((P^2)^T dO^2),

(dK / dV terms summed over the G query heads of the kv head), the visible keys per dQ row n_q, the visible query rows
per dK / dV row n_k, the reference lse on the dQ rows, and over every visited row the largest |lse| and the
Cauchy-Schwarz bound L = scale |q_i| max |k_j| on any visible |logit|.

Bounds, u = 2^-24 (half an fp32 ulp), r the reference, g the kernel:

  P:   relative error eps_p = 2u (d L + 2 |lse| + 16) + LSE_RATIO u (2 L + 2 |lse| + 8 + sqrt(n)): the wgmma sum of d
       products (at most d L relative ulps), the fmaf and ex2, and the forward's lse error (tests/attn_fwd_ref.py);
  dP, delta:  absolute error at most d 2u (|dO| |V|^T)_ij and d 2u rowsum|dO * O|, which reach dQ / dK through
       P scale |K| / |Q| as d 2u E_q / E_k;
  elementwise (hard):
       |g - r| <= ulp_bf16(r) + (1 + 2^-7) [(2^-8 + eps_p + 2^-21) A + 2u d E + 2^-22 (N / 16 + 32) A]
       with N = n_q for dQ and G n_k for dK / dV (the fp32 accumulation, as in the forward), and no E term for dV.
       2^-8 A is the bf16 rounding of dS (of P for dV), 2^-21 A the fp32 products and difference in dS, ulp_bf16(r) the
       output rounding; 1 + 2^-7 covers the terms' own bf16 / fp32 perturbation.  Any O(1) error fails it.
  per row:  Z = rms over the columns of (g - r) / sqrt(var) <= Z_ROW, per (row, head) of dQ and per (key row, kv head)
       of dK / dV, var = 2^-16 / 3 sig^2 + ulp_bf16(r)^2 / 12 + (u sqrt(d) E)^2 + (LSE_RATIO u (2L + 2|lse| + 8 +
       sqrt(n)) r)^2: the bf16 rounding of dS (P) as in the forward, the output rounding, the fp32 dP / delta roundings
       (a random walk over d terms) and the forward's lse error (a common factor on a row's P).  A correct kernel gives
       Z about 1, up to ~2 on rows dominated by one term (a planted key's dK / dV: one rounding, the same relative
       error on every column); a missing 64-key tile of one query tile, a head's or tile's missing share of a dK / dV
       sum give many.
  exact edges:  every value finite; dQ = 0 exactly on rows that see no key, dK = dV = 0 exactly on key rows no query
       sees (past the last visible position, before kv_pos0, past a zig-zag rank's last chunk, past a document end).
  aggregate:  relative Frobenius error in excess of the bf16 floor, sqrt(e^2 - e_floor^2) < 3e-3, as in
       tests/test_gpu_attention_bwd.py.

Z_ROW is at least twice the worst figure measured on an H100 (DESIGN.md, "Tolerances"); the other limits are derived.

Paired plants (`plant_pairs`) make a one-key mask error O(1) in every gradient.  The forward's saturating plant
(tests/attn_fwd_ref.py `plant_keys`) does not: with P = 1 on the target, dS = P (dP - delta) = 0, so dQ and dK do not
depend on it.  Here key t (the edge key) and a partner key p are rescaled to norm 2 sqrt(d) and query row i becomes
c (k_t + k_p), c chosen so that both logits beat every other logit of the row by >= PLANT_GAP.  If t is visible, P is
about 1/2 on each and dQ_i = scale dS_it (k_t - k_p), dK_t, dV_t all depend at O(1) on t's visibility (with p a copy of
t, dQ_i would cancel to 0).  If t is hidden, P is about 1 on p, and a pass that shows t gets P about 1 on it through the
forward's lse: an O(1) change in dQ_i, dK_t and dV_t.
"""
import math
from typing import Optional

import torch

Z_ROW = 5.0
EXCESS = 3e-3


def _sample_rows(n_rows, local_len, seed, boundaries=(128, 256)):
    """Local row indices: ends, both sides of 128- / 256-row tile boundaries, random rows."""
    rows = {0, 1, local_len - 1, local_len - 2, local_len // 2 - 1, local_len // 2}
    for b in boundaries:
        for m in (1, 7, local_len // b // 2, local_len // b - 1):
            for off in (-1, 0):
                r = m * b + off
                if 0 <= r < local_len:
                    rows.add(r)
    g = torch.Generator().manual_seed(seed)
    while len(rows) < n_rows:
        rows.add(int(torch.randint(0, local_len, (1,), generator=g)))
    return torch.tensor(sorted(rows), dtype=torch.int64)


def attention_grads(q, k, v, d_out, *, causal: bool, scale: Optional[float] = None, q_pos=None, kv_pos=None,
                    kv_lo=None, q_rows=None, kv_rows=None, out=None, terms: bool = False, block_bytes: int = 1 << 30):
    """q / d_out [b, sq, hq, d], k / v [b, sk, hkv, d], any float dtype, all on one device.  `q_pos` [sq] / `kv_pos`
    [sk] are the global positions (defaults: bottom-right aligned, q_pos = i + sk - sq, kv_pos = j).  `kv_lo` [sq]: the
    first key row each query row may see (documents, tests/attn_fwd_ref.py `doc_lo`), None = 0.  `q_rows` / `kv_rows`
    select the rows whose dQ / dK, dV are wanted (sorted int64 indices; None = all rows, an empty tensor = none).
    `out` [b, sq, hq, d], if given, is the forward output the backward reads: delta = rowsum(dO * out) is then taken
    from it instead of from the exact O = P V, as lv_attn_bwd and flash-attn's backward do.  Returns float64
    (dq [b, |q_rows|, hq, d], dk [b, |kv_rows|, hkv, d], dv [b, |kv_rows|, hkv, d]); with `terms`, a dict of those
    and the magnitude terms of the module docstring (A_*, E_*, sig_* shaped like their gradient, n_q [|q_rows|], n_k
    [|kv_rows|], lse [b, hq, |q_rows|], and the floats L, lse_max, n_max)."""
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
    J = torch.arange(sk, device=dev) if kv_rows is None else torch.as_tensor(kv_rows).to(dev, torch.int64)
    nJ = J.numel()
    dq = torch.zeros((b, R.numel(), hq, d), dtype=f64, device=dev)
    dk = torch.zeros((b, nJ, hkv, d), dtype=f64, device=dev)
    dv = torch.zeros((b, nJ, hkv, d), dtype=f64, device=dev)
    if terms:
        T = {name: torch.zeros_like(dq) for name in ("A_q", "E_q", "sig_q")}
        T.update({name: torch.zeros_like(dk) for name in ("A_k", "E_k", "sig_k", "A_v", "sig_v")})
        T["n_q"] = torch.zeros(R.numel(), dtype=torch.int64, device=dev)
        T["n_k"] = torch.zeros(nJ, dtype=torch.int64, device=dev)
        T["lse"] = torch.full((b, hq, R.numel()), float("-inf"), dtype=f64, device=dev)
        T["L"], T["lse_max"], T["n_max"] = 0.0, 0.0, 0
        T["q_rows"], T["kv_rows"] = R, J

    # query rows to visit: the dQ rows and every row that sees some requested key; dq_slot[i] = slot of row i in dq
    want_dq = torch.zeros(sq, dtype=torch.bool, device=dev)
    want_dq[R] = True
    visit = want_dq.clone()
    if nJ:
        sees = q_pos >= kv_pos[J[0]] if causal else torch.ones_like(visit)
        if lo_all is not None:
            sees &= lo_all <= J[-1]
        visit |= sees
    rows = torch.nonzero(visit).view(-1)
    dq_slot = torch.full((sq,), -1, dtype=torch.int64, device=dev)
    dq_slot[R] = torch.arange(R.numel(), device=dev)
    qc = max(1, block_bytes // (8 * b * G * sk))

    for h in range(hkv):
        heads = slice(h * G, (h + 1) * G)
        kf, vf = k[:, :, h].to(f64), v[:, :, h].to(f64)                        # [b, sk, d]
        for r0 in range(0, rows.numel(), qc):
            idx = rows[r0 : r0 + qc]
            pos = q_pos[idx]
            # keys [k0, k1) hold every key a row of this chunk can see
            k1 = int(torch.searchsorted(kv_pos, pos.max(), right=True)) if causal else sk
            lo = None if lo_all is None else lo_all[idx]
            k0 = 0 if lo is None else min(int(lo.min()), k1)
            if k1 == k0:
                continue
            hidden = torch.zeros((idx.numel(), k1 - k0), dtype=torch.bool, device=dev)
            if causal:
                hidden |= kv_pos[None, k0:k1] > pos[:, None]
            if lo is not None:
                hidden |= torch.arange(k0, k1, device=dev)[None, :] < lo[:, None]
            kc, vc = kf[:, k0:k1], vf[:, k0:k1]
            qf = q[:, idx, heads].to(f64).permute(0, 2, 1, 3)                   # [b, G, n, d]
            dof = d_out[:, idx, heads].to(f64).permute(0, 2, 1, 3)
            s = torch.matmul(qf * scale, kc.unsqueeze(1).transpose(-1, -2))    # [b, G, n, nk]
            s.masked_fill_(hidden, float("-inf"))
            lse = torch.logsumexp(s, dim=-1, keepdim=True)
            p = torch.exp(s - torch.where(torch.isinf(lse), torch.zeros_like(lse), lse))   # a row seeing nothing: 0
            del s
            if out is None:
                o = torch.matmul(p, vc.unsqueeze(1))
            else:
                o = out[:, idx, heads].to(f64).permute(0, 2, 1, 3)
            delta = (dof * o).sum(-1, keepdim=True)                            # [b, G, n, 1]
            if terms:
                dlabs = (dof * o).abs().sum(-1, keepdim=True)
                fin = torch.isfinite(lse)
                T["lse_max"] = max(T["lse_max"], float(lse[fin].abs().max()) if bool(fin.any()) else 0.0)
                T["L"] = max(T["L"], scale * float(qf.norm(dim=-1).max()) * float(kc.norm(dim=-1).max()))
                T["n_max"] = max(T["n_max"], int((~hidden).sum(-1).max()))
            del o
            slot = dq_slot[idx]
            sel = slot >= 0
            if bool(sel.any()):
                all_rows = bool(sel.all())
                pr, dor, dlr = (p, dof, delta) if all_rows else (p[:, :, sel], dof[:, :, sel], delta[:, :, sel])
                dp = torch.matmul(dor, vc.unsqueeze(1).transpose(-1, -2))
                ds = pr * (dp - dlr)
                dq[:, slot[sel], heads] = (scale * torch.matmul(ds, kc.unsqueeze(1))).permute(0, 2, 1, 3)
                if terms:
                    kabs = kc.abs().unsqueeze(1)
                    dla = dlabs if all_rows else dlabs[:, :, sel]
                    e = pr * (torch.matmul(dor.abs(), vc.abs().unsqueeze(1).transpose(-1, -2)) + dla)
                    for name, x in (("A_q", torch.matmul(pr * (dp - dlr).abs(), kabs)), ("E_q", torch.matmul(e, kabs)),
                                    ("sig_q", torch.matmul(ds.square(), kc.square().unsqueeze(1)).sqrt())):
                        T[name][:, slot[sel], heads] = scale * x.permute(0, 2, 1, 3)
                    del e
                    T["lse"][:, heads, slot[sel]] = lse[..., 0][:, :, sel]
                    if h == 0:
                        T["n_q"][slot[sel]] = (~hidden[sel]).sum(-1)
                del dp, ds
            # requested keys inside [k0, k1): slots [j0, j1) of dk / dv (J sorted)
            j0, j1 = int(torch.searchsorted(J, k0)), int(torch.searchsorted(J, k1))
            if j1 > j0:
                cols = J[j0:j1] - k0
                pj = p[..., cols]
                vj = vc[:, cols].unsqueeze(1)
                dpj = torch.matmul(dof, vj.transpose(-1, -2))
                dsj = pj * (dpj - delta)
                dv[:, j0:j1, h] += torch.matmul(pj.transpose(-1, -2), dof).sum(1)
                dk[:, j0:j1, h] += scale * torch.matmul(dsj.transpose(-1, -2), qf).sum(1)
                if terms:
                    qabs = qf.abs()
                    T["A_v"][:, j0:j1, h] += torch.matmul(pj.transpose(-1, -2), dof.abs()).sum(1)
                    T["sig_v"][:, j0:j1, h] += torch.matmul(pj.square().transpose(-1, -2), dof.square()).sum(1)
                    T["A_k"][:, j0:j1, h] += scale * torch.matmul((pj * (dpj - delta).abs()).transpose(-1, -2), qabs).sum(1)
                    e = pj * (torch.matmul(dof.abs(), vj.abs().transpose(-1, -2)) + dlabs)
                    T["E_k"][:, j0:j1, h] += scale * torch.matmul(e.transpose(-1, -2), qabs).sum(1)
                    T["sig_k"][:, j0:j1, h] += scale * scale * torch.matmul(dsj.square().transpose(-1, -2), qf.square()).sum(1)
                    if h == 0:
                        T["n_k"][j0:j1] += (~hidden[:, cols]).sum(0)
                del pj, dpj, dsj
            del p
    if not terms:
        return dq, dk, dv
    T["sig_v"].sqrt_()
    T["sig_k"].sqrt_()
    T.update(dq=dq, dk=dk, dv=dv)
    return T


def _ulp_bf16(r):
    """Spacing of bf16 numbers at |r| (0 at r = 0)."""
    _, e = torch.frexp(r)
    return torch.where(r == 0, torch.zeros_like(r), torch.ldexp(torch.ones_like(r), (e - 8).to(torch.int32)))


def _worst(t):
    """Index and value of the largest entry of t (for assertion messages)."""
    i = int(t.argmax())
    return tuple(int(x) for x in torch.unravel_index(torch.tensor(i), t.shape)), float(t.reshape(-1)[i])


def check_attn_bwd(got, ref, *, excess_limit: float = EXCESS, label: str = ""):
    """`got` = (dq, dk, dv) of the kernel on the reference's rows ([b, n, h, d] each), against `ref` of
    attention_grads(..., terms=True); any device.  Asserts the bounds of the module docstring and returns the
    measured figures (elem_ratio, z_row, excess per gradient, e.g. "z_row_dq")."""
    from tests.attn_fwd_ref import LSE_RATIO   # (attn_fwd_ref imports this module)

    u = 2.0 ** -24
    d = ref["dq"].shape[-1]
    G = ref["dq"].shape[2] // max(ref["dk"].shape[2], 1)
    L, lm, nm = ref["L"], ref["lse_max"], ref["n_max"]
    eps_lse = LSE_RATIO * u * (2 * L + 2 * lm + 8 + math.sqrt(nm))
    eps_p = 2 * u * (d * L + 2 * lm + 16) + eps_lse
    dev = ref["dq"].device
    stats = {}
    for name in ("dq", "dk", "dv"):
        g = got[("dq", "dk", "dv").index(name)].to(dev, torch.float64)
        r = ref[name]
        assert g.shape == r.shape, (label, name, g.shape, r.shape)
        assert bool(torch.isfinite(g).all()), (label, name, "non-finite gradient")
        c = name[1]
        A = ref["A_" + c]
        E = ref["E_" + c] if c != "v" else torch.zeros_like(A)
        sig = ref["sig_" + c]
        if c == "q":
            n = ref["n_q"].to(torch.float64)[None, :, None, None]
        else:
            n = G * ref["n_k"].to(torch.float64)[None, :, None, None]
        blind = (n == 0).expand_as(r)
        assert not bool(g[blind].any()), (label, name, "not exactly 0 on rows the mask hides from everything")
        ulp = _ulp_bf16(r)
        terms = (2.0 ** -8 + eps_p + 2.0 ** -21) * A + 2 * u * d * E + 2.0 ** -22 * (n / 16 + 32) * A
        bound = ulp + (1 + 2.0 ** -7) * terms
        err = (g - r).abs()
        elem = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                           torch.where(err > 0, float("inf"), 0.0))
        stats["elem_ratio_" + name] = float(elem.max()) if elem.numel() else 0.0
        assert stats["elem_ratio_" + name] <= 1.0, (label, name, "elementwise", stats["elem_ratio_" + name],
                                                    _worst(elem.amax(-1)))
        var = 2.0 ** -16 / 3 * sig.square() + ulp.square() / 12 + (u * math.sqrt(d) * E).square() + (eps_lse * r).square()
        z2 = torch.where(var > 0, err.square() / torch.where(var > 0, var, torch.ones_like(var)),
                         torch.where(err > 0, float("inf"), 0.0))
        z_row = z2.mean(-1).sqrt()                                                   # [b, n, h]
        stats["z_row_" + name] = float(z_row.max()) if z_row.numel() else 0.0
        assert stats["z_row_" + name] <= Z_ROW, (label, name, "per-row Z", stats["z_row_" + name], _worst(z_row))
        rn = float(r.norm())
        if rn > 0:
            e_tot = float((g - r).norm()) / rn
            e_floor = float((r.to(torch.bfloat16).to(torch.float64) - r).norm()) / rn
            stats["excess_" + name] = math.sqrt(max(e_tot * e_tot - e_floor * e_floor, 0.0))
            assert stats["excess_" + name] < excess_limit, (label, name, "excess", stats["excess_" + name], e_tot, e_floor)
    return stats


def plant_pairs(q, k, rows, targets, partners, *, scale: Optional[float] = None):
    """In place, for every batch entry and head: key rows targets[m] and partners[m] are rescaled to norm 2 sqrt(d),
    then query row rows[m] becomes c (k_t + k_p) (kv head h // G for query head h), with
    c = PLANT_GAP / (scale (k_t . (k_t + k_p) - 7 |k_t + k_p|)), so that both logits (equal, as |k_t| = |k_p|) beat every
    other logit of the row by at least PLANT_GAP (another Gaussian key's projection on a unit vector is below 7); a
    small multiple of k_t - k_p keeps the two logits equal after the bf16 rounding of the keys.  A
    key may serve several rows; rows must be distinct and each target differ from its partner."""
    from tests.attn_fwd_ref import PLANT_GAP   # (attn_fwd_ref imports this module)

    d = q.shape[-1]
    G = q.shape[2] // k.shape[2]
    scale = 1.0 / math.sqrt(d) if scale is None else float(scale)
    rows, targets, partners = (torch.as_tensor(x, dtype=torch.int64).to(q.device) for x in (rows, targets, partners))
    assert rows.unique().numel() == rows.numel(), "planted rows must be distinct"
    assert not bool((targets == partners).any()), "a partner must be another key"
    keys = torch.unique(torch.cat([targets, partners]))
    kk = k[:, keys].float()
    k[:, keys] = (kk * (2 * math.sqrt(d) / kk.norm(dim=-1, keepdim=True))).to(k.dtype)
    kt, kp = k[:, targets].double(), k[:, partners].double()                     # [b, m, hkv, d]
    ks, kd = kt + kp, kt - kp
    den = (kt * ks).sum(-1, keepdim=True) - 7.0 * ks.norm(dim=-1, keepdim=True)
    assert bool((den > 0).all()), "target and partner too far apart to plant"
    c = PLANT_GAP / (scale * den)
    # + lam (k_t - k_p) evens out what the bf16 rounding of the two norms left: q . k_t = q . k_p
    lam = -c * (kt.square().sum(-1, keepdim=True) - kp.square().sum(-1, keepdim=True)) / kd.square().sum(-1, keepdim=True)
    q[:, rows] = (c * ks + lam * kd).repeat_interleave(G, dim=2).to(q.dtype)


def check_pairs(q, k, ref, rows, targets, partners, visible: bool, *, scale: Optional[float] = None, label: str = ""):
    """Sanity of paired plants, on the reference alone (`ref` of attention_grads with terms, whose dQ rows include the
    planted query rows `rows`).  Visible targets: P on target and partner each in [0.45, 0.55].  Hidden targets: the
    partner carries P > 0.98, and the target's weight exp(s_t - lse), 0 in the reference, would be > 0.5 in a pass
    that showed it (not 1: the bf16 rounding of q moves the two logits apart by up to ~0.1)."""
    d = q.shape[-1]
    G = q.shape[2] // k.shape[2]
    scale = 1.0 / math.sqrt(d) if scale is None else float(scale)
    dev = ref["lse"].device
    rows, targets, partners = (torch.as_tensor(x, dtype=torch.int64).to(dev) for x in (rows, targets, partners))
    slots = torch.searchsorted(ref["q_rows"], rows)
    assert bool((ref["q_rows"][slots.clamp_max(ref["q_rows"].numel() - 1)] == rows).all()), (label, "plants not in ref")
    lse = ref["lse"][:, :, slots].transpose(1, 2)                                    # [b, m, hq]
    qr, kd = q.to(dev)[:, rows].to(torch.float64), k.to(dev)
    pt, pp = (torch.exp(scale * (qr * kd[:, t].to(torch.float64).repeat_interleave(G, 2)).sum(-1) - lse)
              for t in (targets, partners))                                         # [b, m, hq]
    if visible:
        lo, hi = float(torch.minimum(pt, pp).min()), float(torch.maximum(pt, pp).max())
        assert 0.45 <= lo and hi <= 0.55, (label, "visible pair weights", lo, hi)
    else:
        assert float(pp.min()) > 0.98 and float(pt.min()) > 0.5, (label, "hidden pair weights", float(pp.min()),
                                                                   float(pt.min()))


def plant_edge_pairs(q, k, rows, targets, *, q_pos, kv_pos, kv_lo=None, scale: Optional[float] = None):
    """plant_pairs for query rows `rows` (local indices) aimed at key rows `targets`, visible or not, each with the
    middle key of the row's visible range [first, last] as partner (its last visible key if the middle is the target).
    Rows that see fewer than two keys, or whose target is outside the keys, are skipped.  Returns {"visible": (rows,
    targets, partners), "hidden": (...)} for check_pairs."""
    sk = k.shape[1]
    rows, targets = torch.as_tensor(rows, dtype=torch.int64), torch.as_tensor(targets, dtype=torch.int64)
    qp, kp = torch.as_tensor(q_pos, dtype=torch.int64).cpu(), torch.as_tensor(kv_pos, dtype=torch.int64).cpu()
    first = torch.zeros_like(rows) if kv_lo is None else torch.as_tensor(kv_lo, dtype=torch.int64).cpu()[rows]
    last = torch.searchsorted(kp, qp[rows], right=True) - 1
    part = (first + last) // 2
    part = torch.where(part == targets, last, part)
    ok = (last > first) & (targets >= 0) & (targets < sk) & (part != targets)
    vis = (targets >= first) & (targets <= last)
    rows, targets, part, vis = rows[ok], targets[ok], part[ok], vis[ok]
    plant_pairs(q, k, rows, targets, part, scale=scale)
    return {"visible": (rows[vis], targets[vis], part[vis]), "hidden": (rows[~vis], targets[~vis], part[~vis])}


def check_planted_pairs(q, k, ref, planted, *, scale: Optional[float] = None, label: str = ""):
    """check_pairs on both kinds of plant_edge_pairs' result."""
    for kind in ("visible", "hidden"):
        r, t, p = planted[kind]
        if r.numel():
            check_pairs(q, k, ref, r, t, p, kind == "visible", scale=scale, label=label)


def edge_targets(rows, q_pos, kv_pos0: int = 0):
    """The mask edge of each query row: even rows its first hidden key (position + 1), odd rows its diagonal key."""
    rows = torch.as_tensor(rows, dtype=torch.int64)
    diag = torch.as_tensor(q_pos, dtype=torch.int64).cpu()[rows] - kv_pos0
    return torch.where(rows % 2 == 0, diag + 1, diag)


def check_rows(got, q, k, v, d_out, out, *, causal: bool, q_rows=None, kv_rows=None, planted=None, worst=None,
               label: str = "", **kw):
    """attention_grads(terms=True) on `q_rows` / `kv_rows` (None = all), check_attn_bwd of the kernel's whole gradients
    `got` there, and check_planted_pairs of `planted`; prints the figures and folds them into `worst`.  Returns them."""
    ref = attention_grads(q, k, v, d_out, causal=causal, q_rows=q_rows, kv_rows=kv_rows, out=out, terms=True, **kw)
    dq, dk, dv = got
    if q_rows is not None:
        dq = dq[:, torch.as_tensor(q_rows).to(dq.device)]
    if kv_rows is not None:
        kr = torch.as_tensor(kv_rows).to(dk.device)
        dk, dv = dk[:, kr], dv[:, kr]
    if planted is not None:
        check_planted_pairs(q, k, ref, planted, scale=kw.get("scale"), label=label)
    st = check_attn_bwd((dq, dk, dv), ref, label=label)
    print(label, {k_: f"{v_:.3g}" for k_, v_ in st.items()})
    if worst is not None:
        for k_, v_ in st.items():
            worst[k_] = max(worst.get(k_, 0.0), v_)
    return st
