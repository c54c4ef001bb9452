"""Float64 reference for the gradients of the fused attention, at training lengths.

`attention_grads` computes dQ on a set of query rows and dK / dV on a set of key rows of

    out = softmax(scale * q k^T + mask) v,   mask: key hidden iff kv_pos > q_pos (causal),

the attention `lv_attn_fwd` / `lv_attn_bwd` define (query head h reads kv head h // G, G = hq / hkv; positions are
global, so zig-zag context-parallel segments and `kv_pos0` are just other `q_pos` / `kv_pos`).  It runs on the device
of its inputs, CPU or CUDA, in float64, with the textbook formulas per query row i:

    s = scale q_i K^T (masked), lse, P = exp(s - lse), O_i = P V, delta_i = rowsum(dO_i * O_i),
    dQ_i = scale (P * (dO_i V^T - delta_i)) K,   dV_j = sum_i P_ij dO_i,   dK_j = scale sum_i dS_ij q_i.

Rows are independent, so work goes in (query chunk x query heads of one kv group) blocks sized to keep the score
block near `block_bytes`.  For dK / dV only the query chunks that can see some requested key are visited, each with
its own lse and delta.  With a causal mask a chunk's scores stop at the last key it can see (kv_pos must be
non-decreasing).  A query row that sees no key has P = 0 and gets dQ = 0, never NaN.

Why `out=`: the backward reads the forward's bf16 output, and delta = rowsum(dO * O) taken from it differs from the
exact delta by the output rounding.  In dS = P (dP - delta) that difference is not damped where dP - delta is small
against dP (rows that see few keys, a peaked softmax), so at bf16 precision the gradient of the exact function is the
wrong target for those rows; flash-attn 2's backward shows the same difference.  With `out` the reference computes the
gradient the backward is asked for, given its inputs.
"""
import math
from typing import Optional

import torch


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
                    q_rows=None, kv_rows=None, out=None, block_bytes: int = 1 << 30):
    """q / d_out [b, sq, hq, d], k / v [b, sk, hkv, d], any float dtype, all on one device.  `q_pos` [sq] / `kv_pos`
    [sk] are the global positions (defaults: bottom-right aligned, q_pos = i + sk - sq, kv_pos = j).  `q_rows` /
    `kv_rows` select the rows whose dQ / dK, dV are wanted (sorted int64 indices; None = all rows, an empty tensor =
    none).  `out` [b, sq, hq, d], if given, is the forward output the backward reads: delta = rowsum(dO * out) is then
    taken from it instead of from the exact O = P V, as lv_attn_bwd and flash-attn's backward do.  Returns float64
    (dq [b, |q_rows|, hq, d], dk [b, |kv_rows|, hkv, d], dv [b, |kv_rows|, hkv, d])."""
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
    R = torch.arange(sq, device=dev) if q_rows is None else torch.as_tensor(q_rows).to(dev, torch.int64)
    J = None if kv_rows is None else torch.as_tensor(kv_rows).to(dev, torch.int64)
    nJ = sk if J is None else J.numel()
    dq = torch.zeros((b, R.numel(), hq, d), dtype=f64, device=dev)
    dk = torch.zeros((b, nJ, hkv, d), dtype=f64, device=dev)
    dv = torch.zeros((b, nJ, hkv, d), dtype=f64, device=dev)

    # query rows to visit: the dQ rows and every row that sees some requested key; dq_slot[i] = slot of row i in dq
    want_dq = torch.zeros(sq, dtype=torch.bool, device=dev)
    want_dq[R] = True
    visit = want_dq.clone()
    if nJ and causal:
        visit |= q_pos >= kv_pos[J[0] if J is not None else 0]
    elif nJ:
        visit[:] = True
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
            # keys [0, nk) hold every key a row of this chunk can see
            nk = int(torch.searchsorted(kv_pos, pos.max(), right=True)) if causal else sk
            if nk == 0 and not bool(want_dq[idx].any()):
                continue
            kc, vc = kf[:, :nk], vf[:, :nk]
            qf = q[:, idx, heads].to(f64).permute(0, 2, 1, 3)                   # [b, G, n, d]
            dof = d_out[:, idx, heads].to(f64).permute(0, 2, 1, 3)
            s = torch.matmul(qf * scale, kc.unsqueeze(1).transpose(-1, -2))    # [b, G, n, nk]
            if causal:
                s.masked_fill_(kv_pos[None, :nk] > pos[:, None], float("-inf"))
            lse = torch.logsumexp(s, dim=-1, keepdim=True)
            p = torch.exp(s - torch.where(torch.isinf(lse), torch.zeros_like(lse), lse))   # a row seeing nothing: 0
            del s
            if out is None:
                o = torch.matmul(p, vc.unsqueeze(1))
            else:
                o = out[:, idx, heads].to(f64).permute(0, 2, 1, 3)
            delta = (dof * o).sum(-1, keepdim=True)                            # [b, G, n, 1]
            del o
            slot = dq_slot[idx]
            sel = slot >= 0
            ds = None
            if bool(sel.any()):
                all_rows = bool(sel.all())
                pr, dor, dlr = (p, dof, delta) if all_rows else (p[:, :, sel], dof[:, :, sel], delta[:, :, sel])
                ds = pr * (torch.matmul(dor, vc.unsqueeze(1).transpose(-1, -2)) - dlr)
                g = scale * torch.matmul(ds, kc.unsqueeze(1))                     # [b, G, n_sel, d]
                dq[:, slot[sel], heads] = g.permute(0, 2, 1, 3)
                if not all_rows:
                    ds = None
            if nJ:
                if J is None:
                    cols, n_in = slice(0, nk), nk
                else:
                    n_in = int(torch.searchsorted(J, nk))                        # requested keys below nk (J sorted)
                    cols = J[:n_in]
                pj = p[..., cols]
                if ds is not None and J is None:
                    dsj = ds
                else:
                    dsj = pj * (torch.matmul(dof, vc[:, cols].unsqueeze(1).transpose(-1, -2)) - delta)
                dv[:, :n_in, h] += torch.matmul(pj.transpose(-1, -2), dof).sum(1)
                dk[:, :n_in, h] += scale * torch.matmul(dsj.transpose(-1, -2), qf).sum(1)
            del p, ds
    return dq, dk, dv
