"""The `lv_attn_params` the attention entry points hand to the C ABI, on CPU.

`ops.attention_fwd`, `ops.attention_bwd` and `cp.CPContext._launch` pack their views through `ops.attn_params`.  Here
the library is replaced by a stub that records the structs it receives, so the pointers, shapes, strides and mask
fields each call site writes are checked without a GPU: a dense forward on strided views of a fused QKV GEMM output,
the backward of one context-parallel rank (two query segments at their global positions), and the fused
context-parallel launch (zig-zag query segments, K/V in the global-order staging buffers).
"""
import math
import types

import pytest
import torch

from long_vita_b200 import cp as CP
from long_vita_b200 import ops

T, HQ, HKV, D = 256, 4, 2, 64
ROW = (HQ + 2 * HKV) * D
E = 2       # bytes per bf16 element


def _fields(p):
    return {"q": p.q, "k": p.k, "v": p.v, "out": p.out, "lse": p.lse,
            "dims": (p.batch, p.sq, p.sk, p.hq, p.hkv, p.d),
            "q_strides": tuple(p.q_strides), "k_strides": tuple(p.k_strides), "v_strides": tuple(p.v_strides),
            "o_strides": tuple(p.o_strides), "scale": p.scale, "causal": p.causal,
            "q_seg_len": p.q_seg_len, "q_seg_pos": tuple(p.q_seg_pos), "kv_pos0": p.kv_pos0}


class _Lib:
    """Records what the attention entry points receive and reports success."""

    def __init__(self):
        self.calls = []

    def lv_attn_fwd(self, p, stream):
        self.calls.append(("fwd", _fields(p._obj)))
        return 0

    def lv_attn_bwd(self, p, stream):
        b = p._obj
        self.calls.append(("bwd", _fields(b.fwd), {
            "ptrs": (b.d_out, b.dq, b.dk, b.dv),
            "strides": tuple(tuple(getattr(b, n)) for n in ("do_strides", "dq_strides", "dk_strides", "dv_strides"))}))
        return 0

    def lv_attn_cp_fwd(self, a, cpp, stream):
        self.calls.append(("cp", _fields(a._obj)))
        return 0


@pytest.fixture
def lib(monkeypatch):
    fake = _Lib()
    monkeypatch.setattr(ops._lib, "lib", lambda: fake)
    monkeypatch.setattr(ops, "_stream", lambda: 0)
    monkeypatch.setattr(ops, "_need_cuda_bf16", lambda *ts: None)
    monkeypatch.setattr(ops, "_need_cuda", lambda t, dtype: None)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: types.SimpleNamespace(cuda_stream=0))
    return fake


def _bf16(*shape):
    return torch.zeros(*shape, dtype=torch.bfloat16)


def test_dense_forward_reads_the_fused_qkv_views_in_place(lib):
    qkv = _bf16(T, ROW)
    q = qkv[:, : HQ * D].view(T, HQ, D)
    k = qkv[:, HQ * D : (HQ + HKV) * D].view(T, HKV, D)
    v = qkv[:, (HQ + HKV) * D :].view(T, HKV, D)
    out = ops.attention_fwd(q.unsqueeze(0), k.unsqueeze(0), v.unsqueeze(0), causal=True)
    base = qkv.data_ptr()
    (kind, f), = lib.calls
    assert kind == "fwd"
    assert (f["q"], f["k"], f["v"], f["out"], f["lse"]) == (base, base + HQ * D * E, base + (HQ + HKV) * D * E,
                                                            out.data_ptr(), None)
    assert f["dims"] == (1, T, T, HQ, HKV, D)
    assert f["q_strides"] == f["k_strides"] == f["v_strides"] == (T * ROW, ROW, D)
    assert f["o_strides"] == (T * HQ * D, HQ * D, D)
    assert (f["scale"], f["causal"], f["q_seg_len"], f["q_seg_pos"], f["kv_pos0"]) == (0.125, 1, T, (0, 0), 0)

    # a chunk of 128 new rows over 384 keys: the mask is aligned to the last key; Megatron's [s, b, h, d] layout
    lib.calls.clear()
    qs, ks = _bf16(128, 1, HQ, D), _bf16(384, 1, HKV, D)
    out, lse = ops.attention_fwd(qs, ks, ks, causal=True, scale=0.5, layout="sbhd", return_lse=True)
    (_, f), = lib.calls
    assert f["dims"] == (1, 128, 384, HQ, HKV, D) and f["lse"] == lse.data_ptr() and lse.shape == (1, HQ, 128)
    assert f["q_strides"] == (HQ * D, HQ * D, D) and f["k_strides"] == (HKV * D, HKV * D, D)
    assert f["o_strides"] == (HQ * D, HQ * D, D) and out.shape == qs.shape
    assert (f["scale"], f["q_seg_len"], f["q_seg_pos"]) == (0.5, 128, (256, 0))


def test_backward_of_a_context_parallel_rank(lib):
    S, cp, rank = 4 * T, 2, 1
    c = S // (2 * cp)
    q, out, d_out = _bf16(1, T, HQ, D), _bf16(1, T, HQ, D), _bf16(1, T, HQ, D)
    K, V = _bf16(1, S, HKV, D), _bf16(1, S, HKV, D)
    lse = torch.zeros(1, HQ, T)
    odd = _bf16(1, T, HQ, D + 4)[..., :D]                     # row stride not a multiple of 8: copied first
    dq, dk, dv = ops.attention_bwd(d_out, odd, K, V, out, lse, causal=True, q_seg_len=c,
                                   q_seg_pos=(rank * c, (2 * cp - 1 - rank) * c))
    (kind, f, b), = lib.calls
    assert kind == "bwd"
    assert f["q"] != odd.data_ptr() and (f["k"], f["v"], f["out"], f["lse"]) == (K.data_ptr(), V.data_ptr(),
                                                                                   out.data_ptr(), lse.data_ptr())
    assert f["dims"] == (1, T, S, HQ, HKV, D)
    assert f["q_strides"] == f["o_strides"] == (T * HQ * D, HQ * D, D)
    assert f["k_strides"] == f["v_strides"] == (S * HKV * D, HKV * D, D)
    assert (f["scale"], f["causal"], f["q_seg_len"], f["q_seg_pos"], f["kv_pos0"]) == (0.125, 1, c, (c, 2 * c), 0)
    assert b["ptrs"] == (d_out.data_ptr(), dq.data_ptr(), dk.data_ptr(), dv.data_ptr())
    assert b["strides"] == ((T * HQ * D, HQ * D, D), (T * HQ * D, HQ * D, D), (S * HKV * D, HKV * D, D),
                            (S * HKV * D, HKV * D, D))


def _cp_context(fused_qkv: bool, cp: int, rank: int, lib) -> CP.CPContext:
    ctx = CP.CPContext.__new__(CP.CPContext)      # the peer-mapped buffers stand in as host tensors
    ctx.lib, ctx._check = lib, lambda rc, what: None
    ctx.cp, ctx.rank, ctx.epoch, ctx.device = cp, rank, 0, "cpu"
    ctx.S, ctx.T, ctx.hq, ctx.hkv, ctx.d = cp * T, T, HQ, HKV, D
    ctx.fused_qkv = fused_qkv
    ctx.row = ROW if fused_qkv else 2 * HKV * D
    ctx.k_col = HQ * D if fused_qkv else 0
    ctx.qkv = [_bf16(T, ctx.row), _bf16(T, ctx.row)]
    ctx.qkv_bytes = T * ctx.row * E
    ctx.base = ctx.ready_ptr = 0
    ctx.peer_base = [0] * cp
    ctx.k_full, ctx.v_full = _bf16(ctx.S, HKV * D), _bf16(ctx.S, HKV * D)
    ctx.blk_flags, ctx.fault = torch.zeros(ctx.S // 128, dtype=torch.int32), torch.zeros(1, dtype=torch.int32)
    return ctx


@pytest.mark.parametrize("cp,rank", [(2, 0), (4, 3)])
def test_context_parallel_launch(lib, cp, rank):
    ctx = _cp_context(True, cp, rank, lib)
    S, c = cp * T, T // 2
    out = ctx.attention()
    ctx.attention()                                            # the next epoch reads the other buffer
    (_, f), (_, f2) = lib.calls
    assert (f["q"], f2["q"]) == (ctx.qkv[0].data_ptr(), ctx.qkv[1].data_ptr())
    assert (f["k"], f["v"], f["out"], f["lse"]) == (ctx.k_full.data_ptr(), ctx.v_full.data_ptr(), out.data_ptr(), None)
    assert f["dims"] == (1, T, S, HQ, HKV, D)
    assert f["q_strides"] == (T * ROW, ROW, D)
    assert f["k_strides"] == f["v_strides"] == (S * HKV * D, HKV * D, D)
    assert f["o_strides"] == (T * HQ * D, HQ * D, D)
    assert f["scale"] == pytest.approx(1 / math.sqrt(D)) and f["causal"] == 1 and f["kv_pos0"] == 0
    assert f["q_seg_len"] == c and f["q_seg_pos"] == (rank * c, (2 * cp - 1 - rank) * c)

    # K|V copied into the exchange buffer, Q read in place unless its strides break the TMA rule
    lib.calls.clear()
    ctx = _cp_context(False, cp, rank, lib)
    qkv = _bf16(T, ROW)
    q, k, v = (qkv[:, : HQ * D].view(T, HQ, D), qkv[:, HQ * D : (HQ + HKV) * D].view(T, HKV, D),
               qkv[:, (HQ + HKV) * D :].view(T, HKV, D))
    _, lse = ctx.attention_separate(q, k, v, scale=0.25, return_lse=True)
    ctx.attention_separate(_bf16(T, HQ, D + 4)[..., :D], k, v)
    (_, f), (_, f2) = lib.calls
    assert f["q"] == qkv.data_ptr() and f["q_strides"] == (T * ROW, ROW, D) and f["lse"] == lse.data_ptr()
    assert f["scale"] == 0.25 and f["q_seg_pos"] == (rank * c, (2 * cp - 1 - rank) * c)
    assert f2["q_strides"] == (T * HQ * D, HQ * D, D)
