"""CPU tests of the streamed decoder layer (hf.modeling.STREAM_THRESHOLD / DecoderLayer._forward_streamed), of the
per-chunk image scatter (hf.modeling.scatter_images, ops.row_scatter) and of the attention FLOP count of a query chunk.

* The plan at the product lengths: the 16K, 128K and 1M bench prompts keep their plans, the 2M prompt streams, and
  only the plain causal attention step declares that it may be called per query chunk.
* The call sequence, with the recording stub library of test_ops_args_host.py: per span, the norm, the QKV GEMM as
  a Q launch into a span buffer and a K|V launch into the span's rows of the K|V buffer, RoPE on both, attention of
  the span's queries over k[:r1], and the MLP ending in x[r0:r1] += MLP output; no buffer of T rows but x and K|V.
* Bit-identity of the composition on the CPU oracle (tests/hostlogic.py), the constants patched down: the HF model
  with images, inputs_embeds, B200GPTVLModel with a logit mask and the `--spec` layer give torch.equal results
  streamed, whole and row-chunked; K/V-cache, packed-row and context-parallel (gloo) runs make the same operator calls
  with the stream threshold patched below their length as without.  The oracle's GEMM and attention sum in float64 so
  that a row's result cannot depend on how many rows or keys share the call.  The GPU twin is
  tests/test_gpu_stream_layer.py.
"""
import contextlib
import math
import socket
import types
from functools import partial

import pytest
import torch

from long_vita_b200 import ops
from long_vita_b200.config import LongVITAConfig
from long_vita_b200.hf import modeling
from long_vita_b200.hf.modeling import attention_step, query_chunked, row_chunks, streams
from long_vita_b200.megatron import checkpoint as ck
from long_vita_b200.weights import synthetic_state_dict
from tests import packed_oracle
from tests.hostlogic import oracle_ops
from tests.test_ops_args_host import P, _bf16, _i64, lib  # noqa: F401  (lib is the recording-stub fixture)
from tests.test_row_chunks_host import _inputs, _stub_layer, exact_oracle_ops


# ------------------------------------------------------------------------------------------------
# the plan
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,plan", [(18432, "whole"), (131072, "whole"), (1058816, "row-chunked"),
                                    (2115584, "streamed")])
def test_plan_at_product_lengths(T, plan):
    """bench.py --frames 64 / 512 / 4096 / 8192."""
    step = attention_step()
    got = "streamed" if streams(T, step) else ("row-chunked" if len(row_chunks(T)) > 1 else "whole")
    assert got == plan
    if plan == "streamed":
        assert all(r0 % 128 == 0 for r0, _ in row_chunks(T)) and min(r1 - r0 for r0, r1 in row_chunks(T)) > 4


def test_only_the_plain_causal_step_declares_query_chunks():
    from long_vita_b200.cp import exchange_attention

    T = 2115584
    assert query_chunked(attention_step()) and query_chunked(partial(attention_step(), 3))
    assert streams(T, partial(partial(attention_step(), 0)))
    assert not streams(modeling.STREAM_THRESHOLD, attention_step())
    assert not streams(T, attention_step(cu_seqlens=torch.tensor([0, 5, T], dtype=torch.int32)))
    assert not streams(T, attention_step(cache=types.SimpleNamespace()))
    assert not streams(T, exchange_attention(types.SimpleNamespace()))
    assert not streams(T, lambda q, k, v: q)


# ------------------------------------------------------------------------------------------------
# the streamed layer's C-call sequence (recording stub)
# ------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _constants(threshold=None, chunk=None, stream=None):
    names = ("ROW_CHUNK_THRESHOLD", "ROW_CHUNK", "STREAM_THRESHOLD")
    saved = [getattr(modeling, n) for n in names]
    for n, v in zip(names, (threshold, chunk, stream)):
        if v is not None:
            setattr(modeling, n, v)
    try:
        yield
    finally:
        for n, v in zip(names, saved):
            setattr(modeling, n, v)


@contextlib.contextmanager
def _allocations(T):
    """Records the shape of every torch.empty / empty_like with T rows."""
    seen, empty, empty_like = [], torch.empty, torch.empty_like

    def rec(t):
        if t.dim() and t.shape[0] == T:
            seen.append(tuple(t.shape))
        return t

    torch.empty = lambda *a, **kw: rec(empty(*a, **kw))
    torch.empty_like = lambda *a, **kw: rec(empty_like(*a, **kw))
    try:
        yield seen
    finally:
        torch.empty, torch.empty_like = empty, empty_like


@pytest.mark.parametrize("inplace", [False, True])
def test_streamed_layer_calls_run_span_by_span(lib, inplace):  # noqa: F811
    """T = 300 over spans of 128, 128, 44 (stub layer: H 256, 2 q heads, 1 kv head of 128, intermediate 256)."""
    T, H, row, kv_row = 300, 256, 256 * 2, 256 * 2
    cfg, L = _stub_layer()
    x, cos, sin = _bf16(T, H), _bf16(T, 128), _bf16(T, 128)
    att = _bf16(T, 2 * 128)

    def attend(li, q, k, v):
        lib.calls.append(("attend", q.data_ptr(), q.shape[0], k.data_ptr(), k.shape[0], k.stride(0), v.data_ptr(),
                          v.shape[0]))
        return att[: q.shape[0]]

    attend.query_chunks = True
    with _constants(200, 128, 200), _allocations(T) as big:
        xo, m = L.forward(x, None, cos, sin, partial(attend, 0), inplace=inplace)
    spans = [(0, 128), (128, 256), (256, 300)]
    assert row_chunks(T) == [(0, T)] and m is None and (P(xo) == P(x)) == inplace
    assert sorted(big) == sorted([(T, 2 * 128)] + ([] if inplace else [(T, H)]))     # K|V (and a new x)
    c = lib.calls
    per = ["lv_rmsnorm", "lv_gemm_bias_act", "lv_gemm_bias_act", "lv_rope", "lv_rope", "attend", "lv_gemm_bias_act",
           "lv_rmsnorm", "lv_gemm_bias_act", "lv_gemm_bias_act", "lv_ls_residual"]
    assert [k[0] for k in c] == per * 3
    kv = c[2][4]
    for i, (r0, r1) in enumerate(spans):
        n = r1 - r0
        a = c[11 * i : 11 * i + 11]
        assert a[0][1:3] == (P(x) + r0 * row, None) and a[0][6] == n
        h = a[0][4]
        # Q columns into a span buffer, K|V columns into rows r0:r1 of the K|V buffer: two launches, ldc = their width
        assert a[1][1:4] == (h, P(L.wqkv), P(L.bqkv)) and a[1][5:] == (n, 256, H, H, H, 256, 0)
        assert a[2][1:5] == (h, P(L.wqkv) + 256 * H * 2, P(L.bqkv) + 256 * 2, kv + r0 * kv_row)
        assert a[2][5:] == (n, 256, H, H, H, 256, 0)
        q = a[1][4]
        assert a[3][1:5] == (q, q, P(cos) + r0 * 256, P(sin) + r0 * 256) and a[3][5:9] == (n, 2, 128, 256)
        assert a[4][1:5] == (kv + r0 * kv_row, kv + r0 * kv_row, P(cos) + r0 * 256, P(sin) + r0 * 256)
        assert a[4][5:9] == (n, 1, 128, 256)
        assert a[5] == ("attend", q, n, kv, r1, 256, kv + 128 * 2, r1)                   # k[:r1], v[:r1]
        assert a[6][1:3] == (P(att), P(L.wo)) and a[6][5] == n
        assert a[7][1:3] == (a[6][4], P(x) + r0 * row) and a[7][5:7] == (P(xo) + r0 * row, n)
        assert a[8][1:3] == (a[7][4], P(L.w_gate_up)) and a[8][5] == n
        assert a[10][1:3] == (P(xo) + r0 * row, a[9][4]) and a[10][5:] == (P(xo) + r0 * row, n, H)


def test_run_layers_shares_one_kv_buffer(lib):  # noqa: F811
    T = 300
    layers = [_stub_layer()[1] for _ in range(3)]
    x, cos, sin, att = _bf16(T, 256), _bf16(T, 128), _bf16(T, 128), _bf16(T, 256)
    seen = []

    def attend(li, q, k, v):
        seen.append((li, k.data_ptr()))
        return att[: q.shape[0]]

    attend.query_chunks = True
    with _constants(200, 128, 200), _allocations(T) as big:
        modeling.run_layers(layers, x, cos, sin, attend, _bf16(256), 1e-6, donate=True)
    assert [li for li, _ in seen] == [0, 0, 0, 1, 1, 1, 2, 2, 2] and len({p for _, p in seen}) == 1
    assert big == [(T, 256)]                       # the K|V buffer; x is donated and the final norm writes it per span
    assert [c[0] for c in lib.calls[-3:]] == ["lv_rmsnorm"] * 3


# ------------------------------------------------------------------------------------------------
# row_scatter and the attention FLOP count (recording stub)
# ------------------------------------------------------------------------------------------------
def test_row_scatter_call_and_refusals(lib):  # noqa: F811
    out, x, idx = _bf16(10, 64), _bf16(2, 2, 64), _i64(4)
    assert ops.row_scatter(x, idx, out) is out
    assert lib.calls == [("lv_row_scatter", P(x), P(idx), P(out), 4, 10, 64)]
    lib.calls.clear()
    with pytest.raises(ValueError, match="row_scatter: idx"):
        ops.row_scatter(x, _i64(3), out)
    with pytest.raises(ValueError, match="row_scatter: out"):
        ops.row_scatter(x, idx, _bf16(10, 128)[:, :64])
    with pytest.raises(ValueError, match="row_scatter: idx"):
        ops.row_scatter(x, idx.int(), out)
    assert lib.calls == []


@pytest.mark.parametrize("sq,sk,kw,pairs", [
    (256, 1024, {}, 256 * 768 + 256 * 257 / 2),               # a query chunk over its key prefix: the visible pairs
    (1024, 1024, {}, 1024 * 1025 / 2),                          # self-attention: unchanged
    (256, 1024, {"q_seg_pos": (0, 0)}, 256 * 1024),             # explicit segments: the upper bound, unchanged
    (256, 1024, {"kv_pos0": 128}, 256 * 1024),
])
def test_attention_flop_count(lib, monkeypatch, sq, sk, kw, pairs):  # noqa: F811
    rec = []
    timer = types.SimpleNamespace(start=lambda: "ev", stop=lambda kind, fl, ev: rec.append((kind, fl)))
    monkeypatch.setattr(ops, "_TIMER", timer)
    q, k, v = _bf16(1, sq, 8, 128), _bf16(1, sk, 2, 128), _bf16(1, sk, 2, 128)
    ops.attention_fwd(q, k, v, causal=True, **kw)
    assert rec == [("attn_fwd", 4.0 * 8 * 128 * pairs)]


# ------------------------------------------------------------------------------------------------
# bit-identity on the CPU oracle
# ------------------------------------------------------------------------------------------------
def _attention_fwd64(q, k, v, *, causal, scale=None, layout="bshd", return_lse=False, out=None, cu_seqlens=None,
                     **kw):
    """Attention in float64, each query row on its own: a row's result does not depend on the rows or the masked
    keys that share the call."""
    if cu_seqlens is not None or layout != "bshd" or kw or return_lse:
        return packed_oracle._attention_fwd(q, k, v, causal=causal, scale=scale, layout=layout, return_lse=return_lse,
                                            out=out, cu_seqlens=cu_seqlens, **kw)
    sq, hq, d = q.shape[1:]
    sk, hkv = k.shape[1:3]
    g = hq // hkv
    s = torch.einsum("bqhd,bkhd->bhqk", q.double(), k.double().repeat_interleave(g, dim=2))
    s = s * (1.0 / math.sqrt(d) if scale is None else scale)
    if causal:
        s = s.masked_fill(torch.arange(sk)[None, :] > torch.arange(sq)[:, None] + (sk - sq), float("-inf"))
    p = torch.nan_to_num(torch.softmax(s, dim=-1), nan=0.0)
    o = torch.einsum("bhqk,bkhd->bqhd", p, v.double().repeat_interleave(g, dim=2)).to(torch.bfloat16).contiguous()
    if out is not None:
        out.copy_(o)
        o = out
    return o


def _row_scatter(x, idx, out):
    out[idx.view(-1)] = x.reshape(-1, out.shape[1])
    return out


@contextlib.contextmanager
def stream_oracle_ops():
    """exact_oracle_ops() with a float64 attention and ops.row_scatter on the CPU."""
    with exact_oracle_ops() as o:
        o.attention_fwd = _attention_fwd64           # restored by oracle_ops on exit
        saved, o.row_scatter = o.row_scatter, _row_scatter
        try:
            yield o
        finally:
            o.row_scatter = saved


def _attention_calls(o):
    """Counts the decoder attention calls whose queries are fewer than their keys (query chunks)."""
    n, fn = [0], o.attention_fwd

    def wrapped(q, k, v, **kw):
        n[0] += q.shape[1] < k.shape[1]
        return fn(q, k, v, **kw)
    o.attention_fwd = wrapped
    return n


def _three_plans(fn, T, scatters=None):
    """fn() whole, row-chunked (128-row chunks) and streamed (the same spans); asserts the plans are what they say and,
    if `scatters` is given, that only the streamed run makes that many per-chunk image scatters (ops.row_scatter)."""
    with stream_oracle_ops() as o:
        n = _attention_calls(o)
        rows, scatter = [0], o.row_scatter

        def counted(*a, **kw):
            rows[0] += 1
            return scatter(*a, **kw)
        o.row_scatter = counted                    # stream_oracle_ops restores the wrapper on exit
        whole = fn()
        assert n[0] == 0
        with _constants(256, 128):
            chunked = fn()
        assert n[0] == 0 and rows[0] == 0
        with _constants(256, 128, 256):
            assert streams(T, attention_step())
            streamed = fn()
        assert n[0] > 0
        assert scatters is None or rows[0] == scatters, rows[0]
    return whole, chunked, streamed


def _equal(a, b):
    if isinstance(a, torch.Tensor):
        return torch.equal(a, b)
    return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))


@pytest.fixture(scope="module")
def tiny():
    cfg = LongVITAConfig.tiny(layers=2, vit_layers=1)
    w = synthetic_state_dict(cfg, seed=31, dtype=torch.bfloat16, perturb=True)
    return cfg, w


def test_hf_model_with_images(tiny):
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w)
    model.model.vision_chunk = 1                   # one scatter per frame above the threshold
    ids, images, idx = _inputs(cfg)

    def run():
        a = model(input_ids=ids, images=images, image_indices=idx, num_logits_to_keep=100)
        b = model(input_ids=ids, images=images, image_indices=idx, output_hidden_states=True)
        return a.logits, b.logits, b.hidden_states

    whole, chunked, streamed = _three_plans(run, ids.shape[1], scatters=2 * 2)
    assert _equal(streamed, whole) and _equal(chunked, whole)
    assert torch.equal(whole[0][0], whole[1][0, -100:])


def test_inputs_embeds_are_not_overwritten(tiny):
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w)
    emb = torch.randn(1, 600, cfg.hidden_size, generator=torch.Generator().manual_seed(4)).to(torch.bfloat16)
    keep = emb.clone()
    whole, chunked, streamed = _three_plans(lambda: model(inputs_embeds=emb).logits, 600)
    assert torch.equal(streamed, whole) and torch.equal(chunked, whole) and torch.equal(emb, keep)


def test_megatron_model_with_logit_mask(tiny):
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel

    cfg, w = tiny
    with oracle_ops():
        model = B200GPTVLModel(cfg, ck.hf_to_mcore(w, cfg))
    model.vision_chunk = 1
    ids, images, idx = _inputs(cfg)
    s = ids.shape[1]
    mask = torch.zeros(1, s, dtype=torch.bool)
    mask[0, [3, 130, 257, 699]] = True
    whole, chunked, streamed = _three_plans(lambda: model(ids, torch.arange(s).unsqueeze(0), None, logit_mask=mask,
                                                          external_inputs={"images": images, "indices": idx}), s,
                                            scatters=2)
    assert whole.shape == (1, 4, cfg.vocab_size) and torch.equal(streamed, whole) and torch.equal(chunked, whole)


def test_megatron_model_through_inference_params_without_kv_cache(tiny):
    """Megatron's generation loop without --use-kv-cache: external inputs and the logit mask come in
    inference_params, with use_kv_cache False.  That is no cache, so the vision phase streams with the decoder."""
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel

    cfg, w = tiny
    with oracle_ops():
        model = B200GPTVLModel(cfg, ck.hf_to_mcore(w, cfg))
    model.vision_chunk = 1
    ids, images, idx = _inputs(cfg)
    s = ids.shape[1]
    mask = torch.zeros(1, s, dtype=torch.bool)
    mask[0, [3, 130, 257, 699]] = True

    def run():
        ip = types.SimpleNamespace(external_inputs={"images": images, "indices": idx}, key_value_memory_dict={},
                                   logit_mask=mask, use_kv_cache=False)
        return model(ids, torch.arange(s).unsqueeze(0), None, inference_params=ip)

    whole, chunked, streamed = _three_plans(run, s, scatters=2)
    assert whole.shape == (1, 4, cfg.vocab_size) and torch.equal(streamed, whole) and torch.equal(chunked, whole)


def test_megatron_model_external_inputs_none(tiny):
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel

    cfg, w = tiny
    with oracle_ops():
        model = B200GPTVLModel(cfg, ck.hf_to_mcore(w, cfg))
    ids = _inputs(cfg)[0]
    pos = torch.arange(ids.shape[1]).unsqueeze(0)
    with stream_oracle_ops(), _constants(256, 128, 256):
        assert torch.equal(model(ids, pos, None, external_inputs=None), model(ids, pos, None))


def test_spec_layer(tiny):
    """The `--spec` layer streams too, adds the MLP output itself and leaves Megatron's hidden_states untouched."""
    from long_vita_b200.megatron.transformer_layer import B200TransformerLayer
    from oracle import ops as O

    cfg, w = tiny
    mc = ck.hf_to_mcore(w, cfg)
    mcfg = types.SimpleNamespace(hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_attention_heads,
                                 num_query_groups=cfg.num_key_value_heads, kv_channels=cfg.head_dim,
                                 ffn_hidden_size=cfg.intermediate_size, layernorm_epsilon=cfg.rms_norm_eps,
                                 hidden_dropout=0.0, attention_dropout=0.0, params_dtype=torch.bfloat16)
    layer = B200TransformerLayer(mcfg, layer_number=1)
    layer.load_state_dict({k[len("decoder.layers.0."):]: v for k, v in mc.items() if k.startswith("decoder.layers.0.")})
    s = 520
    x = torch.randn(s, 1, cfg.hidden_size, generator=torch.Generator().manual_seed(8)).to(torch.bfloat16)
    keep = x.clone()
    freqs = torch.outer(torch.arange(s).float(), O.rope_inv_freq(cfg.head_dim, cfg.rope_theta))
    rotary = torch.cat((freqs, freqs), dim=-1).view(s, 1, 1, cfg.head_dim)
    whole, chunked, streamed = _three_plans(lambda: layer(hidden_states=x, rotary_pos_emb=rotary)[0], s)
    assert torch.equal(streamed, whole) and torch.equal(chunked, whole) and torch.equal(x, keep)


# -- the surfaces that keep their plan: the same operator calls with the stream threshold below their length --------
_RECORDED = ("rmsnorm", "linear", "rope", "attention_fwd", "attention_decode", "ls_residual", "embed_scatter",
             "row_scatter")


def _shapes(a):
    if isinstance(a, torch.Tensor):
        return (tuple(a.shape), a.stride())
    if isinstance(a, (tuple, list)):
        return tuple(_shapes(x) for x in a)
    return a


@contextlib.contextmanager
def _recording(o):
    """Records (operator, argument shapes and strides) of every call of the _RECORDED operators of `o`."""
    calls, saved = [], {n: getattr(o, n) for n in _RECORDED if hasattr(o, n)}

    def wrap(name, fn):
        def run(*a, **kw):
            calls.append((name, _shapes(a), tuple(sorted((k, _shapes(v)) for k, v in kw.items()))))
            return fn(*a, **kw)
        return run
    for n, fn in saved.items():
        setattr(o, n, wrap(n, fn))
    try:
        yield calls
    finally:
        for n, fn in saved.items():
            setattr(o, n, fn)


def _same_calls(fn, T):
    """fn() with the row-chunk constants patched down, then also with STREAM_THRESHOLD below T: same calls, same
    results."""
    with stream_oracle_ops() as o, _constants(256, 128):
        with _recording(o) as before:
            a = fn()
        with _constants(stream=128), _recording(o) as after:
            assert T > modeling.STREAM_THRESHOLD
            b = fn()
    assert len(before) > 20 and after == before
    return a, b


def test_kv_cache_keeps_its_calls(tiny):
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w)
    ids, images, idx = _inputs(cfg)
    ids, images, idx = ids[:, :600], images[:1], idx[:, :1]

    def run():
        out = model(input_ids=ids, images=images, image_indices=idx, use_cache=True, num_logits_to_keep=1,
                    max_cache_len=ids.shape[1] + 4)
        cache, logits = out.past_key_values, [out.logits]
        for _ in range(3):
            tok = logits[-1][0, -1].float().argmax().view(1, 1)
            logits.append(model(input_ids=tok, past_key_values=cache, use_cache=True, num_logits_to_keep=1).logits)
        return logits

    a, b = _same_calls(run, 600)
    assert _equal(a, b)


def test_packed_rows_keep_their_calls(tiny):
    """Images included: a packed row's vision phase keeps its one-shot embedding, as its decoder keeps its plan."""
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w)
    ids, images, idx = _inputs(cfg)
    pos = torch.cat([torch.arange(450), torch.arange(250)]).unsqueeze(0)
    a, b = _same_calls(lambda: model(input_ids=ids, images=images, image_indices=idx, position_ids=pos).logits, 700)
    assert torch.equal(a, b)


def test_megatron_packed_rows_and_kv_cache_keep_their_calls(tiny):
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel

    cfg, w = tiny
    with oracle_ops():
        model = B200GPTVLModel(cfg, ck.hf_to_mcore(w, cfg))
    ids, images, idx = _inputs(cfg)
    s = ids.shape[1]
    ext = {"images": images, "indices": idx}
    pos = torch.cat([torch.arange(450), torch.arange(250)]).unsqueeze(0)
    a, b = _same_calls(lambda: model(ids, pos, None, external_inputs=ext), s)
    assert torch.equal(a, b)

    def cached():
        ip = types.SimpleNamespace(external_inputs=ext, key_value_memory_dict={}, max_sequence_length=s + 4)
        return model(ids, torch.arange(s).unsqueeze(0), None, inference_params=ip)
    a, b = _same_calls(cached, s)
    assert torch.equal(a, b)


def test_streamed_layer_refuses_a_qkv_buffer(lib):  # noqa: F811
    T = 300
    _, L = _stub_layer()
    attend = types.SimpleNamespace(query_chunks=True)
    with _constants(200, 128, 200), pytest.raises(ValueError, match="takes no qkv_out"):
        L.forward(_bf16(T, 256), None, None, None, attend, qkv_out=_bf16(T, 512))
    assert lib.calls == []


def _cp_worker(rank, world, port, path):
    import os

    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from long_vita_b200 import cp as CP
        from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel
        from long_vita_b200.synthetic import build_prompt
        from tests.test_megatron_model_host import _GlooCPContext

        torch.set_num_threads(2)
        cfg = LongVITAConfig.tiny(layers=2, vit_layers=1)
        mc = ck.hf_to_mcore(synthetic_state_dict(cfg, seed=31, dtype=torch.bfloat16, perturb=True), cfg)
        ids, idx = build_prompt(cfg, 2, n_text=20, pad_multiple=2 * world * 128)
        images = torch.randn(2, 3, 448, 448, generator=torch.Generator().manual_seed(3)).to(torch.bfloat16)
        sh = CP.shard_prompt(ids, idx, world, rank, cfg.visual.tokens_per_image)
        tpi = cfg.visual.tokens_per_image
        ext = {"images": images[sh.image_sel], "src_indices": (sh.src_idx // tpi, sh.src_idx % tpi),
               "tgt_indices": (torch.zeros_like(sh.dst_idx), sh.dst_idx)}
        with oracle_ops():
            model = B200GPTVLModel(cfg, mc, cp=_GlooCPContext(ids.shape[1], cfg.num_attention_heads,
                                                               cfg.num_key_value_heads, cfg.head_dim))
        a, b = _same_calls(lambda: model(sh.input_ids, sh.position_ids.unsqueeze(0), None, external_inputs=ext),
                           sh.input_ids.shape[1])
        torch.save({"equal": torch.equal(a, b), "T": sh.input_ids.shape[1]}, f"{path}.{rank}")
    finally:
        dist.destroy_process_group()


def test_context_parallel_keeps_its_calls(tmp_path):
    """2 ranks, the K/V exchange emulated by a gloo all-gather: each rank's operator calls and logits are the same
    with the stream threshold below its shard's length."""
    import torch.multiprocessing as mp

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    path = str(tmp_path / "cp")
    mp.spawn(_cp_worker, args=(2, port, path), nprocs=2, join=True)
    for r in range(2):
        res = torch.load(f"{path}.{r}")
        assert res["equal"] and res["T"] > 128, res


# ------------------------------------------------------------------------------------------------
# the per-chunk image scatter
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", [1, 2, 3])
def test_scatter_images_equals_the_one_shot_embedding(tiny, chunk):
    """Three frames, their rows in a shuffled order across the prompt: every chunking gives the bits of
    embed_scatter(encode_images(...))."""
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w).model
    g = torch.Generator().manual_seed(6)
    tpi, s = cfg.visual.tokens_per_image, 1000
    ids = torch.randint(0, cfg.vocab_size, (1, s), generator=g)
    images = torch.randn(3, 3, 448, 448, generator=g).to(torch.bfloat16)
    dst = torch.randperm(s, generator=g)[: 3 * tpi]
    with stream_oracle_ops() as o:
        whole = o.embed_scatter(ids, model.embed_tokens,
                                modeling.encode_images(model.vision_model, model.vision_projection, images), dst)
        x = o.embed_scatter(ids, model.embed_tokens)
        got = modeling.scatter_images(x, model.vision_model, model.vision_projection, images, dst, chunk)
        assert got is x and torch.equal(got, whole)
        with pytest.raises(ValueError, match="scatter_images"):
            modeling.scatter_images(x, model.vision_model, model.vision_projection, images, dst[:-1], chunk)
