"""CPU tests of questions about a prefilled context (kv_cache.ContextCache / ContextSession, ops.attention_host_rows).

* The decode rule of csrc/fp8_core.h (lv_kv8_decode), built with gcc: every e4m3 code under scales from 0 to the
  largest float, through subnormal products and bf16 ties, equals (fp8.float() * scale).to(bfloat16) byte for byte.
* The C-call sequence of attention_host_rows, with the recording stub library and a recording stand-in for CUDA
  streams and events: one copy per chunk on the side stream, lv_kv_rows_dequant_fp8 for FP8 rows, one lv_attn_fwd per
  chunk over the staged rows (sk the chunk or the remainder), one merge; the stream rules (the side stream waits for
  the call's entry, a buffer is refilled only after the call that read it, each chunk is read only after its copy).
  Every refusal launches nothing.
* On the CPU oracle, the tiny model with one host layer: a question asked of the context gives the ids of a plain
  generate() over prompt + question; two questions give the same results in either order; the context's rows do not
  change.  Passing the context itself, packed rows and an overflowing question are refused before anything runs.
The GPU twin is tests/test_gpu_context_questions.py.
"""
import contextlib
import ctypes
import itertools

import numpy as np
import pytest
import torch

from long_vita_b200 import ops
from long_vita_b200.hf import modeling
from long_vita_b200.kv_cache import ContextCache, ContextSession, KVCache, OffloadedKVCache
from tests.fp8_ref import E4M3, build_shim
from tests.test_offloaded_cache_host import _oracle_host_tier, _offload, tiny  # noqa: F401  (tiny is a fixture)
from tests.test_ops_args_host import P, _bf16, lib  # noqa: F401  (lib is the recording-stub fixture)
from tests.test_row_chunks_host import _inputs
from tests.test_stream_layer_host import _constants

# ------------------------------------------------------------------------------------------------
# the decode rule, built with gcc
# ------------------------------------------------------------------------------------------------
DECODE_SHIM = r"""
#include "fp8_core.h"
void decode(const uint8_t* q, const float* s, uint16_t* out, long long n) {
  for (long long i = 0; i < n; ++i) out[i] = lv_kv8_decode(lv_e4m3_to_f32(q[i]), s[i]);
}
"""


def decode_ref(q: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """The torch statement of the rule: e4m3 bits q (uint8) with fp32 scales -> bf16 (fp8.float() * scale)."""
    return (q.view(E4M3).float() * scale).to(torch.bfloat16)


def test_decode_rule_every_code_and_scale(tmp_path):
    lib = build_shim(tmp_path, DECODE_SHIM)
    lib.decode.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_longlong]
    special = [0.0, 2.0 ** -149, 1e-40, 2.0 ** -126, 1e-30, 1e-3, 1 / 448, 0.5, 1.0, 1 + 2 ** -8, 1 + 3 * 2 ** -8,
               3 * (1 + 2 ** -8), 1.0 + 2 ** -9, 7.0, 1e30, 3e38, float(np.finfo(np.float32).max)]
    g = torch.Generator().manual_seed(5)
    rand = torch.exp(torch.empty(200).uniform_(-80.0, 80.0, generator=g)).tolist()
    scales = torch.tensor(special + rand, dtype=torch.float32)
    codes = torch.arange(256, dtype=torch.int32).to(torch.uint8)
    q = codes.repeat(scales.numel())
    s = scales.repeat_interleave(256)
    out = np.zeros(q.numel(), dtype=np.uint16)
    lib.decode(q.numpy().ctypes.data_as(ctypes.c_void_p), s.numpy().ctypes.data_as(ctypes.c_void_p),
               out.ctypes.data_as(ctypes.c_void_p), q.numel())
    got = torch.from_numpy(out.view(np.int16))
    ref = decode_ref(q, s)
    nan = ref.isnan()
    assert int(nan.sum()) == 2 * scales.numel()                          # 0x7F and 0xFF
    assert bool(got.view(torch.bfloat16)[nan].isnan().all())
    bad = (got != ref.view(torch.int16)) & ~nan
    assert not bool(bad.any()), (int(bad.sum()), q[bad][:4], s[bad][:4], got[bad][:4], ref.view(torch.int16)[bad][:4])
    prod = (q.view(E4M3).float() * s)[~nan]
    ties = (prod.view(torch.int32) & 0xFFFF) == 0x8000                  # exactly halfway between two bf16 values
    assert int(ties.sum()) > 50
    assert bool(((prod != 0) & (prod.abs() < 2.0 ** -126)).any()) and bool(prod.isinf().any())


# ------------------------------------------------------------------------------------------------
# attention_host_rows: the C-call sequence and the stream rules (recording stub)
# ------------------------------------------------------------------------------------------------
class _Timeline:
    """Stand-ins for torch.cuda streams and events that log, in program order, each record / wait / copy together
    with the number of kernel calls the stub library has recorded by then."""

    def __init__(self, lib):
        self.lib, self.log, self.active = lib, [], "cur"
        self.ids = itertools.count()
        tl = self

        class Stream:
            def __init__(self, name="side", **kw):
                self.name = name

            def wait_event(self, ev):
                tl.log.append(("wait", self.name, ev.id, len(tl.lib.calls)))

        class Event:
            def __init__(self, **kw):
                self.id = next(tl.ids)

            def record(self, stream):
                tl.log.append(("record", stream.name, self.id, len(tl.lib.calls)))

        self.Stream, self.Event, self.cur = Stream, Event, Stream("cur")

    @contextlib.contextmanager
    def stream(self, s):
        saved, self.active = self.active, s.name
        try:
            yield
        finally:
            self.active = saved

    def copy(self, dst, src):
        self.log.append(("copy", self.active, P(dst), P(src), src.shape[0], len(self.lib.calls)))


@pytest.fixture
def timeline(lib, monkeypatch):  # noqa: F811
    tl = _Timeline(lib)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: tl.cur)
    monkeypatch.setattr(torch.cuda, "Stream", tl.Stream)
    monkeypatch.setattr(torch.cuda, "Event", tl.Event)
    monkeypatch.setattr(torch.cuda, "stream", tl.stream)
    monkeypatch.setattr(ops, "_copy_to_device", tl.copy)
    monkeypatch.setattr(ops, "_is_pinned", lambda t: not t.is_cuda)
    return tl


HQ, HKV, D = 4, 2, 128


def _host(cap, fp8):
    if fp8:
        return torch.zeros(cap, ops.kv_fp8_row_bytes(HKV, D), dtype=torch.uint8)
    return _bf16(cap, 2 * HKV * D)


@pytest.mark.parametrize("fp8", [False, True], ids=["bf16", "fp8"])
@pytest.mark.parametrize("M,length,chunk", [(2, 300, 128), (5, 256, 128), (1, 1, 65536), (3, 1000, 384),
                                            (2, 129, 128)])
def test_host_rows_calls_and_stream_rules(lib, timeline, M, length, chunk, fp8):  # noqa: F811
    host = _host(length + 7, fp8)
    q = _bf16(M, HQ, D)
    out, lse = ops.attention_host_rows(q, host, length, chunk_rows=chunk, return_lse=True)
    assert out.shape == (M, HQ, D) and lse.shape == (HQ, M)
    spans = [(r, min(r + chunk, length)) for r in range(0, length, chunk)]
    n = len(spans)
    names = [c[0] for c in lib.calls]
    per_chunk = ["lv_kv_rows_dequant_fp8", "lv_attn_fwd"] if fp8 else ["lv_attn_fwd"]
    assert names == per_chunk * n + ["lv_attn_decode_merge"]
    row_bytes = host.shape[1] * host.element_size()
    copies = [e for e in timeline.log if e[0] == "copy"]
    assert [(c[1], c[3], c[4]) for c in copies] == [("side", P(host) + r0 * row_bytes, r1 - r0) for r0, r1 in spans]
    stage = [copies[i][2] for i in range(min(n, 2))]
    assert len(set(stage)) == len(stage)                                  # two staging buffers, used in turn
    step = len(per_chunk)
    for i, (r0, r1) in enumerate(spans):
        assert copies[i][2] == stage[i % 2]
        attn = lib.calls[step * i + step - 1]
        p = attn[1]._obj
        assert (p.sq, p.sk, p.hq, p.hkv, p.d, p.causal, p.batch) == (M, r1 - r0, HQ, HKV, D, 0, 1)
        assert (p.k_strides[1] == 2 * HKV * D or r1 - r0 == 1) and p.v == p.k + HKV * D * 2 and p.lse
        if fp8:
            dq = lib.calls[step * i]
            assert dq[1] == stage[i % 2] and dq[3:] == (r1 - r0, HKV, D)
            assert p.k == dq[2]                                             # attention reads the decoded rows
        else:
            assert p.k == stage[i % 2]
    merge = lib.calls[-1]
    assert merge[5:] == (n, M * HQ, 1, D)
    # stream rules, on the logged order of events
    log = timeline.log
    first = log.index(next(e for e in log if e[0] == "copy"))
    entry = log[0]
    assert entry[:2] == ("record", "cur") and entry[3] == 0
    assert ("wait", "side", entry[2]) in [e[:3] for e in log[:first]]
    recorded = {e[2]: e for e in log if e[0] == "record"}
    for i in range(n):
        ci = log.index(copies[i])
        consumer = step * i + step - 1 if not fp8 else step * i           # the kernel that reads the staged buffer
        # the current stream waits for the event recorded behind copy i before the kernel that reads it
        after_copy = [e[2] for e in log[ci + 1 :] if e[0] == "record" and e[1] == "side"][0]
        waits = [e for e in log if e[0] == "wait" and e[1] == "cur" and e[2] == after_copy]
        assert waits and waits[0][3] <= consumer
        if i >= 2:
            # copy i refills buffer i % 2 only after an event recorded behind chunk i - 2's reader
            prior = step * (i - 2) + (step - 1 if not fp8 else 0)
            side_waits = [e for e in log[:ci] if e[0] == "wait" and e[1] == "side"]
            assert any(recorded[w[2]][1] == "cur" and recorded[w[2]][3] > prior for w in side_waits)


def test_host_rows_merges_in_groups_when_the_parts_are_large(lib, timeline, monkeypatch):  # noqa: F811
    """10 chunks whose results exceed HOST_ROWS_PARTS_BYTES: merged in groups of 4, 4 and 2, then once more."""
    M, length = 3, 10 * 128 - 5
    monkeypatch.setattr(ops, "HOST_ROWS_PARTS_BYTES", 9 * M * HQ * D * 2)
    ops.attention_host_rows(_bf16(M, HQ, D), _host(length, False), length, chunk_rows=128)
    names = [c[0] for c in lib.calls]
    merge = "lv_attn_decode_merge"
    assert names == ["lv_attn_fwd"] * 4 + [merge] + ["lv_attn_fwd"] * 4 + [merge] + ["lv_attn_fwd"] * 2 + [merge] * 2
    assert [c[5] for c in lib.calls if c[0] == merge] == [4, 4, 2, 3]
    assert [c[1]._obj.sk for c in lib.calls if c[0] == "lv_attn_fwd"] == [128] * 9 + [123]


def test_host_rows_refusals_launch_nothing(lib, timeline):  # noqa: F811
    host, q = _host(1000, False), _bf16(3, HQ, D)
    fp8 = _host(1000, True)
    big = torch.zeros(1, 1, D, dtype=torch.bfloat16).expand((1 << 20) // HQ, HQ, D)
    cases = [(dict(kv_host=host.float()), "contiguous bfloat16"), (dict(kv_host=host[:, : 3 * D]), "contiguous"),
             (dict(kv_host=_bf16(1000, 3 * D)), "not K\\|V"),
             (dict(kv_host=fp8[:, :-16].contiguous()), "not FP8 K\\|V"),
             (dict(q=_bf16(3, HQ * D)), "q must be"), (dict(length=0), "length 0 outside"),
             (dict(length=1001), "length 1001 outside"), (dict(chunk_rows=0), "chunk_rows 0"),
             (dict(chunk_rows=100), "chunk_rows 100"), (dict(chunk_rows=-128), "chunk_rows -128"),
             (dict(q=big), "2\\^20")]
    for bad, msg in cases:
        a = dict(q=q, kv_host=host, length=10, chunk_rows=128)
        a.update(bad)
        with pytest.raises(ValueError, match=msg):
            ops.attention_host_rows(a["q"], a["kv_host"], a["length"], chunk_rows=a["chunk_rows"])
    ops._is_pinned = lambda t: False                                          # restored by the fixture
    with pytest.raises(ValueError, match="kv_host must be pinned host memory"):
        ops.attention_host_rows(q, host, 10)
    assert lib.calls == [] and timeline.log == []


# ------------------------------------------------------------------------------------------------
# questions on the CPU oracle, the tiny model with its layer 1 on the host
# ------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _oracle_context(monkeypatch):
    """_oracle_host_tier() with attention_host_rows restated as attention over the K and V halves of the host rows."""
    def host_rows(q, kv, length, return_lse=False, **kw):
        d = q.shape[-1]
        hkv = kv.shape[1] // (2 * d)
        k, v = kv[:length, : hkv * d].view(length, hkv, d), kv[:length, hkv * d :].view(length, hkv, d)
        calls.append((q.shape[0], length))
        return ops.attention_fwd(q.unsqueeze(0), k.unsqueeze(0), v.unsqueeze(0), causal=False, return_lse=return_lse)

    calls = []
    with _oracle_host_tier(monkeypatch) as decodes:
        monkeypatch.setattr(ops, "attention_host_rows", host_rows)
        yield calls, decodes


def test_questions_about_a_context(monkeypatch, tiny):  # noqa: F811
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w)
    model.model.vision_chunk = 1
    ids, images, idx = _inputs(cfg)
    s = ids.shape[1]
    g = torch.Generator().manual_seed(9)
    q1 = torch.randint(0, cfg.vocab_size, (1, 37), generator=g)
    q2 = torch.randint(0, cfg.vocab_size, (1, 12), generator=g)
    with _oracle_context(monkeypatch) as (host_calls, decodes), _constants(256, 128):
        refs = [model.generate(torch.cat([ids, qq], 1), images=images, image_indices=idx, max_new_tokens=5)
                for qq in (q1, q2)]
        with monkeypatch.context() as m:
            _offload(m, cfg, 1)
            ctx = model.prefill_context(ids, images, idx)
            plain = model(input_ids=ids, images=images, image_indices=idx, use_cache=True, num_logits_to_keep=1,
                          max_cache_len=s)
        assert isinstance(ctx, ContextCache) and isinstance(ctx.cache, OffloadedKVCache) and len(ctx) == s
        assert ctx.cache.capacity == s and torch.equal(ctx.logits, plain.logits)
        rows = (ctx.cache.k[0].clone(), ctx.cache.v[0].clone(), ctx.cache.host[0].clone())
        assert not hasattr(ctx, "append")
        got = {}
        for order in ((0, 1), (1, 0)):
            for i in order:
                qq = (q1, q2)[i]
                host_calls.clear()
                decodes.clear()
                out = model.generate(qq, context=ctx, max_new_tokens=5)
                assert host_calls == [(qq.shape[1], s)]                     # the question over the host layer's rows
                assert decodes == [s] * 4                                   # each answer token over the same rows
                assert torch.equal(out, refs[i][:, s:]), (i, out, refs[i][:, s:])
                got.setdefault(i, []).append(out)
                assert len(ctx) == s
        assert all(torch.equal(a, b) for a, b in got.values())
        sess = ctx.session(40)
        out = model(input_ids=q1, past_key_values=sess, use_cache=True, num_logits_to_keep=1)
        assert out.past_key_values is sess and len(sess) == s + 37 and sess.get_seq_length() == s + 37
        assert int(out.logits[0, -1].float().argmax()) == int(refs[0][0, s + 37])
    assert torch.equal(ctx.cache.k[0], rows[0]) and torch.equal(ctx.cache.v[0], rows[1])
    assert torch.equal(ctx.cache.host[0], rows[2])


def test_context_refusals(lib, tiny):  # noqa: F811
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w)
    cache = KVCache(2, 64, 1, 128, "cpu")
    cache._len = 10
    ctx = ContextCache(cache, _bf16(1, 1, cfg.vocab_size), 1, 128)
    ids = torch.zeros(1, 3, dtype=torch.int64)
    with pytest.raises(TypeError, match=r"session\("):
        model(input_ids=ids, past_key_values=ctx, use_cache=True)
    with pytest.raises(NotImplementedError, match="packed samples"):
        model(input_ids=torch.zeros(1, 6, dtype=torch.int64), position_ids=torch.tensor([[0, 1, 2, 0, 1, 2]]),
              past_key_values=ctx.session(8), use_cache=True)
    sess = ctx.session(2)
    assert isinstance(sess, ContextSession) and len(sess) == 10
    with pytest.raises(RuntimeError, match="KV cache overflow: 3 tokens > capacity 2"):
        model(input_ids=ids, past_key_values=sess, use_cache=True)
    with pytest.raises(ValueError, match="images belong"):
        model.generate(ids, images=_bf16(1, 3, 448, 448), context=ctx)
    assert lib.calls == []
    with pytest.raises(ValueError, match="no prompt"):
        ContextCache(KVCache(2, 64, 1, 128, "cpu"), _bf16(1, 1, 8), 1, 128)
