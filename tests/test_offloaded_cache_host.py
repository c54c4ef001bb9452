"""CPU tests of the K/V cache partly in pinned host memory (kv_cache.OffloadedKVCache, ops.attention_decode_host).

* Placement (kv_cache.device_layers): the 16K and 128K prompts keep the plain device cache on an 80 GB card with the
  14B weights resident, the 1M and 2M prompts offload, and the edges of the budget.
* The C-call sequence, with the recording stub library of test_ops_args_host.py: an offloaded prefill makes the
  attention calls of the step without a cache plus one device-to-host row copy per layer call (whole, row-chunked
  and streamed plans); a decode step runs lv_attn_fwd + merge on device layers, and the row copy,
  lv_attn_decode_host and the merge on host layers.
* Refusals, with nothing launched: the wrapper's argument errors, the C ABI's null and size checks, a multi-token
  call on a filled offloaded cache, packed rows.
* On the CPU oracle (tests/hostlogic.py): generate() gives the same tokens with a device cache and an offloaded one,
  for the HF model with images and for B200GPTVLModel through inference_params, with the constants patched so that
  the offloaded prefill streams.  The GPU twin is tests/test_gpu_offloaded_cache.py.
"""
import contextlib
import ctypes
import types

import pytest
import torch

from long_vita_b200 import kv_cache, ops
from long_vita_b200.config import LongVITAConfig
from long_vita_b200.hf import modeling
from long_vita_b200.kv_cache import KVCache, OffloadedKVCache, device_layers
from long_vita_b200.megatron import checkpoint as ck
from long_vita_b200.weights import synthetic_state_dict
from tests.test_ops_args_host import P, _bf16, lib  # noqa: F401  (lib is the recording-stub fixture)
from tests.test_row_chunks_host import _inputs, _stub_layer
from tests.test_stream_layer_host import _constants, stream_oracle_ops

GB = 10 ** 9


# ------------------------------------------------------------------------------------------------
# placement
# ------------------------------------------------------------------------------------------------
def _weight_bytes(cfg):
    H, I, V = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size
    qkv = (cfg.num_attention_heads + 2 * cfg.num_key_value_heads) * cfg.head_dim
    layer = qkv * H + qkv + H * cfg.num_attention_heads * cfg.head_dim + 3 * H * I + 2 * H
    return 2 * (cfg.num_hidden_layers * layer + 2 * V * H + H)


def _free_on_80gb(cfg):
    """An H100 80GB (85.0e9 bytes) with the 14B decoder weights and ~1 GB of ViT weights and context resident."""
    return int(85.0 * GB) - _weight_bytes(cfg) - GB


def _placement(T, new=1024):
    cfg = LongVITAConfig()
    streamed = T > modeling.STREAM_THRESHOLD
    return device_layers(_free_on_80gb(cfg), T + new, cfg.num_hidden_layers, 2 * 2 * cfg.num_key_value_heads * 128,
                         T * modeling.prefill_bytes_per_token(cfg, T, False),
                         T * modeling.prefill_bytes_per_token(cfg, T, streamed))


def test_prefill_bytes_per_token_at_the_14b_geometry():
    cfg = LongVITAConfig()
    assert modeling.prefill_bytes_per_token(cfg, 131072, False) == 103_936
    assert modeling.prefill_bytes_per_token(cfg, 1058816, False) == 35_328
    assert modeling.prefill_bytes_per_token(cfg, 2115584, True) == 14_848


@pytest.mark.parametrize("T,n_dev", [(18432, 48), (131072, 48), (1058816, 2), (2115584, 2)])
def test_placement_at_product_lengths(T, n_dev):
    """16K and 128K keep the whole device cache; 1M keeps 2 layers beside the row-chunked prefill, 2M 2 beside the
    streamed one (4.34 and 8.67 GB per layer)."""
    assert 40 * GB < _free_on_80gb(LongVITAConfig()) < 60 * GB
    assert _placement(T) == n_dev


def test_placement_edges():
    L, cap, row, pre, off, res = 4, 1000, 4096, 10_000, 6_000, kv_cache.KV_RESERVE
    fit = L * cap * row + pre + res
    assert device_layers(fit, cap, L, row, pre, off) == L                       # exactly fits: the plain cache
    assert device_layers(None, cap, L, row, pre, off) == L                      # no budget (a CPU cache)
    assert device_layers(fit - 1, cap, L, row, pre, off) == L - 1                # one byte short: at most L - 1
    assert device_layers(off + res + 2 * cap * row, cap, L, row, pre, off) == 2
    assert device_layers(off + res + 2 * cap * row - 1, cap, L, row, pre, off) == 1
    assert device_layers(off + res, cap, L, row, pre, off) == 0
    assert device_layers(0, cap, L, row, pre, off) == 0


def test_make_cache_chooses_the_plain_cache_when_it_fits(monkeypatch):
    monkeypatch.setattr(kv_cache, "device_free_bytes", lambda dev: None)
    c = kv_cache.make_cache(3, 100, 1, 128, "cpu", prefill_bytes=0, offloaded_prefill_bytes=0)
    assert type(c) is KVCache and len(c.k) == 3
    with _host_memory(monkeypatch):
        monkeypatch.setattr(kv_cache, "device_free_bytes", lambda dev: kv_cache.KV_RESERVE + 100 * 512)
        c = kv_cache.make_cache(3, 100, 1, 128, "cpu", prefill_bytes=0, offloaded_prefill_bytes=0)
    assert type(c) is OffloadedKVCache and c.n_dev == 1 and len(c.host) == 2
    assert c.host[0].shape == (100, 256) and c.host_bytes() == 2 * 100 * 512 and c.bytes() == 100 * 512


# ------------------------------------------------------------------------------------------------
# the C-call sequence (recording stub)
# ------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _host_memory(monkeypatch):
    """Host buffers as plain CPU tensors that the wrappers take for pinned ones."""
    monkeypatch.setattr(ops, "pinned_rows", lambda rows, cols: torch.zeros(rows, cols, dtype=torch.bfloat16))
    monkeypatch.setattr(ops, "_is_pinned", lambda t: not t.is_cuda)
    yield


_ATTN = ("lv_attn_fwd", "lv_attn_decode_merge", "lv_attn_decode_host", "lv_rows_to_host")


def _attn_calls(calls):
    return [c for c in calls if c[0] in _ATTN]


def _run(layers, T, cache, rows=None):
    x, cos, sin = _bf16(T, 256), _bf16(T, 128), _bf16(T, 128)
    attend = modeling.attention_step(cache, rows=T if rows is None else rows)
    modeling.run_layers(layers, x, cos, sin, attend, _bf16(256), 1e-6, cache=cache, donate=True)


@pytest.mark.parametrize("plan", ["whole", "row-chunked", "streamed"])
def test_offloaded_prefill_and_decode_calls(lib, monkeypatch, plan):  # noqa: F811
    """Stub layers (2 q heads, 1 kv head of 128): layer 0 on the device, layer 1 on the host, T = 300."""
    T, row = 300, 2 * 128 * 2
    layers = [_stub_layer()[1] for _ in range(2)]
    consts = {"whole": (), "row-chunked": (200, 128), "streamed": (200, 128, 200)}[plan]
    with _host_memory(monkeypatch), _constants(*consts):
        lib.calls.clear()
        _run(layers, T, None)
        plain = _attn_calls(lib.calls)
        cache = OffloadedKVCache(2, 1, T + 4, 1, 128, "cpu")
        assert modeling.streams(T, modeling.attention_step(cache, rows=T)) == (plan == "streamed")
        lib.calls.clear()
        _run(layers, T, cache)
        got = _attn_calls(lib.calls)
    host = P(cache.host[0])
    spans = [(0, 128), (128, 256), (256, 300)] if plan == "streamed" else [(0, T)]
    # the device layer's attention calls, then for each of the host layer's: its rows to the host, then the call of
    # the step without a cache, over the same k (the source of the copy)
    n = len(spans)
    assert [c[0] for c in got] == ["lv_attn_fwd"] * n + ["lv_rows_to_host", "lv_attn_fwd"] * n
    assert [c[0] for c in plain] == ["lv_attn_fwd"] * 2 * n
    pitch = row if plan == "streamed" else (2 + 2) * 128 * 2
    for i, (r0, r1) in enumerate(spans):
        cp, at = got[n + 2 * i], got[n + 2 * i + 1]
        p, p0 = at[1]._obj, plain[n + i][1]._obj
        assert cp[1] == host + r0 * row and cp[3:] == (r1 - r0, row, pitch)
        assert cp[2] == p.k + r0 * pitch                      # the span's K|V rows of the layer's own k
        assert (p.sq, p.sk, p.causal, p.k_strides[1], p.q_seg_pos[0]) == (p0.sq, p0.sk, p0.causal, p0.k_strides[1],
                                                                          p0.q_seg_pos[0])
        assert p.k_strides[1] == p0.k_strides[1] and p.sk == r1
        d = got[i][1]._obj
        assert d.k == P(cache.k[0]) and (d.sq, d.sk) == (r1 - r0, r1)   # the device layer: today's call
    assert len(cache) == T

    lib.calls.clear()
    with _host_memory(monkeypatch):
        _run(layers, 1, cache)
    got = _attn_calls(lib.calls)
    assert [c[0] for c in got] == ["lv_attn_fwd", "lv_attn_fwd", "lv_attn_decode_merge",
                                   "lv_rows_to_host", "lv_attn_decode_host", "lv_attn_decode_merge"]
    assert got[3][1] == host + T * row and got[3][3:] == (1, row, row)
    dh = got[4]
    assert dh[2] == host and dh[5:11] == (T + 1, T + 4, 2, 1, 128, 3)      # length, capacity, hq, hkv, d, splits
    assert got[5][5:] == (3, 2, 1, 128)                                     # merge of 3 splits, G 2, hkv 1, d 128
    assert len(cache) == T + 1


def test_decode_host_wrapper_call_and_refusals(lib, monkeypatch):  # noqa: F811
    q, kv = _bf16(40, 128), _bf16(1000, 2 * 8 * 128)
    with pytest.raises(ValueError, match="kv_host must be pinned host memory.*not pinned"):
        ops.attention_decode_host(q, kv, 10)
    with pytest.raises(ValueError, match="kv_host must be pinned host memory, got cuda"):
        ops.attention_decode_host(q, types.SimpleNamespace(is_cuda=True, device="cuda:0"), 10)
    monkeypatch.setattr(ops, "_is_pinned", lambda t: not t.is_cuda)
    out, lse = ops.attention_decode_host(q, kv, 700, n_splits=3, return_lse=True)
    assert out.shape == (40, 128) and lse.shape == (40,)
    (name, *args), merge = lib.calls
    assert name == "lv_attn_decode_host" and args[:2] == [P(q), P(kv)]
    assert args[4:] == [700, 1000, 40, 8, 128, 3, pytest.approx(128 ** -0.5)]
    assert merge[0] == "lv_attn_decode_merge" and merge[5:] == (3, 5, 8, 128)
    lib.calls.clear()
    for bad, msg in ((dict(kv_host=kv.float()), "contiguous bfloat16"), (dict(kv_host=kv[:, :1000]), "contiguous"),
                     (dict(kv_host=kv.view(1000, 2, 1024)), "contiguous bfloat16"),
                     (dict(kv_host=_bf16(1000, 3 * 128)), "not K\\|V"), (dict(kv_host=_bf16(1000, 6 * 128)), "not K\\|V"),
                     (dict(q=_bf16(1, 40, 128)), "q must be"), (dict(length=0), "length 0 outside"),
                     (dict(length=1001), "length 1001 outside")):
        a = dict(q=q, kv_host=kv, length=10)
        a.update(bad)
        with pytest.raises(ValueError, match=msg):
            ops.attention_decode_host(a["q"], a["kv_host"], a["length"])
    assert lib.calls == []


def test_rows_to_host_call_and_refusals(lib, monkeypatch):  # noqa: F811
    qkv, dst = _bf16(6, (5 + 2) * 128), _bf16(6, 2 * 128)
    k, v = qkv[:, 5 * 128 : 6 * 128].view(6, 1, 128), qkv[:, 6 * 128 :].view(6, 1, 128)
    with pytest.raises(ValueError, match="dst must be pinned"):
        ops.kv_rows_to_host(k, v, dst)
    monkeypatch.setattr(ops, "_is_pinned", lambda t: not t.is_cuda)
    assert ops.kv_rows_to_host(k, v, dst) is dst
    assert lib.calls == [("lv_rows_to_host", P(dst), P(k), 6, 512, 7 * 128 * 2)]
    lib.calls.clear()
    for kk, vv, d, msg in ((k, qkv[:, :128].view(6, 1, 128), dst, "not the K and V halves"),
                           (k, v, _bf16(5, 256), "dst has 5 rows"), (k, v, _bf16(6, 512), "contiguous bfloat16"),
                           (k, v, dst.float(), "contiguous bfloat16")):
        with pytest.raises(ValueError, match=msg):
            ops.kv_rows_to_host(kk, vv, d)
    assert lib.calls == []


def test_abi_null_and_size_checks_without_a_gpu(lib_built):
    """Run on a thread of its own: the error text it leaves is thread-local."""
    from concurrent.futures import ThreadPoolExecutor

    with ThreadPoolExecutor(1) as ex:
        ex.submit(_abi_checks).result()


def _abi_checks():
    from long_vita_b200 import _lib

    h = _lib.lib()
    ok = dict(q=1, kv=1, o=1, lse=1, length=10, cap=10, hq=40, hkv=8, d=128, n=4, scale=0.088)
    for kw, msg in ((dict(q=None), b"null pointer"), (dict(kv=None), b"null pointer"), (dict(lse=None), b"null pointer"),
                    (dict(d=64), b"head_dim 64 not supported"), (dict(hq=41), b"bad heads"),
                    (dict(hq=24, hkv=3), b"must divide 16"), (dict(hq=72, hkv=8), b"at most 8"),
                    (dict(length=11), b"length 11 outside"), (dict(length=0), b"length 0 outside"),
                    (dict(n=0), b"bad n_splits"), (dict(scale=float("nan")), b"finite")):
        a = dict(ok, **kw)
        rc = h.lv_attn_decode_host(a["q"], a["kv"], a["o"], a["lse"], a["length"], a["cap"], a["hq"], a["hkv"], a["d"],
                                   a["n"], a["scale"], None)
        assert rc == -1 and msg in h.lv_last_error(), (kw, h.lv_last_error())
    assert h.lv_rows_to_host(None, 1, 4, 512, 512, None) == -1 and b"null pointer" in h.lv_last_error()
    assert h.lv_rows_to_host(1, 1, 4, 512, 256, None) == -1 and b"bad shape" in h.lv_last_error()
    assert h.lv_rows_to_host(1, 1, 0, 512, 512, None) == -1 and b"bad shape" in h.lv_last_error()
    p = ctypes.c_void_p()
    assert h.lv_host_alloc(0, ctypes.byref(p)) == -1 and b"bad arguments" in h.lv_last_error()


# ------------------------------------------------------------------------------------------------
# refusals of the surfaces, nothing launched
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    cfg = LongVITAConfig.tiny(layers=2, vit_layers=1)
    w = synthetic_state_dict(cfg, seed=31, dtype=torch.bfloat16, perturb=True)
    return cfg, w


def _offload(monkeypatch, cfg, n_dev):
    """Patches the device budget so that a cache keeps `n_dev` of its layers on the device (for any capacity up to
    ~1000 rows at the tiny geometry)."""
    row = 2 * 2 * cfg.num_key_value_heads * cfg.head_dim
    monkeypatch.setattr(kv_cache, "KV_RESERVE", 0)
    monkeypatch.setattr(kv_cache, "device_free_bytes", lambda dev: 10 ** 12)
    real = kv_cache.device_layers
    monkeypatch.setattr(kv_cache, "device_layers", lambda free, cap, L, *a, **kw: min(n_dev, real(free, cap, L, *a)))
    assert row == 512


def test_offloaded_cache_refusals(lib, monkeypatch, tiny):  # noqa: F811
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w)
    _offload(monkeypatch, cfg, 1)
    with _host_memory(monkeypatch):
        cache = kv_cache.make_cache(2, 64, 1, 128, "cpu", prefill_bytes=0, offloaded_prefill_bytes=0)
        assert isinstance(cache, OffloadedKVCache) and cache.n_dev == 1
        cache._len = 10                                  # a filled cache
        ids = torch.zeros(1, 3, dtype=torch.int64)
        lib.calls.clear()
        with pytest.raises(NotImplementedError, match="multi-token call on a filled cache"):
            model(input_ids=ids, past_key_values=cache, use_cache=True)
        with pytest.raises(NotImplementedError, match="packed samples"):
            model(input_ids=torch.zeros(1, 6, dtype=torch.int64), position_ids=torch.tensor([[0, 1, 2, 0, 1, 2]]),
                  use_cache=True)
        assert lib.calls == []
        assert not modeling.streams(2 ** 22, modeling.attention_step(cache, rows=1))   # only an empty cache streams


def test_megatron_refusals(lib, monkeypatch, tiny):  # noqa: F811
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel

    cfg, w = tiny
    model = B200GPTVLModel(cfg, ck.hf_to_mcore(w, cfg))
    _offload(monkeypatch, cfg, 1)
    with _host_memory(monkeypatch):
        ip = types.SimpleNamespace(key_value_memory_dict={}, max_sequence_length=64)
        ids = torch.zeros(1, 5, dtype=torch.int64)
        lib.calls.clear()
        model(ids, None, None, inference_params=ip)
        cache = ip.key_value_memory_dict["b200_kv_cache"]
        assert isinstance(cache, OffloadedKVCache) and len(cache) == 5
        lib.calls.clear()
        with pytest.raises(NotImplementedError, match="multi-token call on a filled cache"):
            model(ids[:, :2], None, None, inference_params=ip)
        model.cp = object()                              # context parallelism keeps its sharded-cache runner
        with pytest.raises(NotImplementedError, match="ContextParallelRunner"):
            model(ids, None, None, inference_params=types.SimpleNamespace(key_value_memory_dict={}))
        assert lib.calls == []


# ------------------------------------------------------------------------------------------------
# generate() on the CPU oracle: device cache and offloaded cache give the same tokens
# ------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _oracle_host_tier(monkeypatch):
    """stream_oracle_ops() with the host-tier operators restated on the CPU: the row copy is a copy, and the decode
    over host rows is ops.attention_decode over the K and V halves of those rows (the oracle's decode)."""
    def rows_to_host(k, v, dst):
        n = k.shape[0]
        dst.copy_(torch.cat([k.reshape(n, -1), v.reshape(n, -1)], dim=1))
        return dst

    def decode_host(q, kv, length, **kw):
        hkv = kv.shape[1] // (2 * q.shape[1])
        k = kv[:, : hkv * q.shape[1]].view(kv.shape[0], hkv, -1)
        v = kv[:, hkv * q.shape[1] :].view(kv.shape[0], hkv, -1)
        calls.append(length)
        return ops.attention_decode(q, k, v, length, **kw)

    calls = []
    with stream_oracle_ops():
        monkeypatch.setattr(ops, "pinned_rows", lambda rows, cols: torch.full((rows, cols), float("nan"),
                                                                               dtype=torch.bfloat16))
        monkeypatch.setattr(ops, "kv_rows_to_host", rows_to_host)
        monkeypatch.setattr(ops, "attention_decode_host", decode_host)
        yield calls


def test_hf_generate_with_an_offloaded_cache(monkeypatch, tiny):
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w)
    model.model.vision_chunk = 1
    ids, images, idx = _inputs(cfg)
    with _oracle_host_tier(monkeypatch) as host_calls, _constants(256, 128):
        ref = model.generate(ids, images=images, image_indices=idx, max_new_tokens=5)
        assert host_calls == []
        for stream in (None, 256):
            with monkeypatch.context() as m, _constants(stream=stream):
                _offload(m, cfg, 1)
                got = model.generate(ids, images=images, image_indices=idx, max_new_tokens=5)
            assert torch.equal(got, ref)
        assert host_calls == list(range(701, 705)) * 2            # layer 1 on the host, one decode per new token
        # the cache object of a generation: the host layer's rows are the device layer's layout of the same rows
        with monkeypatch.context() as m:
            _offload(m, cfg, 1)
            out = model(input_ids=ids, images=images, image_indices=idx, use_cache=True, max_cache_len=704)
        dev = model(input_ids=ids, images=images, image_indices=idx, use_cache=True, max_cache_len=704)
    c, d = out.past_key_values, dev.past_key_values
    assert isinstance(c, OffloadedKVCache) and type(d) is KVCache and len(c) == len(d) == 700
    assert torch.equal(out.logits, dev.logits)
    assert torch.equal(c.k[0][:700], d.k[0][:700]) and torch.equal(c.v[0][:700], d.v[0][:700])
    assert torch.equal(c.host[0][:700], torch.cat([d.k[1][:700].reshape(700, -1), d.v[1][:700].reshape(700, -1)], 1))
    assert c.host[0][700:].isnan().all()                                 # rows past the prompt never written


def test_megatron_generate_with_an_offloaded_cache(monkeypatch, tiny):
    """Megatron's --use-kv-cache loop: the prompt, then one token per call with its position."""
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel
    from tests.hostlogic import oracle_ops

    cfg, w = tiny
    with oracle_ops():
        model = B200GPTVLModel(cfg, ck.hf_to_mcore(w, cfg))
    model.vision_chunk = 1
    ids, images, idx = _inputs(cfg)
    s = ids.shape[1]

    def generate(n=4):
        ip = types.SimpleNamespace(external_inputs={"images": images, "indices": idx}, key_value_memory_dict={},
                                   logit_mask=None, use_kv_cache=True, max_sequence_length=s + n)
        logits = model(ids, torch.arange(s).unsqueeze(0), None, inference_params=ip)
        toks = [logits[0, -1].float().argmax().view(1, 1)]
        for i in range(n - 1):
            logits = model(toks[-1], torch.tensor([[s + i]]), None, inference_params=ip)
            toks.append(logits[0, -1].float().argmax().view(1, 1))
        return torch.cat(toks, 1), type(ip.key_value_memory_dict["b200_kv_cache"])

    with _oracle_host_tier(monkeypatch) as host_calls, _constants(256, 128):
        ref, kind = generate()
        assert kind is KVCache
        for n_dev, stream in ((1, None), (0, 256)):
            with monkeypatch.context() as m, _constants(stream=stream):
                _offload(m, cfg, n_dev)
                got, kind = generate()
            assert kind is OffloadedKVCache and torch.equal(got, ref)
    assert len(host_calls) == 3 + 2 * 3
