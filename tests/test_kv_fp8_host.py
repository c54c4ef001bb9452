"""CPU tests of the FP8 (e4m3) host tier of the K/V cache (kv_cache.OffloadedKVCache(host_dtype=torch.float8_e4m3fn)).

* The row quantiser of csrc/fp8_core.h, the text the kernels compile, built with gcc: byte for byte the torch
  restatement of tests/fp8_ref.py (`quant_rows_ref`) for every finite bf16 value x paired with several amax >= |x|
  (x = +-amax, subnormals and underflow to zero included) in e4m3 and e5m2, zero heads and heads too small to scale.
* The wrappers' argument checks with the recording stub library: what they pass to lv_rows_to_host_fp8 and
  lv_attn_decode_host_fp8, and that nothing reaches the library on bad input.
* Placement: the device-layer count does not depend on the host format at the product lengths, and an FP8 host tier
  takes 2112 / 4096 of the pinned bytes of a bf16 one.
* `kv_host_dtype` reaches the cache from forward, generate and B200GPTVLModel; any other value is a ValueError.
* On the CPU oracle, generate() with an FP8 host tier runs the FP8 row copy and decode (restated with `fp8_rows` /
  `dequantise_rows` of tests/fp8_ref.py) and its prefill logits equal the bf16 offloaded cache's.

The GPU twin is tests/test_gpu_kv_fp8_host.py.
"""
import contextlib
import types

import pytest
import torch

from long_vita_b200 import kv_cache, ops
from long_vita_b200.config import LongVITAConfig
from long_vita_b200.hf import modeling
from long_vita_b200.kv_cache import KVCache, OffloadedKVCache
from long_vita_b200.megatron import checkpoint as ck
from tests.fp8_ref import E4M3, E5M2, FP8_MAX, build_rows_shim, check_rows, dequantise_rows, finite_bf16, fp8_rows
from tests.test_offloaded_cache_host import _free_on_80gb, _offload, tiny  # noqa: F401  (tiny is a fixture)
from tests.test_ops_args_host import P, _bf16, lib  # noqa: F401  (lib is the recording-stub fixture)
from tests.test_row_chunks_host import _inputs
from tests.test_stream_layer_host import _constants, stream_oracle_ops

FP8 = torch.float8_e4m3fn


# ------------------------------------------------------------------------------------------------
# the shared quantiser built with gcc, against the restatement
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return build_rows_shim(tmp_path_factory.mktemp("kv8_host"))


@pytest.mark.parametrize("dtype", [E4M3, E5M2], ids=["e4m3", "e5m2"])
def test_every_finite_bf16_value_against_several_amax(core, dtype):
    """Heads of two values [x, amax]: amax is the head's max, so x is quantised with inv = M / amax exactly as in a
    128-wide head.  amax = |x| (the +-amax edge, q = +-M), the next bf16 above, 3|x|, and 2^8 .. 2^24 |x| (subnormals
    of the format and underflow to +-0)."""
    mx = FP8_MAX[dtype]
    top = {E4M3: 0x7E, E5M2: 0x7B}[dtype]                           # the code of M
    x = finite_bf16()
    ax = x.float().abs()
    for f in (1.0, None, 3.0, 2.0 ** 8, 2.0 ** 16, 2.0 ** 20, 2.0 ** 24):
        if f is None:                                               # one bf16 step above |x|
            amax = ((x.view(torch.int16) & 0x7FFF) + 1).view(torch.bfloat16)
        else:
            amax = (ax * f).to(torch.bfloat16)
        keep = torch.isfinite(amax.float()) & (amax.float() >= ax)
        heads = torch.stack([x[keep], amax[keep]], dim=1)
        q, _ = check_rows(core, heads, dtype)
        big = (heads[:, 1].float() >= 1e-30)                                              # inv finite
        if f == 1.0:
            assert bool((q[big, 1] == top).all())                                          # amax -> M
            assert bool(((q[big, 0] & 0x7F) == top)[heads[big, 0].float() != 0].all())    # x = +-amax -> +-M
    # amax = M (inv = 1): every finite code is reached, subnormals included, and none is NaN or inf
    x = x[x.float().abs() <= mx]
    q, _ = check_rows(core, torch.stack([x, torch.full_like(x, mx)], dim=1), dtype)
    assert set(q[:, 0].tolist()) == {c for c in range(256) if c & 0x7F <= top}


def test_zero_heads_and_heads_too_small_to_scale(core):
    d = 128
    tiny = torch.tensor([0, 1, 0x8001, 0x7F], dtype=torch.int32).to(torch.int16).view(torch.bfloat16)  # subnormals
    heads = torch.zeros(6, d, dtype=torch.bfloat16)
    heads[1] = -0.0
    heads[2, 5] = tiny[1]                                           # amax 9.2e-41: M / amax overflows
    heads[3, :4] = tiny
    heads[4] = torch.randn(d).to(torch.bfloat16) * 1e-36            # amax ~ 3e-36: inv finite
    heads[5, 7] = 2.0 ** -119                                       # just above M / FLT_MAX: inv = M * 2^119
    q, scale = check_rows(core, heads)
    assert bool((q[:4] == 0).all()) and bool((scale[:4] == 0).all())
    assert scale[4] > 0 and scale[5] > 0 and q[5, 7] == 0x7E


def test_random_heads_and_rows(core):
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(4096, 128, generator=g) * torch.logspace(-20, 20, 4096).unsqueeze(1)).to(torch.bfloat16)
    x[::7, :3] = 0
    check_rows(core, x)
    assert core.kv8_row_bytes(8, 128) == ops.kv_fp8_row_bytes(8, 128) == 2112
    for hkv in (1, 2, 3, 4, 16):
        assert core.kv8_row_bytes(hkv, 128) == ops.kv_fp8_row_bytes(hkv, 128)
        assert ops.kv_fp8_row_bytes(hkv, 128) % 16 == 0
    k, v = x[:64].view(16, 4, 128), x[64:128].view(16, 4, 128)
    rows = fp8_rows(k, v)
    assert rows.shape == (16, ops.kv_fp8_row_bytes(4, 128))
    dk, dv = dequantise_rows(rows, 4, 128)
    for a, b in ((dk, k), (dv, v)):                                 # e4m3 keeps 3 mantissa bits: <= 2^-4 relative
        err = (a - b.float()).abs() / b.float().abs().amax(-1, keepdim=True).clamp_min(1e-30)
        assert float(err.max()) <= 2.0 ** -4


# ------------------------------------------------------------------------------------------------
# wrappers: recorded calls and refusals (recording stub library)
# ------------------------------------------------------------------------------------------------
def _pinned(monkeypatch):
    monkeypatch.setattr(ops, "_is_pinned", lambda t: not t.is_cuda)


def test_kv_rows_to_host_fp8_calls(lib, monkeypatch):  # noqa: F811
    _pinned(monkeypatch)
    row = ops.kv_fp8_row_bytes(8, 128)
    qkv = _bf16(5, 56 * 128)                                        # a QKV buffer row: 40 q heads, 8 k, 8 v
    k, v = qkv[:, 40 * 128 : 48 * 128].view(5, 8, 128), qkv[:, 48 * 128 :].view(5, 8, 128)
    dst = torch.zeros(7, row, dtype=torch.uint8)
    assert ops.kv_rows_to_host_fp8(k, v, dst[2:]) is not None
    kvb = _bf16(5, 2, 8, 128)                                       # the streamed layer's K|V buffer
    ops.kv_rows_to_host_fp8(kvb[:, 0], kvb[:, 1], dst[:5])
    assert lib.calls == [("lv_rows_to_host_fp8", P(dst[2:]), P(k), 5, 8, 128, 56 * 128 * 2),
                         ("lv_rows_to_host_fp8", P(dst), P(kvb), 5, 8, 128, 2 * 8 * 128 * 2)]


def test_kv_rows_to_host_fp8_refusals(lib, monkeypatch):  # noqa: F811
    row = ops.kv_fp8_row_bytes(8, 128)
    kvb = _bf16(5, 2, 8, 128)
    k, v = kvb[:, 0], kvb[:, 1]
    with pytest.raises(ValueError, match="pinned host memory"):
        ops.kv_rows_to_host_fp8(k, v, torch.zeros(5, row, dtype=torch.uint8))          # not pinned
    _pinned(monkeypatch)
    bad = [
        (torch.zeros(5, 2 * 8 * 128, dtype=torch.bfloat16), "contiguous uint8"),         # a bf16 host layer
        (torch.zeros(5, row - 16, dtype=torch.uint8), "contiguous uint8"),               # wrong row size
        (torch.zeros(5, 2 * row, dtype=torch.uint8)[:, :row], "contiguous uint8"),       # rows not contiguous
        (torch.zeros(4, row, dtype=torch.uint8), "dst has 4 rows for 5"),
    ]
    for dst, msg in bad:
        with pytest.raises(ValueError, match=msg):
            ops.kv_rows_to_host_fp8(k, v, dst)
    dst = torch.zeros(5, row, dtype=torch.uint8)
    with pytest.raises(ValueError, match="not the K and V halves"):
        ops.kv_rows_to_host_fp8(v, k, dst)
    with pytest.raises(ValueError, match="not the K and V halves"):
        ops.kv_rows_to_host_fp8(k, _bf16(5, 8, 128), dst)
    assert lib.calls == []


def test_attention_decode_host_fp8_calls(lib, monkeypatch):  # noqa: F811
    _pinned(monkeypatch)
    kv = torch.zeros(1000, ops.kv_fp8_row_bytes(8, 128), dtype=torch.uint8)
    q = _bf16(40, 128)
    ops.attention_decode_host_fp8(q, kv, 700)
    ops.attention_decode_host_fp8(q, kv, 1000, n_splits=3, scale=0.5)
    (n0, a0), (m0, *_), (n1, a1), (m1, *_) = [(c[0], c[1:]) for c in lib.calls]
    assert (n0, m0, n1, m1) == ("lv_attn_decode_host_fp8", "lv_attn_decode_merge") * 2
    assert a0[1] == P(kv) and a0[4:] == (700, 1000, 40, 8, 128, 6, pytest.approx(128 ** -0.5))
    assert a1[4:] == (1000, 1000, 40, 8, 128, 3, 0.5)
    kv1 = torch.zeros(10, ops.kv_fp8_row_bytes(1, 128), dtype=torch.uint8)     # one kv head: 272-byte rows
    lib.calls.clear()
    ops.attention_decode_host_fp8(_bf16(5, 128), kv1, 10)
    assert lib.calls[0][5:10] == (10, 10, 5, 1, 128)


def test_attention_decode_host_fp8_refusals(lib, monkeypatch):  # noqa: F811
    row = ops.kv_fp8_row_bytes(8, 128)
    q = _bf16(40, 128)
    with pytest.raises(ValueError, match="pinned host memory"):
        ops.attention_decode_host_fp8(q, torch.zeros(100, row, dtype=torch.uint8), 10)
    _pinned(monkeypatch)
    kv = torch.zeros(100, row, dtype=torch.uint8)
    cases = [
        ((q, torch.zeros(100, 2 * 8 * 128, dtype=torch.bfloat16), 10), "contiguous uint8"),   # a bf16 layer
        ((q, torch.zeros(100, 2 * row, dtype=torch.uint8)[:, :row], 10), "contiguous uint8"),
        ((q, torch.zeros(100, 4096, dtype=torch.uint8), 10), "not FP8 K|V rows"),            # bf16 row size
        ((q, torch.zeros(100, row + 16, dtype=torch.uint8), 10), "not FP8 K|V rows"),
        ((q, torch.zeros(100, 64, dtype=torch.uint8), 10), "not FP8 K|V rows"),
        ((_bf16(36, 128), kv, 10), "not FP8 K|V rows"),                                         # hq % hkv
        ((q, kv, 0), "outside the cache"),
        ((q, kv, 101), "outside the cache"),
        ((_bf16(1, 40, 128), kv, 10), r"q must be \[hq, d\]"),
    ]
    for args, msg in cases:
        with pytest.raises(ValueError, match=msg):
            ops.attention_decode_host_fp8(*args)
    assert lib.calls == []


# ------------------------------------------------------------------------------------------------
# placement and size
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,n_dev", [(18432, 48), (131072, 48), (1058816, 2), (2115584, 2)])
def test_host_dtype_keeps_the_placement_and_halves_the_host_bytes(monkeypatch, T, n_dev):
    """The 14B cache at the product lengths on an 80 GB card (meta tensors: nothing is allocated)."""
    cfg = LongVITAConfig()
    monkeypatch.setattr(kv_cache, "device_free_bytes", lambda dev: _free_on_80gb(cfg))
    monkeypatch.setattr(ops, "pinned_rows", lambda rows, cols, dtype=torch.bfloat16:
                        torch.empty(rows, cols, dtype=dtype, device="meta"))
    caches = {dt: modeling.new_cache(cfg, cfg.num_hidden_layers, T + 1024, T, "meta", dt) for dt in kv_cache.HOST_DTYPES}
    bf, f8 = caches[torch.bfloat16], caches[FP8]
    if n_dev == cfg.num_hidden_layers:
        assert type(bf) is KVCache and type(f8) is KVCache            # the device cache ignores the option
        assert bf.bytes() == f8.bytes() and f8.k[0].dtype == torch.bfloat16
        return
    assert isinstance(f8, OffloadedKVCache) and bf.n_dev == f8.n_dev == n_dev
    assert bf.host_dtype == torch.bfloat16 and f8.host_dtype == FP8
    assert f8.host[0].shape == (T + 1024, 2112) and f8.host[0].dtype == torch.uint8
    assert f8.host_bytes() * 4096 == bf.host_bytes() * 2112
    assert f8.host_bytes() == (cfg.num_hidden_layers - n_dev) * (T + 1024) * 2112
    assert f8.bytes() == bf.bytes() and all(t.dtype == torch.bfloat16 for t in f8.k + f8.v)


def test_bad_host_dtype_is_refused():
    for bad in (torch.float16, torch.float32, torch.uint8, torch.float8_e5m2, "fp8", None):
        with pytest.raises(ValueError, match="host dtype"):
            kv_cache.make_cache(2, 10, 1, 128, "cpu", prefill_bytes=0, offloaded_prefill_bytes=0, host_dtype=bad)
        with pytest.raises(ValueError, match="host dtype"):
            OffloadedKVCache(2, 1, 10, 1, 128, "cpu", host_dtype=bad)


# ------------------------------------------------------------------------------------------------
# kv_host_dtype reaches the cache from every surface
# ------------------------------------------------------------------------------------------------
class _Made(Exception):
    pass


@contextlib.contextmanager
def _record_make_cache(monkeypatch):
    """make_cache records its host_dtype (after its own check) and stops the forward there."""
    seen = []
    real = kv_cache.make_cache

    def make(*a, host_dtype=torch.bfloat16, **kw):
        kv_cache.check_host_dtype(host_dtype)
        seen.append(host_dtype)
        raise _Made

    monkeypatch.setattr(kv_cache, "make_cache", make)
    yield seen
    monkeypatch.setattr(kv_cache, "make_cache", real)


def test_kv_host_dtype_reaches_the_cache(lib, monkeypatch, tiny):  # noqa: F811
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel

    cfg, w = tiny
    lm = modeling.LongVITAForCausalLM(cfg, w)
    ids = torch.zeros(1, 5, dtype=torch.int64)
    with _record_make_cache(monkeypatch) as seen:
        for call in (lambda **kw: lm(input_ids=ids, use_cache=True, **kw),
                     lambda **kw: lm.model(input_ids=ids, use_cache=True, **kw),
                     lambda **kw: lm.generate(ids, max_new_tokens=2, **kw),
                     lambda **kw: B200GPTVLModel(cfg, ck.hf_to_mcore(w, cfg), **kw)(
                         ids, None, None, inference_params=types.SimpleNamespace(key_value_memory_dict={}))):
            for kw, want in (({}, torch.bfloat16), ({"kv_host_dtype": FP8}, FP8),
                             ({"kv_host_dtype": torch.bfloat16}, torch.bfloat16)):
                seen.clear()
                with pytest.raises(_Made):
                    call(**kw)
                assert seen == [want]
            seen.clear()
            with pytest.raises(ValueError, match="host dtype"):
                call(kv_host_dtype=torch.float16)
            assert seen == []
    assert lib.calls == []


# ------------------------------------------------------------------------------------------------
# generate() on the CPU oracle with an FP8 host tier
# ------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _oracle_fp8_host_tier(monkeypatch):
    """stream_oracle_ops() with the FP8 host-tier operators restated on the CPU: the row copy writes fp8_rows, the
    decode is the oracle's attention_decode over the dequantised rows (rounded to bf16, the oracle's input type)."""
    def rows_to_host(k, v, dst):
        dst.copy_(fp8_rows(k, v))
        calls.append("rows")
        return dst

    def decode_host(q, kv, length, **kw):
        hkv = kv.shape[1] // (2 * q.shape[1] + 8)
        k, v = dequantise_rows(kv[:length], hkv, q.shape[1])
        calls.append(length)
        return ops.attention_decode(q, k.to(torch.bfloat16), v.to(torch.bfloat16), length, **kw)

    calls = []
    with stream_oracle_ops():
        monkeypatch.setattr(ops, "pinned_rows", lambda rows, cols, dtype=torch.bfloat16:
                            torch.full((rows, cols), 0xFF if dtype == torch.uint8 else float("nan"), dtype=dtype))
        monkeypatch.setattr(ops, "kv_rows_to_host_fp8", rows_to_host)
        monkeypatch.setattr(ops, "attention_decode_host_fp8", decode_host)
        monkeypatch.setattr(ops, "kv_rows_to_host", None)            # the bf16 host operators are not called
        monkeypatch.setattr(ops, "attention_decode_host", None)
        yield calls


def test_hf_generate_with_an_fp8_host_tier(monkeypatch, tiny):
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w)
    model.model.vision_chunk = 1
    ids, images, idx = _inputs(cfg)
    s = ids.shape[1]
    with stream_oracle_ops(), _constants(256, 128), monkeypatch.context() as m:
        monkeypatch.setattr(ops, "pinned_rows", lambda rows, cols, dtype=torch.bfloat16: torch.zeros(rows, cols,
                                                                                                      dtype=dtype))
        monkeypatch.setattr(ops, "kv_rows_to_host", lambda k, v, dst: dst.copy_(
            torch.cat([k.reshape(k.shape[0], -1), v.reshape(k.shape[0], -1)], 1)))
        _offload(m, cfg, 1)
        ref = model(input_ids=ids, images=images, image_indices=idx, use_cache=True, max_cache_len=s + 4)
    with _oracle_fp8_host_tier(monkeypatch) as calls, _constants(256, 128):
        for stream in (None, 256):
            with monkeypatch.context() as m, _constants(stream=stream):
                _offload(m, cfg, 1)
                out = model(input_ids=ids, images=images, image_indices=idx, use_cache=True, max_cache_len=s + 4,
                            kv_host_dtype=FP8)
                c = out.past_key_values
                assert isinstance(c, OffloadedKVCache) and c.host_dtype == FP8 and c.n_dev == 1
                assert torch.equal(out.logits, ref.logits)              # the prefill never reads the host rows
                want = fp8_rows(ref.past_key_values.host[0][:s, :128].view(s, 1, 128),
                                ref.past_key_values.host[0][:s, 128:].view(s, 1, 128))
                assert torch.equal(c.host[0][:s], want) and bool((c.host[0][s:] == 0xFF).all())
                calls.clear()
                toks = model.generate(ids, images=images, image_indices=idx, max_new_tokens=4, kv_host_dtype=FP8)
                assert toks.shape == (1, s + 4)
                assert calls.count("rows") >= 4 and [c for c in calls if c != "rows"] == [s + 1, s + 2, s + 3]
