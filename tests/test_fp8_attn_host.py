"""CPU tests of the FP8 attention forward (ops.attention_fwd_fp8, attn_dtype=torch.float8_e4m3fn).

* The operand rule of csrc/attn_fp8_core.h, the text the kernels compile, built with gcc: K8, Vt8 and the scales of
  each block are byte for byte the torch restatement of tests/attn_fp8_ref.py (`quant_kv`), with the transpose and key
  permutation of Vt8, ragged last blocks, all-zero blocks, blocks of bf16 subnormals (scale 0) and a 1000x outlier.
* Routing, on the CPU oracle (tests/hostlogic.py) with a recording twin of ops.attention_fwd_fp8: the bf16 default
  never reaches it and makes the same attention calls as before; attn_dtype=FP8 sends the whole-tensor, row-chunked,
  streamed and cache-prefill calls to it, and decode and ViT calls to the bf16 ops.
* Bad attn_dtype values and packed rows with FP8 attention are refused before any operator runs.
* prefill_bytes_per_token changes only with FP8 attention, by the quantised K / V of one call.
"""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch

from long_vita_b200 import ops
from long_vita_b200.config import LongVITAConfig
from long_vita_b200.hf import modeling
from long_vita_b200.weights import synthetic_state_dict
from tests import attn_fp8_ref as R
from tests.fp8_ref import E4M3, FP8_MAX, build_shim
from tests.test_stream_layer_host import _constants, stream_oracle_ops

FP8 = torch.float8_e4m3fn

_SHIM = r"""
#include "attn_fp8_core.h"
int key_of(int kappa) { return lv_attn8_key_of(kappa); }
/* x [n, hkv, d] bf16 rows (one batch entry) -> k8 [hkv][nt*128][d], vt8 [hkv][nt][d][128], scales [hkv][nt] */
void quant_kv(const uint16_t* k, const uint16_t* v, int n, int hkv, int d, uint8_t* k8, uint8_t* vt8, float* ks,
              float* vs, uint16_t* work, uint8_t* wq) {
  const int nt = (int)lv_attn8_blocks(n);
  for (int h = 0; h < hkv; ++h)
    for (int t = 0; t < nt; ++t) {
      const int rows = n - t * 128 < 128 ? n - t * 128 : 128;
      const long long blk = (long long)h * nt + t;
      ks[blk] = lv_attn8_quant_k_block(k + ((long long)t * 128 * hkv + h) * d, (long long)hkv * d, rows, d,
                                       k8 + blk * 128 * d, work, wq);
      vs[blk] = lv_attn8_quant_v_block(v + ((long long)t * 128 * hkv + h) * d, (long long)hkv * d, rows, d,
                                       vt8 + blk * 128 * d, work, wq);
    }
}
"""


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    lib = build_shim(tmp_path_factory.mktemp("attn8_host"), _SHIM)
    lib.key_of.argtypes = [C.c_int]
    lib.quant_kv.argtypes = [C.c_void_p] * 2 + [C.c_int] * 3 + [C.c_void_p] * 6
    return lib


def _header_quant(core, k, v):
    n, hkv, d = k.shape
    nt = -(-n // 128)
    k8 = np.zeros((hkv, nt * 128, d), np.uint8)
    vt8 = np.zeros((hkv, nt, d, 128), np.uint8)
    ks = np.zeros((hkv, nt), np.float32)
    vs = np.zeros((hkv, nt), np.float32)
    work = np.zeros(128 * d, np.uint16)
    wq = np.zeros(128 * d, np.uint8)
    kn, vn = k.contiguous().view(torch.int16).numpy(), v.contiguous().view(torch.int16).numpy()
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    core.quant_kv(ptr(kn), ptr(vn), n, hkv, d, ptr(k8), ptr(vt8), ptr(ks), ptr(vs), ptr(work), ptr(wq))
    return [torch.from_numpy(a) for a in (k8, vt8, ks, vs)]


def test_key_permutation(core):
    perm = [core.key_of(i) for i in range(128)]
    assert perm == R.key_of(torch.arange(128)).tolist()
    assert sorted(perm) == list(range(128))
    # the accumulator layout packs into the A fragment: thread t % 4 = c holds keys 2c, 2c + 1 of every 8-column group,
    # the fragment wants k = 4c .. 4c + 3 and 16 + 4c .. 16 + 4c + 3 of each 32-key step
    for c in range(4):
        held = sorted({8 * j + 2 * c + e for j in range(4) for e in range(2)})
        assert sorted(perm[4 * c + i] for i in range(4)) + sorted(perm[16 + 4 * c + i] for i in range(4)) == held


@pytest.mark.parametrize("n", [1, 127, 128, 129, 300, 517])
def test_header_matches_restatement(core, n):
    g = torch.Generator().manual_seed(n)
    hkv, d = 3, 128
    k = torch.randn((n, hkv, d), generator=g).to(torch.bfloat16)
    v = torch.randn((n, hkv, d), generator=g).to(torch.bfloat16)
    if n > 256:
        k[128:256, 1] = 0                                                       # all-zero block
        v[256:, 2] = (torch.randn((n - 256, d), generator=g) * 1e-39).to(torch.bfloat16)   # subnormal amax: scale 0
        v[130, 0, 5] = 1000.0                                                   # outlier
        k[3, 2, 77] = -1000.0
    got = _header_quant(core, k, v)
    want = R.quant_kv(k.unsqueeze(0), v.unsqueeze(0))
    for name, a, b in zip(("k8", "vt8", "k_scale", "v_scale"), got, want):
        b = b[0]
        if a.dtype == torch.float32:
            a, b = a.view(torch.int32), b.view(torch.int32)
        assert a.shape == b.shape and torch.equal(a, b), (name, n)
    if n > 256:
        assert float(got[2][1, 1]) == 0.0 and float(got[3][2, 2]) == 0.0
        assert float(got[3][0, 1]) == float(torch.tensor(1000.0) / FP8_MAX[E4M3])
        assert not got[0][1, 128:256].any()
    # padding rows / keys are zero bytes
    nt = -(-n // 128)
    assert not got[0][:, n:].any()
    last = got[1][:, nt - 1]
    pad = R.key_of(torch.arange(128)) >= n - (nt - 1) * 128
    assert not last[..., pad].any()
    # the dequantised operands are the bf16 ones within the e4m3 rounding
    kf, vf = R.dequant_kv(*[t.unsqueeze(0) for t in got], n)
    for x, xf in ((k, kf[0]), (v, vf[0])):
        tol = x.float().abs().amax(dim=(0, 2)).view(1, hkv, 1) / FP8_MAX[E4M3] * 2.0 ** -6   # below the e4m3 normals
        assert bool(((xf - x.float()).abs() <= 2.0 ** -4 * x.float().abs() + tol).all())


# ------------------------------------------------------------------------------------------------
# routing on the CPU oracle
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    cfg = LongVITAConfig.tiny(layers=2, vit_layers=1)
    return cfg, synthetic_state_dict(cfg, seed=31, dtype=torch.bfloat16, perturb=True)


@contextlib.contextmanager
def recording():
    """stream_oracle_ops() (tests/hostlogic.py's CPU oracle) with a recording twin of ops.attention_fwd_fp8 (the float64 reference of the FP8 kernel, rounded to
    bf16) and recorders on the bf16 attention ops; yields the list of (op, sq, sk, causal)."""
    calls = []
    with stream_oracle_ops() as o:
        fwd, dec = o.attention_fwd, o.attention_decode

        def fwd_rec(q, k, v, *, causal, **kw):
            calls.append(("attention_fwd", q.shape[1], k.shape[1], causal))
            return fwd(q, k, v, causal=causal, **kw)

        def fp8_rec(q, k, v, causal=True, return_lse=False, **kw):
            calls.append(("attention_fwd_fp8", q.shape[1], k.shape[1], causal))
            ref = R.reference(q, k, v)
            out = ref["out"].to(torch.bfloat16)
            return (out, ref["lse"].float()) if return_lse else out

        def dec_rec(q, k, v, length, **kw):
            calls.append(("attention_decode", 1, length, True))
            return dec(q, k, v, length, **kw)

        saved = o.attention_fwd_fp8, o.attention_decode
        o.attention_fwd, o.attention_fwd_fp8, o.attention_decode = fwd_rec, fp8_rec, dec_rec
        try:
            yield calls
        finally:
            o.attention_fwd_fp8, o.attention_decode = saved


def _decoder(calls):
    return [c for c in calls if c[3]]


def _ids(cfg, s, seed=1):
    return torch.randint(0, cfg.vocab_size, (1, s), generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("plan", ["whole", "row-chunked", "streamed"])
def test_routing_prefill_plans(tiny, plan):
    cfg, w = tiny
    consts = {"whole": (), "row-chunked": (200, 128), "streamed": (200, 128, 200)}[plan]
    s = 300
    ids = _ids(cfg, s)
    out = {}
    for dt in (torch.bfloat16, FP8):
        model = modeling.LongVITAForCausalLM(cfg, w, attn_dtype=dt)
        with _constants(*consts), recording() as calls:
            out[dt] = model(input_ids=ids, num_logits_to_keep=5).logits
        ops_used = {c[0] for c in _decoder(calls)}
        assert ops_used == ({"attention_fwd"} if dt == torch.bfloat16 else {"attention_fwd_fp8"}), (plan, calls)
        n_calls = 2 * (3 if plan == "streamed" else 1)        # two layers; streamed: spans 128, 128, 44
        assert len(_decoder(calls)) == n_calls, calls
        if plan == "streamed":
            assert [c[1:3] for c in _decoder(calls)[:3]] == [(128, 128), (128, 256), (44, 300)]
    assert torch.isfinite(out[FP8].float()).all() and not torch.equal(out[FP8], out[torch.bfloat16])


def test_bf16_default_calls_unchanged(tiny):
    """attn_dtype defaults to bf16: the default model and an explicit bf16 one make the same calls and logits."""
    cfg, w = tiny
    ids = _ids(cfg, 200, seed=2)
    res = []
    for kw in ({}, {"attn_dtype": torch.bfloat16}):
        model = modeling.LongVITAForCausalLM(cfg, w, **kw)
        with recording() as calls:
            logits = model(input_ids=ids, num_logits_to_keep=3).logits
        res.append((calls, logits))
    assert res[0][0] == res[1][0] and torch.equal(res[0][1], res[1][1])
    assert all(c[0] == "attention_fwd" for c in res[0][0])


def test_routing_cache_prefill_decode_and_vit(tiny):
    """generate() with FP8 attention: the prefill of the empty cache and a multi-token forward on the filled cache go
    to the FP8 op, the single-token steps to ops.attention_decode, the ViT (non-causal) to ops.attention_fwd."""
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w, attn_dtype=FP8)
    from tests.test_row_chunks_host import _inputs

    ids, images, idx = _inputs(cfg, s=300, n_img=1)
    with recording() as calls:
        out = model.generate(inputs=ids, images=images, image_indices=idx, max_new_tokens=3)
    assert out.shape == (1, 303)
    vit = [c for c in calls if not c[3]]
    assert vit and all(c[0] == "attention_fwd" for c in vit)
    dec = _decoder(calls)
    assert [c[0] for c in dec[:2]] == ["attention_fwd_fp8"] * 2 and dec[0][1:3] == (300, 300)
    assert [c[0] for c in dec[2:]] == ["attention_decode"] * 4
    # a multi-token forward on the filled cache: FP8 over cache + new rows
    with recording() as calls:
        first = model(input_ids=ids[:, :200], use_cache=True, num_logits_to_keep=1)
        model(input_ids=ids[:, 200:203], past_key_values=first.past_key_values, use_cache=True, num_logits_to_keep=1)
    dec = _decoder(calls)
    assert [c[0] for c in dec] == ["attention_fwd_fp8"] * 4 and dec[2][1:3] == (3, 203)


def test_refusals_before_any_launch(tiny):
    cfg, w = tiny
    for bad in (torch.float16, torch.float32, torch.float8_e5m2, "fp8", None):
        with pytest.raises(ValueError):
            modeling.LongVITAForCausalLM(cfg, w, attn_dtype=bad)
        with pytest.raises(ValueError):
            modeling.LongVITAForCausalLM.from_synthetic(cfg, device="cpu", attn_dtype=bad)
        with pytest.raises(ValueError):
            modeling.LongVITAForCausalLM.from_pretrained("/nonexistent", attn_dtype=bad)
        with pytest.raises(ValueError):
            modeling.attention_step(attn_dtype=bad)
    model = modeling.LongVITAForCausalLM(cfg, w, attn_dtype=FP8)
    pos = torch.cat([torch.arange(100), torch.arange(100)]).unsqueeze(0)     # two packed samples
    with recording() as calls:
        with pytest.raises(NotImplementedError):
            model(input_ids=_ids(cfg, 200), position_ids=pos)
    assert calls == []
    with pytest.raises(NotImplementedError):
        modeling.attention_step(cu_seqlens=torch.tensor([0, 100, 200], dtype=torch.int32), attn_dtype=FP8)


def test_prefill_bytes_change_only_with_fp8_attention():
    cfg = LongVITAConfig.long_vita_14b()
    hkv, d = cfg.num_key_value_heads, cfg.head_dim
    for T, streamed in ((18432, False), (131072, False), (1058816, False), (2115584, True)):
        bf = modeling.prefill_bytes_per_token(cfg, T, streamed)
        assert modeling.prefill_bytes_per_token(cfg, T, streamed, torch.bfloat16, torch.bfloat16) == bf
        extra = modeling.prefill_bytes_per_token(cfg, T, streamed, torch.bfloat16, FP8) - bf
        assert extra == -(-ops.attn_fp8_kv_bytes(T, hkv, d) // T)
        assert 2 * hkv * d <= extra <= 2 * hkv * d + 2 + 2 * hkv * d * 127 // T
        both = modeling.prefill_bytes_per_token(cfg, T, streamed, FP8, FP8)
        assert both == modeling.prefill_bytes_per_token(cfg, T, streamed, FP8) + extra
    assert ops.attn_fp8_kv_bytes(300, 8, 128) == 8 * 3 * (2 * 128 * 128 + 8)
