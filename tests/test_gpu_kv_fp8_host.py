"""The FP8 (e4m3) host tier of the K/V cache on the H100 (lv_rows_to_host_fp8, lv_attn_decode_host_fp8).

* Quantiser: the rows lv_rows_to_host_fp8 writes from a QKV-buffer view and from a K|V buffer are byte for byte the
  CPU restatement (tests/fp8_ref.fp8_rows), for 8 kv heads (2112-byte rows) and 1 (272-byte rows, padded
  scales), with zero heads; rows outside the destination view are untouched.
* Decode kernel: against float64 attention over the dequantised rows (tests/attn_fwd_ref.check_attn_fwd,
  merged=True) from 1 to 1 058 816 rows, for the split counts of the bf16 test and G = 5 and 8.  Host bytes at and
  past `length` are 0xFF (NaN codes and NaN scales: never read), and planted keys sit on split borders, so a split
  that drops or repeats a border row is an O(1) error.
* A 4-layer 14B-geometry model at 18 432 tokens with 2 host layers, FP8 against bf16: prefill logits equal, host rows
  the quantised bf16 rows, 16 teacher-forced decode steps within a stated logit bound, greedy agreement printed.
  The weights are synthetic: how the FP8 host tier changes the output of a trained checkpoint is NOT measured here.
"""
import pytest
import torch

from tests.attn_fwd_ref import attention_fwd_ref, check_attn_fwd
from tests.test_gpu_attention_fwd_ref import _plant_decode, _randn
from tests.test_gpu_offloaded_cache import _model, _need_host, _placed
from tests.fp8_ref import dequantise_rows, fp8_rows

pytestmark = pytest.mark.gpu

HKV, D = 8, 128
ROW8 = 2112
WORST = {}
# worst relative logit deviation of 16 FP8 decode steps from the bf16 host tier, synthetic 14B-geometry weights
# (measured 0.0078 on an H100 80GB HBM3)
FP8_LOGIT_LIMIT = 0.02


@pytest.fixture(scope="module")
def L(lib_built):
    from long_vita_b200 import ops

    yield ops
    print(f"\n[decode_host_fp8] worst figures {({k: round(v, 4) for k, v in WORST.items()})}")


@pytest.mark.parametrize("hkv", [8, 1])
@pytest.mark.parametrize("n", [1, 2, 3, 1000, 65537])
def test_rows_to_host_fp8_is_the_restatement(L, hkv, n):
    g = torch.Generator(device="cuda").manual_seed(n + hkv)
    hq = 5 * hkv
    row = L.kv_fp8_row_bytes(hkv, D)
    # per-head magnitudes from 1e-3 to 1e3, one zero head per 5 rows
    mag = torch.logspace(-3, 3, 7, device="cuda")[torch.randint(0, 7, (n, hq + 2 * hkv, 1), device="cuda",
                                                                generator=g)]
    qkv = (torch.randn((n, hq + 2 * hkv, D), device="cuda", generator=g) * mag).to(torch.bfloat16)
    qkv[::5, hq] = 0
    qkv = qkv.view(n, -1)
    kvb = (torch.randn((n, 2, hkv, D), device="cuda", generator=g) * 3).to(torch.bfloat16)
    dst = L.pinned_fp8_rows(n + 2, hkv, D)
    for k, v in ((qkv[:, hq * D : (hq + hkv) * D].view(n, hkv, D), qkv[:, (hq + hkv) * D :].view(n, hkv, D)),
                 (kvb[:, 0], kvb[:, 1])):
        dst.fill_(0xAB)
        L.kv_rows_to_host_fp8(k, v, dst[1 : n + 1])
        torch.cuda.synchronize()
        assert dst.shape == (n + 2, row)
        assert torch.equal(dst[1 : n + 1], fp8_rows(k, v))
        assert bool((dst[0] == 0xAB).all()) and bool((dst[n + 1] == 0xAB).all())


def _fill_fp8(L, host, k, v):
    """Quantise the device rows k / v [cap, hkv, d] into host through the kernel, 65 536 rows at a time."""
    for r0 in range(0, k.shape[0], 65536):
        r1 = min(r0 + 65536, k.shape[0])
        L.kv_rows_to_host_fp8(k[r0:r1], v[r0:r1], host[r0:r1])
    torch.cuda.synchronize()


@pytest.mark.parametrize("G", [5, 8])
@pytest.mark.parametrize("length", [1, 127, 128, 129, 131072, 1058816])
def test_decode_host_fp8_kernel(L, length, G):
    hq = G * HKV
    cap = length + 300
    _need_host(cap * ROW8, f"length {length}")
    g = torch.Generator(device="cuda").manual_seed(length + G)
    q = _randn((hq, D), g)
    kv = _randn((cap, 2, HKV, D), g)
    host = L.pinned_fp8_rows(cap, HKV, D)
    for n_splits in (None, 1, 7, 64, 264):
        ns = n_splits if n_splits is not None else max(1, min(L._sm_count(q.device), -(-length // 128)))
        per = -(-length // ns)
        borders = sorted({t for c0 in range(per, length, per) for t in (c0 - 1, c0)} | {0, length - 1})
        qq, kvp = q.clone(), kv.clone()                    # kvp: a K|V buffer, V following K in each row
        targets = {h: borders[(h // 2 * 7) % len(borders)] for h in range(0, hq, 2)}
        _plant_decode(qq, kvp[:, 0], targets)
        _fill_fp8(L, host, kvp[:, 0], kvp[:, 1])
        host[length:] = 0xFF                                 # e4m3 NaN codes and NaN scales: never read
        out, lse = L.attention_decode_host_fp8(qq, host, length, n_splits=n_splits, return_lse=True)
        label = f"decode_host_fp8 {length} G {G} splits {n_splits}"
        kd, vd = dequantise_rows(host[:length].cuda(), HKV, D)
        ref = attention_fwd_ref(qq.view(1, 1, hq, D), kd.unsqueeze(0), vd.unsqueeze(0), causal=False)
        st = check_attn_fwd(out.view(1, 1, hq, D), lse.view(1, hq, 1), ref, merged=True, label=label)
        print(label, {k: f"{v:.3g}" for k, v in st.items()})
        for k, v in st.items():
            WORST[k] = max(WORST.get(k, 0.0), v)
        hs = torch.tensor(sorted(targets))
        vt = vd[torch.tensor([targets[h] for h in hs.tolist()]), hs // G].double()
        dist = (ref["out"][0, 0, hs] - vt).norm(dim=-1) / vt.norm(dim=-1)
        assert float(dist.max()) < 1e-2, ("plant", length, n_splits, float(dist.max()))
        out2, lse2 = L.attention_decode_host_fp8(qq, host, length, n_splits=n_splits, return_lse=True)
        assert torch.equal(out2, out) and torch.equal(lse2, lse)
        del ref, kd, vd


def test_two_fp8_host_layers_against_the_bf16_host_tier(lib_built, monkeypatch):
    from long_vita_b200.kv_cache import OffloadedKVCache

    s, steps = 18432, 16
    _need_host(2 * (s + steps) * (4096 + ROW8), "the 18 432-token model")
    model = _model(4)
    g = torch.Generator(device="cuda").manual_seed(3)
    ids = torch.randint(0, model.config.vocab_size, (1, s), device="cuda", generator=g)
    with torch.no_grad(), monkeypatch.context() as m:
        _placed(m, 2)
        bf = model(input_ids=ids, use_cache=True, num_logits_to_keep=1, max_cache_len=s + steps)
        f8 = model(input_ids=ids, use_cache=True, num_logits_to_keep=1, max_cache_len=s + steps,
                   kv_host_dtype=torch.float8_e4m3fn)
        bc, fc = bf.past_key_values, f8.past_key_values
        assert isinstance(fc, OffloadedKVCache) and fc.host_dtype == torch.float8_e4m3fn and fc.n_dev == 2
        assert bc.host_dtype == torch.bfloat16 and fc.host_bytes() * 4096 == bc.host_bytes() * 2112
        assert torch.equal(f8.logits, bf.logits)                 # the prefill attends over its own bf16 k, v
        for j in range(2):
            assert torch.equal(fc.k[j][:s], bc.k[j][:s]) and torch.equal(fc.v[j][:s], bc.v[j][:s])
            hb = bc.host[j][:s]
            want = fp8_rows(hb[:, : HKV * D].reshape(s, HKV, D), hb[:, HKV * D :].reshape(s, HKV, D))
            assert torch.equal(fc.host[j][:s], want)
        tok = bf.logits[0, -1].float().argmax().view(1, 1)
        worst, agree = 0.0, 0
        for i in range(steps):
            a = model(input_ids=tok, past_key_values=bc, use_cache=True, num_logits_to_keep=1).logits[0, -1].float()
            b = model(input_ids=tok, past_key_values=fc, use_cache=True, num_logits_to_keep=1).logits[0, -1].float()
            rel = float((a - b).norm() / a.norm())
            worst = max(worst, rel)
            agree += int(a.argmax()) == int(b.argmax())
            tok = a.argmax().view(1, 1)                 # teacher forcing: both caches take the bf16 run's token
    print(f"[fp8 host 18432] {steps} decode steps against the bf16 host tier: worst relative logit deviation "
          f"{worst:.3g} (limit {FP8_LOGIT_LIMIT}), greedy tokens agree {agree}/{steps}; synthetic weights, quality on "
          f"a trained checkpoint not measured")
    assert worst <= FP8_LOGIT_LIMIT and len(bc) == len(fc) == s + steps
