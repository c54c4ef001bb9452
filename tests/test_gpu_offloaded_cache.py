"""The K/V cache partly in pinned host memory on the H100 (kv_cache.OffloadedKVCache, lv_attn_decode_host).

* The kernel against float64 (tests/attn_fwd_ref.check_attn_fwd, merged=True) from 1 to 1 058 816 rows, for several
  split counts: host rows at and past `length` are NaN (never read), and the even heads want a key on a split border
  (the last row of one split or the first of the next), so a split that drops or repeats its border row is an O(1)
  error.  The worst figures are printed (`pytest -s`).
* A 4-layer 14B-geometry model at 18 432 tokens with 2 device and 2 host layers against the device cache: prefill
  logits and host rows bit-identical; 16 teacher-forced decode steps within 1e-2; greedy agreement reported.
* 1 058 816 tokens, 2 layers both on the host: the prefill logits are those of the prefill without a cache, the peak
  device memory is that of the prefill without a cache, and the cache pins exactly its rows.

Pinned host memory is at most ~9 GB per case; a case whose need exceeds half of MemAvailable is skipped.
"""
import pytest
import torch

from tests.attn_fwd_ref import attention_fwd_ref, check_attn_fwd
from tests.test_gpu_attention_fwd_ref import _plant_decode, _randn

pytestmark = pytest.mark.gpu

HQ, HKV, D = 40, 8, 128
ROW = 2 * HKV * D * 2
WORST = {}


def _need_host(nbytes, what):
    avail = 0
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                avail = int(line.split()[1]) * 1024
    if avail < 2 * nbytes:
        pytest.skip(f"{what} pins {nbytes / 1e9:.1f} GB of host memory; MemAvailable is {avail / 1e9:.1f} GB, "
                    f"less than twice that")


@pytest.fixture(scope="module")
def L(lib_built):
    from long_vita_b200 import ops

    yield ops
    print(f"\n[decode_host] worst figures {({k: round(v, 4) for k, v in WORST.items()})}")


@pytest.mark.parametrize("length", [1, 127, 128, 129, 2047, 2049, 33000, 131073, 1058816])
def test_decode_host_kernel(L, length):
    cap = length + 300
    _need_host(cap * ROW, f"length {length}")
    g = torch.Generator(device="cuda").manual_seed(length)
    q = _randn((HQ, D), g)
    kv = _randn((cap, 2, HKV, D), g)
    host = L.pinned_rows(cap, 2 * HKV * D)
    G = HQ // HKV
    for n_splits in (None, 1, 7, 64, 264):
        ns = n_splits if n_splits is not None else max(1, min(L._sm_count(q.device), -(-length // 128)))
        per = -(-length // ns)
        borders = sorted({t for c0 in range(per, length, per) for t in (c0 - 1, c0)} | {0, length - 1})
        qq, kk = q.clone(), kv[:, 0].clone()
        targets = {h: borders[(h // 2 * 7) % len(borders)] for h in range(0, HQ, 2)}
        _plant_decode(qq, kk, targets)
        host.view(cap, 2, HKV, D)[:, 0].copy_(kk)
        host.view(cap, 2, HKV, D)[:, 1].copy_(kv[:, 1])
        host[length:] = float("nan")
        out, lse = L.attention_decode_host(qq, host, length, n_splits=n_splits, return_lse=True)
        label = f"decode_host {length} splits {n_splits}"
        ref = attention_fwd_ref(qq.view(1, 1, HQ, D), kk[:length].unsqueeze(0), kv[:length, 1].unsqueeze(0),
                                causal=False)
        st = check_attn_fwd(out.view(1, 1, HQ, D), lse.view(1, HQ, 1), ref, merged=True, label=label)
        print(label, {k: f"{v:.3g}" for k, v in st.items()})
        for k, v in st.items():
            WORST[k] = max(WORST.get(k, 0.0), v)
        hs = torch.tensor(sorted(targets))
        vt = kv[torch.tensor([targets[h] for h in hs.tolist()]), 1, hs // G].double()
        dist = (ref["out"][0, 0, hs] - vt).norm(dim=-1) / vt.norm(dim=-1)
        assert float(dist.max()) < 1e-2, ("plant", length, n_splits, float(dist.max()))
        out2, lse2 = L.attention_decode_host(qq, host, length, n_splits=n_splits, return_lse=True)
        assert torch.equal(out2, out) and torch.equal(lse2, lse)
        del ref


def _model(layers):
    from long_vita_b200.config import LongVITAConfig
    from long_vita_b200.hf.modeling import LongVITAForCausalLM

    return LongVITAForCausalLM.from_synthetic(LongVITAConfig(), seed=7, device="cuda", num_layers=layers)


def _placed(monkeypatch, n_dev):
    from long_vita_b200 import kv_cache

    monkeypatch.setattr(kv_cache, "device_layers", lambda *a, **kw: n_dev)


def test_two_device_two_host_layers_against_the_device_cache(lib_built, monkeypatch):
    from long_vita_b200.kv_cache import KVCache, OffloadedKVCache

    s, steps = 18432, 16
    _need_host(2 * (s + steps) * ROW, "the 18 432-token model")
    model = _model(4)
    g = torch.Generator(device="cuda").manual_seed(3)
    ids = torch.randint(0, model.config.vocab_size, (1, s), device="cuda", generator=g)
    with torch.no_grad():
        dev = model(input_ids=ids, use_cache=True, num_logits_to_keep=1, max_cache_len=s + steps)
        with monkeypatch.context() as m:
            _placed(m, 2)
            off = model(input_ids=ids, use_cache=True, num_logits_to_keep=1, max_cache_len=s + steps)
        dc, oc = dev.past_key_values, off.past_key_values
        assert type(dc) is KVCache and isinstance(oc, OffloadedKVCache) and oc.n_dev == 2 and len(oc.host) == 2
        assert torch.equal(off.logits, dev.logits)
        for j in range(2):
            assert torch.equal(oc.k[j][:s], dc.k[j][:s]) and torch.equal(oc.v[j][:s], dc.v[j][:s])
            want = torch.cat([dc.k[2 + j][:s].reshape(s, -1), dc.v[2 + j][:s].reshape(s, -1)], dim=1).cpu()
            assert torch.equal(oc.host[j][:s], want)
        tok = dev.logits[0, -1].float().argmax().view(1, 1)
        worst, agree = 0.0, 0
        for i in range(steps):
            a = model(input_ids=tok, past_key_values=dc, use_cache=True, num_logits_to_keep=1).logits[0, -1].float()
            b = model(input_ids=tok, past_key_values=oc, use_cache=True, num_logits_to_keep=1).logits[0, -1].float()
            rel = float((a - b).norm() / a.norm())
            worst = max(worst, rel)
            agree += int(a.argmax()) == int(b.argmax())
            tok = a.argmax().view(1, 1)                 # teacher forcing: both caches take the device run's token
    print(f"[offload 18432] {steps} decode steps: worst relative logit difference {worst:.3g}, "
          f"greedy tokens agree {agree}/{steps}")
    assert worst <= 1e-2 and len(dc) == len(oc) == s + steps


def test_million_token_prompt_with_both_layers_on_the_host(lib_built, monkeypatch):
    from long_vita_b200.kv_cache import OffloadedKVCache

    T = 1058816
    _need_host(2 * T * ROW, "the 1 058 816-token prompt")
    model = _model(2)
    g = torch.Generator(device="cuda").manual_seed(5)
    ids = torch.randint(0, model.config.vocab_size, (1, T), device="cuda", generator=g)
    with torch.no_grad():
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        ref = model(input_ids=ids, num_logits_to_keep=1).logits
        peak_ref = torch.cuda.max_memory_allocated() - base
        with monkeypatch.context() as m:
            _placed(m, 0)
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            out = model(input_ids=ids, use_cache=True, num_logits_to_keep=1, max_cache_len=T)
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
    c = out.past_key_values
    print(f"[offload 1M] peak device memory above the model: {peak / 2**30:.2f} GiB with the host cache, "
          f"{peak_ref / 2**30:.2f} GiB without a cache; pinned {c.host_bytes() / 1e9:.2f} GB")
    assert isinstance(c, OffloadedKVCache) and c.n_dev == 0 and len(c) == T
    assert torch.equal(out.logits, ref)
    assert c.host_bytes() == 2 * T * 4096 and c.bytes() == 0
    assert peak <= peak_ref + 64 * 2**20
    assert peak_ref <= 35328 * T * 1.05 + 2**30          # the row-chunked layer's bound, plus the logits and spans
