"""CPU tests of packed training samples (`--reset-position-ids --reset-attention-mask`):

* pinning: the oracle's document mask is the mask the reference's own get_ltor_masks_and_position_ids builds, and
  ops.packed_cu_seqlens agrees with the reference's compute_actual_seq_len and with transformers'
  prepare_fa_kwargs_from_position_ids - from tests/golden/ref_packed_docs.pt, and live where the reference is mounted;
* the C ABI of the document kernels rejects every unsupported call with LV_EINVAL and a message (no GPU needed);
* host logic: a packed prompt through B200GPTVLModel, the `--spec` layer, the Megatron core-attention slot, the
  b200_fa interface and LongVITAModel gives, on the oracle swap (tests/packed_oracle.py), the per-document results;
* packing under context parallelism, with a KV cache, or without a causal mask raises.
"""
import ctypes
import os
import sys
import types

import pytest
import torch

from oracle import model as OM
from oracle import ops as O
from oracle import ref_loader
from tests import packed_oracle as PO
from tests.packed_oracle import packed_oracle_ops
from tests.util import rel_fro

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "ref_packed_docs.pt")
EOD = 7
SEQ = 128


def golden_token_rows():
    """Seeded EOD-delimited rows: random samples, an EOD first, two EODs in a row, an EOD last, and no EOD at all."""
    g = torch.Generator().manual_seed(2024)
    rows = []
    for _ in range(3):
        r = torch.randint(8, 100, (SEQ,), generator=g)
        r[torch.randint(0, SEQ, (5,), generator=g)] = EOD
        rows.append(r)
    r = torch.randint(8, 100, (SEQ,), generator=g)
    r[[0, 40, 41, SEQ - 1]] = EOD
    rows.append(r)
    rows.append(torch.randint(8, 100, (SEQ,), generator=g))
    return torch.stack(rows)


def reference_packed_docs():
    """The reference's own get_ltor_masks_and_position_ids (reset_position_ids / reset_attention_mask, as every shipped
    fine-tuning script sets them) and compute_actual_seq_len on golden_token_rows()."""
    utils, _ = ref_loader.load_megatron_training_utils(1, 0, SEQ)
    tokens = golden_token_rows()
    out = {"tokens": tokens, "eod": EOD, "mask": [], "position_ids": [], "actual_seq_len": []}
    for row in tokens:
        mask, _, pos = utils.get_ltor_masks_and_position_ids(row.view(1, -1), EOD, True, True, False)
        out["mask"].append(mask[0, 0].clone())
        out["position_ids"].append(pos[0].clone())
        out["actual_seq_len"].append(list(utils.compute_actual_seq_len(pos[0])))
    return out


def _check_against(rec):
    from long_vita_b200 import ops
    from transformers.modeling_flash_attention_utils import prepare_fa_kwargs_from_position_ids

    for mask, pos, ends in zip(rec["mask"], rec["position_ids"], rec["actual_seq_len"]):
        cu = [0] + [int(e) for e in ends]
        assert torch.equal(PO.document_mask(cu, SEQ), mask)
        got = ops.packed_cu_seqlens(pos.view(1, -1))
        assert (got is None) == (len(ends) == 1)
        if got is not None:
            assert got.dtype == torch.int32 and got.tolist() == cu
        assert ops.packed_cu_seqlens(actual_seq_len=ends, device="cpu") is None or got.tolist() == cu
        (cu_q, cu_k), _ = prepare_fa_kwargs_from_position_ids(pos.view(1, -1))
        assert cu_q.tolist() == cu and cu_k.tolist() == cu


def test_document_mask_and_boundaries_match_the_reference_fixture():
    _check_against(torch.load(GOLDEN))


@pytest.mark.skipif(not ref_loader.available(), reason="the reference is not mounted here")
def test_document_mask_and_boundaries_match_the_reference_live():
    rec = reference_packed_docs()
    gold = torch.load(GOLDEN)
    assert torch.equal(rec["tokens"], gold["tokens"])
    for a, b in zip(rec["mask"], gold["mask"]):
        assert torch.equal(a, b)
    assert rec["actual_seq_len"] == gold["actual_seq_len"]
    _check_against(rec)


# ------------------------------------------------------------------------------------------------
# packed_cu_seqlens
# ------------------------------------------------------------------------------------------------
def test_packed_cu_seqlens_rules():
    from long_vita_b200 import ops

    assert ops.packed_cu_seqlens(torch.arange(50).view(1, -1)) is None
    assert ops.packed_cu_seqlens(torch.cat([torch.arange(0, 16), torch.arange(48, 64)]).view(1, -1)) is None  # zig-zag
    pos = torch.cat([torch.arange(10), torch.arange(5), torch.arange(1)])
    for shape in ((1, -1), (-1, 1), (-1,)):
        assert ops.packed_cu_seqlens(pos.view(*shape)).tolist() == [0, 10, 15, 16]
    assert ops.packed_cu_seqlens(actual_seq_len=[10, 15, 16], device="cpu", seq_len=16).tolist() == [0, 10, 15, 16]
    assert ops.packed_cu_seqlens(actual_seq_len=[16], device="cpu", seq_len=16) is None
    with pytest.raises(ValueError, match="micro-batch"):
        ops.packed_cu_seqlens(torch.stack([pos, pos]))
    with pytest.raises(ValueError, match="start at 0"):
        ops.packed_cu_seqlens(torch.cat([torch.arange(3, 10), torch.arange(5)]).view(1, -1))
    with pytest.raises(ValueError, match="strictly|0 = c0"):
        ops.packed_cu_seqlens(actual_seq_len=[10, 10, 16], device="cpu")
    with pytest.raises(ValueError, match="ends at"):
        ops.packed_cu_seqlens(actual_seq_len=[10, 15], device="cpu", seq_len=16)


# ------------------------------------------------------------------------------------------------
# C ABI
# ------------------------------------------------------------------------------------------------
def _params(**kw):
    from long_vita_b200._lib import AttnBwdParams

    b = AttnBwdParams()
    p = b.fwd
    p.q = p.k = p.v = p.out = p.lse = 0x1000          # never dereferenced: every case fails validation first
    p.batch, p.sq, p.sk, p.hq, p.hkv, p.d = 1, 256, 256, 8, 2, 128
    for arr, row in ((p.q_strides, 8 * 128), (p.k_strides, 2 * 128), (p.v_strides, 2 * 128), (p.o_strides, 8 * 128)):
        arr[0], arr[1], arr[2] = 256 * row, row, 128
    p.scale, p.causal, p.q_seg_len, p.kv_pos0 = 0.088, 1, 256, 0
    b.d_out = b.dq = b.dk = b.dv = b.delta_ws = 0x1000
    for arr, row in ((b.do_strides, 8 * 128), (b.dq_strides, 8 * 128), (b.dk_strides, 2 * 128), (b.dv_strides, 2 * 128)):
        arr[0], arr[1], arr[2] = 256 * row, row, 128
    for k, v in kw.items():
        if k == "q_seg_pos":
            p.q_seg_pos[0], p.q_seg_pos[1] = v
        else:
            setattr(p, k, v)
    return b


@pytest.mark.parametrize("kw,docs,msg", [
    (dict(batch=2), None, b"batch 1"),
    (dict(sk=384), None, b"sq == sk"),
    (dict(causal=0), None, b"causal = 1"),
    (dict(q_seg_len=128), None, b"q_seg_len == sq"),
    (dict(kv_pos0=5), None, b"kv_pos0 = 0"),
    (dict(q_seg_pos=(3, 0)), None, b"q_seg_pos = {0, 0}"),
    ({}, (0x2000, 0), b"n_docs=0 out of range"),
    ({}, (None, 3), b"null cu_seqlens"),
])
def test_document_entry_points_reject_unsupported_calls(lib_built, kw, docs, msg):
    from long_vita_b200 import _lib
    from long_vita_b200._lib import AttnDocs

    h = _lib.lib()
    b = _params(**kw)
    d = AttnDocs()
    d.cu_seqlens, d.n_docs = docs if docs is not None else (0x2000, 2)
    rc = h.lv_attn_docs_fwd(ctypes.byref(b.fwd), ctypes.byref(d), None)
    assert rc == -1 and msg in h.lv_last_error(), h.lv_last_error()
    rc = h.lv_attn_docs_bwd(ctypes.byref(b), ctypes.byref(d), None)
    assert rc == -1 and msg in h.lv_last_error(), h.lv_last_error()
    assert h.lv_attn_docs_fwd(ctypes.byref(b.fwd), None, None) == -1 and b"null docs" in h.lv_last_error()


def test_document_symbols_are_exported_and_bound(lib_built):
    from long_vita_b200 import _lib

    h = _lib.lib()
    assert h.lv_version() == 1001
    for name in ("lv_attn_docs_fwd", "lv_attn_docs_bwd"):
        assert name in _lib.SIGNATURES and hasattr(ctypes.CDLL(lib_built), name)
    assert ctypes.sizeof(_lib.AttnDocs) == 16
    assert ctypes.sizeof(_lib.AttnParams) == 5 * 8 + 6 * 8 + 12 * 8 + 4 + 4 + 8 + 16 + 8


# ------------------------------------------------------------------------------------------------
# host-logic composition on the oracle swap
# ------------------------------------------------------------------------------------------------
LENGTHS = [70, 130, 1, 99]


def _packed_pos():
    return torch.cat([torch.arange(n) for n in LENGTHS]).view(1, -1)


def _bounds():
    cu = [0]
    for n in LENGTHS:
        cu.append(cu[-1] + n)
    return list(zip(cu, cu[1:]))


@pytest.fixture(scope="module")
def tiny():
    from tests.test_megatron_model_host import tiny_setup

    return tiny_setup()


def _per_doc_oracle_logits(cfg, hf, ids):
    w32 = OM.cast_weights(hf, torch.float32)
    return torch.cat([OM.long_vita_forward(cfg, w32, ids[:, a:b], None, None)[0] for a, b in _bounds()])


def _same_as_alone(packed, alone):
    """Packed rows against each document run alone through the same model: equal up to the bf16 rounding of GEMMs
    over a different number of rows (an argmax may flip only where two logits tie to that rounding)."""
    assert rel_fro(packed, alone) < 3e-3, rel_fro(packed, alone)
    assert float((packed.float().argmax(-1) == alone.float().argmax(-1)).float().mean()) >= 0.99


def test_gptvl_model_packed_prompt_equals_per_document_oracle(tiny):
    from tests.test_megatron_model_host import build_model

    cfg, hf, mc = tiny
    model = build_model(mc, cfg)
    s = sum(LENGTHS)
    ids = torch.randint(0, cfg.vocab_size, (1, s), generator=torch.Generator().manual_seed(3))
    with packed_oracle_ops():
        out = model(ids, _packed_pos(), None)
    ref = _per_doc_oracle_logits(cfg, hf, ids)
    assert rel_fro(out[0], ref) < 1.5e-2
    with packed_oracle_ops():
        alone = torch.cat([model(ids[:, a:b], torch.arange(b - a).view(1, -1), None)[0] for a, b in _bounds()])
    _same_as_alone(out[0], alone)
    # the same rows without packing see the earlier documents: a different result
    with packed_oracle_ops():
        dense = model(ids, torch.arange(s).view(1, -1), None)
    assert rel_fro(dense[0, LENGTHS[0]:], ref[LENGTHS[0]:]) > 0.05
    # packing is refused with a KV cache and under context parallelism
    ip = types.SimpleNamespace(key_value_memory_dict={}, max_sequence_length=2 * s)
    with packed_oracle_ops(), pytest.raises(NotImplementedError, match="KV cache"):
        model(ids, _packed_pos(), None, inference_params=ip)
    model.cp = object()
    try:
        with packed_oracle_ops(), pytest.raises(NotImplementedError, match="context parallelism"):
            model(ids, _packed_pos(), None)
    finally:
        model.cp = None


def test_hf_model_packed_prompt_equals_per_document_oracle():
    from long_vita_b200.config import LongVITAConfig
    from long_vita_b200.hf.modeling import LongVITAForCausalLM
    from long_vita_b200.weights import synthetic_state_dict

    cfg = LongVITAConfig.tiny(layers=2, vit_layers=1)
    w = synthetic_state_dict(cfg, seed=31, dtype=torch.bfloat16, perturb=True)
    model = LongVITAForCausalLM(cfg, w)
    s = sum(LENGTHS)
    ids = torch.randint(0, cfg.vocab_size, (1, s), generator=torch.Generator().manual_seed(4))
    with packed_oracle_ops():
        out = model(input_ids=ids, position_ids=_packed_pos()).logits
    ref = _per_doc_oracle_logits(cfg, w, ids)
    assert rel_fro(out[0].float(), ref) < 1.5e-2
    with packed_oracle_ops():
        alone = torch.cat([model(input_ids=ids[:, a:b]).logits[0] for a, b in _bounds()])
    _same_as_alone(out[0], alone)
    with packed_oracle_ops(), pytest.raises(NotImplementedError, match="KV cache"):
        model(input_ids=ids, position_ids=_packed_pos(), use_cache=True)


@pytest.fixture
def megatron_packed(monkeypatch):
    """Stand-in for `long_vita_megatron.training.utils` with the actual_seq_len of a packed micro-batch."""
    mod = types.ModuleType("long_vita_megatron.training.utils")
    state = {"ends": None}
    mod.get_actual_seq_len = lambda: state["ends"]
    monkeypatch.setitem(sys.modules, "long_vita_megatron.training.utils", mod)
    return state


def _spec_layer(cfg, mc, **extra):
    from long_vita_b200.megatron.transformer_layer import B200TransformerLayer

    mcfg = types.SimpleNamespace(hidden_size=cfg.hidden_size, num_attention_heads=cfg.num_attention_heads,
                                 num_query_groups=cfg.num_key_value_heads, kv_channels=cfg.head_dim,
                                 ffn_hidden_size=cfg.intermediate_size, layernorm_epsilon=cfg.rms_norm_eps,
                                 hidden_dropout=0.0, attention_dropout=0.0, params_dtype=torch.bfloat16, **extra)
    layer = B200TransformerLayer(mcfg, layer_number=1)
    sd = {k[len("decoder.layers.0."):]: v for k, v in mc.items() if k.startswith("decoder.layers.0.")}
    layer.load_state_dict(sd, strict=True)
    return layer


def _rotary(cfg, pos):
    inv = O.rope_inv_freq(cfg.head_dim, cfg.rope_theta)
    freqs = torch.outer(pos.float(), inv)
    return torch.cat((freqs, freqs), dim=-1).view(-1, 1, 1, cfg.head_dim)


def test_spec_layer_forward_and_training_with_actual_seq_len(tiny, megatron_packed):
    cfg, hf, mc = tiny
    layer = _spec_layer(cfg, mc)
    s = sum(LENGTHS)
    x = torch.randn(s, 1, cfg.hidden_size, generator=torch.Generator().manual_seed(5)).to(torch.bfloat16)
    pos = _packed_pos().view(-1)
    call = dict(attention_mask=None, context=None, context_mask=None, inference_params=None, packed_seq_params=None)

    def per_doc(train):
        outs, grads = [], []
        megatron_packed["ends"] = None
        for a, b in _bounds():
            xi = x[a:b].clone().requires_grad_(train)
            with packed_oracle_ops():
                o, _ = layer(hidden_states=xi, rotary_pos_emb=_rotary(cfg, pos[a:b]), **call)
                if train:
                    o.float().square().sum().backward()
            outs.append(o.detach())
            grads.append(xi.grad if train else None)
        return torch.cat(outs), (torch.cat(grads) if train else None)

    for train in (False, True):
        ref, gref = per_doc(train)
        megatron_packed["ends"] = [b for _, b in _bounds()]
        xp = x.clone().requires_grad_(train)
        with packed_oracle_ops():
            out, _ = layer(hidden_states=xp, rotary_pos_emb=_rotary(cfg, pos), **call)
            if train:
                out.float().square().sum().backward()
        assert rel_fro(out.detach(), ref) < 1e-2, (train, rel_fro(out.detach(), ref))
        if train:
            assert rel_fro(xp.grad, gref) < 2e-2, rel_fro(xp.grad, gref)
    # context parallelism + packing is refused
    cp_layer = _spec_layer(cfg, mc, context_parallel_size=2)
    with packed_oracle_ops(), pytest.raises(NotImplementedError, match="context parallelism"):
        cp_layer(hidden_states=x, rotary_pos_emb=_rotary(cfg, pos), **call)


@pytest.mark.parametrize("np_,ng", [(5, 1), (40, 8)])
def test_core_attention_slot_uses_actual_seq_len(megatron_packed, np_, ng):
    """The TP8 head slice of the 14B model (5 query heads, 1 kv head) and the whole 40:8 layer."""
    from long_vita_b200.megatron import stub
    from long_vita_b200.megatron.core_attention import B200DotProductAttention

    hn, s = 16, sum(LENGTHS)
    cfg = stub.TransformerConfig(hidden_size=np_ * hn, num_attention_heads=np_, num_query_groups=ng)
    attn = stub.build_module(stub.ModuleSpec(module=B200DotProductAttention), config=cfg, layer_number=1,
                             attn_mask_type=stub.AttnMaskType.causal, attention_type="self")
    g = torch.Generator().manual_seed(np_)
    q, k, v = (torch.randn(s, 1, h, hn, generator=g).to(torch.bfloat16) for h in (np_, ng, ng))
    cu = [0] + [b for _, b in _bounds()]
    ref, _ = PO.attention(q.permute(1, 0, 2, 3), k.permute(1, 0, 2, 3), v.permute(1, 0, 2, 3), cu)
    ref = ref.permute(1, 0, 2, 3).reshape(s, 1, np_ * hn)
    megatron_packed["ends"] = cu[1:]
    with packed_oracle_ops():
        out = attn(q, k, v, None, attn_mask_type=stub.AttnMaskType.causal, packed_seq_params=None)
        assert rel_fro(out, ref) < 1e-2
        # training branch
        qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
        o2 = attn(qg, kg, vg, None)
        o2.float().sum().backward()
        assert rel_fro(o2.detach(), ref) < 1e-2 and qg.grad is not None
        with pytest.raises(NotImplementedError, match="causal"):
            attn(q, k, v, None, attn_mask_type=stub.AttnMaskType.no_mask)
    cp_attn = stub.build_module(stub.ModuleSpec(module=B200DotProductAttention),
                                config=stub.TransformerConfig(hidden_size=np_ * hn, num_attention_heads=np_,
                                                              num_query_groups=ng, context_parallel_size=2),
                                layer_number=1, attn_mask_type=stub.AttnMaskType.causal, attention_type="self")
    with packed_oracle_ops(), pytest.raises(NotImplementedError, match="context parallelism"):
        cp_attn(q, k, v, None)


def test_hf_attention_interface_honours_packing():
    from long_vita_b200.hf.attention_interface import b200_attention_forward

    s, hq, hkv, d = sum(LENGTHS), 4, 2, 32
    g = torch.Generator().manual_seed(8)
    q, k, v = (torch.randn(1, h, s, d, generator=g).to(torch.bfloat16) for h in (hq, hkv, hkv))
    cu = [0] + [b for _, b in _bounds()]
    ref, _ = PO.attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), cu)
    mod = types.SimpleNamespace(is_causal=True)
    with packed_oracle_ops():
        a, _ = b200_attention_forward(mod, q, k, v, None, position_ids=_packed_pos())
        cut = torch.tensor(cu, dtype=torch.int32)
        b, _ = b200_attention_forward(mod, q, k, v, None, cu_seq_lens_q=cut, cu_seq_lens_k=cut, max_length_q=130,
                                      max_length_k=130)
        plain, _ = b200_attention_forward(mod, q, k, v, None, position_ids=torch.arange(s).view(1, -1))
        with pytest.raises(NotImplementedError, match="cu_seq_lens_q == cu_seq_lens_k"):
            b200_attention_forward(mod, q, k, v, None, cu_seq_lens_q=cut, cu_seq_lens_k=cut + 0 * cut - cut)
    assert rel_fro(a, ref) < 1e-2 and torch.equal(a, b)
    assert rel_fro(plain[:, LENGTHS[0]:], ref[:, LENGTHS[0]:]) > 0.05


def test_context_parallel_entry_points_refuse_packing():
    from long_vita_b200 import cp

    t = torch.zeros(4, 2, 8)
    with pytest.raises(NotImplementedError, match="context parallelism"):
        cp.cp_attention(t, t, t, None, cu_seqlens=torch.tensor([0, 2, 4]))
    with pytest.raises(NotImplementedError, match="context parallelism"):
        cp.CPContext.attention_separate(None, t, t, t, cu_seqlens=torch.tensor([0, 2, 4]))
    with pytest.raises(NotImplementedError, match="context parallelism"):
        cp.CPContext.attention(None, cu_seqlens=torch.tensor([0, 2, 4]))
