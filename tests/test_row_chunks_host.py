"""CPU tests of the row-chunked decoder layer (hf.modeling.row_chunks / DecoderLayer.forward) and of the in-place
`out=` of ops.rmsnorm / ops.ls_residual.

* The chunk plan, on a table of row counts: one chunk up to the threshold, 128-row aligned chunks above it, no chunk
  short enough for the GEMV path, and the chunks tile [0, T) exactly.
* The call sequence, with the recording stub library of test_ops_args_host.py: a one-chunk layer makes the same C
  calls as the whole-tensor layer always made, and a chunked layer makes them chunk by chunk on the right rows.
* Bit-identity of the composition: with the constants patched down to a few hundred rows, every surface (plain rows,
  packed rows, K/V-cache prefill + decode, B200GPTVLModel, the `--spec` layer, the context-parallel layer step over
  gloo) gives torch.equal results with and without chunking, on the CPU oracle ops (tests/hostlogic.py).  The oracle's
  GEMM here sums in float64 so that its own result cannot depend on the row count.  The GPU twin of these checks is
  tests/test_gpu_row_chunks.py.
"""
import contextlib
import socket
import types

import pytest
import torch

from long_vita_b200 import ops
from long_vita_b200.config import LongVITAConfig
from long_vita_b200.hf import modeling
from long_vita_b200.hf.modeling import DecoderLayer, row_chunks
from long_vita_b200.megatron import checkpoint as ck
from long_vita_b200.weights import synthetic_state_dict
from tests.hostlogic import oracle_ops
from tests.packed_oracle import packed_oracle_ops
from tests.test_ops_args_host import P, _bf16, lib  # noqa: F401  (lib is the recording-stub fixture)


# ------------------------------------------------------------------------------------------------
# the chunk plan
# ------------------------------------------------------------------------------------------------
def _check_plan(T, spans, threshold, chunk):
    assert spans[0][0] == 0 and spans[-1][1] == T
    assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))          # contiguous, in order: [0, T) exactly
    sizes = [r1 - r0 for r0, r1 in spans]
    if T <= threshold:
        assert spans == [(0, T)]
        return
    assert all(r0 % 128 == 0 for r0, _ in spans)
    assert all(s % 128 == 0 for s in sizes[:-1])
    assert min(sizes) > 4                                               # never the GEMV path (M <= 4)
    assert max(sizes) < chunk + 128 + 5                                 # about `chunk` rows each
    assert max(sizes[:-1], default=0) - min(sizes[:-1], default=0) == 0  # near-equal: one size, and a last remainder


@pytest.mark.parametrize("T", [1, 4, 5, 16384, 18432, 131072, 133120, 262143, 262144, 262145, 300000, 524288, 530432,
                               1058816, 2 ** 21 + 3])
def test_chunk_plan_at_product_lengths(T):
    spans = row_chunks(T)
    _check_plan(T, spans, modeling.ROW_CHUNK_THRESHOLD, modeling.ROW_CHUNK)
    assert (len(spans) == 1) == (T <= 262144)


def test_chunk_plan_with_small_constants(monkeypatch):
    """Every T up to 3 000 with a 128-row chunk: includes the cases whose remainder would be <= 4 rows (merged)."""
    monkeypatch.setattr(modeling, "ROW_CHUNK_THRESHOLD", 200)
    monkeypatch.setattr(modeling, "ROW_CHUNK", 128)
    merged = 0
    for T in range(1, 3000):
        spans = row_chunks(T)
        _check_plan(T, spans, 200, 128)
        merged += len(spans) > 1 and spans[-1][1] - spans[-1][0] > 128
    assert merged > 0


# ------------------------------------------------------------------------------------------------
# in-place out= of the residual wrappers (recording stub: the call, and the refusals)
# ------------------------------------------------------------------------------------------------
def test_rmsnorm_out_writes_the_residual_rows_in_place(lib):  # noqa: F811
    x, w, d = _bf16(10, 64), _bf16(64), _bf16(10, 64)
    y, s = ops.rmsnorm(d[2:6], w, 1e-6, residual=x[2:6], out=x[2:6])
    assert lib.calls == [("lv_rmsnorm", P(d) + 2 * 128, P(x) + 2 * 128, P(w), P(y), P(x) + 2 * 128, 4, 64, 1e-6)]
    assert s.data_ptr() == x.data_ptr() + 2 * 128 and s.shape == (4, 64)


def test_ls_residual_out_adds_in_place(lib):  # noqa: F811
    x, d = _bf16(10, 64), _bf16(4, 64)
    o = ops.ls_residual(x[6:], d, out=x[6:])
    assert lib.calls == [("lv_ls_residual", P(x) + 6 * 128, P(d), None, None, P(x) + 6 * 128, 4, 64)]
    assert o.data_ptr() == x.data_ptr() + 6 * 128


REFUSED = [
    ("rmsnorm out without residual", lambda x: ops.rmsnorm(x[:4], _bf16(64), out=x[4:8]), "rmsnorm: out receives"),
    ("rmsnorm out shifted by a row", lambda x: ops.rmsnorm(x[:4], _bf16(64), residual=x[4:8], out=x[5:9]),
     "rmsnorm: out overlaps"),
    ("rmsnorm out rows", lambda x: ops.rmsnorm(x[:4], _bf16(64), residual=x[4:8], out=_bf16(3, 64)), "rmsnorm: out"),
    ("ls_residual out strided", lambda x: ops.ls_residual(x[:4, :32], x[4:8, :32], out=_bf16(4, 64)[:, :32]),
     "ls_residual: out"),
    ("ls_residual out shifted", lambda x: ops.ls_residual(x[:4], x[4:8], out=x[1:5]), "ls_residual: out overlaps"),
]


@pytest.mark.parametrize("call,match", [r[1:] for r in REFUSED], ids=[r[0] for r in REFUSED])
def test_out_refusals_launch_nothing(lib, call, match):  # noqa: F811
    with pytest.raises(ValueError, match=match):
        call(_bf16(10, 64))
    assert lib.calls == []


# ------------------------------------------------------------------------------------------------
# the layer's C-call sequence (recording stub)
# ------------------------------------------------------------------------------------------------
def _stub_layer(H=256, hq=2, hkv=1, d=128, inter=256):
    cfg = types.SimpleNamespace(num_attention_heads=hq, num_key_value_heads=hkv, head_dim=d, rms_norm_eps=1e-6)
    p = "model.layers.0."
    n = {"self_attn.q_proj": hq * d, "self_attn.k_proj": hkv * d, "self_attn.v_proj": hkv * d}
    w = {p + k + ".weight": _bf16(r, H) for k, r in n.items()}
    w.update({p + k + ".bias": _bf16(r) for k, r in n.items()})
    w.update({p + "self_attn.o_proj.weight": _bf16(H, hq * d), p + "mlp.gate_proj.weight": _bf16(inter, H),
              p + "mlp.up_proj.weight": _bf16(inter, H), p + "mlp.down_proj.weight": _bf16(H, inter),
              p + "input_layernorm.weight": _bf16(H), p + "post_attention_layernorm.weight": _bf16(H)})
    return cfg, DecoderLayer(cfg, w, 0)


def _record_layer(lib, T, with_delta, inplace=False):  # noqa: F811
    cfg, L = _stub_layer()
    H, nq = 256, (2 + 2) * 128
    x, delta, cos, sin = _bf16(T, H), _bf16(T, H), _bf16(T, 128), _bf16(T, 128)
    att = _bf16(T, 2 * 128)

    def attend(q, k, v):
        lib.calls.append(("attend", q.data_ptr(), q.shape[0]))
        return att

    out = L.forward(x, delta if with_delta else None, cos, sin, attend, inplace=inplace)
    return L, x, delta, cos, sin, att, out, nq


@pytest.mark.parametrize("with_delta", [False, True])
def test_one_chunk_layer_makes_the_whole_tensor_calls_and_nothing_more(lib, with_delta):  # noqa: F811
    """T at the threshold: the sequence the layer has always made (norm, QKV GEMM, 2 x RoPE in place, attention, O GEMM,
    fused add + norm, gate|up GEMM with SwiGLU, down GEMM), the MLP output handed on as delta."""
    T, H = 300, 256
    with _constants(threshold=300, chunk=128):
        L, x, delta, cos, sin, att, (xo, m), nq = _record_layer(lib, T, with_delta)
    c = lib.calls
    names = [k[0] for k in c]
    assert names == ["lv_rmsnorm", "lv_gemm_bias_act", "lv_rope", "lv_rope", "attend", "lv_gemm_bias_act",
                     "lv_rmsnorm", "lv_gemm_bias_act", "lv_gemm_bias_act"]
    qkv = c[1][4]
    if with_delta:
        assert c[0][1:3] == (P(delta), P(x)) and c[0][5] not in (0, None, P(x)) and c[0][6:] == (T, H, 1e-6)
        x1 = c[0][5]
    else:
        assert c[0][1:3] == (P(x), None) and c[0][5] is None and c[0][6:] == (T, H, 1e-6)
        x1 = P(x)
    assert c[1][:4] == ("lv_gemm_bias_act", c[0][4], P(L.wqkv), P(L.bqkv)) and c[1][5:] == (T, nq, H, H, H, nq, 0)
    assert c[2][1:3] == (qkv, qkv) and c[2][3:5] == (P(cos), P(sin)) and c[2][5:8] == (T, 2, 128)
    assert c[3][1:3] == (qkv + 2 * 128 * 2, qkv + 2 * 128 * 2) and c[3][5:8] == (T, 1, 128)
    assert c[4] == ("attend", qkv, T)
    assert c[5][1:3] == (P(att), P(L.wo)) and c[5][5:] == (T, H, 256, 256, 256, H, 0)
    assert c[6][1:3] == (c[5][4], x1) and c[6][5] == P(xo) and P(xo) not in (P(x), x1)
    assert c[7][1:3] == (c[6][4], P(L.w_gate_up)) and c[7][5:] == (T, 512, H, H, H, 256, 3)
    assert c[8][1:3] == (c[7][4], P(L.w_down)) and c[8][4] == P(m) and c[8][5:] == (T, H, 256, 256, 256, H, 0)


@pytest.mark.parametrize("inplace", [False, True])
def test_chunked_layer_calls_run_chunk_by_chunk_on_their_rows(lib, inplace):  # noqa: F811
    """T = 300 over chunks of 128, 128, 44: pre-attention calls per chunk on rows r0.. of x, the QKV buffer and the
    RoPE tables; one attention call over all rows; post-attention calls per chunk ending in x[r0:r1] += MLP output
    (in x itself with `inplace`, else in a new residual buffer); no delta is handed on."""
    T, H, row = 300, 256, 256 * 2
    with _constants(threshold=200, chunk=128):
        L, x, _, cos, sin, att, (xo, m), nq = _record_layer(lib, T, False, inplace=inplace)
    spans = [(0, 128), (128, 256), (256, 300)]
    assert m is None and (P(xo) == P(x)) == inplace
    c = lib.calls
    assert [k[0] for k in c] == (["lv_rmsnorm", "lv_gemm_bias_act", "lv_rope", "lv_rope"] * 3 + ["attend"]
                                 + ["lv_gemm_bias_act", "lv_rmsnorm", "lv_gemm_bias_act", "lv_gemm_bias_act",
                                    "lv_ls_residual"] * 3)
    qkv = c[1][4]
    for i, (r0, r1) in enumerate(spans):
        n = r1 - r0
        a = c[4 * i : 4 * i + 4]
        assert a[0][1] == P(x) + r0 * row and a[0][6] == n
        assert a[1][4] == qkv + r0 * nq * 2 and a[1][5] == n and a[1][10] == nq
        assert a[2][1] == a[2][2] == qkv + r0 * nq * 2 and a[2][3] == P(cos) + r0 * 256 and a[2][5] == n
        assert a[3][4] == P(sin) + r0 * 256 and a[3][5] == n
        b = c[13 + 5 * i : 18 + 5 * i]
        assert b[0][1] == P(att) + r0 * row and b[0][5] == n
        assert b[1][2] == P(x) + r0 * row and b[1][5] == P(xo) + r0 * row and b[1][6] == n
        assert b[4][1:3] == (P(xo) + r0 * row, b[3][4]) and b[4][5:] == (P(xo) + r0 * row, n, H)
    assert c[12] == ("attend", qkv, T)


# ------------------------------------------------------------------------------------------------
# bit-identity of the chunked composition on the CPU oracle
# ------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _constants(threshold, chunk):
    saved = modeling.ROW_CHUNK_THRESHOLD, modeling.ROW_CHUNK
    modeling.ROW_CHUNK_THRESHOLD, modeling.ROW_CHUNK = threshold, chunk
    try:
        yield
    finally:
        modeling.ROW_CHUNK_THRESHOLD, modeling.ROW_CHUNK = saved


def _bf(t):
    return t.to(torch.bfloat16)


def _rmsnorm(x, weight, eps=1e-6, residual=None, out=None):
    from oracle import ops as O

    if residual is None:
        return O.rmsnorm(x, weight, eps)
    s = _bf(x.float() + residual.float())
    y = O.rmsnorm(s, weight, eps)
    if out is None:
        return y, s
    out.copy_(s)
    return y, out


def _ls_residual(x, y, ls=None, bias=None, out=None):
    from oracle import ops as O

    r = _bf(O.ls_residual(x.float(), y.float(), None if ls is None else ls.float(), None if bias is None else bias.float()))
    if out is None:
        return r
    out.copy_(r)
    return out


def _linear(x, weight, bias=None, act=None, out=None):
    import torch.nn.functional as F

    y = x.double().reshape(-1, x.shape[-1]) @ weight.double().t()
    if bias is not None:
        y = y + bias.double()
    if act == "swiglu":
        y = F.silu(_bf(y[:, 0::2]).float()) * _bf(y[:, 1::2]).float()
    elif act is not None:
        y = F.gelu(y.float(), approximate="tanh" if act == "gelu_tanh" else "none")
    y = _bf(y)
    if out is not None:
        out.view(y.shape).copy_(y)
        y = out
    return y.view(*x.shape[:-1], y.shape[-1])


@contextlib.contextmanager
def exact_oracle_ops():
    """packed_oracle_ops() (the oracle ops, attention with `cu_seqlens`) with `out=` on the residual wrappers and a
    GEMM whose per-row result cannot depend on M."""
    with packed_oracle_ops() as o:
        o.rmsnorm, o.ls_residual, o.linear = _rmsnorm, _ls_residual, _linear      # restored by oracle_ops on exit
        yield o


CHUNKINGS = [(256, 128), (200, 300)]          # (threshold, chunk): 128-row chunks; 256-row chunks and a ragged end


@pytest.fixture(scope="module")
def tiny():
    cfg = LongVITAConfig.tiny(layers=2, vit_layers=1)
    w = synthetic_state_dict(cfg, seed=31, dtype=torch.bfloat16, perturb=True)
    return cfg, w


def _inputs(cfg, s=700, n_img=2, seed=1):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, cfg.vocab_size, (1, s), generator=g)
    images = torch.randn(n_img, 3, 448, 448, generator=g).to(torch.bfloat16)
    idx_s = torch.stack([torch.arange(5 + i * 300, 5 + i * 300 + 256) for i in range(n_img)])
    return ids, images, torch.stack([torch.zeros_like(idx_s), idx_s])


def _each_chunking(fn):
    """fn() with one chunk, then under each of CHUNKINGS; asserts the chunked plans really have several chunks."""
    with exact_oracle_ops():
        whole = fn()
        outs = []
        for threshold, chunk in CHUNKINGS:
            with _constants(threshold, chunk):
                outs.append(fn())
    return whole, outs


def _equal(a, b):
    if isinstance(a, torch.Tensor):
        return torch.equal(a, b)
    return len(a) == len(b) and all(_equal(x, y) for x, y in zip(a, b))


def test_plain_rows_with_images(tiny):
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w)
    ids, images, idx = _inputs(cfg)
    assert len(row_chunks(ids.shape[1])) == 1
    with _constants(256, 128):
        assert len(row_chunks(ids.shape[1])) == 6

    def run():
        a = model(input_ids=ids, images=images, image_indices=idx, num_logits_to_keep=100)
        b = model(input_ids=ids, images=images, image_indices=idx, output_hidden_states=True)
        return a.logits, b.logits, b.hidden_states

    whole, outs = _each_chunking(run)
    for o in outs:
        assert _equal(o, whole)
    assert torch.equal(whole[0][0], whole[1][0, -100:])


def test_inputs_embeds_are_not_overwritten(tiny):
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w)
    emb = torch.randn(1, 600, cfg.hidden_size, generator=torch.Generator().manual_seed(4)).to(torch.bfloat16)
    keep = emb.clone()
    whole, outs = _each_chunking(lambda: model(inputs_embeds=emb).logits)
    assert all(torch.equal(o, whole) for o in outs) and torch.equal(emb, keep)


def test_packed_rows(tiny):
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w)
    ids, images, idx = _inputs(cfg)
    pos = torch.cat([torch.arange(450), torch.arange(250)]).unsqueeze(0)      # two samples, attention inside each
    whole, outs = _each_chunking(lambda: model(input_ids=ids, images=images, image_indices=idx, position_ids=pos).logits)
    assert all(torch.equal(o, whole) for o in outs)


def test_kv_cache_prefill_then_decode(tiny):
    cfg, w = tiny
    model = modeling.LongVITAForCausalLM(cfg, w)
    ids, images, idx = _inputs(cfg)

    def run():
        out = model(input_ids=ids, images=images, image_indices=idx, use_cache=True, num_logits_to_keep=1,
                    max_cache_len=ids.shape[1] + 8)
        cache, logits = out.past_key_values, [out.logits]
        for _ in range(6):
            tok = logits[-1][0, -1].float().argmax().view(1, 1)
            logits.append(model(input_ids=tok, past_key_values=cache, use_cache=True, num_logits_to_keep=1).logits)
        return logits, [cache.k[i][: len(cache)] for i in range(len(cache.k))]

    whole, outs = _each_chunking(run)
    assert all(_equal(o, whole) for o in outs)


def test_megatron_model_with_logit_mask(tiny):
    from long_vita_b200.megatron.gpt_vl_model import B200GPTVLModel

    cfg, w = tiny
    with oracle_ops():
        model = B200GPTVLModel(cfg, ck.hf_to_mcore(w, cfg))
    ids, images, idx = _inputs(cfg)
    s = ids.shape[1]
    mask = torch.zeros(1, s, dtype=torch.bool)
    mask[0, [3, 130, 257, 699]] = True
    whole, outs = _each_chunking(lambda: model(ids, torch.arange(s).unsqueeze(0), None, logit_mask=mask,
                                               external_inputs={"images": images, "indices": idx}))
    assert whole.shape == (1, 4, cfg.vocab_size) and all(torch.equal(o, whole) for o in outs)


def test_spec_layer(tiny):
    """The `--spec` layer adds the MLP output itself when chunked, and leaves Megatron's hidden_states untouched."""
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
    whole, outs = _each_chunking(lambda: layer(hidden_states=x, rotary_pos_emb=rotary)[0])
    assert all(torch.equal(o, whole) for o in outs) and torch.equal(x, keep)


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
        S = ids.shape[1]
        images = torch.randn(2, 3, 448, 448, generator=torch.Generator().manual_seed(3)).to(torch.bfloat16)
        sh = CP.shard_prompt(ids, idx, world, rank, cfg.visual.tokens_per_image)
        tpi = cfg.visual.tokens_per_image
        ext = {"images": images[sh.image_sel], "src_indices": (sh.src_idx // tpi, sh.src_idx % tpi),
               "tgt_indices": (torch.zeros_like(sh.dst_idx), sh.dst_idx)}
        with oracle_ops():
            model = B200GPTVLModel(cfg, mc, cp=_GlooCPContext(S, cfg.num_attention_heads, cfg.num_key_value_heads,
                                                               cfg.head_dim))
        whole, outs = _each_chunking(lambda: model(sh.input_ids, sh.position_ids.unsqueeze(0), None, external_inputs=ext))
        with _constants(*CHUNKINGS[0]):
            n_chunks = len(row_chunks(sh.input_ids.shape[1]))
        torch.save({"equal": all(torch.equal(o, whole) for o in outs), "chunks": n_chunks, "T": sh.input_ids.shape[1]},
                   f"{path}.{rank}")
    finally:
        dist.destroy_process_group()


def test_context_parallel_layer_step_over_gloo(tmp_path):
    """2 ranks, the K/V exchange emulated by a gloo all-gather: the chunked QKV GEMM fills the rank's QKV buffer row
    chunk by row chunk before the (one) attention call, and each rank's logits are bit-identical to one chunk."""
    import torch.multiprocessing as mp

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    path = str(tmp_path / "cp")
    mp.spawn(_cp_worker, args=(2, port, path), nprocs=2, join=True)
    for r in range(2):
        res = torch.load(f"{path}.{r}")
        assert res["equal"] and res["chunks"] > 1, res
