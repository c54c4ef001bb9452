/*
 * lvb200.h - C ABI of the H100-native Long-VITA hot path (long-context forward / backward).
 *
 * This is the drop-in boundary (SURVEY.md section 8, row B5).  The reference has no native layer: on
 * GPU it reaches flash-attn 2, TransformerEngine, apex and cuBLAS through Python.  Every entry
 * point below replaces one of those third-party calls; the comment on each cites the reference
 * call site (path:line relative to the Long-VITA repository) whose arithmetic it reproduces.
 *
 * Conventions
 *   - plain device pointers and sizes only; no framework types cross this boundary;
 *   - the caller owns every buffer (inputs, outputs, workspace); nothing is allocated here
 *     except per-process tensor-map caches;
 *   - every call takes the CUDA stream to launch on and is asynchronous with respect to the host;
 *   - return value: 0 on success, a negative LV_E* code otherwise; lv_last_error() returns a
 *     thread-local description of the last failure on the calling thread;
 *   - activations are bfloat16 unless stated otherwise ("bf16" below), statistics are float;
 *   - all functions are re-entrant and keep no mutable global state other than the
 *     peer-mapped allocations made through lv_ipc_alloc().
 */
#ifndef LVB200_H_
#define LVB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* lv_stream_t; /* cudaStream_t */

#define LV_OK 0
#define LV_EINVAL (-1)    /* bad argument (shape, stride, alignment)            */
#define LV_ECUDA (-2)     /* a CUDA runtime / driver call failed                */
#define LV_ENOTSUP (-3)   /* valid request this build does not implement        */
#define LV_ESTATE (-4)    /* context-parallel heap not registered / bad epoch   */

/* ABI version: major * 1000 + minor. */
int lv_version(void);
/* Thread-local text of the last error returned on this thread ("" if none). */
const char* lv_last_error(void);
/* Number of kernels this library has launched in this process (all threads). */
int64_t lv_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Attention (forward).
 *
 * Replaces flash_attn_func / _flash_attention_forward as called from
 *   long_vita_megatron/core/transformer/dot_product_attention.py:318-326 (ViT, non-causal) and
 *   :374-390 (LLM, causal, GQA kv heads not pre-expanded, :176-184), and from
 *   long_vita/models/long_vita_qwen2_intern/flash_attention.py:52-74 (HF ViT).
 *
 * out[b, i, h, :] = sum_j softmax_j(scale * q[b,i,h,:] . k[b,j,h/(hq/hkv),:]) v[b,j,h/(hq/hkv),:]
 * lse[b, h, i]    = log sum_j exp(scale * q.k)          (natural log; float; may be NULL)
 *
 * Strides are in elements; the head dimension is contiguous (stride 1).  Supported head_dim: 64,
 * 128.  q_pos0 / causal: query row i has global position q_seg_pos[i / q_seg_len] + i % q_seg_len
 * and key row j has position kv_pos0 + j; with causal != 0 a key is visible iff
 * key_pos <= query_pos.  For a plain causal call use q_seg_len = sq, q_seg_pos = {sk - sq, 0},
 * kv_pos0 = 0 (bottom-right aligned, the flash-attn >= 2.1 convention the reference relies on).
 * The zig-zag context-parallel layout (training/utils.py:329-341) is q_seg_len = sq / 2,
 * q_seg_pos = {r * c, (2 cp - 1 - r) * c}.
 * ------------------------------------------------------------------------------------------ */
typedef struct lv_attn_params {
  const void* q;  /* bf16 [b, sq, hq, d]  (any strides, d contiguous) */
  const void* k;  /* bf16 [b, sk, hkv, d] */
  const void* v;  /* bf16 [b, sk, hkv, d] */
  void* out;      /* bf16 [b, sq, hq, d]  */
  float* lse;     /* float [b, hq, sq] contiguous, or NULL */
  int64_t batch, sq, sk, hq, hkv, d;
  int64_t q_strides[3];   /* batch, seq, head */
  int64_t k_strides[3];
  int64_t v_strides[3];
  int64_t o_strides[3];
  float scale;            /* softmax scale, e.g. 1/sqrt(d); finite and > 0, else LV_EINVAL */
  int32_t causal;         /* 0 / 1 */
  int64_t q_seg_len;      /* rows per query segment (sq if one segment); multiple of 128 if < sq */
  int64_t q_seg_pos[2];   /* global position of the first row of each query segment */
  int64_t kv_pos0;        /* global position of key row 0 */
} lv_attn_params;

int lv_attn_fwd(const lv_attn_params* p, lv_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Attention (backward): dQ, dK, dV of lv_attn_fwd.
 *
 * Replaces flash-attn 2's backward, which the reference reaches through autograd of
 * flash_attn_func / _flash_attention_forward (dot_product_attention.py:318-326, 374-390) during
 * pretrain_long_vita.py.  `fwd` repeats the forward call's arguments with `out` and `lse` holding the
 * forward results (lse is required).  d_out has the layout of out; dq / dk / dv have the shapes of
 * q / k / v (GQA: dk, dv are summed over the query heads of each group).  delta_ws is caller
 * workspace of lv_attn_bwd_ws_bytes(batch, hq, sq) bytes (batch*hq*sq floats).  Deterministic (no atomics): two tensor-core passes, one for
 * dK/dV and one for dQ.
 * ------------------------------------------------------------------------------------------ */
typedef struct lv_attn_bwd_params {
  lv_attn_params fwd;
  const void* d_out;      /* bf16 [b, sq, hq, d]  */
  void* dq;               /* bf16 [b, sq, hq, d]  */
  void* dk;               /* bf16 [b, sk, hkv, d] */
  void* dv;               /* bf16 [b, sk, hkv, d] */
  int64_t do_strides[3];  /* batch, seq, head */
  int64_t dq_strides[3];
  int64_t dk_strides[3];
  int64_t dv_strides[3];
  float* delta_ws;        /* float [b, hq, sq] */
} lv_attn_bwd_params;

int64_t lv_attn_bwd_ws_bytes(int64_t batch, int64_t hq, int64_t sq);
int lv_attn_bwd(const lv_attn_bwd_params* p, lv_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Document-masked attention over one packed row of training samples (`--reset-attention-mask`),
 * forward and backward.
 *
 * Replaces the packed-sample attention of the reference: on GPU, _flash_attention_forward called
 * with the reset position ids (long_vita_megatron/core/transformer/dot_product_attention.py:374-390),
 * which transformers turns into flash_attn_varlen_func over the documents; on NPU, the varlen flash
 * attention fed with actual_seq_len as the document ends (long_vita_modellink/core/transformer/
 * dot_product_attention.py:334-365, 373-382, 460-470).  Same mask as Megatron's
 * get_ltor_masks_and_position_ids(reset_attention_mask=True) (training/utils.py:192-249).
 *
 * The row holds n_docs documents with boundaries cu_seqlens = {0 = c_0 < c_1 < ... < c_n = sk}
 * (int32, device memory; the layout of flash-attn varlen, Megatron's PackedSeqParams and
 * transformers; the reference's actual_seq_len is c_1 .. c_n).  Key j is visible to query i iff
 * both lie in the same document and j <= i.  `a` / `p` are filled as for lv_attn_fwd / lv_attn_bwd
 * with batch = 1, sq = sk, causal = 1, q_seg_len = sq, q_seg_pos = {0, 0}, kv_pos0 = 0; any other
 * value returns LV_EINVAL.  Key tiles that lie wholly in earlier documents are skipped, so the cost
 * follows the visible pairs sum_i L_i (L_i + 1) / 2 rather than S (S + 1) / 2.  With n_docs = 1 the
 * results are bit-identical to lv_attn_fwd / lv_attn_bwd with causal = 1.  No workspace beyond
 * lv_attn_bwd's; deterministic (no atomics).  The kernels clamp every index they derive from
 * cu_seqlens (memory-safe on a malformed table), but the result is only defined for a valid one.
 * ------------------------------------------------------------------------------------------ */
typedef struct lv_attn_docs {
  const int32_t* cu_seqlens;  /* device, [n_docs + 1]: 0 = c0 < c1 < ... < c_n = sk */
  int64_t n_docs;
} lv_attn_docs;

int lv_attn_docs_fwd(const lv_attn_params* a, const lv_attn_docs* docs, lv_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * The FP8 row rule (csrc/fp8_core.h), which every FP8 entry point below quantises with.  fmt: 0 = e4m3 (largest
 * finite value M = 448), 1 = e5m2 (M = 57344).  A row of values x is quantised in fp32: amax = max|x|,
 * inv = M / amax, q = fp8_rn_satfinite(x * inv), scale = amax / M, read back as q * scale; a row whose inv is not
 * finite (amax = 0, or a bf16 subnormal amax) is zero bytes and scale 0.
 * ------------------------------------------------------------------------------------------ */

/* ------------------------------------------------------------------------------------------
 * FP8 (e4m3) attention forward (opt-in, lossy; csrc/attn_fwd_fp8.cu, rule in csrc/attn_fp8_core.h): causal
 * attention on the FP8 tensor cores with K and V quantised once per call.
 *
 * With nt = ceil(sk / 128) key blocks of 128 rows, aligned to key row 0 (the last one zero-padded):
 *   k8       e4m3 [b][hkv][nt * 128][d]   the quantised keys
 *   vt8      e4m3 [b][hkv][nt][d][128]    each block of values transposed; inside each 32-key chunk, byte
 *                                         32 c + 16 h + 4 t + i of a row holds key 32 c + 16 h + 8 (i / 2) + 2 t + i % 2
 *   k_scale, v_scale  float [b][hkv][nt]
 * A block's values are quantised as one e4m3 row of the FP8 row rule.
 *
 * lv_attn_fp8_quant_kv: bf16 K and V of `a` (a->k, a->v, batch, sk, hkv, d, k_strides, v_strides; the other fields
 *   are not read) -> the four buffers of `kv`, one pass.  d = 128; k, v, k8, vt8 16-byte aligned.
 * lv_attn_fwd_fp8: lv_attn_fwd over the quantised K / V of `kv` (a->k and a->v are not read).  Q is quantised inside
 *   the kernel, one scale per (batch, query head, 64-row group aligned to query row 0); the scores are
 *   s_q s_k (q8 . k8) in fp32, p = exp2 of the log2-domain score minus the running max in fp32, the row sum takes
 *   p, and P V takes e4m3(p * 2^8) * v8 with the 2^-8 in the block's V scale, accumulated in fp32 per key block
 *   (out of the tensor cores every 128 keys).  Only d = 128 and causal = 1 with sq <= sk, q_seg_len = sq,
 *   q_seg_pos = {sk - sq, 0}, kv_pos0 = 0 are built; anything else (documents, query segments, context
 *   parallelism) is LV_EINVAL.  A call over query rows [r0, r1) and keys [0, r1), r0 a multiple of 128, returns
 *   exactly those rows of the call over all rows. lse as for lv_attn_fwd (may be NULL).
 * ------------------------------------------------------------------------------------------ */
typedef struct lv_attn_fp8_kv {
  void* k8;
  void* vt8;
  float* k_scale;
  float* v_scale;
} lv_attn_fp8_kv;

int lv_attn_fp8_quant_kv(const lv_attn_params* a, const lv_attn_fp8_kv* kv, lv_stream_t stream);
int lv_attn_fwd_fp8(const lv_attn_params* a, const lv_attn_fp8_kv* kv, lv_stream_t stream);
int lv_attn_docs_bwd(const lv_attn_bwd_params* p, const lv_attn_docs* docs, lv_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Context-parallel attention (forward): zig-zag sequence sharding with the K/V exchange inside the
 * attention kernel.
 *
 * Replaces TransformerEngine's ring attention (`TEDotProductAttention` with cp_group,
 * long_vita_megatron/core/models/gpt/gpt_layer_specs.py:35-45; un-vendored `AttnFuncWithCP`:
 * cp steps of flash-attn on zig-zag half-chunks + NCCL P2P + LSE merge) and uses the data layout
 * of long_vita_megatron/training/utils.py:329-341: the S-token sequence is cut into 2*cp chunks
 * of c = S/(2 cp) tokens, rank r owns chunks {r, 2cp-1-r} (sq = 2c local rows).
 *
 * Every rank keeps its K|V rows (this epoch's, after RoPE) in a peer-mapped buffer obtained from
 * lv_ipc_alloc(); `peer_kv[p]` is the (peer-mapped) address of rank p's K of local token 0, with
 * V following K inside the row and `peer_tok_stride` elements between tokens - for the fused QKV
 * GEMM output [T, (hq + 2 hkv) d] that is the K column of the buffer itself, so no copy precedes
 * the exchange.  Copier warps inside the kernel wait for the owner's ready flag (system-scope
 * acquire), pull the visible chunks over NVLink into the caller's staging buffers
 * k_full / v_full [S, hkv*d] in global order and publish per-128-token flags the TMA producer
 * polls; the math of already-staged blocks overlaps the transfer of later ones.  No NCCL call is
 * on this path.  `epoch` must increase by one per call, identically on all ranks; buffers alternate
 * by epoch parity (two K|V buffers per rank) so that no barrier is needed between layers.
 * `a` describes the local queries against the staging buffers: k = k_full, v = v_full, sk = S,
 * q_seg_len = c, q_seg_pos = {r c, (2cp-1-r) c}, kv_pos0 = 0, causal = 1, batch = 1, d = 128.
 * ------------------------------------------------------------------------------------------ */
typedef struct lv_cp_params {
  int32_t rank, cp;          /* 2 <= cp <= 8 */
  int64_t seq_total;         /* S */
  uint32_t epoch;            /* call counter (same on every rank) */
  int64_t peer_tok_stride;   /* elements */
  const void* peer_kv[8];    /* [cp] peer-mapped K row-0 address of rank p for this epoch's parity */
  void* peer_ready[8];       /* [cp] peer-mapped base of rank p's ready words: uint32[2][8] */
  void* my_ready;            /* local base of the same array */
  void* k_full;              /* bf16 [S, hkv*d] staging (local) */
  void* v_full;
  void* blk_flags;           /* uint32 [S/128], zero-initialised once; private to the kernel (it counts
                              * staged 32-token units: 4 * (epoch + 1) when block b of this epoch is whole) */
  void* fault;               /* uint32, zero-initialised once (local device memory): sticky fault word */
} lv_cp_params;

int lv_attn_cp_fwd(const lv_attn_params* a, const lv_cp_params* c, lv_stream_t stream);
/* Every in-kernel wait on another GPU's progress is bounded (LV_CP_TIMEOUT_MS, default 120 000): on expiry the kernel
 * sets the sticky fault word, stops waiting and finishes with undefined output instead of hanging the node.
 * lv_cp_check_fault synchronises the stream and returns LV_ESTATE (+ lv_last_error text) once the word is set. */
int lv_cp_check_fault(const void* fault, lv_stream_t stream);

/* Peer-mappable device memory (cudaMalloc + CUDA IPC).  The 64-byte handle is exchanged by the
 * host (torch.distributed) and opened on the other ranks of the node. */
int lv_ipc_alloc(int64_t bytes, void** ptr);
int lv_ipc_free(void* ptr);
int lv_ipc_get_handle(void* ptr, void* handle64);
int lv_ipc_open_handle(const void* handle64, void** ptr);
int lv_ipc_close_handle(void* ptr);

/* ------------------------------------------------------------------------------------------
 * Token-wise memory-bound operators (HBM roofline).
 * ------------------------------------------------------------------------------------------ */

/* RMSNorm: y = bf16( bf16(x_f32 * rsqrt(mean(x^2) + eps)) * w ).
 * long_vita_megatron/core/transformer/custom_layers/transformer_engine.py:74-79 (and the HF
 * Qwen2RMSNorm the reference instantiates, modeling_long_vita.py:57).  If `residual` is not NULL
 * the kernel first forms h = x + residual (bf16 rounding), writes h to `sum_out`, and normalises
 * h (the bias-dropout-add of transformer_layer.py:211-213 fused with the following norm). */
int lv_rmsnorm(const void* x, const void* residual, const void* w, void* y, void* sum_out, int64_t rows,
               int64_t cols, float eps, lv_stream_t stream);

/* LayerNorm with affine weight/bias (ViT norm1/norm2, eps 1e-6: modeling_intern_vit.py:205-206;
 * pre-projection LayerNorm over 4096: resampler_projector.py:17,30). fp32 statistics. */
int lv_layernorm(const void* x, const void* w, const void* b, void* y, int64_t rows, int64_t cols, float eps,
                 lv_stream_t stream);

/* Rotary table: cos/sin (bf16, [n, dim]) of pos[i] * inv_freq[j % (dim/2)], the
 * cat(freqs, freqs) layout of rotary_pos_embedding.py:102-106; pos is int64 (position_ids gather
 * of :114-117 and the zig-zag slice of :36-47 are both expressed by passing the right pos). */
int lv_rope_table(const int64_t* pos, const float* inv_freq, void* cos_out, void* sin_out, int64_t n,
                  int64_t dim, lv_stream_t stream);

/* Rotary embedding, non-interleaved (rotate_half): t = t*cos + rotate_half(t)*sin with the bf16
 * rounding sequence of apply_rotary_pos_emb_bshd, rotary_pos_embedding.py:181-204 (== HF
 * apply_rotary_pos_emb).  x is [n_tok, heads, dim] with element strides (tok, head), dim
 * contiguous; out may alias x. */
int lv_rope(const void* x, void* out, const void* cos_t, const void* sin_t, int64_t n_tok, int64_t heads,
            int64_t dim, int64_t x_tok_stride, int64_t x_head_stride, int64_t o_tok_stride,
            int64_t o_head_stride, lv_stream_t stream);

/* SwiGLU: out[r, i] = silu(gu[r, i]) * gu[r, inter + i]; fc1 = cat(gate, up)
 * (tools/hf2mcore_long_vita.py:502-504), HF Qwen2MLP act_fn(gate_proj(x)) * up_proj(x). */
int lv_swiglu(const void* gate_up, void* out, int64_t rows, int64_t inter, lv_stream_t stream);

/* y = gelu(x + bias); approx = 0: exact erf GELU (InternViT, pretrain_long_vita.py:206,
 * resampler_projector.py:21); approx = 1: tanh GELU (SigLIP, pretrain_long_vita.py:291).
 * bias may be NULL. */
int lv_bias_gelu(const void* x, const void* bias, void* y, int64_t rows, int64_t cols, int32_t approx,
                 lv_stream_t stream);

/* Layer-scale residual: out = x + (y + bias) * ls   (intern_vit_model.py:63,77;
 * modeling_intern_vit.py:224-226).  bias may be NULL; ls may be NULL (plain residual add). */
int lv_ls_residual(const void* x, const void* y, const void* bias, const void* ls, void* out, int64_t rows,
                   int64_t cols, lv_stream_t stream);

/* Pixel-shuffle x0.5 of ViT tokens without the class token:
 * in [n, 1 + hw*hw, c] (cls at index 0, dropped: modeling_long_vita.py:97) ->
 * out [n, (hw/2)^2, 4c]; pure permutation, bit-exact with resampler_projector.py:36-46 /
 * pretrain_long_vita.py:572-582.  has_cls selects whether row 0 is skipped. */
int lv_pixel_shuffle(const void* x, void* out, int64_t n, int64_t hw, int64_t c, int32_t has_cls,
                     lv_stream_t stream);

/* Embedding gather + image-feature scatter:
 * out[t, :] = table[ids[t], :]; then out[dst_idx[i], :] = feat[src_idx[i], :] (src_idx NULL =>
 * identity).  language_model_embedding.py:102-131, modeling_long_vita.py:138-147.  Index
 * arithmetic is int64 and bit-exact.  Duplicate dst_idx are applied in increasing i order only
 * if `n_scatter` is small; callers pass unique targets (the reference has unique targets). */
int lv_embed_scatter(const int64_t* ids, const void* table, int64_t vocab, const void* feat,
                     const int64_t* src_idx, const int64_t* dst_idx, int64_t n_scatter, void* out,
                     int64_t n_tok, int64_t hidden, lv_stream_t stream);

/* Row gather / scatter used by the logit-masked LM head:
 * gather:  out[i, :] = x[idx[i], :]                     (masked_select, layers.py:402-407)
 * scatter: out[idx[i], :] = x[i, :], other rows zero    (masked_scatter, layers.py:446-451)
 * lv_row_scatter: out[idx[i], :] = x[i, :] into an existing [n_rows_out, cols] out, other rows untouched (one
 * chunk of image features into the embedded prompt); a bit-exact copy, targets outside [0, n_rows_out) dropped. */
int lv_row_gather(const void* x, const int64_t* idx, void* out, int64_t n_idx, int64_t cols,
                  lv_stream_t stream);
int lv_row_scatter_zero(const void* x, const int64_t* idx, void* out, int64_t n_idx, int64_t n_rows_out,
                        int64_t cols, lv_stream_t stream);
int lv_row_scatter(const void* x, const int64_t* idx, void* out, int64_t n_idx, int64_t n_rows_out, int64_t cols,
                   lv_stream_t stream);

/* Backward of the token-wise operators (training through the `--spec` layer, SURVEY.md 8f-1).
 * RMSNorm: g = dy*w, dx = rstd*(g - xhat*mean(g*xhat)) (+ add_in, the gradient arriving on the residual stream),
 * dw partial sums in `dw_partials` [lv_rmsnorm_bwd_partials(rows, cols), cols] float - the caller adds the rows
 * (no atomics: bit-reproducible).  x is the tensor that was normalised (after the fused residual add).
 * SwiGLU: gate_up = cat(gate, up) as in lv_swiglu; d_gate_up in the same layout. */
int64_t lv_rmsnorm_bwd_partials(int64_t rows, int64_t cols);
int lv_rmsnorm_bwd(const void* x, const void* w, const void* dy, const void* add_in, void* dx, float* dw_partials,
                   int64_t rows, int64_t cols, float eps, lv_stream_t stream);
int lv_swiglu_bwd(const void* gate_up, const void* dh, void* d_gate_up, int64_t rows, int64_t inter, lv_stream_t stream);

/* Backward of the vision-tower operators (training InternViT and the projector through MegatronVisionModel,
 * long_vita_megatron/pretrain_long_vita.py:310-596).  All reductions are deterministic: per-CTA fp32 partial rows that
 * the caller adds, no atomics.
 * LayerNorm (forward lv_layernorm): mean / rstd are recomputed from x in fp32; xhat = (x - mean) * rstd, g = dy * w,
 *   dx = rstd * (g - mean(g) - xhat * mean(g * xhat)) (+ add_in, the gradient arriving on the residual stream);
 *   dw / db partial sums of dy * xhat / dy in dw_partials / db_partials, each [lv_layernorm_bwd_partials(rows, cols), cols]
 *   float.  cols <= 8192 (ViT norms: 1024; pre-projection LayerNorm: 4096).  dx may be NULL (then add_in must be NULL
 *   too): only the dw / db partials are written, for a norm whose input needs no gradient.
 * GELU: dx = dy * gelu'(pre) where pre is the bf16 pre-activation; approx as in lv_bias_gelu (0 erf, 1 tanh).
 * Layer-scale residual, bias-free (out = x + y * ls): dy = bf16(dout * ls); dls partial sums of dout * y in
 *   dls_partials [lv_ls_residual_bwd_partials(rows, cols), cols] float.  dx = dout needs no kernel.
 * Pixel shuffle: dx [n, (1 +) hw*hw, c] from dout [n, (hw/2)^2, 4c], the exact inverse permutation of lv_pixel_shuffle
 *   (bit-exact); with has_cls the class-token rows of dx are written as zeros. */
int64_t lv_layernorm_bwd_partials(int64_t rows, int64_t cols);
int lv_layernorm_bwd(const void* x, const void* w, const void* dy, const void* add_in, void* dx, float* dw_partials,
                     float* db_partials, int64_t rows, int64_t cols, float eps, lv_stream_t stream);
int lv_gelu_bwd(const void* pre, const void* dy, void* dx, int64_t rows, int64_t cols, int32_t approx, lv_stream_t stream);
int64_t lv_ls_residual_bwd_partials(int64_t rows, int64_t cols);
int lv_ls_residual_bwd(const void* dout, const void* y, const void* ls, void* dy, float* dls_partials, int64_t rows,
                       int64_t cols, lv_stream_t stream);
int lv_pixel_shuffle_bwd(const void* dout, void* dx, int64_t n, int64_t hw, int64_t c, int32_t has_cls, lv_stream_t stream);

/* Merge of split-key partial attention results (flash-decoding, one new token against a K/V cache; the
 * reference has no such path - it re-prefills every generated token, generation.py:127-135).
 * o_part bf16 [n, G, hkv, d] and lse_part float [n, hkv, G] are what lv_attn_fwd returns when the G = hq/hkv
 * query heads of a kv group are laid out as G query rows and the key range as n batch entries;
 * out[h = kvh*G + g, :] = sum_s w_s o_part[s, g, kvh, :], w_s = exp(lse_s - LSE), LSE = logsumexp_s lse_s;
 * lse_out float [hq] (may be NULL) receives LSE. */
int lv_attn_decode_merge(const void* o_part, const float* lse_part, void* out, float* lse_out, int64_t n_splits,
                         int64_t group, int64_t hkv, int64_t d, lv_stream_t stream);

/* Flash-decoding of one query token over K/V rows in pinned host memory (the host tier of the K/V cache, for
 * prompts whose cache does not fit in HBM).  q bf16 [hq, d] on the device; kv_host bf16 [capacity, 2 * hkv * d],
 * token-major, row = K of the hkv heads then V of the hkv heads, allocated pinned and mapped (lv_host_alloc); the
 * kernel reads rows [0, length) in place over PCIe, never a row at or past `length`.  Split s of n_splits takes
 * the rows [s * per, min((s + 1) * per, length)), per = ceil(length / n_splits), and writes o_part bf16
 * [n_splits, G, hkv, d] and lse_part float [n_splits, hkv, G] (G = hq / hkv, natural log, -inf for an empty
 * split): the inputs of lv_attn_decode_merge.  d = 128 only; hkv must divide 16 and G be at most 8.  kv_host is
 * checked to be pinned host memory (cudaPointerGetAttributes) before anything launches. */
int lv_attn_decode_host(const void* q, const void* kv_host, void* o_part, float* lse_part, int64_t length,
                        int64_t capacity, int64_t hq, int64_t hkv, int64_t d, int64_t n_splits, float scale,
                        lv_stream_t stream);
/* Pinned host memory mapped into the device address space (cudaHostAlloc, mapped | portable), and its release.
 * The host tier's buffers come from here: an exact size, where a caching pinned allocator may round a
 * multi-gigabyte buffer up to the next power of two. */
int lv_host_alloc(int64_t bytes, void** ptr);
int lv_host_free(void* ptr);
/* Copy `rows` rows of row_bytes from device memory (src_pitch bytes apart) to contiguous pinned host rows, in
 * stream order (one cudaMemcpy2DAsync): the K|V columns of a QKV buffer go to the host tier without a device
 * temporary.  host_dst must be pinned host memory. */
int lv_rows_to_host(void* host_dst, const void* src, int64_t rows, int64_t row_bytes, int64_t src_pitch,
                    lv_stream_t stream);

/* FP8 host tier (opt-in, lossy: it halves the PCIe bytes and the pinned memory of a host layer).  A row holds K of
 * the hkv heads, e4m3 [hkv][d]; V of the hkv heads, e4m3 [hkv][d]; then the scales, float [2][hkv] (K scales, then V
 * scales), zero-padded to a multiple of 16 bytes: 2 * hkv * d + ceil(8 * hkv / 16) * 16 bytes, 2112 at 8:128.  Each
 * head is one e4m3 row of the FP8 row rule.
 *
 * lv_rows_to_host_fp8: quantise `rows` bf16 K|V rows of the device (2 * hkv * d values each, V following K, src_pitch
 * bytes apart: the K|V columns of a QKV buffer row or the streamed layer's K|V buffer) into contiguous FP8 host rows,
 * in stream order.  The kernel stores straight into the mapped host memory with 16-byte stores: no device temporary.
 * d = 128, hkv divides 16, src, src_pitch and host_dst 16-byte aligned; host_dst must be pinned host memory.
 *
 * lv_attn_decode_host_fp8: lv_attn_decode_host over FP8 rows, kv_host uint8 [capacity, row bytes] from lv_host_alloc:
 * the same arguments, split rule (never a row at or past `length`) and outputs for lv_attn_decode_merge.  Each score
 * is s_k * sum_i q_i k8_i and each value row enters as (p * s_v) v8, in fp32.  d = 128 only; hkv must divide 16 and
 * G be at most 8.  kv_host is checked to be pinned host memory before anything launches. */
int lv_rows_to_host_fp8(void* host_dst, const void* src, int64_t rows, int64_t hkv, int64_t d, int64_t src_pitch,
                        lv_stream_t stream);
int lv_attn_decode_host_fp8(const void* q, const void* kv_host, void* o_part, float* lse_part, int64_t length,
                            int64_t capacity, int64_t hq, int64_t hkv, int64_t d, int64_t n_splits, float scale,
                            lv_stream_t stream);

/* lv_kv_rows_dequant_fp8: FP8 host rows staged in device memory, src uint8 [rows, row bytes] (the format above, copied
 * as they are), -> bf16 K|V rows dst [rows, 2 * hkv * d] (K of the hkv heads, then V), by the decode rule of
 * csrc/fp8_core.h: each value becomes bf16_rn(float(q) * scale) with its head's scale, one fp32 multiply rounded to
 * nearest.  The attention over host rows for several query tokens copies each chunk of rows to the device and runs
 * lv_attn_fwd over it; this makes an FP8 chunk that call's bf16 operands.  HBM-bound.  d = 128, hkv divides 16, src
 * and dst 16-byte aligned device memory. */
int lv_kv_rows_dequant_fp8(const void* src, void* dst, int64_t rows, int64_t hkv, int64_t d, lv_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Dense linears (tensor-core roofline).  C[M,N] = act(A[M,K] . W[N,K]^T + bias[N]), bf16 in,
 * fp32 accumulate, bf16 out.  Replaces torch.matmul / te.Linear at layers.py:270,409, the ViT
 * qkv/proj/fc1/fc2 (modeling_intern_vit.py:131,141,190-191) and the projector
 * (resampler_projector.py:19-23).  K must be a multiple of 8 (16-byte rows).
 * act: 0 none, 1 exact GELU, 2 tanh GELU, 3 fused SwiGLU: W rows are interleaved (gate_i, up_i), C is
 * [M, N/2] with C[:, i] = bf16(silu(bf16 gate_i)) * bf16(up_i) - the rounding sequence of act 0 followed
 * by lv_swiglu - so the [M, 2*inter] intermediate never reaches HBM (bias must be NULL).
 * lda / ldw / ldc are row strides in elements.
 * ------------------------------------------------------------------------------------------ */
int lv_gemm_bias_act(const void* A, const void* W, const void* bias, void* C, int64_t M, int64_t N,
                     int64_t K, int64_t lda, int64_t ldw, int64_t ldc, int32_t act, lv_stream_t stream);

/* lv_gemm_bias_act with a layout flag per operand, for the backward products dX = dY . W and dW = dY^T . X, which
 * contract over a dimension that is not contiguous in memory.  a_mn_major = 0: A is [M, K] (row stride lda);
 * 1: A is stored [K, M] with M contiguous (A^T, row stride lda >= M).  w_mn_major likewise: W [N, K] or stored
 * [K, N] (ldw >= N).  An MN-major operand needs no padding: its contraction extent K may be any value >= 1 (tails
 * are zero-filled); K must be a multiple of 8 only while an operand is K-major.  All leading dimensions are multiples
 * of 8 and A, W, C 16-byte aligned.  Epilogues (bias, act) are those of lv_gemm_bias_act; results equal
 * lv_gemm_bias_act on transposed copies of the MN-major operands, bit for bit.  With both flags 0 the call is
 * lv_gemm_bias_act. */
int lv_gemm_ex(const void* A, const void* W, const void* bias, void* C, int64_t M, int64_t N, int64_t K,
               int64_t lda, int64_t ldw, int64_t ldc, int32_t a_mn_major, int32_t w_mn_major, int32_t act,
               lv_stream_t stream);

/* Weight-gradient accumulation into an fp32 master gradient (Megatron's gradient_accumulation_fusion, the
 * `main_grad` of layers.py:486-518): C[M, N] += A . W^T in fp32, with the operands, layouts, mainloop and k-order of
 * lv_gemm_ex, so the accumulator added is exactly the value lv_gemm_ex rounds to bf16.  Each element becomes one IEEE
 * fp32 round-to-nearest add prior + acc (subnormals kept), deterministic.  Only a_mn_major = w_mn_major = 1 is built
 * (dW = dY^T . X with dY and X read in place); K may be any value >= 0 (K = 0 or M = 0: no launch).  C is fp32 with
 * row stride ldc (a multiple of 4, >= N), N a multiple of 4, lda / ldw multiples of 8, A, W, C 16-byte aligned;
 * columns and rows outside [M, N] are not touched. */
int lv_gemm_wgrad_acc_f32(const void* A, const void* W, float* C, int64_t M, int64_t N, int64_t K, int64_t lda,
                          int64_t ldw, int64_t ldc, int32_t a_mn_major, int32_t w_mn_major, lv_stream_t stream);

/* FP8 linears of the decoder (csrc/gemm_fp8.cu).
 * lv_quant_rows_fp8_fmt: x bf16 [M, K] (row stride ldx elements, a multiple of 8) -> q [M, K] contiguous in format fmt
 * and scale fp32 [M], each row quantised by the FP8 row rule.  K a positive multiple of 16; x and q 16-byte aligned.
 * lv_gemm_fp8: C[M, N] = act(bf16((A . W^T) * a_scale[m] * w_scale[n] + bias[n])) with A e4m3 [M, K] (row stride
 * lda bytes) and W e4m3 [N, K] (ldw bytes), both K-major, fp32 accumulation promoted out of the tensor cores every
 * 128 k-values, C bf16 with row stride ldc elements.  act: 0 none (bias optional), 3 fused SwiGLU over interleaved
 * (gate_i, up_i) W rows as in lv_gemm_bias_act (C is [M, N/2], bias NULL), each of gate and up scaled and rounded to
 * bf16 before bf16(silu(gate)) * up.  K a multiple of 16, N of 8 (16 for SwiGLU), lda / ldw multiples of 16, ldc of
 * 8; A, W, C 16-byte aligned.  For M <= 4 the product runs as a weight-stream GEMV (the rule of lv_gemm_bias_act). */
int lv_quant_rows_fp8_fmt(const void* x, void* q, float* scale, int64_t M, int64_t K, int64_t ldx, int32_t fmt,
                          lv_stream_t stream);
int lv_gemm_fp8(const void* A, const float* a_scale, const void* W, const float* w_scale, const void* bias, void* C,
                int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldw, int64_t ldc, int32_t act,
                lv_stream_t stream);

/* FP8 training of the decoder's linears (csrc/gemm_fp8.cu), fmt as in the FP8 row rule.
 * lv_quant_cols_fp8_t: cast-transpose.  x bf16 [R, C] (row stride ldx elements, a multiple of 8; C a multiple of 8)
 * -> q [C, R16] contiguous, R16 = R rounded up to 16, with q[c, r] = x[r, c] quantised by the scale of column c,
 * scale fp32 [C]; columns R..R16 of q are zero.  amax_ws is a workspace of C unsigned words.  x and q 16-byte aligned.
 * lv_gemm_fp8_grad: the backward products.  C[M, N] = bf16((A . B^T) * a_scale[m] * b_scale[n]) with A [M, K] in
 * format a_fmt and B e4m3 [N, K] (row strides lda / ldb bytes, multiples of 16), K-major, accumulation promoted out of
 * the tensor cores every 128 k-values as in lv_gemm_fp8; C bf16 with row stride ldc (a multiple of 8).  With
 * accumulate = 1, C is fp32 (ldc a multiple of 4) and each element becomes one IEEE round-to-nearest add
 * C + (acc * a_scale[m]) * b_scale[n], the value whose bf16 rounding accumulate = 0 stores (Megatron's fp32
 * main_grad, gradient-accumulation fusion).  K a multiple of 16, N of 8; A, B, C 16-byte aligned. */
int lv_quant_cols_fp8_t(const void* x, void* q, float* scale, unsigned* amax_ws, int64_t R, int64_t C, int64_t ldx,
                        int32_t fmt, lv_stream_t stream);
int lv_gemm_fp8_grad(const void* A, int32_t a_fmt, const float* a_scale, const void* B, const float* b_scale, void* C,
                     int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int32_t accumulate,
                     lv_stream_t stream);

/* Patch embedding of 14x14 non-overlapping patches (Conv2d(3, C, k=14, s=14),
 * modeling_intern_vit.py:79-81,98; intern_vit_model.py:139-145,203) + class token + learned
 * position embedding (modeling_intern_vit.py:100-107):
 * out[n, 0, :] = cls + pos[0]; out[n, 1 + p, :] = bf16(W . patch(n, p) + bias) + pos[1 + p].
 * images bf16 [n, 3, img, img]; W bf16 [C, Kpad] = the conv weight flattened to [C, 3*ps*ps] and
 * zero-padded per row to Kpad = 3*ps*ps rounded up to a multiple of 64 (done once at load time);
 * out bf16 [n, 1 + (img/ps)^2, C].  cls == NULL selects the class-token-free form of SigLIP
 * (long_vita_megatron/core/models/vision/siglip_vit_model.py:165-176): out [n, (img/ps)^2, C],
 * out[n, p] = bf16(W . patch + bias) + pos[p].  `ws` is caller workspace of lv_patch_embed_ws_bytes() bytes
 * (the im2col matrix and the un-offset GEMM result). */
int64_t lv_patch_embed_ws_bytes(int64_t n, int64_t img, int64_t ps, int64_t C);
int lv_patch_embed(const void* images, const void* W, const void* bias, const void* cls, const void* pos,
                   void* out, void* ws, int64_t n, int64_t img, int64_t ps, int64_t C,
                   lv_stream_t stream);

/* The im2col step of lv_patch_embed on its own: col bf16 [n * (img/ps)^2, kpad], row p of image i = the patch's
 * 3*ps*ps pixels in (channel, y, x) order, zero-padded to kpad (a multiple of 8, >= 3*ps*ps).  With it the conv weight
 * gradient is one lv_gemm_ex call: dW[C, kpad] = dP^T . col, both operands MN-major (read in place) so that the
 * token dimension is the contraction. */
int lv_patch_im2col(const void* images, void* col, int64_t n, int64_t img, int64_t ps, int64_t kpad, lv_stream_t stream);

/* Cross-entropy over vocabulary CHUNKS, fused with the logit-masked LM head (SURVEY.md 8f-3): replaces
 * `compute_language_model_loss(labels, logits)` = vocab_parallel_cross_entropy(logits.float(), labels) on a
 * materialised [M, vocab] tensor (long_vita_megatron/core/models/multimodal/gpt_vl_model.py:371-414; Megatron
 * core_r0.7.0 tensor_parallel/cross_entropy.py, un-vendored).  The caller runs lv_gemm_bias_act per chunk of W rows.
 * lv_ce_accumulate: logits bf16 [rows, cols] (row stride ld) = columns [col0, col0 + cols) of the full logits;
 *   folds the chunk into run_max / run_sum (float [rows], initialise to -inf / 0) and writes tgt[r] = logit of
 *   labels[r] when it falls inside the chunk.  After the last chunk: loss[r] = log(run_sum[r]) + run_max[r] - tgt[r].
 * lv_ce_grad: dlogits[r, c] = bf16((exp(logits[r, c] - lse[r]) - [col0 + c == labels[r]]) * dloss[r]); rows with a
 *   negative label produce zeros.  dlogits may alias logits. */
int lv_ce_accumulate(const void* logits, int64_t ld, const int64_t* labels, float* run_max, float* run_sum, float* tgt,
                     int64_t rows, int64_t cols, int64_t col0, lv_stream_t stream);
int lv_ce_grad(const void* logits, int64_t ld, void* dlogits, int64_t ldd, const int64_t* labels, const float* lse,
               const float* dloss, int64_t rows, int64_t cols, int64_t col0, lv_stream_t stream);

/* Frame preprocessing (SURVEY.md 8f-4): decoded uint8 RGB frames [n, H, W, 3] -> bf16 [n, 3, S, S], bit-identical to
 * ImageProcessor.process_images (long_vita/data/processor/image_processor.py:183-223: expand2square with the mean
 * colour, PIL BICUBIC resize to S x S, * 1/255, (x - mean) / std in float32, channel-first) followed by .to(bfloat16).
 * win_min / win_cnt int32 [S] and coeff int32 [S, ksize] are Pillow's resampling windows and 22-bit fixed-point
 * weights for max(H, W) -> S pixels (device memory; computed once per geometry by the host, see
 * long_vita_b200/preprocess.py); background int32[3], mean / std float[3] are HOST arrays; ws is device workspace of
 * lv_frame_preprocess_ws_bytes() bytes (the uint8 intermediate of the horizontal pass). */
int64_t lv_frame_preprocess_ws_bytes(int64_t n_frames, int64_t H, int64_t W, int64_t S);
int lv_frame_preprocess(const void* frames, void* out, void* ws, const int32_t* win_min, const int32_t* win_cnt,
                        const int32_t* coeff, int64_t ksize, int64_t n_frames, int64_t H, int64_t W, int64_t S,
                        const int32_t* background, const float* mean, const float* std, lv_stream_t stream);

/* Dynamic-patch tiling of one image (same survey row): uint8 RGB image [H, W, 3] -> bf16 tiles [*, 3, S, S], bit-identical
 * to ImageProcessor.process_dynamic (long_vita/data/processor/image_processor.py:263-285) = dynamic_preprocess (:404-448:
 * PIL BICUBIC resize to out_w x out_h = a grid of S x S tiles chosen by the host, aspect ratio not kept; crop boxes
 * row-major over the grid) + process_images on the tiles (:211-221) + .to(bfloat16).  The resized pixel (oy, ox) lands in
 * tile tile_base + (oy / S) * (out_w / S) + ox / S.  The thumbnail tile the reference puts first (:442-447) is a second
 * call with out_h = out_w = S and tile_base = 0.  x_* / y_* are the resampling tables for W -> out_w and H -> out_h
 * (device memory, long_vita_b200/preprocess.py::resample_table); mean / std float[3] are HOST arrays; ws is device
 * workspace of lv_image_tiles_ws_bytes(H, out_w) bytes. */
int64_t lv_image_tiles_ws_bytes(int64_t H, int64_t out_w);
int lv_image_tiles_preprocess(const void* image, void* out, void* ws, const int32_t* x_min, const int32_t* x_cnt,
                              const int32_t* x_coeff, int64_t x_ksize, const int32_t* y_min, const int32_t* y_cnt,
                              const int32_t* y_coeff, int64_t y_ksize, int64_t H, int64_t W, int64_t out_h, int64_t out_w,
                              int64_t S, int64_t tile_base, const float* mean, const float* std, lv_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* LVB200_H_ */
