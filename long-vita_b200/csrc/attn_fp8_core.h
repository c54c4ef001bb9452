// The FP8 (e4m3) operand rule of the FP8 attention forward (csrc/attn_fwd_fp8.cu), shared by the kernels and the host
// compiler: tests/test_fp8_attn_host.py builds this text with gcc (LV_FP8_HD = static inline) and checks it, byte for
// byte, against the torch restatement of tests/attn_fp8_ref.py.  Each block below is one e4m3 row of the rule of
// csrc/fp8_core.h (lv_fp8_quant_row).
//
// K and V: one fp32 scale per (batch, kv head, 128-row key block), blocks aligned to key row 0; the ragged last block
// holds the rows [128 (nt - 1), sk) and is zero-padded to 128 rows (nt = ceil(sk / 128)).
//   K8  e4m3 [b][hkv][nt * 128][d]    the quantised key rows, padding rows zero
//   Vt8 e4m3 [b][hkv][nt][d][128]     each 128-key block transposed (FP8 wgmma reads only K-major operands, and P V
//                                     contracts over the keys); byte kappa of a row holds key lv_attn8_key_of(kappa)
//                                     of the block, padding keys zero
//   k_scale, v_scale fp32 [b][hkv][nt]
// Inside each 32-key chunk the keys are permuted so that the fp32 accumulator of S = Q K^T (m64n128: thread t holds
// columns 8 j + 2 (t % 4) + 0..1 of its rows) packs, four e4m3 values per register and in register order, into the A
// fragment of wgmma m64n128k32 e4m3 (k = 4 (t % 4) + 0..3 and 16 + 4 (t % 4) + 0..3): no shuffle between the two.
//
// Q: quantised inside the attention kernel from the bf16 tile it loads, one scale per (batch, query head, 64-row group
// aligned to query row 0 of the call).  P: p = exp2(s - m) in fp32; the row sum takes the fp32 p and P V takes
// e4m3(p * 2^8), the 2^-8 going into the block's V scale.
//
// Blocks are aligned to key row 0 and query groups to query row 0, so a call over the query rows [r0, r1) and the keys
// [0, r1) with r0 a multiple of 128 quantises exactly the blocks of the call over all rows.
#ifndef LV_ATTN_FP8_CORE_H_
#define LV_ATTN_FP8_CORE_H_

#include "fp8_core.h"

#define LV_ATTN8_BLOCK 128  /* key rows per K / V block (the kernel's key tile) */
#define LV_ATTN8_QROWS 64   /* query rows per Q scale (one consumer warpgroup) */

// Key (0..127, within its block) whose value sits at byte kappa of a transposed V row: kappa = 32 c + 16 h + 4 t + i
// holds key 32 c + 16 h + 8 (i / 2) + 2 t + i % 2.
LV_FP8_HD int lv_attn8_key_of(int kappa) {
  return (kappa & ~15) | (((kappa >> 1) & 1) << 3) | (((kappa >> 2) & 3) << 1) | (kappa & 1);
}

// Number of key blocks of sk keys.
LV_FP8_HD int64_t lv_attn8_blocks(int64_t sk) { return (sk + LV_ATTN8_BLOCK - 1) / LV_ATTN8_BLOCK; }

#ifndef __CUDA_ARCH__
// One (kv head, key block) of K and of V: rows x [n][d] bf16 bits with row stride ld elements (n <= 128 valid rows)
// -> k8 [128][d] (padding rows zero) and vt8 [d][128] (the permuted transpose, padding keys zero); returns the scales.
// `work` holds n * d bf16 values and n * d bytes.
static inline float lv_attn8_quant_k_block(const uint16_t* x, int64_t ld, int n, int d, uint8_t* k8, uint16_t* work,
                                           uint8_t* wq) {
  for (int r = 0; r < n; ++r)
    for (int c = 0; c < d; ++c) work[(int64_t)r * d + c] = x[r * ld + c];
  const float s = lv_fp8_quant_row(LV_FP8_E4M3, work, wq, (int64_t)n * d);
  for (int64_t i = 0; i < (int64_t)LV_ATTN8_BLOCK * d; ++i) k8[i] = i < (int64_t)n * d ? wq[i] : 0;
  return s;
}

static inline float lv_attn8_quant_v_block(const uint16_t* x, int64_t ld, int n, int d, uint8_t* vt8, uint16_t* work,
                                           uint8_t* wq) {
  for (int r = 0; r < n; ++r)
    for (int c = 0; c < d; ++c) work[(int64_t)r * d + c] = x[r * ld + c];
  const float s = lv_fp8_quant_row(LV_FP8_E4M3, work, wq, (int64_t)n * d);
  for (int c = 0; c < d; ++c)
    for (int kappa = 0; kappa < LV_ATTN8_BLOCK; ++kappa) {
      const int key = lv_attn8_key_of(kappa);
      vt8[c * LV_ATTN8_BLOCK + kappa] = key < n ? wq[(int64_t)key * d + c] : 0;
    }
  return s;
}
#endif

#endif  // LV_ATTN_FP8_CORE_H_
