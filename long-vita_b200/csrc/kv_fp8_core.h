// The FP8 (e4m3) quantiser of the project and the row format of the host tier of the K/V cache, shared by the kernels
// (csrc/attn_decode_host.cu: rows_to_host_fp8_kernel, attn_decode_host_fp8_kernel; csrc/gemm_fp8.cu:
// quant_rows_fp8_kernel) and the host compiler: tests/test_kv_fp8_host.py and tests/test_fp8_linear_host.py build this
// text with gcc (LV_KV8_HD = static inline) and check it, bit for bit, against the torch.float8_e4m3fn restatement of
// the same rule.
//
// The rule quantises a row of n values with one fp32 scale: a K/V head (n = d), or a whole row of a linear layer's
// operand (n = K: one scale per output channel of W [N, K], one per token of A [M, K]).
//
// A row of an FP8 layer holds, in this order: K of the hkv heads, e4m3 [hkv][d]; V of the hkv heads, e4m3 [hkv][d];
// the scales, fp32 [2][hkv] (K scales, then V scales), zero-padded to a multiple of 16 bytes.  At hkv = 8, d = 128 a
// row is 1024 + 1024 + 64 = 2112 bytes, against 4096 for bf16.
//
// A row's n values x are quantised in fp32: amax = max|x|; inv = 448 / amax (IEEE division, round to nearest);
// q = e4m3_rn_satfinite(x * inv); scale = amax / 448, and x is read back as float(q) * scale.  A row whose inv is
// not finite - amax is 0, or below 448 / FLT_MAX ~ 1.3e-36 (bf16 subnormals only) - is all-zero bytes with scale 0.
#ifndef LV_KV_FP8_CORE_H_
#define LV_KV_FP8_CORE_H_

#include <stdint.h>

#ifdef __CUDACC__
#define LV_KV8_HD __host__ __device__ __forceinline__
#else
#include <math.h>
#define LV_KV8_HD static inline
#endif

#define LV_KV8_MAX 448.0f /* largest finite e4m3 value */

// Bytes of one FP8 row: 2 * hkv * d e4m3 values, then 2 * hkv fp32 scales padded to 16 bytes.
LV_KV8_HD int64_t lv_kv8_scale_bytes(int64_t hkv) { return (8 * hkv + 15) / 16 * 16; }
LV_KV8_HD int64_t lv_kv8_row_bytes(int64_t hkv, int64_t d) { return 2 * hkv * d + lv_kv8_scale_bytes(hkv); }

// bf16 bits -> float (exact).
LV_KV8_HD float lv_kv8_bf16_to_f32(uint16_t b) {
  union {
    uint32_t u;
    float f;
  } c;
  c.u = (uint32_t)b << 16;
  return c.f;
}

// 448 / amax and amax / 448, each one IEEE fp32 division rounded to nearest (amax > 0).
LV_KV8_HD float lv_kv8_inv(float amax) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(LV_KV8_MAX, amax);
#else
  volatile float r = LV_KV8_MAX / amax;
  return r;
#endif
}

// A head stored as zeros: 448 / amax is not finite (amax = 0, or a subnormal amax below ~1.3e-36).
LV_KV8_HD int lv_kv8_zero_head(float inv) { return !(inv <= 3.40282347e38f); }

LV_KV8_HD float lv_kv8_scale(float amax) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(amax, LV_KV8_MAX);
#else
  volatile float r = amax / LV_KV8_MAX;
  return r;
#endif
}

#ifdef __CUDACC__
// Two products x * inv -> two e4m3 bytes (lo in the low byte): PTX cvt.rn.satfinite.e4m3x2.f32, which for |v| < 464
// gives exactly lv_kv8_e4m3.
__device__ __forceinline__ uint16_t lv_kv8_pack2(float lo, float hi) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
#endif

#ifndef __CUDA_ARCH__
// fp32 -> e4m3 bits, round to nearest even, finite values above 448 saturate to 448 (PTX cvt.rn.satfinite).  The
// kernels convert two at a time with the PTX instruction (lv_kv8_pack2); this is the host statement of the same rule.
static inline uint8_t lv_kv8_e4m3(float f) {
  union {
    float f;
    uint32_t u;
  } c;
  c.f = f;
  const uint8_t sign = (uint8_t)((c.u >> 24) & 0x80u);
  c.u &= 0x7FFFFFFFu;
  const float a = c.f;
  if (a != a) return 0x7F;                      // NaN
  if (a >= LV_KV8_MAX) return sign | 0x7E;      // satfinite
  if (a < 0.015625f) {                          // below 2^-6: subnormal steps of 2^-9 (8 steps reach 2^-6 = 0x08)
    return sign | (uint8_t)rintf(a * 512.0f);   // a * 2^9 is exact; rintf rounds half to even
  }
  int e;
  frexpf(a, &e);                                // a = m * 2^e, m in [0.5, 1): 2^(e-1) <= a < 2^e
  const int q = (int)rintf(ldexpf(a, 4 - e));   // a / 2^(e-4) in [8, 16], exact scaling; 16 carries the exponent
  return sign | (uint8_t)(((e + 6) << 3) + (q - 8));
}

// Quantise one row: x [n] bf16 bits -> q [n] e4m3, returns the scale.  The kernels split a row over lanes, reduce
// amax with shuffles (max is exact in any order) and multiply with __fmul_rn.
static inline float lv_fp8_quant_row(const uint16_t* x, uint8_t* q, int64_t n) {
  float amax = 0.0f;
  for (int64_t i = 0; i < n; ++i) {
    const float v = fabsf(lv_kv8_bf16_to_f32(x[i]));
    amax = v > amax ? v : amax;
  }
  const float inv = lv_kv8_inv(amax);
  if (lv_kv8_zero_head(inv)) {
    for (int64_t i = 0; i < n; ++i) q[i] = 0;
    return 0.0f;
  }
  for (int64_t i = 0; i < n; ++i) {
    volatile float t = lv_kv8_bf16_to_f32(x[i]) * inv;
    q[i] = lv_kv8_e4m3(t);
  }
  return lv_kv8_scale(amax);
}

// One K/V head of d values is one row of the rule.
static inline float lv_kv8_quant_head(const uint16_t* x, uint8_t* q, int d) { return lv_fp8_quant_row(x, q, d); }
#endif

#endif  // LV_KV_FP8_CORE_H_
