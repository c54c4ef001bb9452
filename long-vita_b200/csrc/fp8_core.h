// The FP8 quantisation rule of the project, for both formats, and the row layout of the FP8 host tier of the K/V cache.
// Every FP8 kernel includes it (csrc/attn_decode_host.cu, csrc/attn_fwd_fp8.cu, csrc/gemm_fp8.cu), and the host
// compiler builds the same text (LV_FP8_HD = static inline): tests/fp8_ref.py compiles it with gcc and the CPU suite
// checks it, byte for byte, against the torch restatement of the rule in that file.
//
// Formats (`fmt`): 0 = e4m3 (largest finite value M = 448), 1 = e5m2 (M = 57344).
//
// The rule quantises a row of n values x with one fp32 scale: amax = max|x|; inv = M / amax (IEEE division, round to
// nearest); q = fp8_rn_satfinite(x * inv); scale = amax / M, and x is read back as float(q) * scale.  A row whose inv
// is not finite - amax is 0, or below M / FLT_MAX (bf16 subnormals only) - is all-zero bytes with scale 0.  A row is a
// K/V head (n = d), a whole row of a linear layer's operand (n = K), a column of a cast-transposed gradient, or a
// 128-key block of the FP8 attention's K / V (csrc/attn_fp8_core.h).
//
// A row of an FP8 host layer of the K/V cache holds, in this order: K of the hkv heads, e4m3 [hkv][d]; V of the hkv
// heads, e4m3 [hkv][d]; the scales, fp32 [2][hkv] (K scales, then V scales), zero-padded to a multiple of 16 bytes.  At
// hkv = 8, d = 128 a row is 1024 + 1024 + 64 = 2112 bytes, against 4096 for bf16.
#ifndef LV_FP8_CORE_H_
#define LV_FP8_CORE_H_

#include <stdint.h>

#ifdef __CUDACC__
#define LV_FP8_HD __host__ __device__ __forceinline__
#else
#include <math.h>
#define LV_FP8_HD static inline
#endif

#define LV_FP8_E4M3 0
#define LV_FP8_E5M2 1

// The largest finite value of a format.
LV_FP8_HD float lv_fp8_max(int fmt) { return fmt == LV_FP8_E5M2 ? 57344.0f : 448.0f; }

// Bytes of one FP8 K/V host row: 2 * hkv * d e4m3 values, then 2 * hkv fp32 scales padded to 16 bytes.
LV_FP8_HD int64_t lv_kv8_scale_bytes(int64_t hkv) { return (8 * hkv + 15) / 16 * 16; }
LV_FP8_HD int64_t lv_kv8_row_bytes(int64_t hkv, int64_t d) { return 2 * hkv * d + lv_kv8_scale_bytes(hkv); }

// bf16 bits -> float (exact).
LV_FP8_HD float lv_bf16_to_f32(uint16_t b) {
  union {
    uint32_t u;
    float f;
  } c;
  c.u = (uint32_t)b << 16;
  return c.f;
}

// M / amax and amax / M, each one IEEE fp32 division rounded to nearest (amax > 0).
LV_FP8_HD float lv_fp8_inv(int fmt, float amax) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(lv_fp8_max(fmt), amax);
#else
  volatile float r = lv_fp8_max(fmt) / amax;
  return r;
#endif
}

LV_FP8_HD float lv_fp8_scale(int fmt, float amax) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(amax, lv_fp8_max(fmt));
#else
  volatile float r = amax / lv_fp8_max(fmt);
  return r;
#endif
}

// A row stored as zeros: M / amax is not finite (amax = 0, or a subnormal amax).
LV_FP8_HD int lv_fp8_zero_row(float inv) { return !(inv <= 3.40282347e38f); }

// The decode rule of an FP8 K/V host row, for attention that runs over the rows in bf16: element x (the exact value of
// its e4m3 byte) of a head whose scale is s becomes bf16_rn(x * s), one fp32 multiply rounded to nearest, then one
// rounding to bf16, nearest even.  Returns the bf16 bits.
#ifndef __CUDA_ARCH__
// float -> bf16 bits, nearest even; a NaN becomes 0x7FC0 (the row format holds none: the quantiser saturates).
LV_FP8_HD uint16_t lv_f32_to_bf16(float f) {
  union {
    float f;
    uint32_t u;
  } c;
  c.f = f;
  if (f != f) return 0x7FC0;
  return (uint16_t)((c.u + 0x7FFFu + ((c.u >> 16) & 1u)) >> 16);
}
#endif

LV_FP8_HD uint16_t lv_kv8_decode(float x, float s) {
#ifdef __CUDA_ARCH__
  uint16_t r;
  asm("cvt.rn.bf16.f32 %0, %1;" : "=h"(r) : "f"(__fmul_rn(x, s)));
  return r;
#else
  volatile float p = x * s;
  return lv_f32_to_bf16(p);
#endif
}

#ifdef __CUDACC__
// Two products x * inv -> two bytes of the format (lo in the low byte): PTX cvt.rn.satfinite.{e4m3x2,e5m2x2}.f32, which
// for the products of the rule (|v| <= M rounded up by the two divisions) gives exactly lv_fp8_encode.
__device__ __forceinline__ uint16_t lv_fp8_pack2(int fmt, float lo, float hi) {
  uint16_t r;
  if (fmt == LV_FP8_E5M2)
    asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  else
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
  return r;
}
#endif

#ifndef __CUDA_ARCH__
// fp32 -> the bits of the format, round to nearest even, finite values above M saturate to M (PTX cvt.rn.satfinite).
// The kernels convert two at a time with the PTX instruction (lv_fp8_pack2); this is the host statement of the same
// rule.  e4m3: 3 mantissa bits, smallest normal 2^-6; e5m2: 2 mantissa bits, smallest normal 2^-14.
static inline uint8_t lv_fp8_encode(int fmt, float f) {
  const int mbits = fmt == LV_FP8_E5M2 ? 2 : 3;
  const int emin = fmt == LV_FP8_E5M2 ? -14 : -6;
  union {
    float f;
    uint32_t u;
  } c;
  c.f = f;
  const uint8_t sign = (uint8_t)((c.u >> 24) & 0x80u);
  c.u &= 0x7FFFFFFFu;
  const float a = c.f;
  if (a != a) return 0x7F;                                                  // NaN
  if (a >= lv_fp8_max(fmt)) return sign | (fmt == LV_FP8_E5M2 ? 0x7B : 0x7E);  // satfinite
  if (a < ldexpf(1.0f, emin)) {                   // subnormal steps of 2^(emin - mbits); the last step reaches 2^emin
    return sign | (uint8_t)rintf(ldexpf(a, mbits - emin));   // exact scaling; rintf rounds half to even
  }
  int e;
  frexpf(a, &e);                                  // a = m * 2^e, m in [0.5, 1): 2^(e-1) <= a < 2^e
  const int q = (int)rintf(ldexpf(a, mbits + 1 - e));   // in [2^mbits, 2^(mbits+1)], exact scaling; the top carries
  return sign | (uint8_t)(((e - emin) << mbits) + (q - (1 << mbits)));
}

// e4m3 bits -> float, exact (0x7F and 0xFF are NaN).  The kernels convert with PTX cvt.rn.f16x2.e4m3x2, also exact.
static inline float lv_e4m3_to_f32(uint8_t b) {
  const int e = (b >> 3) & 15, m = b & 7;
  const float a = (e == 15 && m == 7) ? NAN : e == 0 ? ldexpf((float)m, -9) : ldexpf((float)(8 + m), e - 10);
  return (b & 0x80) ? -a : a;
}

// Quantise one row: x [n] bf16 bits -> q [n] in the format, returns the scale.  The kernels split a row over lanes,
// reduce amax with shuffles (max is exact in any order) and multiply with __fmul_rn.
static inline float lv_fp8_quant_row(int fmt, const uint16_t* x, uint8_t* q, int64_t n) {
  float amax = 0.0f;
  for (int64_t i = 0; i < n; ++i) {
    const float v = fabsf(lv_bf16_to_f32(x[i]));
    amax = v > amax ? v : amax;
  }
  const float inv = lv_fp8_inv(fmt, amax);
  if (lv_fp8_zero_row(inv)) {
    for (int64_t i = 0; i < n; ++i) q[i] = 0;
    return 0.0f;
  }
  for (int64_t i = 0; i < n; ++i) {
    volatile float t = lv_bf16_to_f32(x[i]) * inv;
    q[i] = lv_fp8_encode(fmt, t);
  }
  return lv_fp8_scale(fmt, amax);
}
#endif

#endif  // LV_FP8_CORE_H_
