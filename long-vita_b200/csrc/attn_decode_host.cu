// Flash-decoding over K/V rows that live in pinned host memory, and the two host-memory helpers of the host tier of
// the K/V cache (kv_cache.OffloadedKVCache): a pinned, mapped allocation and a strided device-to-host row copy.
//
// A decode step reads every K/V row of a layer once, so over host memory the step is bound by PCIe, not by HBM or
// arithmetic (~10 000 FMA per 4 KB row).  The kernel reads the rows in place through their device-mapped address:
// no device staging copy of a layer exists.  What it must do is keep enough independent 16-byte reads in flight:
// every 16-lane half-warp owns one kv head of one row (128 columns, 8 per lane, K and V), the half-warps of a CTA
// cover consecutive whole rows, and each half-warp issues the loads of kUnroll rows before it uses any of them.
//
// Host row format: token-major, K | V per row, [capacity, 2 * hkv * 128] bf16 (the streamed decoder layer's K|V
// buffer rows, so a prefill span is one contiguous copy).  CTA s takes rows [s * per, min((s + 1) * per, length))
// over all heads; the G = hq / hkv query heads of a group are its rows.  Output: o_part [n, G, hkv, 128] bf16 and
// lse_part [n, hkv, G] fp32 (natural log), exactly what lv_attn_decode_merge consumes.
//
// The FP8 host tier (opt-in, lossy) halves the bytes per row: e4m3 K | V with one fp32 scale per head and row, the
// format and quantisation rule of fp8_core.h (2112 B per row at 8 kv heads).  rows_to_host_fp8_kernel quantises
// device rows straight into the mapped host rows; attn_decode_host_fp8_kernel is the flash-decoding above over them.
//
// Several query tokens (a question about a prefilled context) do not read host rows in place: the rows are copied to
// the device chunk by chunk (ops.attention_host_rows) and attended by lv_attn_fwd.  kv_rows_dequant_fp8_kernel decodes
// an FP8 chunk, once it is in HBM, into the bf16 K|V rows that call reads.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"
#include "fp8_core.h"

namespace {

constexpr int kD = 128;
constexpr int kThreads = 256;
constexpr int kHalfWarps = kThreads / 16;
constexpr int kMaxG = 8;
constexpr int kUnroll = 4;
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

__device__ __forceinline__ void bf16x8_to_f32(const uint4& u, float* f) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

// Sum over the 16 lanes of a half-warp (xor offsets below 16 stay inside it); every lane of the warp takes part.
__device__ __forceinline__ float half_warp_sum(float x) {
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

template <int G>
__global__ void __launch_bounds__(kThreads) attn_decode_host_kernel(const __nv_bfloat16* __restrict__ q,
                                                                    const __nv_bfloat16* kv,
                                                                    __nv_bfloat16* __restrict__ o_part,
                                                                    float* __restrict__ lse_part, int64_t length,
                                                                    int64_t per_split, int hkv, float scale_log2) {
  __shared__ float sm_acc[kHalfWarps / 2][G][kD];
  __shared__ float sm_m[kHalfWarps / 2][G], sm_l[kHalfWarps / 2][G];

  const int hw = threadIdx.x >> 4, lane = threadIdx.x & 15;
  const int phases = kHalfWarps / hkv;             // half-warps per head: each takes every phases-th row
  const int head = hw % hkv, phase = hw / hkv;
  const int64_t row_elems = 2ll * hkv * kD;
  const int64_t r_begin = (int64_t)blockIdx.x * per_split;
  const int64_t r_end = min(r_begin + per_split, length);  // no row at or past `length` is read

  float qf[G][8];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    bf16x8_to_f32(*reinterpret_cast<const uint4*>(q + ((int64_t)head * G + g) * kD + lane * 8), qf[g]);
#pragma unroll
    for (int e = 0; e < 8; ++e) qf[g][e] *= scale_log2;     // scores in log2 units
  }
  float m[G], l[G], acc[G][8];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    m[g] = -INFINITY;
    l[g] = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[g][e] = 0.f;
  }

  const __nv_bfloat16* kcol = kv + (int64_t)head * kD + lane * 8;
  const __nv_bfloat16* vcol = kcol + (int64_t)hkv * kD;
  for (int64_t base = r_begin; base < r_end; base += (int64_t)phases * kUnroll) {
    uint4 kr[kUnroll], vr[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {                       // all loads first: kUnroll rows in flight per lane
      const int64_t row = base + (int64_t)u * phases + phase;
      if (row < r_end) {
        kr[u] = __ldcs(reinterpret_cast<const uint4*>(kcol + row * row_elems));
        vr[u] = __ldcs(reinterpret_cast<const uint4*>(vcol + row * row_elems));
      } else {
        kr[u] = vr[u] = make_uint4(0u, 0u, 0u, 0u);
      }
    }
#pragma unroll
    for (int u = 0; u < kUnroll; ++u) {
      const bool valid = base + (int64_t)u * phases + phase < r_end;
      float kf[8], vf[8];
      bf16x8_to_f32(kr[u], kf);
      bf16x8_to_f32(vr[u], vf);
#pragma unroll
      for (int g = 0; g < G; ++g) {
        float s = 0.f;
#pragma unroll
        for (int e = 0; e < 8; ++e) s = fmaf(qf[g][e], kf[e], s);
        s = half_warp_sum(s);                                   // outside `valid`: the whole warp shuffles
        if (valid) {
          const float m_new = fmaxf(m[g], s);
          const float corr = exp2f(m[g] - m_new);                 // 0 while m is -inf
          const float p = exp2f(s - m_new);
          l[g] = fmaf(l[g], corr, p);
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[g][e] = fmaf(acc[g][e], corr, p * vf[e]);
          m[g] = m_new;
        }
      }
    }
  }

  // fold the phases of each head into phase 0, one phase at a time through shared memory
  for (int p = 1; p < phases; ++p) {
    if (phase == p) {
#pragma unroll
      for (int g = 0; g < G; ++g) {
#pragma unroll
        for (int e = 0; e < 8; ++e) sm_acc[head][g][lane * 8 + e] = acc[g][e];
        if (lane == 0) sm_m[head][g] = m[g], sm_l[head][g] = l[g];
      }
    }
    __syncthreads();
    if (phase == 0) {
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const float m1 = sm_m[head][g], l1 = sm_l[head][g];
        const float m_new = fmaxf(m[g], m1);
        if (m_new > -INFINITY) {
          const float c0 = exp2f(m[g] - m_new), c1 = exp2f(m1 - m_new);
          l[g] = l[g] * c0 + l1 * c1;
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[g][e] = acc[g][e] * c0 + sm_acc[head][g][lane * 8 + e] * c1;
          m[g] = m_new;
        }
      }
    }
    __syncthreads();
  }

  if (phase == 0) {
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const float inv = l[g] > 0.f ? 1.f / l[g] : 0.f;
      __align__(16) __nv_bfloat16 out[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) out[e] = __float2bfloat16_rn(acc[g][e] * inv);
      *reinterpret_cast<uint4*>(o_part + (((int64_t)blockIdx.x * G + g) * hkv + head) * kD + lane * 8) =
          *reinterpret_cast<const uint4*>(out);
      if (lane == 0)
        lse_part[((int64_t)blockIdx.x * hkv + head) * G + g] = l[g] > 0.f ? (m[g] + log2f(l[g])) * kLn2 : -INFINITY;
    }
  }
}

template <int G>
void launch(const __nv_bfloat16* q, const __nv_bfloat16* kv, __nv_bfloat16* o, float* lse, int64_t length,
            int64_t per, int64_t n_splits, int hkv, float scale_log2, cudaStream_t stream) {
  attn_decode_host_kernel<G><<<(unsigned)n_splits, kThreads, 0, stream>>>(q, kv, o, lse, length, per, hkv,
                                                                          scale_log2);
}

// ------------------------------------------------------------------------------------------------
// FP8 host tier
// ------------------------------------------------------------------------------------------------
constexpr int kQuantThreads = 256;     // 32 groups of 8 lanes: a group quantises one head of K or V of one row
constexpr int kFp8Unroll = 8;          // rows in flight per lane: 256 lanes x 16 B x 8 = 32 KB per CTA, as above

// Row r of the source, K|V of the hkv heads (2 hkv head vectors of 128 bf16, V following K): each group of 8 lanes
// takes one vector, 16 columns per lane, reduces amax over its 8 lanes, and stores its 128 e4m3 bytes as 8 16-byte
// stores straight into the mapped host row (no device temporary).  The 2 hkv scales of a row go through shared
// memory and out as 16-byte stores, zero padding included.  Rows [r0, r0 + 32 / (2 hkv)) per CTA iteration.
__global__ void __launch_bounds__(kQuantThreads) rows_to_host_fp8_kernel(const __nv_bfloat16* __restrict__ src,
                                                                         int64_t src_pitch, uint8_t* dst,
                                                                         int64_t rows, int hkv) {
  __shared__ float sm_scale[kQuantThreads / 8];
  const int grp = threadIdx.x >> 3, lane = threadIdx.x & 7;
  const int vecs = 2 * hkv, rows_per_it = (kQuantThreads / 8) / vecs;
  const int r_in = grp / vecs, j = grp % vecs;
  const int64_t row_bytes = lv_kv8_row_bytes(hkv, kD);
  const int scale_vecs = (int)(lv_kv8_scale_bytes(hkv) / 16);
  for (int64_t r0 = (int64_t)blockIdx.x * rows_per_it; r0 < rows; r0 += (int64_t)gridDim.x * rows_per_it) {
    const int64_t row = r0 + r_in;
    const bool valid = row < rows;
    float x[16];
    if (valid) {
      const uint4* p = reinterpret_cast<const uint4*>(src + row * src_pitch + j * kD + lane * 16);
      bf16x8_to_f32(p[0], x);
      bf16x8_to_f32(p[1], x + 8);
    } else {
#pragma unroll
      for (int e = 0; e < 16; ++e) x[e] = 0.f;
    }
    float amax = 0.f;
#pragma unroll
    for (int e = 0; e < 16; ++e) amax = fmaxf(amax, fabsf(x[e]));
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));  // the 8 lanes
    const float inv = lv_fp8_inv(LV_FP8_E4M3, amax);
    const bool zero = lv_fp8_zero_row(inv);                                 // amax 0: all-zero bytes, scale 0
    uint4 out = make_uint4(0u, 0u, 0u, 0u);
    if (!zero) {
      uint32_t w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
        w[i] = (uint32_t)lv_fp8_pack2(LV_FP8_E4M3, __fmul_rn(x[4 * i], inv), __fmul_rn(x[4 * i + 1], inv)) |
               (uint32_t)lv_fp8_pack2(LV_FP8_E4M3, __fmul_rn(x[4 * i + 2], inv), __fmul_rn(x[4 * i + 3], inv)) << 16;
      out = make_uint4(w[0], w[1], w[2], w[3]);
    }
    if (valid) *reinterpret_cast<uint4*>(dst + row * row_bytes + j * kD + lane * 16) = out;
    if (lane == 0) sm_scale[grp] = zero ? 0.f : lv_fp8_scale(LV_FP8_E4M3, amax);
    __syncthreads();
    if (threadIdx.x < rows_per_it * scale_vecs) {
      const int rr = threadIdx.x / scale_vecs, c = threadIdx.x % scale_vecs;
      if (r0 + rr < rows) {
        float f[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) f[i] = 4 * c + i < vecs ? sm_scale[rr * vecs + 4 * c + i] : 0.f;
        *reinterpret_cast<uint4*>(dst + (r0 + rr) * row_bytes + 2 * hkv * kD + 16 * c) =
            make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
      }
    }
    __syncthreads();
  }
}

// 16 e4m3 bytes -> 16 floats (exact: e4m3 -> f16 with cvt.rn.f16x2.e4m3x2, then f16 -> f32).
__device__ __forceinline__ void e4m3x16_to_f32(const uint4& u, float* f) {
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      uint32_t r;
      asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"((unsigned short)(w[i] >> (16 * h))));
      const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&r));
      f[4 * i + 2 * h] = t.x;
      f[4 * i + 2 * h + 1] = t.y;
    }
  }
}

// attn_decode_host_kernel over FP8 rows.  A 128-column head of K or V is 128 bytes, so a 16-lane half-warp still owns
// one head of one row, now split by role: lanes 0-7 load its K (16 columns each), lanes 8-15 its V.  The register
// array r holds the query (in log2 units) on K lanes and the output accumulator on V lanes.  A score is the
// half-warp sum of the K lanes' partial dot products times s_k (each scale applied once per dot product); the V
// lanes accumulate (p * s_v) * v8.  Each lane also loads its role's scale of the row; s_k and s_v reach the other
// lanes by shuffle.  Split rule, phases and outputs are those of attn_decode_host_kernel.
template <int G>
__global__ void __launch_bounds__(kThreads) attn_decode_host_fp8_kernel(const __nv_bfloat16* __restrict__ q,
                                                                        const uint8_t* kv,
                                                                        __nv_bfloat16* __restrict__ o_part,
                                                                        float* __restrict__ lse_part, int64_t length,
                                                                        int64_t per_split, int hkv, float scale_log2) {
  __shared__ float sm_acc[kHalfWarps / 2][G][kD];
  __shared__ float sm_m[kHalfWarps / 2][G], sm_l[kHalfWarps / 2][G];

  const int hw = threadIdx.x >> 4, lane = threadIdx.x & 15;
  const bool is_k = lane < 8;
  const int col = (lane & 7) * 16;                 // this lane's 16 columns of its head
  const int phases = kHalfWarps / hkv;
  const int head = hw % hkv, phase = hw / hkv;
  const int64_t row_bytes = lv_kv8_row_bytes(hkv, kD);
  const int64_t r_begin = (int64_t)blockIdx.x * per_split;
  const int64_t r_end = min(r_begin + per_split, length);  // no row at or past `length` is read

  float r[G][16];
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const uint4* qp = reinterpret_cast<const uint4*>(q + ((int64_t)head * G + g) * kD + col);
    bf16x8_to_f32(qp[0], r[g]);
    bf16x8_to_f32(qp[1], r[g] + 8);
#pragma unroll
    for (int e = 0; e < 16; ++e) r[g][e] = is_k ? r[g][e] * scale_log2 : 0.f;
  }
  float m[G], l[G];
#pragma unroll
  for (int g = 0; g < G; ++g) m[g] = -INFINITY, l[g] = 0.f;

  const uint8_t* xcol = kv + (int64_t)((is_k ? 0 : hkv) + head) * kD + col;
  const uint8_t* scol = kv + 2ll * hkv * kD + 4ll * ((is_k ? 0 : hkv) + head);
  for (int64_t base = r_begin; base < r_end; base += (int64_t)phases * kFp8Unroll) {
    uint4 xr[kFp8Unroll];
    float sr[kFp8Unroll];
#pragma unroll
    for (int u = 0; u < kFp8Unroll; ++u) {                   // all loads first: kFp8Unroll rows in flight per lane
      const int64_t row = base + (int64_t)u * phases + phase;
      if (row < r_end) {
        xr[u] = __ldcs(reinterpret_cast<const uint4*>(xcol + row * row_bytes));
        sr[u] = __ldcs(reinterpret_cast<const float*>(scol + row * row_bytes));
      } else {
        xr[u] = make_uint4(0u, 0u, 0u, 0u);
        sr[u] = 0.f;
      }
    }
#pragma unroll
    for (int u = 0; u < kFp8Unroll; ++u) {
      const bool valid = base + (int64_t)u * phases + phase < r_end;
      const float sk = __shfl_sync(0xffffffffu, sr[u], 0, 16), sv = __shfl_sync(0xffffffffu, sr[u], 8, 16);
      float xf[16];
      e4m3x16_to_f32(xr[u], xf);
#pragma unroll
      for (int g = 0; g < G; ++g) {
        float s = 0.f;
#pragma unroll
        for (int e = 0; e < 16; ++e) s = fmaf(r[g][e], xf[e], s);
        s = half_warp_sum(is_k ? s : 0.f) * sk;                // outside `valid`: the whole warp shuffles
        if (valid) {
          const float m_new = fmaxf(m[g], s);
          const float corr = exp2f(m[g] - m_new);                 // 0 while m is -inf
          const float p = exp2f(s - m_new);
          l[g] = fmaf(l[g], corr, p);
          if (!is_k) {
            const float pv = p * sv;
#pragma unroll
            for (int e = 0; e < 16; ++e) r[g][e] = fmaf(r[g][e], corr, pv * xf[e]);
          }
          m[g] = m_new;
        }
      }
    }
  }

  // fold the phases of each head into phase 0, one phase at a time through shared memory (V lanes hold the sums)
  for (int p = 1; p < phases; ++p) {
    if (phase == p) {
#pragma unroll
      for (int g = 0; g < G; ++g) {
        if (!is_k) {
#pragma unroll
          for (int e = 0; e < 16; ++e) sm_acc[head][g][col + e] = r[g][e];
        }
        if (lane == 0) sm_m[head][g] = m[g], sm_l[head][g] = l[g];
      }
    }
    __syncthreads();
    if (phase == 0) {
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const float m1 = sm_m[head][g], l1 = sm_l[head][g];
        const float m_new = fmaxf(m[g], m1);
        if (m_new > -INFINITY) {
          const float c0 = exp2f(m[g] - m_new), c1 = exp2f(m1 - m_new);
          l[g] = l[g] * c0 + l1 * c1;
          if (!is_k) {
#pragma unroll
            for (int e = 0; e < 16; ++e) r[g][e] = r[g][e] * c0 + sm_acc[head][g][col + e] * c1;
          }
          m[g] = m_new;
        }
      }
    }
    __syncthreads();
  }

  if (phase == 0) {
#pragma unroll
    for (int g = 0; g < G; ++g) {
      if (!is_k) {
        const float inv = l[g] > 0.f ? 1.f / l[g] : 0.f;
        __align__(16) __nv_bfloat16 out[16];
#pragma unroll
        for (int e = 0; e < 16; ++e) out[e] = __float2bfloat16_rn(r[g][e] * inv);
        uint4* dst = reinterpret_cast<uint4*>(o_part + (((int64_t)blockIdx.x * G + g) * hkv + head) * kD + col);
        dst[0] = reinterpret_cast<const uint4*>(out)[0];
        dst[1] = reinterpret_cast<const uint4*>(out)[1];
      }
      if (lane == 0)
        lse_part[((int64_t)blockIdx.x * hkv + head) * G + g] = l[g] > 0.f ? (m[g] + log2f(l[g])) * kLn2 : -INFINITY;
    }
  }
}

template <int G>
void launch_fp8(const __nv_bfloat16* q, const uint8_t* kv, __nv_bfloat16* o, float* lse, int64_t length, int64_t per,
                int64_t n_splits, int hkv, float scale_log2, cudaStream_t stream) {
  attn_decode_host_fp8_kernel<G><<<(unsigned)n_splits, kThreads, 0, stream>>>(q, kv, o, lse, length, per, hkv,
                                                                              scale_log2);
}

constexpr int kDequantThreads = 256;
constexpr int kDequantUnroll = 4;      // rows in flight per lane

// FP8 host rows staged in device memory -> bf16 K|V rows [rows, 2 hkv 128], by the decode rule of fp8_core.h.  Each
// lane owns 16 e4m3 bytes of a row (one 16-byte load) and writes their 16 bf16 values (two 16-byte stores); the 8
// lanes of a head read its scale (a 4-byte load the L1 serves once for them).  The 16 hkv lanes of a row are consecutive, so a CTA
// covers 256 / (16 hkv) whole rows per step, and each lane issues the loads of kDequantUnroll rows before it converts
// any of them.  HBM-bound: 2112 bytes read and 4096 written per row at 8 kv heads.
__global__ void __launch_bounds__(kDequantThreads) kv_rows_dequant_fp8_kernel(const uint8_t* __restrict__ src,
                                                                             __nv_bfloat16* __restrict__ dst,
                                                                             int64_t rows, int hkv) {
  const int vecs = 2 * hkv * kD / 16;
  const int rows_per_step = kDequantThreads / vecs;
  const int c = threadIdx.x % vecs, head = c / (kD / 16);   // head in [0, 2 hkv): K heads, then V heads
  const int64_t row_bytes = lv_kv8_row_bytes(hkv, kD);
  const int64_t row_elems = 2ll * hkv * kD;
  const int64_t step = (int64_t)gridDim.x * rows_per_step;
  for (int64_t base = (int64_t)blockIdx.x * rows_per_step + threadIdx.x / vecs; base < rows;
       base += step * kDequantUnroll) {
    uint4 x[kDequantUnroll];
    float s[kDequantUnroll];
#pragma unroll
    for (int u = 0; u < kDequantUnroll; ++u) {
      const int64_t row = base + u * step;
      if (row < rows) {
        const uint8_t* p = src + row * row_bytes;
        x[u] = *reinterpret_cast<const uint4*>(p + 16 * c);
        s[u] = *reinterpret_cast<const float*>(p + row_elems + 4 * head);
      } else {
        x[u] = make_uint4(0u, 0u, 0u, 0u);
        s[u] = 0.f;
      }
    }
#pragma unroll
    for (int u = 0; u < kDequantUnroll; ++u) {
      const int64_t row = base + u * step;
      if (row < rows) {
        float f[16];
        e4m3x16_to_f32(x[u], f);
        uint32_t w[8];
#pragma unroll
        for (int i = 0; i < 8; ++i)
          w[i] = (uint32_t)lv_kv8_decode(f[2 * i], s[u]) | (uint32_t)lv_kv8_decode(f[2 * i + 1], s[u]) << 16;
        uint4* o = reinterpret_cast<uint4*>(dst + row * row_elems + 16 * c);
        o[0] = make_uint4(w[0], w[1], w[2], w[3]);
        o[1] = make_uint4(w[4], w[5], w[6], w[7]);
      }
    }
  }
}

// cudaPointerGetAttributes on `p`: LV_OK when it is pinned host memory, else an error naming `what`.
int check_pinned_host(const void* p, const char* what) {
  cudaPointerAttributes a;
  const cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    lv::set_error("%s: cudaPointerGetAttributes failed: %s", what, cudaGetErrorString(e));
    return LV_ECUDA;
  }
  if (a.type != cudaMemoryTypeHost) {
    lv::set_error("%s: %p is not pinned host memory", what, p);
    return LV_EINVAL;
  }
  return LV_OK;
}

}  // namespace

extern "C" {

int lv_attn_decode_host(const void* q, const void* kv_host, void* o_part, float* lse_part, int64_t length,
                        int64_t capacity, int64_t hq, int64_t hkv, int64_t d, int64_t n_splits, float scale,
                        lv_stream_t stream) {
  LV_CHECK_ARG(q && kv_host && o_part && lse_part, "lv_attn_decode_host: null pointer");
  LV_CHECK_ARG(d == kD, "lv_attn_decode_host: head_dim %lld not supported (128 only)", (long long)d);
  LV_CHECK_ARG(hq > 0 && hkv > 0 && hq % hkv == 0, "lv_attn_decode_host: bad heads hq=%lld hkv=%lld", (long long)hq,
               (long long)hkv);
  LV_CHECK_ARG(kHalfWarps % hkv == 0 && hq / hkv <= kMaxG,
               "lv_attn_decode_host: hkv %lld must divide 16 and hq / hkv (%lld) be at most 8", (long long)hkv,
               (long long)(hq / hkv));
  LV_CHECK_ARG(length > 0 && length <= capacity && capacity < (1ll << 40),
               "lv_attn_decode_host: length %lld outside the cache (capacity %lld)", (long long)length,
               (long long)capacity);
  LV_CHECK_ARG(n_splits > 0 && n_splits < (1ll << 20), "lv_attn_decode_host: bad n_splits %lld", (long long)n_splits);
  LV_CHECK_ARG(isfinite(scale) && scale > 0.f, "lv_attn_decode_host: scale must be finite and > 0");
  LV_BIND_DEVICE(q);
  int rc = check_pinned_host(kv_host, "lv_attn_decode_host: K|V rows");
  if (rc != LV_OK) return rc;
  void* kv_dev = nullptr;
  LV_CHECK_CUDA(cudaHostGetDevicePointer(&kv_dev, const_cast<void*>(kv_host), 0));
  const int64_t per = (length + n_splits - 1) / n_splits;
  const auto* qb = static_cast<const __nv_bfloat16*>(q);
  const auto* kvb = static_cast<const __nv_bfloat16*>(kv_dev);
  auto* ob = static_cast<__nv_bfloat16*>(o_part);
  const float sl2 = scale * kLog2e;
  const int h = (int)hkv;
  cudaStream_t s = (cudaStream_t)stream;
  switch (hq / hkv) {
    case 1: launch<1>(qb, kvb, ob, lse_part, length, per, n_splits, h, sl2, s); break;
    case 2: launch<2>(qb, kvb, ob, lse_part, length, per, n_splits, h, sl2, s); break;
    case 3: launch<3>(qb, kvb, ob, lse_part, length, per, n_splits, h, sl2, s); break;
    case 4: launch<4>(qb, kvb, ob, lse_part, length, per, n_splits, h, sl2, s); break;
    case 5: launch<5>(qb, kvb, ob, lse_part, length, per, n_splits, h, sl2, s); break;
    case 6: launch<6>(qb, kvb, ob, lse_part, length, per, n_splits, h, sl2, s); break;
    case 7: launch<7>(qb, kvb, ob, lse_part, length, per, n_splits, h, sl2, s); break;
    default: launch<8>(qb, kvb, ob, lse_part, length, per, n_splits, h, sl2, s); break;
  }
  LV_CHECK_LAUNCH("attn_decode_host_kernel");
  return LV_OK;
}

int lv_host_alloc(int64_t bytes, void** ptr) {
  LV_CHECK_ARG(ptr != nullptr && bytes > 0, "lv_host_alloc: bad arguments");
  *ptr = nullptr;
  LV_CHECK_CUDA(cudaHostAlloc(ptr, (size_t)bytes, cudaHostAllocMapped | cudaHostAllocPortable));
  return LV_OK;
}

int lv_host_free(void* ptr) {
  if (ptr != nullptr) LV_CHECK_CUDA(cudaFreeHost(ptr));
  return LV_OK;
}

int lv_rows_to_host(void* host_dst, const void* src, int64_t rows, int64_t row_bytes, int64_t src_pitch,
                    lv_stream_t stream) {
  LV_CHECK_ARG(host_dst && src, "lv_rows_to_host: null pointer");
  LV_CHECK_ARG(rows > 0 && row_bytes > 0 && src_pitch >= row_bytes, "lv_rows_to_host: bad shape");
  LV_BIND_DEVICE(src);
  int rc = check_pinned_host(host_dst, "lv_rows_to_host: destination");
  if (rc != LV_OK) return rc;
  LV_CHECK_CUDA(cudaMemcpy2DAsync(host_dst, (size_t)row_bytes, src, (size_t)src_pitch, (size_t)row_bytes,
                                  (size_t)rows, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return LV_OK;
}

int lv_attn_decode_host_fp8(const void* q, const void* kv_host, void* o_part, float* lse_part, int64_t length,
                            int64_t capacity, int64_t hq, int64_t hkv, int64_t d, int64_t n_splits, float scale,
                            lv_stream_t stream) {
  LV_CHECK_ARG(q && kv_host && o_part && lse_part, "lv_attn_decode_host_fp8: null pointer");
  LV_CHECK_ARG(d == kD, "lv_attn_decode_host_fp8: head_dim %lld not supported (128 only)", (long long)d);
  LV_CHECK_ARG(hq > 0 && hkv > 0 && hq % hkv == 0, "lv_attn_decode_host_fp8: bad heads hq=%lld hkv=%lld",
               (long long)hq, (long long)hkv);
  LV_CHECK_ARG(kHalfWarps % hkv == 0 && hq / hkv <= kMaxG,
               "lv_attn_decode_host_fp8: hkv %lld must divide 16 and hq / hkv (%lld) be at most 8", (long long)hkv,
               (long long)(hq / hkv));
  LV_CHECK_ARG(length > 0 && length <= capacity && capacity < (1ll << 40),
               "lv_attn_decode_host_fp8: length %lld outside the cache (capacity %lld)", (long long)length,
               (long long)capacity);
  LV_CHECK_ARG(n_splits > 0 && n_splits < (1ll << 20), "lv_attn_decode_host_fp8: bad n_splits %lld",
               (long long)n_splits);
  LV_CHECK_ARG(isfinite(scale) && scale > 0.f, "lv_attn_decode_host_fp8: scale must be finite and > 0");
  LV_CHECK_ARG((uintptr_t)kv_host % 16 == 0, "lv_attn_decode_host_fp8: K|V rows not 16-byte aligned");
  LV_BIND_DEVICE(q);
  int rc = check_pinned_host(kv_host, "lv_attn_decode_host_fp8: K|V rows");
  if (rc != LV_OK) return rc;
  void* kv_dev = nullptr;
  LV_CHECK_CUDA(cudaHostGetDevicePointer(&kv_dev, const_cast<void*>(kv_host), 0));
  const int64_t per = (length + n_splits - 1) / n_splits;
  const auto* qb = static_cast<const __nv_bfloat16*>(q);
  const auto* kv8 = static_cast<const uint8_t*>(kv_dev);
  auto* ob = static_cast<__nv_bfloat16*>(o_part);
  const float sl2 = scale * kLog2e;
  const int h = (int)hkv;
  cudaStream_t s = (cudaStream_t)stream;
  switch (hq / hkv) {
    case 1: launch_fp8<1>(qb, kv8, ob, lse_part, length, per, n_splits, h, sl2, s); break;
    case 2: launch_fp8<2>(qb, kv8, ob, lse_part, length, per, n_splits, h, sl2, s); break;
    case 3: launch_fp8<3>(qb, kv8, ob, lse_part, length, per, n_splits, h, sl2, s); break;
    case 4: launch_fp8<4>(qb, kv8, ob, lse_part, length, per, n_splits, h, sl2, s); break;
    case 5: launch_fp8<5>(qb, kv8, ob, lse_part, length, per, n_splits, h, sl2, s); break;
    case 6: launch_fp8<6>(qb, kv8, ob, lse_part, length, per, n_splits, h, sl2, s); break;
    case 7: launch_fp8<7>(qb, kv8, ob, lse_part, length, per, n_splits, h, sl2, s); break;
    default: launch_fp8<8>(qb, kv8, ob, lse_part, length, per, n_splits, h, sl2, s); break;
  }
  LV_CHECK_LAUNCH("attn_decode_host_fp8_kernel");
  return LV_OK;
}

int lv_rows_to_host_fp8(void* host_dst, const void* src, int64_t rows, int64_t hkv, int64_t d, int64_t src_pitch,
                        lv_stream_t stream) {
  LV_CHECK_ARG(host_dst && src, "lv_rows_to_host_fp8: null pointer");
  LV_CHECK_ARG(d == kD, "lv_rows_to_host_fp8: head_dim %lld not supported (128 only)", (long long)d);
  LV_CHECK_ARG(hkv > 0 && kHalfWarps % hkv == 0, "lv_rows_to_host_fp8: hkv %lld must divide 16", (long long)hkv);
  LV_CHECK_ARG(rows > 0 && src_pitch >= 2 * hkv * d * 2 && src_pitch % 16 == 0, "lv_rows_to_host_fp8: bad shape");
  LV_CHECK_ARG((uintptr_t)src % 16 == 0 && (uintptr_t)host_dst % 16 == 0,
               "lv_rows_to_host_fp8: source and destination must be 16-byte aligned");
  LV_BIND_DEVICE(src);
  int rc = check_pinned_host(host_dst, "lv_rows_to_host_fp8: destination");
  if (rc != LV_OK) return rc;
  void* dst_dev = nullptr;
  LV_CHECK_CUDA(cudaHostGetDevicePointer(&dst_dev, host_dst, 0));
  const int rows_per_it = (kQuantThreads / 8) / (2 * (int)hkv);
  const int64_t need = (rows + rows_per_it - 1) / rows_per_it, cap = 8ll * lv::sm_count();
  const int64_t blocks = need < cap ? need : cap;
  rows_to_host_fp8_kernel<<<(unsigned)blocks, kQuantThreads, 0, (cudaStream_t)stream>>>(
      static_cast<const __nv_bfloat16*>(src), src_pitch / 2, static_cast<uint8_t*>(dst_dev), rows, (int)hkv);
  LV_CHECK_LAUNCH("rows_to_host_fp8_kernel");
  return LV_OK;
}

int lv_kv_rows_dequant_fp8(const void* src, void* dst, int64_t rows, int64_t hkv, int64_t d, lv_stream_t stream) {
  LV_CHECK_ARG(src && dst, "lv_kv_rows_dequant_fp8: null pointer");
  LV_CHECK_ARG(d == kD, "lv_kv_rows_dequant_fp8: head_dim %lld not supported (128 only)", (long long)d);
  LV_CHECK_ARG(hkv > 0 && kHalfWarps % hkv == 0, "lv_kv_rows_dequant_fp8: hkv %lld must divide 16", (long long)hkv);
  LV_CHECK_ARG(rows > 0 && rows < (1ll << 40), "lv_kv_rows_dequant_fp8: bad rows %lld", (long long)rows);
  LV_CHECK_ARG((uintptr_t)src % 16 == 0 && (uintptr_t)dst % 16 == 0,
               "lv_kv_rows_dequant_fp8: source and destination must be 16-byte aligned");
  LV_BIND_DEVICE(dst);
  const int rows_per_step = kDequantThreads / (2 * (int)hkv * kD / 16);
  const int64_t need = (rows + rows_per_step * kDequantUnroll - 1) / (rows_per_step * kDequantUnroll);
  const int64_t cap = 8ll * lv::sm_count();
  kv_rows_dequant_fp8_kernel<<<(unsigned)(need < cap ? need : cap), kDequantThreads, 0, (cudaStream_t)stream>>>(
      static_cast<const uint8_t*>(src), static_cast<__nv_bfloat16*>(dst), rows, (int)hkv);
  LV_CHECK_LAUNCH("kv_rows_dequant_fp8_kernel");
  return LV_OK;
}

}  // extern "C"
