// Token-wise HBM-bound operators of the Long-VITA hot path: RMSNorm(+residual), LayerNorm, RoPE
// table + apply, SwiGLU, bias+GELU, layer-scale residual, pixel-shuffle, embedding gather +
// feature scatter, row gather / scatter.  One pass over the data, 16-byte accesses, fp32 math,
// and the bf16 rounding points of the reference's eager PyTorch sequence (cited per kernel) so
// results match the oracle bit-for-bit wherever the arithmetic is exactly representable.
#include <cuda_bf16.h>
#include <math.h>

#include <iterator>
#include <type_traits>

#include "common.cuh"

namespace lv {

struct alignas(16) Vec8 {
  __nv_bfloat162 h[4];
};

__device__ __forceinline__ Vec8 ldg_vec(const void* p) {
  return *reinterpret_cast<const Vec8*>(p);
}
__device__ __forceinline__ Vec8 ldg_stream(const void* p) {
  Vec8 v;
  uint32_t* u = reinterpret_cast<uint32_t*>(&v);
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(u[0]), "=r"(u[1]), "=r"(u[2]), "=r"(u[3])
               : "l"(p));
  return v;
}
__device__ __forceinline__ void stg_vec(void* p, const Vec8& v) { *reinterpret_cast<Vec8*>(p) = v; }

__device__ __forceinline__ void unpack(const Vec8& v, float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(v.h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ Vec8 pack(const float (&f)[8]) {
  Vec8 v;
#pragma unroll
  for (int i = 0; i < 4; ++i) v.h[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return v;
}
__device__ __forceinline__ float bf16r(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

template <int TPR>
__device__ __forceinline__ float row_reduce_sum(float v, float* smem, int row_in_cta, int tid_in_row) {
  // TPR threads cooperate on one row; TPR is a power of two, <= 32 or a multiple of 32.
  if (TPR <= 32) {
#pragma unroll
    for (int o = TPR / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
  } else {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    constexpr int W = TPR / 32;
    int w = tid_in_row >> 5;
    __syncthreads();  // protect smem reuse across successive reductions
    if ((tid_in_row & 31) == 0) smem[row_in_cta * W + w] = v;
    __syncthreads();
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < W; ++i) t += smem[row_in_cta * W + i];
    return t;
  }
}

// ---------------------------------------------------------------------------------------------
// RMSNorm (+ fused residual add)
// ---------------------------------------------------------------------------------------------
template <int TPR, int VPT>
__global__ void __launch_bounds__(256, 3) rmsnorm_kernel(const __nv_bfloat16* __restrict__ x,
                                                         const __nv_bfloat16* __restrict__ res,
                                                         const __nv_bfloat16* __restrict__ w,
                                                         __nv_bfloat16* __restrict__ y,
                                                         __nv_bfloat16* __restrict__ sum_out, int64_t rows, int cols,
                                                         float eps) {
  constexpr int RPC = 256 / TPR;
  __shared__ float red[RPC * (TPR > 32 ? TPR / 32 : 1)];
  const int row_in_cta = threadIdx.x / TPR;
  const int t = threadIdx.x % TPR;
  const int64_t row = (int64_t)blockIdx.x * RPC + row_in_cta;
  const bool row_ok = row < rows;
  const int nvec = cols / 8;
  // the row stays in registers as packed bf16 (4 registers per 8 elements): all loads are issued
  // up front, occupancy stays high, and the second pass needs no re-read
  Vec8 raw[VPT];
  Vec8 rr[VPT];
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = t + i * TPR;
    if (row_ok && c < nvec) {
      raw[i] = ldg_stream(x + row * cols + c * 8);
      if (res != nullptr) rr[i] = ldg_stream(res + row * cols + c * 8);
    }
  }
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = t + i * TPR;
    if (row_ok && c < nvec) {
      float v[8];
      unpack(raw[i], v);
      if (res != nullptr) {
        float r[8];
        unpack(rr[i], r);
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = v[j] + r[j];
        raw[i] = pack(v);          // bf16(x + residual): the new residual stream
        unpack(raw[i], v);
        if (sum_out != nullptr) stg_vec(sum_out + row * cols + c * 8, raw[i]);
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) ss += v[j] * v[j];
    }
  }
  ss = row_reduce_sum<TPR>(ss, red, row_in_cta, t);
  const float rstd = rsqrtf(ss / (float)cols + eps);
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = t + i * TPR;
    if (row_ok && c < nvec) {
      float v[8], wv[8], o[8];
      unpack(raw[i], v);
      unpack(ldg_vec(w + c * 8), wv);
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = bf16r(v[j] * rstd) * wv[j];
      stg_vec(y + row * cols + c * 8, pack(o));
    }
  }
}

// ---------------------------------------------------------------------------------------------
// RMSNorm backward.  Forward: y = bf16(x * rstd) * w with rstd = rsqrt(mean(x^2) + eps) (the bf16 rounding is
// treated as the identity for the gradient, as autograd does through the reference's `.type_as(x)`).
//   g = dy * w;   dx = rstd * (g - xhat * mean(g * xhat)) [+ add_in];   dw[j] = sum_rows dy[j] * xhat[j]
// Each CTA walks rows with a grid stride and keeps its dw partial sums in registers; partial rows
// [gridDim * RPC, cols] (fp32) are summed by the caller - no atomics, bit-reproducible.
// ---------------------------------------------------------------------------------------------
template <int TPR, int VPT>
__global__ void __launch_bounds__(256) rmsnorm_bwd_kernel(const __nv_bfloat16* __restrict__ x,
                                                          const __nv_bfloat16* __restrict__ w,
                                                          const __nv_bfloat16* __restrict__ dy,
                                                          const __nv_bfloat16* __restrict__ add_in,
                                                          __nv_bfloat16* __restrict__ dx, float* __restrict__ dw_part,
                                                          int64_t rows, int cols, float eps) {
  constexpr int RPC = 256 / TPR;
  __shared__ float red[RPC * (TPR > 32 ? TPR / 32 : 1)];
  const int row_in_cta = threadIdx.x / TPR;
  const int t = threadIdx.x % TPR;
  const int nvec = cols / 8;
  float dw_acc[VPT][8];
#pragma unroll
  for (int i = 0; i < VPT; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) dw_acc[i][j] = 0.f;
  for (int64_t base = (int64_t)blockIdx.x * RPC; base < rows; base += (int64_t)gridDim.x * RPC) {
    const int64_t row = base + row_in_cta;
    const bool row_ok = row < rows;
    Vec8 xr[VPT], gr[VPT];
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = t + i * TPR;
      if (row_ok && c < nvec) {
        xr[i] = ldg_stream(x + row * cols + c * 8);
        gr[i] = ldg_stream(dy + row * cols + c * 8);
      }
    }
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = t + i * TPR;
      if (row_ok && c < nvec) {
        float v[8];
        unpack(xr[i], v);
#pragma unroll
        for (int j = 0; j < 8; ++j) ss += v[j] * v[j];
      }
    }
    ss = row_reduce_sum<TPR>(ss, red, row_in_cta, t);
    const float rstd = rsqrtf(ss / (float)cols + eps);
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = t + i * TPR;
      if (row_ok && c < nvec) {
        float v[8], g[8], wv[8];
        unpack(xr[i], v);
        unpack(gr[i], g);
        unpack(ldg_vec(w + c * 8), wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xh = v[j] * rstd;
          dot += g[j] * wv[j] * xh;
          dw_acc[i][j] += g[j] * xh;
        }
      }
    }
    dot = row_reduce_sum<TPR>(dot, red, row_in_cta, t) / (float)cols;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = t + i * TPR;
      if (row_ok && c < nvec) {
        float v[8], g[8], wv[8], o[8];
        unpack(xr[i], v);
        unpack(gr[i], g);
        unpack(ldg_vec(w + c * 8), wv);
        if (add_in != nullptr) {
          float a[8];
          unpack(ldg_stream(add_in + row * cols + c * 8), a);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = rstd * (g[j] * wv[j] - v[j] * rstd * dot) + a[j];
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] = rstd * (g[j] * wv[j] - v[j] * rstd * dot);
        }
        stg_vec(dx + row * cols + c * 8, pack(o));
      }
    }
  }
  float* part = dw_part + ((int64_t)blockIdx.x * RPC + row_in_cta) * cols;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = t + i * TPR;
    if (c < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) part[c * 8 + j] = dw_acc[i][j];
    }
  }
}

// ---------------------------------------------------------------------------------------------
// LayerNorm
// ---------------------------------------------------------------------------------------------
template <int TPR, int VPT>
__global__ void __launch_bounds__(256) layernorm_kernel(const __nv_bfloat16* __restrict__ x,
                                                        const __nv_bfloat16* __restrict__ w,
                                                        const __nv_bfloat16* __restrict__ b,
                                                        __nv_bfloat16* __restrict__ y, int64_t rows, int cols,
                                                        float eps) {
  constexpr int RPC = 256 / TPR;
  __shared__ float red[RPC * (TPR > 32 ? TPR / 32 : 1)];
  const int row_in_cta = threadIdx.x / TPR;
  const int t = threadIdx.x % TPR;
  const int64_t row = (int64_t)blockIdx.x * RPC + row_in_cta;
  const bool row_ok = row < rows;
  const int nvec = cols / 8;
  float v[VPT][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = t + i * TPR;
    if (row_ok && c < nvec) {
      unpack(ldg_stream(x + row * cols + c * 8), v[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += v[i][j];
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) v[i][j] = 0.f;
    }
  }
  s = row_reduce_sum<TPR>(s, red, row_in_cta, t);
  const float mean = s / (float)cols;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = t + i * TPR;
    if (row_ok && c < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float d = v[i][j] - mean;
        q += d * d;
      }
    }
  }
  q = row_reduce_sum<TPR>(q, red, row_in_cta, t);
  const float rstd = rsqrtf(q / (float)cols + eps);
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = t + i * TPR;
    if (row_ok && c < nvec) {
      float wv[8], bv[8], o[8];
      unpack(ldg_vec(w + c * 8), wv);
      if (b != nullptr) {
        unpack(ldg_vec(b + c * 8), bv);
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) bv[j] = 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = (v[i][j] - mean) * rstd * wv[j] + bv[j];
      stg_vec(y + row * cols + c * 8, pack(o));
    }
  }
}

// ---------------------------------------------------------------------------------------------
// RoPE
// ---------------------------------------------------------------------------------------------
__global__ void rope_table_kernel(const int64_t* __restrict__ pos, const float* __restrict__ inv_freq,
                                  __nv_bfloat16* __restrict__ cos_o, __nv_bfloat16* __restrict__ sin_o, int64_t n,
                                  int dim) {
  const int half = dim / 2;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n * half) return;
  const int64_t i = idx / half;
  const int j = (int)(idx % half);
  // torch.outer(seq, inv_freq) in fp32 (rotary_pos_embedding.py:100), then cos/sin in fp32 and a
  // cast to bf16 (:200-201).
  const float ang = (float)pos[i] * inv_freq[j];
  float sv, cv;
  sincosf(ang, &sv, &cv);
  const __nv_bfloat16 c = __float2bfloat16_rn(cv), s = __float2bfloat16_rn(sv);
  cos_o[i * dim + j] = c;
  cos_o[i * dim + half + j] = c;
  sin_o[i * dim + j] = s;
  sin_o[i * dim + half + j] = s;
}

// one thread: 8 elements of the first half and the matching 8 of the second half, for HPT heads of
// one token (cos / sin are loaded once and reused across those heads)
template <int HPT>
__global__ void __launch_bounds__(256) rope_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ out,
                                                   const __nv_bfloat16* __restrict__ cos_t,
                                                   const __nv_bfloat16* __restrict__ sin_t, int64_t n_tok, int heads,
                                                   int dim, int64_t xts, int64_t xhs, int64_t ots, int64_t ohs) {
  const int vph = dim / 16;  // vectors (of 8) per half
  const int hgroups = heads / HPT;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t total = n_tok * hgroups * vph;
  if (idx >= total) return;
  const int vi = (int)(idx % vph);
  const int hg = (int)((idx / vph) % hgroups);
  const int64_t tok = idx / ((int64_t)vph * hgroups);
  const int half = dim / 2;
  float c1[8], c2[8], s1[8], s2[8];
  unpack(ldg_vec(cos_t + tok * dim + vi * 8), c1);
  unpack(ldg_vec(cos_t + tok * dim + half + vi * 8), c2);
  unpack(ldg_vec(sin_t + tok * dim + vi * 8), s1);
  unpack(ldg_vec(sin_t + tok * dim + half + vi * 8), s2);
  Vec8 a[HPT], b[HPT];
#pragma unroll
  for (int h = 0; h < HPT; ++h) {
    const __nv_bfloat16* xp = x + tok * xts + (int64_t)(hg * HPT + h) * xhs + vi * 8;
    a[h] = ldg_vec(xp);
    b[h] = ldg_vec(xp + half);
  }
#pragma unroll
  for (int h = 0; h < HPT; ++h) {
    float x1[8], x2[8], o1[8], o2[8];
    unpack(a[h], x1);
    unpack(b[h], x2);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      // (t * cos) + (rotate_half(t) * sin), each product and the sum rounded to bf16
      o1[j] = bf16r(x1[j] * c1[j]) + bf16r(-x2[j] * s1[j]);
      o2[j] = bf16r(x2[j] * c2[j]) + bf16r(x1[j] * s2[j]);
    }
    __nv_bfloat16* op = out + tok * ots + (int64_t)(hg * HPT + h) * ohs + vi * 8;
    stg_vec(op, pack(o1));
    stg_vec(op + half, pack(o2));
  }
}

// ---------------------------------------------------------------------------------------------
// SwiGLU, bias+GELU, layer-scale residual
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) swiglu_kernel(const __nv_bfloat16* __restrict__ gu,
                                                     __nv_bfloat16* __restrict__ out, int64_t rows, int64_t inter) {
  const int64_t vpr = inter / 8;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * vpr) return;
  const int64_t r = idx / vpr, c = idx % vpr;
  float g[8], u[8], o[8];
  unpack(ldg_stream(gu + r * 2 * inter + c * 8), g);
  unpack(ldg_stream(gu + r * 2 * inter + inter + c * 8), u);
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = bf16r(__fdividef(g[j], 1.f + __expf(-g[j]))) * u[j];
  stg_vec(out + r * inter + c * 8, pack(o));
}

// d(gate|up) of h = silu(gate) * up:  dgate = dh * up * sig * (1 + gate * (1 - sig)),  dup = dh * silu(gate)
__global__ void __launch_bounds__(256) swiglu_bwd_kernel(const __nv_bfloat16* __restrict__ gu,
                                                         const __nv_bfloat16* __restrict__ dh,
                                                         __nv_bfloat16* __restrict__ dgu, int64_t rows, int64_t inter) {
  const int64_t vpr = inter / 8;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * vpr) return;
  const int64_t r = idx / vpr, c = idx % vpr;
  float g[8], u[8], d[8], og[8], ou[8];
  unpack(ldg_stream(gu + r * 2 * inter + c * 8), g);
  unpack(ldg_stream(gu + r * 2 * inter + inter + c * 8), u);
  unpack(ldg_stream(dh + r * inter + c * 8), d);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float sig = __fdividef(1.f, 1.f + __expf(-g[j]));
    og[j] = d[j] * u[j] * sig * (1.f + g[j] * (1.f - sig));
    ou[j] = d[j] * g[j] * sig;
  }
  stg_vec(dgu + r * 2 * inter + c * 8, pack(og));
  stg_vec(dgu + r * 2 * inter + inter + c * 8, pack(ou));
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float gelu_tanh(float x) {
  const float k = 0.7978845608028654f;
  return 0.5f * x * (1.f + tanhf(k * (x + 0.044715f * x * x * x)));
}

__global__ void __launch_bounds__(256) bias_gelu_kernel(const __nv_bfloat16* __restrict__ x,
                                                        const __nv_bfloat16* __restrict__ bias,
                                                        __nv_bfloat16* __restrict__ y, int64_t rows, int64_t cols,
                                                        int approx) {
  const int64_t vpr = cols / 8;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * vpr) return;
  const int64_t c = idx % vpr;
  float v[8], o[8];
  unpack(ldg_stream(x + idx * 8), v);
  if (bias != nullptr) {
    float b[8];
    unpack(ldg_vec(bias + c * 8), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = bf16r(v[j] + b[j]);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = approx ? gelu_tanh(v[j]) : gelu_erf(v[j]);
  stg_vec(y + idx * 8, pack(o));
}

__global__ void __launch_bounds__(256) ls_residual_kernel(const __nv_bfloat16* __restrict__ x,
                                                          const __nv_bfloat16* __restrict__ y,
                                                          const __nv_bfloat16* __restrict__ bias,
                                                          const __nv_bfloat16* __restrict__ ls,
                                                          __nv_bfloat16* __restrict__ out, int64_t rows,
                                                          int64_t cols) {
  const int64_t vpr = cols / 8;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * vpr) return;
  const int64_t c = idx % vpr;
  float xv[8], yv[8], o[8];
  unpack(ldg_stream(x + idx * 8), xv);
  unpack(ldg_stream(y + idx * 8), yv);
  if (bias != nullptr) {
    float b[8];
    unpack(ldg_vec(bias + c * 8), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) yv[j] = bf16r(yv[j] + b[j]);
  }
  if (ls != nullptr) {
    float l[8];
    unpack(ldg_vec(ls + c * 8), l);
#pragma unroll
    for (int j = 0; j < 8; ++j) yv[j] = bf16r(yv[j] * l[j]);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = xv[j] + yv[j];
  stg_vec(out + idx * 8, pack(o));
}

// ---------------------------------------------------------------------------------------------
// Pixel shuffle (x0.5): out[n, w2*(hw/2)+h2, wi*2c + hi*c + cc] = x[n, cls + (2*w2+wi)*hw + 2*h2+hi, cc]
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) pixel_shuffle_kernel(const __nv_bfloat16* __restrict__ x,
                                                            __nv_bfloat16* __restrict__ out, int64_t n, int hw, int c,
                                                            int has_cls) {
  const int h2n = hw / 2;
  const int64_t otok = blockIdx.x;  // n * h2n * h2n output tokens
  const int64_t img = otok / (h2n * h2n);
  const int rem = (int)(otok % (h2n * h2n));
  const int w2 = rem / h2n, h2 = rem % h2n;
  const int64_t in_tok_per_img = (int64_t)hw * hw + (has_cls ? 1 : 0);
  const int vpc = c / 8;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int wi = q >> 1, hi = q & 1;
    const int64_t itok = img * in_tok_per_img + (has_cls ? 1 : 0) + (int64_t)(2 * w2 + wi) * hw + (2 * h2 + hi);
    const __nv_bfloat16* src = x + itok * c;
    __nv_bfloat16* dst = out + otok * 4 * c + (int64_t)q * c;
    for (int v = threadIdx.x; v < vpc; v += blockDim.x) stg_vec(dst + v * 8, ldg_stream(src + v * 8));
  }
}

// ---------------------------------------------------------------------------------------------
// Row gather kernels (embedding lookup, feature scatter, masked select / scatter)
// ---------------------------------------------------------------------------------------------
// out[dst(i), :] = src[srcrow(i), :];  srcrow(i) = src_idx ? src_idx[i] : i;  dst(i) = dst_idx ? dst_idx[i] : i
__global__ void __launch_bounds__(128) row_copy_kernel(const __nv_bfloat16* __restrict__ src,
                                                       const int64_t* __restrict__ src_idx,
                                                       const int64_t* __restrict__ dst_idx,
                                                       __nv_bfloat16* __restrict__ out, int64_t n, int64_t cols,
                                                       int64_t src_rows, int64_t dst_rows) {
  const int64_t i = blockIdx.x;
  if (i >= n) return;
  const int64_t s = src_idx ? src_idx[i] : i;
  const int64_t d = dst_idx ? dst_idx[i] : i;
  if (s < 0 || s >= src_rows || d < 0 || d >= dst_rows) return;  // out-of-range indices are dropped
  const int64_t vpr = cols / 8;
  for (int64_t v = threadIdx.x; v < vpr; v += blockDim.x) stg_vec(out + d * cols + v * 8, ldg_vec(src + s * cols + v * 8));
}

static inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Flash-decoding merge: one block per query head, one thread per head-dim column; every thread walks the
// n_splits log-sum-exp values itself (n is ~18..150: cheaper than a block reduction).
__global__ void __launch_bounds__(128) decode_merge_kernel(const __nv_bfloat16* __restrict__ o_part,
                                                           const float* __restrict__ lse_part,
                                                           __nv_bfloat16* __restrict__ out, float* __restrict__ lse_out,
                                                           int n, int G, int hkv, int d) {
  const int kvh = blockIdx.x / G, g = blockIdx.x % G;
  const int c = threadIdx.x;
  float m = -INFINITY;
  for (int s = 0; s < n; ++s) m = fmaxf(m, lse_part[((long long)s * hkv + kvh) * G + g]);
  float sum = 0.f, acc = 0.f;
  if (m > -INFINITY) {
    for (int s = 0; s < n; ++s) {
      const float w = __expf(lse_part[((long long)s * hkv + kvh) * G + g] - m);
      sum += w;
      if (c < d) acc = fmaf(w, __bfloat162float(o_part[(((long long)s * G + g) * hkv + kvh) * d + c]), acc);
    }
  }
  if (c < d) out[((long long)kvh * G + g) * d + c] = __float2bfloat16_rn(sum > 0.f ? acc / sum : 0.f);
  if (c == 0 && lse_out != nullptr) lse_out[kvh * G + g] = sum > 0.f ? m + __logf(sum) : -INFINITY;
}


// ---------------------------------------------------------------------------------------------
// Cross-entropy over the vocabulary in chunks, fused with the logit-masked LM head
// (SURVEY.md 8f-3; gpt_vl_model.py:371-414 computes `compute_language_model_loss(labels, logits)` =
// vocab_parallel_cross_entropy(logits.float(), labels) on the full [M, vocab] logits).  The LM-head GEMM
// produces bf16 logits of ONE vocabulary chunk [M, Vc]; `ce_accumulate_kernel` folds the chunk into running
// per-row (max, sum-exp, target logit) in fp32 - the softmax statistics of the whole row without the row ever
// existing - and `ce_grad_kernel` turns a recomputed chunk into d_logits = (softmax - onehot) * d_loss for the
// backward GEMMs.  One CTA per row (grid-stride), two passes over the 2*Vc-byte row (the second from L1/L2).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_reduce(float v, float* red, bool is_max) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float t = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, t) : v + t;
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) r = is_max ? fmaxf(r, red[i]) : r + red[i];
  return r;
}

__global__ void __launch_bounds__(256) ce_accumulate_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld,
                                                            const int64_t* __restrict__ labels, float* __restrict__ run_max,
                                                            float* __restrict__ run_sum, float* __restrict__ tgt,
                                                            int64_t rows, int cols, int64_t col0) {
  __shared__ float red[8];
  const int nvec = cols / 8;
  for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
    const __nv_bfloat16* x = logits + row * ld;
    float mx = -INFINITY;
    for (int c = threadIdx.x; c < nvec; c += blockDim.x) {
      float v[8];
      unpack(ldg_vec(x + c * 8), v);
#pragma unroll
      for (int j = 0; j < 8; ++j) mx = fmaxf(mx, v[j]);
    }
    mx = block_reduce(mx, red, true);
    const float m_old = run_max[row];
    const float m_new = fmaxf(m_old, mx);
    float sum = 0.f;
    for (int c = threadIdx.x; c < nvec; c += blockDim.x) {
      float v[8];
      unpack(ldg_vec(x + c * 8), v);
#pragma unroll
      for (int j = 0; j < 8; ++j) sum += __expf(v[j] - m_new);
    }
    sum = block_reduce(sum, red, false);
    if (threadIdx.x == 0) {
      const float l_old = run_sum[row];
      run_sum[row] = (m_old == -INFINITY ? 0.f : l_old * __expf(m_old - m_new)) + sum;
      run_max[row] = m_new;
      const int64_t lab = labels[row] - col0;
      if (lab >= 0 && lab < cols) tgt[row] = __bfloat162float(x[lab]);
    }
  }
}

// d_logits[row, c] = bf16( (exp(logit - lse) - [c == label]) * d_loss[row] ); rows whose label is `ignore` (< 0) get zeros.
__global__ void __launch_bounds__(256) ce_grad_kernel(const __nv_bfloat16* __restrict__ logits, int64_t ld,
                                                      __nv_bfloat16* __restrict__ dlogits, int64_t ldd,
                                                      const int64_t* __restrict__ labels, const float* __restrict__ lse,
                                                      const float* __restrict__ dloss, int64_t rows, int cols, int64_t col0) {
  const int nvec = cols / 8;
  const int64_t total = rows * nvec;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / nvec;
    const int c = (int)(i - row * nvec);
    float v[8];
    unpack(ldg_stream(logits + row * ld + c * 8), v);
    const int64_t lab = labels[row];
    const float g = lab < 0 ? 0.f : dloss[row];
    const float l = lse[row];
    const int64_t hit = lab - col0 - (int64_t)c * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = (__expf(v[j] - l) - (hit == j ? 1.f : 0.f)) * g;
    stg_vec(dlogits + row * ldd + c * 8, pack(v));
  }
}

// ---------------------------------------------------------------------------------------------
// Backward of the vision-tower operators (training InternViT and the projector).
// ---------------------------------------------------------------------------------------------
// LayerNorm backward.  Forward (layernorm_kernel): y = (x - mean) * rstd * w + b with fp32 statistics of the bf16 row.
// The statistics are recomputed here the same way, then
//   xhat = (x - mean) * rstd;  g = dy * w;  dx = rstd * (g - mean(g) - xhat * mean(g * xhat)) [+ add_in]
//   dw[j] = sum_rows dy[j] * xhat[j];  db[j] = sum_rows dy[j]
// With dx == nullptr only dw / db are produced (the input of the norm needs no gradient).
// Grid-stride over rows with dw / db partial sums in registers, one partial row per (CTA, row slot), summed by the
// caller (no atomics, as rmsnorm_bwd_kernel).
template <int TPR, int VPT>
__global__ void __launch_bounds__(256) layernorm_bwd_kernel(const __nv_bfloat16* __restrict__ x,
                                                            const __nv_bfloat16* __restrict__ w,
                                                            const __nv_bfloat16* __restrict__ dy,
                                                            const __nv_bfloat16* __restrict__ add_in,
                                                            __nv_bfloat16* __restrict__ dx, float* __restrict__ dw_part,
                                                            float* __restrict__ db_part, int64_t rows, int cols, float eps) {
  constexpr int RPC = 256 / TPR;
  __shared__ float red[RPC * (TPR > 32 ? TPR / 32 : 1)];
  const int row_in_cta = threadIdx.x / TPR;
  const int t = threadIdx.x % TPR;
  const int nvec = cols / 8;
  float dw_acc[VPT][8], db_acc[VPT][8];
#pragma unroll
  for (int i = 0; i < VPT; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) dw_acc[i][j] = db_acc[i][j] = 0.f;
  for (int64_t base = (int64_t)blockIdx.x * RPC; base < rows; base += (int64_t)gridDim.x * RPC) {
    const int64_t row = base + row_in_cta;
    const bool row_ok = row < rows;
    Vec8 xr[VPT], gr[VPT];
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = t + i * TPR;
      if (row_ok && c < nvec) {
        xr[i] = ldg_stream(x + row * cols + c * 8);
        gr[i] = ldg_stream(dy + row * cols + c * 8);
      }
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = t + i * TPR;
      if (row_ok && c < nvec) {
        float v[8];
        unpack(xr[i], v);
#pragma unroll
        for (int j = 0; j < 8; ++j) s += v[j];
      }
    }
    const float mean = row_reduce_sum<TPR>(s, red, row_in_cta, t) / (float)cols;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = t + i * TPR;
      if (row_ok && c < nvec) {
        float v[8];
        unpack(xr[i], v);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = v[j] - mean;
          q += d * d;
        }
      }
    }
    const float rstd = rsqrtf(row_reduce_sum<TPR>(q, red, row_in_cta, t) / (float)cols + eps);
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = t + i * TPR;
      if (row_ok && c < nvec) {
        float v[8], g[8], wv[8];
        unpack(xr[i], v);
        unpack(gr[i], g);
        unpack(ldg_vec(w + c * 8), wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xh = (v[j] - mean) * rstd;
          const float gw = g[j] * wv[j];
          sg += gw;
          sgx += gw * xh;
          dw_acc[i][j] += g[j] * xh;
          db_acc[i][j] += g[j];
        }
      }
    }
    if (dx == nullptr) continue;  // uniform across the CTA: the reductions below stay collective
    const float mg = row_reduce_sum<TPR>(sg, red, row_in_cta, t) / (float)cols;
    const float mgx = row_reduce_sum<TPR>(sgx, red, row_in_cta, t) / (float)cols;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
      const int c = t + i * TPR;
      if (row_ok && c < nvec) {
        float v[8], g[8], wv[8], o[8];
        unpack(xr[i], v);
        unpack(gr[i], g);
        unpack(ldg_vec(w + c * 8), wv);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = rstd * (g[j] * wv[j] - mg - (v[j] - mean) * rstd * mgx);
        if (add_in != nullptr) {
          float a[8];
          unpack(ldg_stream(add_in + row * cols + c * 8), a);
#pragma unroll
          for (int j = 0; j < 8; ++j) o[j] += a[j];
        }
        stg_vec(dx + row * cols + c * 8, pack(o));
      }
    }
  }
  const int64_t prow = (int64_t)blockIdx.x * RPC + row_in_cta;
#pragma unroll
  for (int i = 0; i < VPT; ++i) {
    const int c = t + i * TPR;
    if (c < nvec) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        dw_part[prow * cols + c * 8 + j] = dw_acc[i][j];
        db_part[prow * cols + c * 8 + j] = db_acc[i][j];
      }
    }
  }
}

// GELU backward: dx = dy * gelu'(pre), pre = the bf16 pre-activation (fc1 output with its bias).
//   erf:  gelu'(x) = Phi(x) + x * phi(x)
//   tanh: u = k (x + 0.044715 x^3), gelu'(x) = 0.5 (1 + tanh u) + 0.5 x (1 - tanh^2 u) k (1 + 3 * 0.044715 x^2)
__device__ __forceinline__ float gelu_erf_grad(float x) {
  return 0.5f * (1.f + erff(x * 0.70710678118654752440f)) + x * 0.3989422804014327f * __expf(-0.5f * x * x);
}
__device__ __forceinline__ float gelu_tanh_grad(float x) {
  const float k = 0.7978845608028654f;
  const float th = tanhf(k * (x + 0.044715f * x * x * x));
  return 0.5f * (1.f + th) + 0.5f * x * (1.f - th * th) * k * (1.f + 3.f * 0.044715f * x * x);
}

__global__ void __launch_bounds__(256) gelu_bwd_kernel(const __nv_bfloat16* __restrict__ pre,
                                                       const __nv_bfloat16* __restrict__ dy,
                                                       __nv_bfloat16* __restrict__ dx, int64_t total_vec, int approx) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total_vec) return;
  float v[8], g[8], o[8];
  unpack(ldg_stream(pre + idx * 8), v);
  unpack(ldg_stream(dy + idx * 8), g);
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = g[j] * (approx ? gelu_tanh_grad(v[j]) : gelu_erf_grad(v[j]));
  stg_vec(dx + idx * 8, pack(o));
}

// Layer-scale residual backward (out = x + y * ls, bias-free): dy = bf16(dout * ls), dls[j] = sum_rows dout[j] * y[j].
// A CTA covers 32 column vectors (256 columns) x LSB_ROWS row lanes; blockIdx.y strides over the rows.  The 8 row lanes
// are folded through shared memory in a fixed order, so CTA row blockIdx.y writes partial row blockIdx.y of
// dls_partials [gridDim.y, cols] (summed by the caller: deterministic).
constexpr int LSB_ROWS = 8;

__global__ void __launch_bounds__(256) ls_residual_bwd_kernel(const __nv_bfloat16* __restrict__ dout,
                                                              const __nv_bfloat16* __restrict__ y,
                                                              const __nv_bfloat16* __restrict__ ls,
                                                              __nv_bfloat16* __restrict__ dy, float* __restrict__ dls_part,
                                                              int64_t rows, int cols) {
  __shared__ float red[LSB_ROWS][32 * 8 + 1];
  const int nvec = cols / 8;
  const int lane = threadIdx.x % 32, rl = threadIdx.x / 32;
  const int c = blockIdx.x * 32 + lane;
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
  if (c < nvec) {
    float l[8];
    unpack(ldg_vec(ls + c * 8), l);
    for (int64_t r = (int64_t)blockIdx.y * LSB_ROWS + rl; r < rows; r += (int64_t)gridDim.y * LSB_ROWS) {
      float d[8], yv[8], o[8];
      unpack(ldg_stream(dout + r * cols + c * 8), d);
      unpack(ldg_stream(y + r * cols + c * 8), yv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[j] = d[j] * l[j];
        acc[j] += d[j] * yv[j];
      }
      stg_vec(dy + r * cols + c * 8, pack(o));
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[rl][lane * 8 + j] = acc[j];
  __syncthreads();
  // 256 threads, 256 columns of this CTA: thread k sums column k over the row lanes
  const int k = threadIdx.x;
  const int col = blockIdx.x * 256 + k;
  if (col < cols) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < LSB_ROWS; ++i) s += red[i][k];
    dls_part[(int64_t)blockIdx.y * cols + col] = s;
  }
}

// Pixel-shuffle backward: the inverse permutation of pixel_shuffle_kernel.  Blocks [0, n (hw/2)^2) move one output
// token's four c-wide segments back to their input rows; with has_cls, the n blocks after them zero the class-token rows.
__global__ void __launch_bounds__(128) pixel_shuffle_bwd_kernel(const __nv_bfloat16* __restrict__ dout,
                                                                __nv_bfloat16* __restrict__ dx, int64_t n, int hw, int c,
                                                                int has_cls) {
  const int h2n = hw / 2;
  const int64_t in_tok_per_img = (int64_t)hw * hw + (has_cls ? 1 : 0);
  const int vpc = c / 8;
  const int64_t otoks = n * h2n * h2n;
  const int64_t b = blockIdx.x;
  if (b >= otoks) {  // class-token row of image b - otoks
    Vec8 z;
#pragma unroll
    for (int i = 0; i < 4; ++i) z.h[i] = __floats2bfloat162_rn(0.f, 0.f);
    __nv_bfloat16* dst = dx + (b - otoks) * in_tok_per_img * c;
    for (int v = threadIdx.x; v < vpc; v += blockDim.x) stg_vec(dst + v * 8, z);
    return;
  }
  const int64_t img = b / (h2n * h2n);
  const int rem = (int)(b % (h2n * h2n));
  const int w2 = rem / h2n, h2 = rem % h2n;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int wi = q >> 1, hi = q & 1;
    const int64_t itok = img * in_tok_per_img + (has_cls ? 1 : 0) + (int64_t)(2 * w2 + wi) * hw + (2 * h2 + hi);
    const __nv_bfloat16* src = dout + b * 4 * c + (int64_t)q * c;
    __nv_bfloat16* dst = dx + itok * c;
    for (int v = threadIdx.x; v < vpc; v += blockDim.x) stg_vec(dst + v * 8, ldg_stream(src + v * 8));
  }
}

}  // namespace lv

using namespace lv;

#define BF(p) reinterpret_cast<const __nv_bfloat16*>(p)
#define BFM(p) reinterpret_cast<__nv_bfloat16*>(p)

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Row tiling of the norm kernels: TPR threads share a row (256 / TPR rows per CTA) and each holds VPT 16-byte vectors
// of it.  A row of `cols` takes the first entry with cols / 8 <= max_nvec; the last entry takes every wider row.
struct RowTiling {
  int64_t max_nvec;
  int tpr, vpt;
};
constexpr RowTiling NORM_TILING[] = {{32 * 4, 32, 4}, {128 * 4, 128, 4}, {128 * 5, 128, 5}, {INT64_MAX, 256, 8}};
constexpr RowTiling LN_BWD_TILING[] = {{32 * 4, 32, 4}, {128 * 4, 128, 4}, {INT64_MAX, 256, 4}};

// Calls launch(TPR, VPT), both std::integral_constant<int>, with the entry of TABLE that a row of `cols` takes.
template <const auto& TABLE, size_t I = 0, class F>
static void with_tiling(int64_t cols, F&& launch) {
  if constexpr (I + 1 < std::size(TABLE)) {
    if (cols / 8 > TABLE[I].max_nvec) return with_tiling<TABLE, I + 1>(cols, launch);
  }
  launch(std::integral_constant<int, TABLE[I].tpr>{}, std::integral_constant<int, TABLE[I].vpt>{});
}

// Rows of each fp32 partial buffer a norm backward writes: one per row slot of every CTA, ~2 CTAs per SM.
template <const auto& TABLE>
static int64_t bwd_partials(int64_t rows, int64_t cols) {
  int64_t rpc = 0;
  with_tiling<TABLE>(cols, [&](auto TPR, auto) { rpc = 256 / TPR; });
  int64_t grid = (rows + rpc - 1) / rpc;
  const int64_t cap = 2 * (int64_t)lv::sm_count();
  if (grid > cap) grid = cap;
  if (grid < 1) grid = 1;
  return grid * rpc;
}

extern "C" {

int lv_rmsnorm(const void* x, const void* residual, const void* w, void* y, void* sum_out, int64_t rows,
               int64_t cols, float eps, lv_stream_t stream) {
  LV_CHECK_ARG(w && (rows == 0 || (x && y)), "lv_rmsnorm: null pointer");  // an empty tensor may have no storage
  LV_CHECK_ARG(rows >= 0 && cols > 0 && cols % 8 == 0 && cols <= 16384, "lv_rmsnorm: cols=%lld must be a multiple of 8 and <= 16384", (long long)cols);
  LV_CHECK_ARG(aligned16(x) && aligned16(w) && aligned16(y) && aligned16(residual) && aligned16(sum_out), "lv_rmsnorm: pointers must be 16-byte aligned");
  if (rows == 0) return LV_OK;
  cudaStream_t s = (cudaStream_t)stream;
  with_tiling<NORM_TILING>(cols, [&](auto TPR, auto VPT) {
    rmsnorm_kernel<TPR, VPT><<<(unsigned)cdiv(rows, 256 / TPR), 256, 0, s>>>(BF(x), BF(residual), BF(w), BFM(y),
                                                                             BFM(sum_out), rows, (int)cols, eps);
  });
  LV_CHECK_LAUNCH("rmsnorm_kernel");
  return LV_OK;
}

int lv_layernorm(const void* x, const void* w, const void* b, void* y, int64_t rows, int64_t cols, float eps,
                 lv_stream_t stream) {
  LV_CHECK_ARG(w && (rows == 0 || (x && y)), "lv_layernorm: null pointer");
  LV_CHECK_ARG(rows >= 0 && cols > 0 && cols % 8 == 0 && cols <= 16384, "lv_layernorm: cols=%lld must be a multiple of 8 and <= 16384", (long long)cols);
  LV_CHECK_ARG(aligned16(x) && aligned16(w) && aligned16(y) && aligned16(b), "lv_layernorm: pointers must be 16-byte aligned");
  if (rows == 0) return LV_OK;
  cudaStream_t s = (cudaStream_t)stream;
  with_tiling<NORM_TILING>(cols, [&](auto TPR, auto VPT) {
    layernorm_kernel<TPR, VPT><<<(unsigned)cdiv(rows, 256 / TPR), 256, 0, s>>>(BF(x), BF(w), BF(b), BFM(y), rows, (int)cols, eps);
  });
  LV_CHECK_LAUNCH("layernorm_kernel");
  return LV_OK;
}

int lv_rope_table(const int64_t* pos, const float* inv_freq, void* cos_out, void* sin_out, int64_t n, int64_t dim,
                  lv_stream_t stream) {
  LV_CHECK_ARG(inv_freq && (n == 0 || (pos && cos_out && sin_out)), "lv_rope_table: null pointer");
  LV_CHECK_ARG(n >= 0 && dim > 0 && dim % 2 == 0, "lv_rope_table: bad dim %lld", (long long)dim);
  if (n == 0) return LV_OK;
  const int64_t total = n * (dim / 2);
  rope_table_kernel<<<(unsigned)cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(pos, inv_freq, BFM(cos_out),
                                                                                 BFM(sin_out), n, (int)dim);
  LV_CHECK_LAUNCH("rope_table_kernel");
  return LV_OK;
}

int lv_rope(const void* x, void* out, const void* cos_t, const void* sin_t, int64_t n_tok, int64_t heads, int64_t dim,
            int64_t x_tok_stride, int64_t x_head_stride, int64_t o_tok_stride, int64_t o_head_stride,
            lv_stream_t stream) {
  LV_CHECK_ARG(n_tok == 0 || heads == 0 || (x && out && cos_t && sin_t), "lv_rope: null pointer");
  LV_CHECK_ARG(dim > 0 && dim % 16 == 0, "lv_rope: dim=%lld must be a multiple of 16", (long long)dim);
  LV_CHECK_ARG(x_tok_stride % 8 == 0 && x_head_stride % 8 == 0 && o_tok_stride % 8 == 0 && o_head_stride % 8 == 0,
               "lv_rope: strides must be multiples of 8 elements");
  LV_CHECK_ARG(aligned16(x) && aligned16(out) && aligned16(cos_t) && aligned16(sin_t), "lv_rope: pointers must be 16-byte aligned");
  if (n_tok == 0 || heads == 0) return LV_OK;
#define LAUNCH_ROPE(HPT)                                                                                         \
  rope_kernel<HPT><<<(unsigned)cdiv(n_tok * (heads / HPT) * (dim / 16), 256), 256, 0, (cudaStream_t)stream>>>(        \
      BF(x), BFM(out), BF(cos_t), BF(sin_t), n_tok, (int)heads, (int)dim, x_tok_stride, x_head_stride, o_tok_stride, \
      o_head_stride)
  if (heads % 8 == 0)
    LAUNCH_ROPE(8);
  else if (heads % 5 == 0)
    LAUNCH_ROPE(5);
  else if (heads % 2 == 0)
    LAUNCH_ROPE(2);
  else
    LAUNCH_ROPE(1);
#undef LAUNCH_ROPE
  LV_CHECK_LAUNCH("rope_kernel");
  return LV_OK;
}

int lv_swiglu(const void* gate_up, void* out, int64_t rows, int64_t inter, lv_stream_t stream) {
  LV_CHECK_ARG(rows == 0 || (gate_up && out), "lv_swiglu: null pointer");
  LV_CHECK_ARG(inter > 0 && inter % 8 == 0, "lv_swiglu: inter=%lld must be a multiple of 8", (long long)inter);
  LV_CHECK_ARG(aligned16(gate_up) && aligned16(out), "lv_swiglu: pointers must be 16-byte aligned");
  if (rows == 0) return LV_OK;
  const int64_t total = rows * (inter / 8);
  swiglu_kernel<<<(unsigned)cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(BF(gate_up), BFM(out), rows, inter);
  LV_CHECK_LAUNCH("swiglu_kernel");
  return LV_OK;
}

int lv_bias_gelu(const void* x, const void* bias, void* y, int64_t rows, int64_t cols, int32_t approx,
                 lv_stream_t stream) {
  LV_CHECK_ARG(rows == 0 || (x && y), "lv_bias_gelu: null pointer");
  LV_CHECK_ARG(cols > 0 && cols % 8 == 0, "lv_bias_gelu: cols=%lld must be a multiple of 8", (long long)cols);
  LV_CHECK_ARG(aligned16(x) && aligned16(y) && aligned16(bias), "lv_bias_gelu: pointers must be 16-byte aligned");
  if (rows == 0) return LV_OK;
  const int64_t total = rows * (cols / 8);
  bias_gelu_kernel<<<(unsigned)cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(BF(x), BF(bias), BFM(y), rows, cols,
                                                                                approx);
  LV_CHECK_LAUNCH("bias_gelu_kernel");
  return LV_OK;
}

int lv_ls_residual(const void* x, const void* y, const void* bias, const void* ls, void* out, int64_t rows,
                   int64_t cols, lv_stream_t stream) {
  LV_CHECK_ARG(rows == 0 || (x && y && out), "lv_ls_residual: null pointer");
  LV_CHECK_ARG(cols > 0 && cols % 8 == 0, "lv_ls_residual: cols=%lld must be a multiple of 8", (long long)cols);
  LV_CHECK_ARG(aligned16(x) && aligned16(y) && aligned16(out) && aligned16(bias) && aligned16(ls), "lv_ls_residual: pointers must be 16-byte aligned");
  if (rows == 0) return LV_OK;
  const int64_t total = rows * (cols / 8);
  ls_residual_kernel<<<(unsigned)cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(BF(x), BF(y), BF(bias), BF(ls),
                                                                                  BFM(out), rows, cols);
  LV_CHECK_LAUNCH("ls_residual_kernel");
  return LV_OK;
}

int lv_pixel_shuffle(const void* x, void* out, int64_t n, int64_t hw, int64_t c, int32_t has_cls, lv_stream_t stream) {
  LV_CHECK_ARG(x && out, "lv_pixel_shuffle: null pointer");
  LV_CHECK_ARG(hw > 0 && hw % 2 == 0 && c > 0 && c % 8 == 0, "lv_pixel_shuffle: hw=%lld must be even, c=%lld a multiple of 8", (long long)hw, (long long)c);
  LV_CHECK_ARG(aligned16(x) && aligned16(out), "lv_pixel_shuffle: pointers must be 16-byte aligned");
  if (n == 0) return LV_OK;
  const int64_t otoks = n * (hw / 2) * (hw / 2);
  LV_CHECK_ARG(otoks < (1ll << 31), "lv_pixel_shuffle: too many tokens");
  pixel_shuffle_kernel<<<(unsigned)otoks, 128, 0, (cudaStream_t)stream>>>(BF(x), BFM(out), n, (int)hw, (int)c, has_cls);
  LV_CHECK_LAUNCH("pixel_shuffle_kernel");
  return LV_OK;
}

int lv_embed_scatter(const int64_t* ids, const void* table, int64_t vocab, const void* feat, const int64_t* src_idx,
                     const int64_t* dst_idx, int64_t n_scatter, void* out, int64_t n_tok, int64_t hidden,
                     lv_stream_t stream) {
  LV_CHECK_ARG(ids && table && out, "lv_embed_scatter: null pointer");
  LV_CHECK_ARG(hidden > 0 && hidden % 8 == 0, "lv_embed_scatter: hidden=%lld must be a multiple of 8", (long long)hidden);
  LV_CHECK_ARG(n_scatter == 0 || (feat && dst_idx), "lv_embed_scatter: feat/dst_idx required when n_scatter > 0");
  LV_CHECK_ARG(aligned16(table) && aligned16(out) && aligned16(feat), "lv_embed_scatter: pointers must be 16-byte aligned");
  LV_CHECK_ARG(n_tok < (1ll << 31) && n_scatter < (1ll << 31), "lv_embed_scatter: too many rows");
  cudaStream_t s = (cudaStream_t)stream;
  if (n_tok > 0) {
    row_copy_kernel<<<(unsigned)n_tok, 128, 0, s>>>(BF(table), ids, nullptr, BFM(out), n_tok, hidden, vocab, n_tok);
    LV_CHECK_LAUNCH("row_copy_kernel(embed)");
  }
  if (n_scatter > 0) {
    row_copy_kernel<<<(unsigned)n_scatter, 128, 0, s>>>(BF(feat), src_idx, dst_idx, BFM(out), n_scatter, hidden,
                                                       (int64_t)1 << 62, n_tok);
    LV_CHECK_LAUNCH("row_copy_kernel(scatter)");
  }
  return LV_OK;
}

int lv_row_gather(const void* x, const int64_t* idx, void* out, int64_t n_idx, int64_t cols, lv_stream_t stream) {
  if (n_idx == 0) return LV_OK;
  LV_CHECK_ARG(x && idx && out, "lv_row_gather: null pointer");
  LV_CHECK_ARG(cols > 0 && cols % 8 == 0, "lv_row_gather: cols=%lld must be a multiple of 8", (long long)cols);
  LV_CHECK_ARG(aligned16(x) && aligned16(out), "lv_row_gather: pointers must be 16-byte aligned");
  LV_CHECK_ARG(n_idx < (1ll << 31), "lv_row_gather: too many rows");
  if (n_idx == 0) return LV_OK;
  row_copy_kernel<<<(unsigned)n_idx, 128, 0, (cudaStream_t)stream>>>(BF(x), idx, nullptr, BFM(out), n_idx, cols,
                                                                    (int64_t)1 << 62, n_idx);
  LV_CHECK_LAUNCH("row_copy_kernel(gather)");
  return LV_OK;
}

int lv_row_scatter_zero(const void* x, const int64_t* idx, void* out, int64_t n_idx, int64_t n_rows_out, int64_t cols,
                        lv_stream_t stream) {
  LV_CHECK_ARG(out && (n_idx == 0 || (x && idx)), "lv_row_scatter_zero: null pointer");
  LV_CHECK_ARG(cols > 0 && cols % 8 == 0, "lv_row_scatter_zero: cols=%lld must be a multiple of 8", (long long)cols);
  LV_CHECK_ARG(aligned16(x) && aligned16(out), "lv_row_scatter_zero: pointers must be 16-byte aligned");
  LV_CHECK_ARG(n_idx < (1ll << 31), "lv_row_scatter_zero: too many rows");
  cudaStream_t s = (cudaStream_t)stream;
  LV_CHECK_CUDA(cudaMemsetAsync(out, 0, (size_t)n_rows_out * cols * 2, s));
  if (n_idx == 0) return LV_OK;
  row_copy_kernel<<<(unsigned)n_idx, 128, 0, s>>>(BF(x), nullptr, idx, BFM(out), n_idx, cols, n_idx, n_rows_out);
  LV_CHECK_LAUNCH("row_copy_kernel(scatter_zero)");
  return LV_OK;
}

int lv_row_scatter(const void* x, const int64_t* idx, void* out, int64_t n_idx, int64_t n_rows_out, int64_t cols,
                   lv_stream_t stream) {
  LV_CHECK_ARG(n_idx == 0 || (x && idx && out), "lv_row_scatter: null pointer");
  LV_CHECK_ARG(cols > 0 && cols % 8 == 0, "lv_row_scatter: cols=%lld must be a multiple of 8", (long long)cols);
  LV_CHECK_ARG(aligned16(x) && aligned16(out), "lv_row_scatter: pointers must be 16-byte aligned");
  LV_CHECK_ARG(n_idx < (1ll << 31), "lv_row_scatter: too many rows");
  if (n_idx == 0) return LV_OK;
  row_copy_kernel<<<(unsigned)n_idx, 128, 0, (cudaStream_t)stream>>>(BF(x), nullptr, idx, BFM(out), n_idx, cols, n_idx,
                                                                    n_rows_out);
  LV_CHECK_LAUNCH("row_copy_kernel(scatter)");
  return LV_OK;
}

int lv_attn_decode_merge(const void* o_part, const float* lse_part, void* out, float* lse_out, int64_t n_splits,
                         int64_t group, int64_t hkv, int64_t d, lv_stream_t stream) {
  LV_CHECK_ARG(o_part && lse_part && out, "lv_attn_decode_merge: null pointer");
  LV_CHECK_ARG(n_splits > 0 && group > 0 && hkv > 0 && d > 0 && d <= 128, "lv_attn_decode_merge: bad shape");
  LV_CHECK_ARG(n_splits < (1ll << 20) && group * hkv < (1ll << 20), "lv_attn_decode_merge: too large");
  LV_BIND_DEVICE(o_part);
  decode_merge_kernel<<<(unsigned)(group * hkv), 128, 0, (cudaStream_t)stream>>>(BF(o_part), lse_part, BFM(out), lse_out,
                                                                            (int)n_splits, (int)group, (int)hkv, (int)d);
  LV_CHECK_LAUNCH("decode_merge_kernel");
  return LV_OK;
}

int64_t lv_rmsnorm_bwd_partials(int64_t rows, int64_t cols) { return bwd_partials<NORM_TILING>(rows, cols); }

int lv_rmsnorm_bwd(const void* x, const void* w, const void* dy, const void* add_in, void* dx, float* dw_partials,
                   int64_t rows, int64_t cols, float eps, lv_stream_t stream) {
  LV_CHECK_ARG(w && dw_partials && (rows == 0 || (x && dy && dx)), "lv_rmsnorm_bwd: null pointer");
  LV_CHECK_ARG(rows >= 0 && cols > 0 && cols % 8 == 0 && cols <= 16384, "lv_rmsnorm_bwd: cols=%lld must be a multiple of 8 and <= 16384", (long long)cols);
  LV_CHECK_ARG(aligned16(x) && aligned16(w) && aligned16(dy) && aligned16(dx) && aligned16(add_in), "lv_rmsnorm_bwd: pointers must be 16-byte aligned");
  LV_BIND_DEVICE(dw_partials);  // the partial buffer exists (and is zeroed) even with zero rows
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t parts = lv_rmsnorm_bwd_partials(rows, cols);
  if (rows == 0) {
    LV_CHECK_CUDA(cudaMemsetAsync(dw_partials, 0, (size_t)parts * cols * 4, s));
    return LV_OK;
  }
  with_tiling<NORM_TILING>(cols, [&](auto TPR, auto VPT) {
    rmsnorm_bwd_kernel<TPR, VPT><<<(unsigned)(parts / (256 / TPR)), 256, 0, s>>>(BF(x), BF(w), BF(dy), BF(add_in), BFM(dx),
                                                                                  dw_partials, rows, (int)cols, eps);
  });
  LV_CHECK_LAUNCH("rmsnorm_bwd_kernel");
  return LV_OK;
}

int lv_swiglu_bwd(const void* gate_up, const void* dh, void* d_gate_up, int64_t rows, int64_t inter, lv_stream_t stream) {
  LV_CHECK_ARG(rows == 0 || (gate_up && dh && d_gate_up), "lv_swiglu_bwd: null pointer");
  LV_CHECK_ARG(inter > 0 && inter % 8 == 0, "lv_swiglu_bwd: inter=%lld must be a multiple of 8", (long long)inter);
  LV_CHECK_ARG(aligned16(gate_up) && aligned16(dh) && aligned16(d_gate_up), "lv_swiglu_bwd: pointers must be 16-byte aligned");
  if (rows == 0) return LV_OK;
  LV_BIND_DEVICE(gate_up);
  const int64_t total = rows * (inter / 8);
  swiglu_bwd_kernel<<<(unsigned)cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(BF(gate_up), BF(dh), BFM(d_gate_up), rows, inter);
  LV_CHECK_LAUNCH("swiglu_bwd_kernel");
  return LV_OK;
}

int lv_ce_accumulate(const void* logits, int64_t ld, const int64_t* labels, float* run_max, float* run_sum, float* tgt,
                     int64_t rows, int64_t cols, int64_t col0, lv_stream_t stream) {
  LV_CHECK_ARG(logits && labels && run_max && run_sum && tgt, "lv_ce_accumulate: null pointer");
  LV_CHECK_ARG(cols > 0 && cols % 8 == 0 && ld % 8 == 0 && ld >= cols && cols < (1ll << 31), "lv_ce_accumulate: cols=%lld / ld=%lld must be multiples of 8", (long long)cols, (long long)ld);
  LV_CHECK_ARG(aligned16(logits), "lv_ce_accumulate: logits must be 16-byte aligned");
  if (rows == 0) return LV_OK;
  LV_BIND_DEVICE(logits);
  const int64_t cap = 8 * (int64_t)lv::sm_count();
  ce_accumulate_kernel<<<(unsigned)(rows < cap ? rows : cap), 256, 0, (cudaStream_t)stream>>>(BF(logits), ld, labels, run_max, run_sum, tgt,
                                                                                              rows, (int)cols, col0);
  LV_CHECK_LAUNCH("ce_accumulate_kernel");
  return LV_OK;
}

int lv_ce_grad(const void* logits, int64_t ld, void* dlogits, int64_t ldd, const int64_t* labels, const float* lse,
               const float* dloss, int64_t rows, int64_t cols, int64_t col0, lv_stream_t stream) {
  LV_CHECK_ARG(logits && dlogits && labels && lse && dloss, "lv_ce_grad: null pointer");
  LV_CHECK_ARG(cols > 0 && cols % 8 == 0 && ld % 8 == 0 && ldd % 8 == 0 && ld >= cols && ldd >= cols && cols < (1ll << 31),
               "lv_ce_grad: cols=%lld / ld=%lld / ldd=%lld must be multiples of 8", (long long)cols, (long long)ld, (long long)ldd);
  LV_CHECK_ARG(aligned16(logits) && aligned16(dlogits), "lv_ce_grad: pointers must be 16-byte aligned");
  if (rows == 0) return LV_OK;
  LV_BIND_DEVICE(logits);
  const int64_t total = rows * (cols / 8);
  const int64_t cap = 16 * (int64_t)lv::sm_count();
  const int64_t blocks = cdiv(total, 256);
  ce_grad_kernel<<<(unsigned)(blocks < cap ? blocks : cap), 256, 0, (cudaStream_t)stream>>>(BF(logits), ld, BFM(dlogits), ldd, labels, lse,
                                                                                            dloss, rows, (int)cols, col0);
  LV_CHECK_LAUNCH("ce_grad_kernel");
  return LV_OK;
}

int64_t lv_layernorm_bwd_partials(int64_t rows, int64_t cols) { return bwd_partials<LN_BWD_TILING>(rows, cols); }

int lv_layernorm_bwd(const void* x, const void* w, const void* dy, const void* add_in, void* dx, float* dw_partials,
                     float* db_partials, int64_t rows, int64_t cols, float eps, lv_stream_t stream) {
  LV_CHECK_ARG(w && dw_partials && db_partials && (rows == 0 || (x && dy)), "lv_layernorm_bwd: null pointer");
  LV_CHECK_ARG(dx != nullptr || add_in == nullptr, "lv_layernorm_bwd: add_in needs dx");
  LV_CHECK_ARG(rows >= 0 && cols > 0 && cols % 8 == 0 && cols <= 8192, "lv_layernorm_bwd: cols=%lld must be a multiple of 8 and <= 8192", (long long)cols);
  LV_CHECK_ARG(aligned16(x) && aligned16(w) && aligned16(dy) && aligned16(dx) && aligned16(add_in) && aligned16(dw_partials) &&
                   aligned16(db_partials), "lv_layernorm_bwd: pointers must be 16-byte aligned");
  LV_BIND_DEVICE(dw_partials);  // the partial buffer exists (and is zeroed) even with zero rows
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t parts = lv_layernorm_bwd_partials(rows, cols);
  if (rows == 0) {
    LV_CHECK_CUDA(cudaMemsetAsync(dw_partials, 0, (size_t)parts * cols * 4, s));
    LV_CHECK_CUDA(cudaMemsetAsync(db_partials, 0, (size_t)parts * cols * 4, s));
    return LV_OK;
  }
  with_tiling<LN_BWD_TILING>(cols, [&](auto TPR, auto VPT) {
    layernorm_bwd_kernel<TPR, VPT><<<(unsigned)(parts / (256 / TPR)), 256, 0, s>>>(
        BF(x), BF(w), BF(dy), BF(add_in), BFM(dx), dw_partials, db_partials, rows, (int)cols, eps);
  });
  LV_CHECK_LAUNCH("layernorm_bwd_kernel");
  return LV_OK;
}

int lv_gelu_bwd(const void* pre, const void* dy, void* dx, int64_t rows, int64_t cols, int32_t approx, lv_stream_t stream) {
  LV_CHECK_ARG(rows == 0 || (pre && dy && dx), "lv_gelu_bwd: null pointer");
  LV_CHECK_ARG(rows >= 0 && cols > 0 && cols % 8 == 0, "lv_gelu_bwd: cols=%lld must be a multiple of 8", (long long)cols);
  LV_CHECK_ARG(approx == 0 || approx == 1, "lv_gelu_bwd: approx=%d must be 0 (erf) or 1 (tanh)", approx);
  LV_CHECK_ARG(aligned16(pre) && aligned16(dy) && aligned16(dx), "lv_gelu_bwd: pointers must be 16-byte aligned");
  if (rows == 0) return LV_OK;
  LV_BIND_DEVICE(pre);
  const int64_t total = rows * (cols / 8);
  gelu_bwd_kernel<<<(unsigned)cdiv(total, 256), 256, 0, (cudaStream_t)stream>>>(BF(pre), BF(dy), BFM(dx), total, approx);
  LV_CHECK_LAUNCH("gelu_bwd_kernel");
  return LV_OK;
}

int64_t lv_ls_residual_bwd_partials(int64_t rows, int64_t cols) {
  // rows of dls_partials the kernel writes (gridDim.y of the launch below): ~2 CTAs per SM, at least one row lane each
  const int64_t gx = cdiv(cols, 256);
  int64_t gy = 2 * (int64_t)lv::sm_count() / (gx > 0 ? gx : 1);
  const int64_t need = cdiv(rows, LSB_ROWS);
  if (gy > need) gy = need;
  if (gy > 65535) gy = 65535;
  if (gy < 1) gy = 1;
  return gy;
}

int lv_ls_residual_bwd(const void* dout, const void* y, const void* ls, void* dy, float* dls_partials, int64_t rows,
                       int64_t cols, lv_stream_t stream) {
  LV_CHECK_ARG(ls && dls_partials && (rows == 0 || (dout && y && dy)), "lv_ls_residual_bwd: null pointer");
  LV_CHECK_ARG(rows >= 0 && cols > 0 && cols % 8 == 0, "lv_ls_residual_bwd: cols=%lld must be a multiple of 8", (long long)cols);
  LV_CHECK_ARG(aligned16(dout) && aligned16(y) && aligned16(ls) && aligned16(dy) && aligned16(dls_partials),
               "lv_ls_residual_bwd: pointers must be 16-byte aligned");
  LV_BIND_DEVICE(dls_partials);  // the partial buffer exists (and is zeroed) even with zero rows
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t gy = lv_ls_residual_bwd_partials(rows, cols);
  if (rows == 0) {
    LV_CHECK_CUDA(cudaMemsetAsync(dls_partials, 0, (size_t)gy * cols * 4, s));
    return LV_OK;
  }
  const dim3 grid((unsigned)cdiv(cols, 256), (unsigned)gy);
  ls_residual_bwd_kernel<<<grid, 256, 0, s>>>(BF(dout), BF(y), BF(ls), BFM(dy), dls_partials, rows, (int)cols);
  LV_CHECK_LAUNCH("ls_residual_bwd_kernel");
  return LV_OK;
}

int lv_pixel_shuffle_bwd(const void* dout, void* dx, int64_t n, int64_t hw, int64_t c, int32_t has_cls, lv_stream_t stream) {
  LV_CHECK_ARG(dout && dx, "lv_pixel_shuffle_bwd: null pointer");
  LV_CHECK_ARG(n >= 0 && hw > 0 && hw % 2 == 0 && c > 0 && c % 8 == 0, "lv_pixel_shuffle_bwd: hw=%lld must be even, c=%lld a multiple of 8", (long long)hw, (long long)c);
  LV_CHECK_ARG(aligned16(dout) && aligned16(dx), "lv_pixel_shuffle_bwd: pointers must be 16-byte aligned");
  if (n == 0) return LV_OK;
  const int64_t blocks = n * (hw / 2) * (hw / 2) + (has_cls ? n : 0);
  LV_CHECK_ARG(blocks < (1ll << 31), "lv_pixel_shuffle_bwd: too many tokens");
  LV_BIND_DEVICE(dout);
  pixel_shuffle_bwd_kernel<<<(unsigned)blocks, 128, 0, (cudaStream_t)stream>>>(BF(dout), BFM(dx), n, (int)hw, (int)c, has_cls);
  LV_CHECK_LAUNCH("pixel_shuffle_bwd_kernel");
  return LV_OK;
}

}  // extern "C"
