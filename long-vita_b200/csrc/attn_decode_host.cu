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
#include <cuda_bf16.h>
#include <math.h>

#include "common.cuh"

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

}  // extern "C"
