// FP8 (e4m3) linear layers of the decoder on the Hopper tensor cores:
//   C[M, N] = act(bf16((A_q . W_q^T) * s_a[m] * s_w[n] + bias[n]))
// with A_q / W_q e4m3, both K-major, and one fp32 scale per row of each (the rule of csrc/fp8_core.h applied to a whole
// row).  Three kernels:
//   quant_rows_fp8_kernel  bf16 rows -> e4m3 rows + fp32 scales (weights at load, the A operand before each product)
//   gemm_fp8_kernel        the persistent warp-specialised structure of gemm_bf16_kernel (gemm.cu): one TMA producer
//                          thread, two consumer warpgroups, a shared-memory ring of 128-byte-swizzled rows, grouped
//                          rasterisation, a TMA-store epilogue.  A 128-byte row holds 128 e4m3 k-values, so each k-block
//                          is four wgmma m64n128k32 e4m3 steps.
//   gemv_fp8_kernel        the decode path (M <= 4): a weight stream at half the bytes of gemv_bf16_kernel
//
// Accumulation.  Hopper's FP8 wgmma does not keep a full fp32 sum across many k-steps (DeepSeek-V3 §3.3.2 measures
// ~14 bits of the accumulator on H800), so each consumer keeps two fp32 register sets: the wgmma accumulator, restarted
// at every 128-deep k-block, and the sum it is added into after that k-block has retired.  Two sets of a 64 x 256 tile
// (2 x 128 registers per thread) do not fit beside the addressing, so the tile is 128 x 128 (2 x 64 registers).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>
#include <string.h>

#include "common.cuh"
#include "fp8_core.h"
#include "ptx.cuh"

namespace lv {

constexpr int F_BM = 128, F_BN = 128, F_BK = 128, F_STAGES = 6;   // F_BK e4m3 values = one 128-byte row
constexpr int F_A_BYTES = F_BM * F_BK;              // 16 KB
constexpr int F_B_BYTES = F_BN * F_BK;              // 16 KB
constexpr int F_C_BYTES = 64 * 64 * 2;              // 8 KB staging per 64 x 64 bf16 output chunk (two per consumer)
constexpr int F_THREADS = 384;
constexpr int F_SMEM = F_STAGES * (F_A_BYTES + F_B_BYTES) + 4 * F_C_BYTES + 256 + 1024;  // + barriers + align slack

__device__ __forceinline__ void fp8_tile_coords(int tile, int num_m, int num_n, int GM, int& mb, int& nb) {
  const int per_group = GM * num_n;
  const int g = tile / per_group;
  const int first_m = g * GM;
  const int gsz = min(num_m - first_m, GM);
  const int r = tile % per_group;
  mb = first_m + r % gsz;
  nb = r / gsz;
}

// The epilogue value of one output element before its bf16 rounding: (sum * s_a) * s_w + bias, one rounding each.
// The GEMM and the GEMV share it.
__device__ __forceinline__ float fp8_out(float sum, float sa, float sw, float b) {
  return __fmaf_rn(__fmul_rn(sum, sa), sw, b);
}

// One k32 step of a consumer: A e4m3 or (A_E5M2, a gradient of the backward products) e5m2; B e4m3.
template <bool A_E5M2>
__device__ __forceinline__ void fp8_mma(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  if constexpr (A_E5M2)
    wgmma_ss_n128_e5m2_e4m3(d, adesc, bdesc, accumulate);
  else
    wgmma_ss_n128_e4m3(d, adesc, bdesc, accumulate);
}

// act: 0 = none (bias optional), 3 = fused SwiGLU over interleaved (gate_i, up_i) W rows, no bias.
// ACC selects the gradient-accumulation epilogue (lv_gemm_fp8_grad): accC[M, N] (fp32, row stride ldacc) +=
// (sum * s_a) * s_w, the value whose bf16 rounding the plain epilogue stores; tmC, bias and act are then unused.
template <bool A_E5M2, bool ACC>
__global__ void __launch_bounds__(F_THREADS, 1)
    gemm_fp8_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmC, const float* __restrict__ sa_g,
                    const float* __restrict__ sw_g, const __nv_bfloat16* __restrict__ bias, int M, int N, int K,
                    int act, int gm, float* __restrict__ accC, long long ldacc) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + F_STAGES * F_A_BYTES;
  uint8_t* sC = sB + F_STAGES * F_B_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sC + 4 * F_C_BYTES);
  uint64_t* full = bars;                  // [F_STAGES]
  uint64_t* empty = bars + F_STAGES;      // [F_STAGES]: one arrival per consumer warpgroup

  const int wg = threadIdx.x >> 7;
  const int num_m = (M + F_BM - 1) / F_BM, num_n = (N + F_BN - 1) / F_BN;
  const int num_tiles = num_m * num_n;
  const int num_kb = (K + F_BK - 1) / F_BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if constexpr (!ACC) tma_prefetch_desc(&tmC);
    for (int i = 0; i < F_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ------------------------------- TMA producer -------------------------------
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int mb, nb;
        fp8_tile_coords(tile, num_m, num_n, gm, mb, nb);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full[stage], F_A_BYTES + F_B_BYTES);
          // the maps count k in pairs of e4m3 bytes (encode_fp8_operand): a 128-byte row is 64 of them
          tma_load_2d(sA + stage * F_A_BYTES, &tmA, &full[stage], kb * (F_BK / 2), mb * F_BM, kEvictNormal);
          tma_load_2d(sB + stage * F_B_BYTES, &tmB, &full[stage], kb * (F_BK / 2), nb * F_BN, kEvictNormal);
          if (++stage == F_STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ------------------------------- consumers ----------------------------------
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = wg - 1;                          // 64-row half of the tile
    const int wg_tid = threadIdx.x & 127;
    const int warp = wg_tid >> 5, lane = wg_tid & 31;
    const int r_lo = warp * 16 + (lane >> 2);       // accumulator rows r_lo and r_lo + 8 (of 64)
    const int cq = 2 * (lane & 3);                  // first of the two columns of each 8-column group
    uint8_t* stg_base = sC + cw * 2 * F_C_BYTES;
    // 128 B rows of 128 k, 8-row groups 1024 B apart, a k32 step is +32 B; a consumer's 64 rows start 8 KB into A
    const uint64_t adesc0 = make_smem_desc(smem_u32(sA) + cw * 8192, 16, 1024);
    const uint64_t bdesc0 = make_smem_desc(smem_u32(sB), 16, 1024);
    int stage = 0;
    uint32_t phase = 0;
    uint32_t chunk_counter = 0;
    float acc[64], sum[64];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int mb, nb;
      fp8_tile_coords(tile, num_m, num_n, gm, mb, nb);
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        const uint64_t adesc = adesc0 + (uint64_t)((stage * F_A_BYTES) >> 4);
        const uint64_t bdesc = bdesc0 + (uint64_t)((stage * F_B_BYTES) >> 4);
#ifdef LV_FP8_NO_PROMOTION
        // experiment build (LV_EXTRA_DEFINES=-DLV_FP8_NO_PROMOTION): the whole K accumulates inside the tensor cores,
        // the unpromoted accumulation whose error tests/test_gpu_fp8_linear.py must tell apart
#pragma unroll
        for (int kk = 0; kk < F_BK / 32; ++kk)
          fp8_mma<A_E5M2>(sum, adesc + 2 * kk, bdesc + 2 * kk, (kb | kk) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_keep(sum);
        if (wg_tid == 0) mbar_arrive(&empty[stage]);
#else
#pragma unroll
        for (int kk = 0; kk < F_BK / 32; ++kk) fp8_mma<A_E5M2>(acc, adesc + 2 * kk, bdesc + 2 * kk, kk != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_keep(acc);
        if (wg_tid == 0) mbar_arrive(&empty[stage]);
        // promotion: this k-block's partial product joins the fp32 sum (the first one starts it)
#pragma unroll
        for (int i = 0; i < 64; ++i) sum[i] = kb == 0 ? acc[i] : sum[i] + acc[i];
#endif
        if (++stage == F_STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }

      // ------------------------------- epilogue -----------------------------------
      const int grow = mb * F_BM + cw * 64 + r_lo;
      const float sa0 = grow < M ? sa_g[grow] : 0.f, sa1 = grow + 8 < M ? sa_g[grow + 8] : 0.f;
      if constexpr (ACC) {
        // accC += value as a read-add-write from registers with one IEEE round-to-nearest add (add.rn.f32, subnormals
        // kept), as the bf16 accumulate epilogue of gemm.cu does it; one writer per element, deterministic.  A quad's
        // column pairs span one 32-byte sector per row.  Per 64-column chunk the 16 loads go before the adds.
#pragma unroll
        for (int c = 0; c < F_BN / 64; ++c) {
          float2 prior[16];
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int col = nb * F_BN + 64 * c + 8 * jj + cq;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = grow + 8 * h;
              prior[2 * jj + h] = make_float2(0.f, 0.f);
              if (row < M && col < N) prior[2 * jj + h] = *reinterpret_cast<const float2*>(accC + row * ldacc + col);
            }
          }
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = c * 8 + jj;
            const int col = nb * F_BN + 64 * c + 8 * jj + cq;
            const float sw0 = col < N ? sw_g[col] : 0.f, sw1 = col + 1 < N ? sw_g[col + 1] : 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = grow + 8 * h;
              if (row < M && col < N) {
                const float sa = h ? sa1 : sa0;
                float2 v = prior[2 * jj + h];
                const float p0 = fp8_out(sum[4 * j + 2 * h], sa, sw0, 0.f), p1 = fp8_out(sum[4 * j + 2 * h + 1], sa, sw1, 0.f);
                asm("add.rn.f32 %0, %0, %1;" : "+f"(v.x) : "f"(p0));
                asm("add.rn.f32 %0, %0, %1;" : "+f"(v.y) : "f"(p1));
                *reinterpret_cast<float2*>(accC + row * ldacc + col) = v;
              }
            }
          }
        }
        continue;
      }
      auto stage_begin = [&]() -> uint8_t* {
        uint8_t* stg = stg_base + (chunk_counter & 1) * F_C_BYTES;
        // the TMA store that last read this staging buffer (two chunks ago) must have drained
        if (wg_tid == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
        named_bar_sync(1 + cw, 128);
        return stg;
      };
      auto stage_end = [&](uint8_t* stg, int col0) {
        fence_proxy_async_smem();
        named_bar_sync(1 + cw, 128);
        if (wg_tid == 0) {
          tma_store_2d(&tmC, stg, col0, mb * F_BM + cw * 64);
          tma_store_commit();
        }
        ++chunk_counter;
      };
      if (act == 3) {
        // (gate_i, up_i) are accumulator columns (2i, 2i + 1) of one thread; each is scaled and rounded to bf16 as the
        // bf16 GEMM rounds it, then out = bf16(bf16(silu(gate)) * up).  The tile's 64 output columns are one chunk.
        uint8_t* stg = stage_begin();
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = nb * F_BN + 8 * j + cq;
          const float swg = col < N ? sw_g[col] : 0.f, swu = col + 1 < N ? sw_g[col + 1] : 0.f;
          const int oc = 4 * j + (lane & 3);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float sa = h ? sa1 : sa0;
            const float g = __bfloat162float(__float2bfloat16_rn(fp8_out(sum[4 * j + 2 * h], sa, swg, 0.f)));
            const float u = __bfloat162float(__float2bfloat16_rn(fp8_out(sum[4 * j + 2 * h + 1], sa, swu, 0.f)));
            const float o = __bfloat162float(__float2bfloat16_rn(__fdividef(g, 1.f + __expf(-g)))) * u;
            const int row = r_lo + 8 * h;
            *reinterpret_cast<__nv_bfloat16*>(stg + row * 128 + (((oc >> 3) ^ (row & 7)) << 4) + (oc & 7) * 2) =
                __float2bfloat16_rn(o);
          }
        }
        stage_end(stg, nb * (F_BN / 2));
      } else {
#pragma unroll
        for (int c = 0; c < F_BN / 64; ++c) {
          uint8_t* stg = stage_begin();
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = c * 8 + jj;
            const int col = nb * F_BN + 8 * j + cq;
            const float sw0 = col < N ? sw_g[col] : 0.f, sw1 = col + 1 < N ? sw_g[col + 1] : 0.f;
            float b0 = 0.f, b1 = 0.f;
            if (bias != nullptr) {
              b0 = col < N ? __bfloat162float(bias[col]) : 0.f;
              b1 = col + 1 < N ? __bfloat162float(bias[col + 1]) : 0.f;
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float sa = h ? sa1 : sa0;
              const float v0 = fp8_out(sum[4 * j + 2 * h], sa, sw0, b0), v1 = fp8_out(sum[4 * j + 2 * h + 1], sa, sw1, b1);
              const int row = r_lo + 8 * h;
              *reinterpret_cast<uint32_t*>(stg + row * 128 + ((jj ^ (row & 7)) << 4) + cq * 2) = pack_bf16(v0, v1);
            }
          }
          stage_end(stg, nb * F_BN + c * 64);
        }
      }
    }
    if constexpr (!ACC) {
      if (wg_tid == 0) tma_store_wait_all0();
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Row quantiser: one CTA of 256 threads per row, so that a decode-sized call (1-4 rows) is not one warp walking a
// 13 824-wide row; 16 values per thread and step (two 16-byte loads, one 16-byte store).  The first pass finds amax
// (max is exact in any order: warp shuffles, then the 8 warps through shared memory), the second reads the row again
// (from L1 / L2) and stores q; thread 0 stores the scale.  Same arithmetic as lv_fp8_quant_row of fp8_core.h, in e4m3
// or (E5M2, hybrid training's gradients) e5m2.
// ---------------------------------------------------------------------------------------------
constexpr int Q_THREADS = 256;

__device__ __forceinline__ void bf16x8(const uint4& v, float (&f)[8]) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 p = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]));
    f[2 * i] = p.x;
    f[2 * i + 1] = p.y;
  }
}

template <bool E5M2>
__global__ void __launch_bounds__(Q_THREADS)
    quant_rows_fp8_kernel(const __nv_bfloat16* __restrict__ X, uint8_t* __restrict__ Q, float* __restrict__ S, int K,
                          long long ldx) {
  __shared__ float warp_max[Q_THREADS / 32];
  const long long row = blockIdx.x;
  const __nv_bfloat16* x = X + row * ldx;
  uint8_t* q = Q + row * (long long)K;
  float amax = 0.f;
  for (int k = threadIdx.x * 16; k < K; k += Q_THREADS * 16) {
    float f[8];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      bf16x8(*reinterpret_cast<const uint4*>(x + k + 8 * h), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(f[i]));
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, off));
  if ((threadIdx.x & 31) == 0) warp_max[threadIdx.x >> 5] = amax;
  __syncthreads();
#pragma unroll
  for (int w = 0; w < Q_THREADS / 32; ++w) amax = fmaxf(amax, warp_max[w]);
  const float inv = lv_fp8_inv(E5M2, amax);
  const bool zero = lv_fp8_zero_row(inv);
  for (int k = threadIdx.x * 16; k < K; k += Q_THREADS * 16) {
    uint32_t o[4] = {0u, 0u, 0u, 0u};
    if (!zero) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float f[8];
        bf16x8(*reinterpret_cast<const uint4*>(x + k + 8 * h), f);
#pragma unroll
        for (int i = 0; i < 2; ++i)
          o[2 * h + i] =
              (uint32_t)lv_fp8_pack2(E5M2, __fmul_rn(f[4 * i], inv), __fmul_rn(f[4 * i + 1], inv)) |
              ((uint32_t)lv_fp8_pack2(E5M2, __fmul_rn(f[4 * i + 2], inv), __fmul_rn(f[4 * i + 3], inv)) << 16);
      }
    }
    *reinterpret_cast<uint4*>(q + k) = make_uint4(o[0], o[1], o[2], o[3]);
  }
  if (threadIdx.x == 0) S[row] = zero ? 0.f : lv_fp8_scale(E5M2, amax);
}

// ---------------------------------------------------------------------------------------------
// Cast-transpose (the backward operands): x bf16 [R, C] -> q [C, R16] with one scale per column of x (a row of q),
// R16 = R rounded up to 16, columns R..R16 of q zero.  Two passes, both reading x with 16-byte loads along its rows:
//   col_amax_kernel        per column max|x| over a band of CT_AMAX_ROWS rows, merged with atomicMax on the fp32 bits
//                          (non-negative floats order as their bits; max is exact in any order)
//   cast_transpose_kernel  a 128-row x 64-column tile per CTA: quantised as read, transposed through shared memory,
//                          stored as 64 rows of 128 bytes with 16-byte stores.  A tile row c holds its eight 16-byte
//                          chunks in the order chunk ^ (c / 8 % 8): a warp's byte stores (columns 8g + i of the
//                          tile, g = 0..7) then fall on eight different banks instead of one
// ---------------------------------------------------------------------------------------------
constexpr int CT_R = 128, CT_C = 64, CT_THREADS = 256, CT_AMAX_ROWS = 256;

__global__ void __launch_bounds__(CT_THREADS)
    col_amax_kernel(const __nv_bfloat16* __restrict__ X, unsigned* __restrict__ amax_bits, int R, int C, long long ldx) {
  // 32 threads x 8 columns across, 8 row lanes down
  __shared__ float part[8][CT_THREADS];
  const int cv = threadIdx.x & 31, rl = threadIdx.x >> 5;
  const int c = (blockIdx.x * 32 + cv) * 8;
  const int r_end = min(R, (int)(blockIdx.y + 1) * CT_AMAX_ROWS);
  float m[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (c < C) {
    for (int r = blockIdx.y * CT_AMAX_ROWS + rl; r < r_end; r += 8) {
      float f[8];
      bf16x8(*reinterpret_cast<const uint4*>(X + (long long)r * ldx + c), f);
#pragma unroll
      for (int i = 0; i < 8; ++i) m[i] = fmaxf(m[i], fabsf(f[i]));
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) part[i][threadIdx.x] = m[i];
  __syncthreads();
  if (rl == 0 && c < C) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float v = m[i];
#pragma unroll
      for (int l = 1; l < 8; ++l) v = fmaxf(v, part[i][l * 32 + cv]);
      atomicMax(amax_bits + c + i, __float_as_uint(v));
    }
  }
}

template <bool E5M2>
__global__ void __launch_bounds__(CT_THREADS)
    cast_transpose_kernel(const __nv_bfloat16* __restrict__ X, const unsigned* __restrict__ amax_bits,
                          uint8_t* __restrict__ Q, float* __restrict__ S, int R, int R16, int C, long long ldx) {
  __shared__ __align__(16) uint8_t tile[CT_C][CT_R];   // [column of x][row of x, chunk-swizzled] = a row of q
  const int r0 = blockIdx.x * CT_R, c0 = blockIdx.y * CT_C;
  // read: 8 threads x 8 columns across a row, 32 rows per step
  const int g = threadIdx.x & 7, rr = threadIdx.x >> 3;
  const int c = c0 + 8 * g;
  float inv[8];
  bool zero[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float amax = c + i < C ? __uint_as_float(amax_bits[c + i]) : 0.f;
    inv[i] = lv_fp8_inv(E5M2, amax);
    zero[i] = lv_fp8_zero_row(inv[i]);
  }
  if (blockIdx.x == 0 && threadIdx.x < CT_C && c0 + threadIdx.x < C) {
    const float amax = __uint_as_float(amax_bits[c0 + threadIdx.x]);
    S[c0 + threadIdx.x] = lv_fp8_zero_row(lv_fp8_inv(E5M2, amax)) ? 0.f : lv_fp8_scale(E5M2, amax);
  }
#pragma unroll
  for (int step = 0; step < CT_R / 32; ++step) {
    const int lr = step * 32 + rr, r = r0 + lr;
    uint8_t b[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (r < R && c < C) {
      float f[8];
      bf16x8(*reinterpret_cast<const uint4*>(X + (long long)r * ldx + c), f);
#pragma unroll
      for (int i = 0; i < 8; i += 2) {
        const uint16_t p = lv_fp8_pack2(E5M2, __fmul_rn(f[i], inv[i]), __fmul_rn(f[i + 1], inv[i + 1]));
        b[i] = zero[i] ? 0 : (uint8_t)(p & 0xFF);
        b[i + 1] = zero[i + 1] ? 0 : (uint8_t)(p >> 8);
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) tile[8 * g + i][(((lr >> 4) ^ g) << 4) | (lr & 15)] = b[i];
  }
  __syncthreads();
  // write: 8 threads x 16 bytes along a row of q, 32 rows of q per step
#pragma unroll
  for (int step = 0; step < CT_C / 32; ++step) {
    const int lc = step * 32 + rr, qc = c0 + lc, qr = r0 + 16 * g;
    if (qc < C && qr < R16)
      *reinterpret_cast<uint4*>(Q + (long long)qc * R16 + qr) =
          *reinterpret_cast<const uint4*>(&tile[lc][(g ^ ((lc >> 3) & 7)) << 4]);
  }
}

// ---------------------------------------------------------------------------------------------
// FP8 GEMV (decode, M <= 4): gemv_bf16_kernel's shape (gemm.cu) over e4m3 A and W.  One warp owns two adjacent output
// columns (W rows r, r + 1: the (gate, up) pair of the fused SwiGLU layout); its lanes stride over K in 16-byte vectors
// of 16 e4m3 values, 4 loads in flight per W row, dequantised with cvt.rn.f16x2.e4m3x2 (exact: every e4m3 value is an
// fp16 value) and summed in fp32; one shuffle reduction, then the epilogue of gemm_fp8_kernel.
// ---------------------------------------------------------------------------------------------
constexpr int FV_WARPS = 8, FV_UNROLL = 4;

__device__ __forceinline__ uint4 ld_stream_v4_fp8(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

__device__ __forceinline__ float2 e4m3x2_to_float2(uint16_t v) {
  uint32_t h;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"(v));
  return __half22float2(*reinterpret_cast<const __half2*>(&h));
}

__device__ __forceinline__ float dot16_e4m3(const uint4& a, const uint4& b, float acc) {
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float2 af = e4m3x2_to_float2((uint16_t)(aw[i] >> (16 * h)));
      const float2 bf = e4m3x2_to_float2((uint16_t)(bw[i] >> (16 * h)));
      acc = fmaf(af.x, bf.x, acc);
      acc = fmaf(af.y, bf.y, acc);
    }
  }
  return acc;
}

template <int MT>
__global__ void __launch_bounds__(FV_WARPS * 32)
    gemv_fp8_kernel(const uint8_t* __restrict__ A, const float* __restrict__ sa_g, const uint8_t* __restrict__ W,
                    const float* __restrict__ sw_g, const __nv_bfloat16* __restrict__ bias,
                    __nv_bfloat16* __restrict__ C, int M, int N, int K, long long lda, long long ldw, long long ldc,
                    int act) {
  const int lane = threadIdx.x & 31;
  const long long r0 = 2ll * ((long long)blockIdx.x * FV_WARPS + (threadIdx.x >> 5));
  if (r0 >= N) return;
  const bool has1 = r0 + 1 < N;
  const uint8_t* w0 = W + r0 * ldw;
  const uint8_t* w1 = W + (has1 ? r0 + 1 : r0) * ldw;
  float acc0[MT], acc1[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) acc0[m] = acc1[m] = 0.f;
  for (int k0 = lane * 16; k0 < K; k0 += 512 * FV_UNROLL) {
    uint4 a[FV_UNROLL], b[FV_UNROLL];
#pragma unroll
    for (int u = 0; u < FV_UNROLL; ++u) {
      const int k = k0 + u * 512;
      if (k < K) {
        a[u] = ld_stream_v4_fp8(w0 + k);
        b[u] = ld_stream_v4_fp8(w1 + k);
      } else {
        a[u] = b[u] = make_uint4(0u, 0u, 0u, 0u);
      }
    }
#pragma unroll
    for (int u = 0; u < FV_UNROLL; ++u) {
      const int k = k0 + u * 512;
      if (k < K) {
#pragma unroll
        for (int m = 0; m < MT; ++m) {
          if (m < M) {
            const uint4 x = __ldg(reinterpret_cast<const uint4*>(A + m * lda + k));
            acc0[m] = dot16_e4m3(a[u], x, acc0[m]);
            acc1[m] = dot16_e4m3(b[u], x, acc1[m]);
          }
        }
      }
    }
  }
#pragma unroll
  for (int m = 0; m < MT; ++m) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      acc0[m] += __shfl_xor_sync(0xffffffffu, acc0[m], off);
      acc1[m] += __shfl_xor_sync(0xffffffffu, acc1[m], off);
    }
  }
  if (lane != 0) return;
  const float sw0 = sw_g[r0], sw1 = has1 ? sw_g[r0 + 1] : 0.f;
  const float b0 = bias != nullptr ? __bfloat162float(bias[r0]) : 0.f;
  const float b1 = (bias != nullptr && has1) ? __bfloat162float(bias[r0 + 1]) : 0.f;
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    if (m >= M) break;
    const float sa = sa_g[m];
    if (act == 3) {   // (gate, up) pair -> one output column
      const float g = __bfloat162float(__float2bfloat16_rn(fp8_out(acc0[m], sa, sw0, 0.f)));
      const float up = __bfloat162float(__float2bfloat16_rn(fp8_out(acc1[m], sa, sw1, 0.f)));
      C[m * ldc + r0 / 2] = __float2bfloat16_rn(__bfloat162float(__float2bfloat16_rn(__fdividef(g, 1.f + __expf(-g)))) * up);
      continue;
    }
    C[m * ldc + r0] = __float2bfloat16_rn(fp8_out(acc0[m], sa, sw0, b0));
    if (has1) C[m * ldc + r0 + 1] = __float2bfloat16_rn(fp8_out(acc1[m], sa, sw1, b1));
  }
}

// TMA map of an e4m3 operand [rows][K] (row stride ld bytes).  It is encoded as bf16 [rows][K / 2]: a box of 64
// "bf16" columns is one 128-byte row of 128 e4m3 values, the 128-byte swizzle acts on bytes either way, and the
// zero fill of out-of-range rows and k is zero bytes, i.e. e4m3 zeros.
static int encode_fp8_operand(CUtensorMap* m, const void* p, int64_t rows, int64_t K, int64_t ld, uint32_t rows_box) {
  const uint64_t dims[2] = {(uint64_t)(K / 2), (uint64_t)rows};
  const uint64_t str[2] = {2, (uint64_t)ld};
  const uint32_t box[2] = {(uint32_t)(F_BK / 2), rows_box};
  return encode_tmap_bf16(m, p, 2, dims, str, box, true);
}

// gemm_fp8_kernel: A e4m3 or (A_E5M2, a gradient of the backward products) e5m2, B e4m3; C bf16 with bias and act,
// or (ACC, lv_gemm_fp8_grad) fp32 accumulated into.
template <bool A_E5M2, bool ACC>
static int launch_gemm_fp8(const void* A, const float* sa, const void* B, const float* sb, const void* bias, void* C,
                           int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int act,
                           cudaStream_t s) {
  CUtensorMap tmA, tmB, tmC;
  int r = encode_fp8_operand(&tmA, A, M, K, lda, F_BM);
  if (r) return r;
  r = encode_fp8_operand(&tmB, B, N, K, ldb, F_BN);
  if (r) return r;
  if constexpr (!ACC) {
    const uint64_t dims[2] = {(uint64_t)(act == 3 ? N / 2 : N), (uint64_t)M};
    const uint64_t str[2] = {2, (uint64_t)ldc * 2};
    const uint32_t box[2] = {64, 64};
    r = encode_tmap_bf16(&tmC, C, 2, dims, str, box, true);
    if (r) return r;
  } else {
    memset(&tmC, 0, sizeof(tmC));
  }
  auto* const kernel = gemm_fp8_kernel<A_E5M2, ACC>;
  static PerDeviceOnce attr_once;
  int attr_dev;
  if (attr_once.needed(&attr_dev)) {
    LV_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, F_SMEM));
    attr_once.done(attr_dev);
  }
  const int64_t tiles = ((M + F_BM - 1) / F_BM) * ((N + F_BN - 1) / F_BN);
  const int grid = (int)(tiles < sm_count() ? tiles : sm_count());
  // M-blocks per rasterisation group, as in gemm.cu: the group's A panel (gm x 128 rows x K bytes) takes ~16 MB of L2
  int gm = (int)((16ll << 20) / (128 * K));
  gm = gm < 8 ? 8 : (gm > 64 ? 64 : gm);
  kernel<<<grid, F_THREADS, F_SMEM, s>>>(tmA, tmB, tmC, sa, sb, reinterpret_cast<const __nv_bfloat16*>(bias), (int)M,
                                         (int)N, (int)K, act, gm, ACC ? reinterpret_cast<float*>(C) : nullptr,
                                         ACC ? (long long)ldc : 0ll);
  LV_CHECK_LAUNCH("gemm_fp8_kernel");
  return LV_OK;
}

static int launch_gemv_fp8(const void* A, const float* sa, const void* W, const float* sw, const void* bias, void* C,
                           int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldw, int64_t ldc, int act,
                           cudaStream_t s) {
  const unsigned grid = (unsigned)(((N + 1) / 2 + FV_WARPS - 1) / FV_WARPS);
  const auto* a = reinterpret_cast<const uint8_t*>(A);
  const auto* w = reinterpret_cast<const uint8_t*>(W);
  const auto* b = reinterpret_cast<const __nv_bfloat16*>(bias);
  auto* c = reinterpret_cast<__nv_bfloat16*>(C);
  if (M == 1)
    gemv_fp8_kernel<1><<<grid, FV_WARPS * 32, 0, s>>>(a, sa, w, sw, b, c, (int)M, (int)N, (int)K, lda, ldw, ldc, act);
  else if (M == 2)
    gemv_fp8_kernel<2><<<grid, FV_WARPS * 32, 0, s>>>(a, sa, w, sw, b, c, (int)M, (int)N, (int)K, lda, ldw, ldc, act);
  else
    gemv_fp8_kernel<4><<<grid, FV_WARPS * 32, 0, s>>>(a, sa, w, sw, b, c, (int)M, (int)N, (int)K, lda, ldw, ldc, act);
  LV_CHECK_LAUNCH("gemv_fp8_kernel");
  return LV_OK;
}

}  // namespace lv

using namespace lv;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" {

int lv_quant_rows_fp8_fmt(const void* x, void* q, float* scale, int64_t M, int64_t K, int64_t ldx, int32_t fmt,
                          lv_stream_t stream) {
  LV_CHECK_ARG(x && q && scale, "lv_quant_rows_fp8_fmt: null pointer");
  LV_CHECK_ARG(fmt == 0 || fmt == 1, "lv_quant_rows_fp8_fmt: format %d is not built (0 = e4m3, 1 = e5m2)", fmt);
  LV_CHECK_ARG(M >= 0 && K > 0 && K % 16 == 0 && M < (1ll << 31) && K < (1ll << 31),
               "lv_quant_rows_fp8_fmt: bad shape M=%lld K=%lld (K must be a positive multiple of 16)", (long long)M,
               (long long)K);
  LV_CHECK_ARG(ldx % 8 == 0 && ldx >= K, "lv_quant_rows_fp8_fmt: ldx=%lld must be a multiple of 8 and >= K=%lld",
               (long long)ldx, (long long)K);
  LV_CHECK_ARG(aligned16(x) && aligned16(q), "lv_quant_rows_fp8_fmt: x and q must be 16-byte aligned");
  if (M == 0) return LV_OK;
  LV_BIND_DEVICE(x);
  auto* const kernel = fmt ? quant_rows_fp8_kernel<true> : quant_rows_fp8_kernel<false>;
  kernel<<<(unsigned)M, Q_THREADS, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __nv_bfloat16*>(x),
                                                              reinterpret_cast<uint8_t*>(q), scale, (int)K,
                                                              (long long)ldx);
  LV_CHECK_LAUNCH("quant_rows_fp8_kernel");
  return LV_OK;
}

int lv_quant_cols_fp8_t(const void* x, void* q, float* scale, unsigned* amax_ws, int64_t R, int64_t C, int64_t ldx,
                        int32_t fmt, lv_stream_t stream) {
  LV_CHECK_ARG(x && q && scale && amax_ws, "lv_quant_cols_fp8_t: null pointer");
  LV_CHECK_ARG(fmt == 0 || fmt == 1, "lv_quant_cols_fp8_t: format %d is not built (0 = e4m3, 1 = e5m2)", fmt);
  LV_CHECK_ARG(R >= 0 && C > 0 && C % 8 == 0 && R < (1ll << 31) - 16 && C < (1ll << 31),
               "lv_quant_cols_fp8_t: bad shape R=%lld C=%lld (C must be a positive multiple of 8)", (long long)R,
               (long long)C);
  LV_CHECK_ARG(ldx % 8 == 0 && ldx >= C, "lv_quant_cols_fp8_t: ldx=%lld must be a multiple of 8 and >= C=%lld",
               (long long)ldx, (long long)C);
  LV_CHECK_ARG(aligned16(x) && aligned16(q), "lv_quant_cols_fp8_t: x and q must be 16-byte aligned");
  LV_BIND_DEVICE(x);
  const cudaStream_t s = (cudaStream_t)stream;
  const int64_t R16 = (R + 15) / 16 * 16;
  LV_CHECK_CUDA(cudaMemsetAsync(amax_ws, 0, C * sizeof(unsigned), s));
  if (R > 0) {
    col_amax_kernel<<<dim3((unsigned)((C + 255) / 256), (unsigned)((R + CT_AMAX_ROWS - 1) / CT_AMAX_ROWS)), CT_THREADS,
                      0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x), amax_ws, (int)R, (int)C, (long long)ldx);
    LV_CHECK_LAUNCH("col_amax_kernel");
  }
  const dim3 grid((unsigned)((R16 + CT_R - 1) / CT_R > 0 ? (R16 + CT_R - 1) / CT_R : 1), (unsigned)((C + CT_C - 1) / CT_C));
  auto* const kernel = fmt ? cast_transpose_kernel<true> : cast_transpose_kernel<false>;
  kernel<<<grid, CT_THREADS, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x), amax_ws, reinterpret_cast<uint8_t*>(q),
                                     scale, (int)R, (int)R16, (int)C, (long long)ldx);
  LV_CHECK_LAUNCH("cast_transpose_kernel");
  return LV_OK;
}

int lv_gemm_fp8(const void* A, const float* a_scale, const void* W, const float* w_scale, const void* bias, void* C,
                int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldw, int64_t ldc, int32_t act,
                lv_stream_t stream) {
  LV_CHECK_ARG(A && a_scale && W && w_scale && C, "lv_gemm_fp8: null pointer");
  LV_CHECK_ARG(M >= 0 && N > 0 && K > 0 && M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31),
               "lv_gemm_fp8: bad shape M=%lld N=%lld K=%lld", (long long)M, (long long)N, (long long)K);
  LV_CHECK_ARG(K % 16 == 0 && N % 8 == 0, "lv_gemm_fp8: K=%lld must be a multiple of 16 and N=%lld of 8", (long long)K,
               (long long)N);
  LV_CHECK_ARG(act == 0 || act == 3, "lv_gemm_fp8: activation %d is not built (0 = none, 3 = SwiGLU)", act);
  LV_CHECK_ARG(act != 3 || (N % 16 == 0 && bias == nullptr), "lv_gemm_fp8: fused SwiGLU needs N %% 16 == 0 and no bias");
  LV_CHECK_ARG(lda % 16 == 0 && lda >= K, "lv_gemm_fp8: lda=%lld must be a multiple of 16 and >= K=%lld",
               (long long)lda, (long long)K);
  LV_CHECK_ARG(ldw % 16 == 0 && ldw >= K, "lv_gemm_fp8: ldw=%lld must be a multiple of 16 and >= K=%lld",
               (long long)ldw, (long long)K);
  const int64_t row = act == 3 ? N / 2 : N;
  LV_CHECK_ARG(ldc % 8 == 0 && ldc >= row, "lv_gemm_fp8: ldc=%lld must be a multiple of 8 and >= the row length %lld",
               (long long)ldc, (long long)row);
  LV_CHECK_ARG(aligned16(A) && aligned16(W) && aligned16(C), "lv_gemm_fp8: A, W and C must be 16-byte aligned");
  if (M == 0) return LV_OK;
  LV_BIND_DEVICE(A);
  const cudaStream_t s = (cudaStream_t)stream;
  // the GEMV for decode-sized M, by the rule of lv_gemm_bias_act: unless a 256-column tiling already has a tile per SM
  if (M <= 4 && (N + 255) / 256 < sm_count())
    return launch_gemv_fp8(A, a_scale, W, w_scale, bias, C, M, N, K, lda, ldw, ldc, act, s);
  return launch_gemm_fp8<false, false>(A, a_scale, W, w_scale, bias, C, M, N, K, lda, ldw, ldc, act, s);
}

int lv_gemm_fp8_grad(const void* A, int32_t a_fmt, const float* a_scale, const void* B, const float* b_scale, void* C,
                     int64_t M, int64_t N, int64_t K, int64_t lda, int64_t ldb, int64_t ldc, int32_t accumulate,
                     lv_stream_t stream) {
  LV_CHECK_ARG(A && a_scale && B && b_scale && C, "lv_gemm_fp8_grad: null pointer");
  LV_CHECK_ARG(a_fmt == 0 || a_fmt == 1, "lv_gemm_fp8_grad: A format %d is not built (0 = e4m3, 1 = e5m2)", a_fmt);
  LV_CHECK_ARG(M >= 0 && N > 0 && K > 0 && M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31),
               "lv_gemm_fp8_grad: bad shape M=%lld N=%lld K=%lld", (long long)M, (long long)N, (long long)K);
  LV_CHECK_ARG(K % 16 == 0 && N % 8 == 0, "lv_gemm_fp8_grad: K=%lld must be a multiple of 16 and N=%lld of 8",
               (long long)K, (long long)N);
  LV_CHECK_ARG(lda % 16 == 0 && lda >= K && ldb % 16 == 0 && ldb >= K,
               "lv_gemm_fp8_grad: lda=%lld and ldb=%lld must be multiples of 16 and >= K=%lld", (long long)lda,
               (long long)ldb, (long long)K);
  LV_CHECK_ARG(ldc % (accumulate ? 4 : 8) == 0 && ldc >= N,
               "lv_gemm_fp8_grad: ldc=%lld must be a multiple of %d and >= N=%lld", (long long)ldc, accumulate ? 4 : 8,
               (long long)N);
  LV_CHECK_ARG(aligned16(A) && aligned16(B) && aligned16(C), "lv_gemm_fp8_grad: A, B and C must be 16-byte aligned");
  if (M == 0) return LV_OK;
  LV_BIND_DEVICE(A);
  const cudaStream_t s = (cudaStream_t)stream;
  auto* const launch = accumulate ? (a_fmt ? launch_gemm_fp8<true, true> : launch_gemm_fp8<false, true>)
                                  : (a_fmt ? launch_gemm_fp8<true, false> : launch_gemm_fp8<false, false>);
  return launch(A, a_scale, B, b_scale, nullptr, C, M, N, K, lda, ldb, ldc, 0, s);
}

}  // extern "C"
