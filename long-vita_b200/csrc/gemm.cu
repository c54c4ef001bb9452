// Dense linear layer on the Hopper tensor cores:  C[M,N] = act(A[M,K] . W[N,K]^T + bias)
//
// Persistent, warp-specialised sm_90a kernel (one CTA per SM, 3 warpgroups):
//   warpgroup 0     TMA producer (one thread): 128x64 A tiles and 256x64 W tiles (128-byte swizzle) into a
//                   4-stage shared-memory ring, completion on mbarriers
//   warpgroups 1-2  consumers: each owns 64 rows of the 128x256 tile, wgmma m64n256k16 (bf16 x bf16 -> fp32,
//                   accumulators in registers) with one k-block of MMAs in flight; then the epilogue - bias,
//                   activation, bf16 pack, swizzled st.shared, TMA store (clips the M / N tails) - while the
//                   producer already fills the ring for the next tile
// Tiles are rasterised in groups of M-blocks so the concurrently resident tiles share A and W panels in L2.
// Either operand may also be MN-major (stored transposed, lv_gemm_ex): the backward products read dY, X and W in place.
//
// Replaces torch.matmul / te.Linear at long_vita_megatron/core/tensor_parallel/layers.py:270,409 and
// the nn.Linear calls of modeling_intern_vit.py:131,141,190-191 / resampler_projector.py:19-23.
#include <cuda_bf16.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "ptx.cuh"

namespace lv {

constexpr int G_BM = 128, G_BN = 256, G_BK = 64, G_STAGES = 4;
constexpr int G_A_BYTES = G_BM * G_BK * 2;          // 16 KB
constexpr int G_B_BYTES = G_BN * G_BK * 2;          // 32 KB
constexpr int G_C_BYTES = 64 * 64 * 2;              // 8 KB staging per 64 x 64 output chunk (two per consumer)
constexpr int G_THREADS = 384;
constexpr int G_ACC_PREFETCH_KB = 8;                // accumulate epilogue: L2 prefetch of accC this many k-blocks early
constexpr int G_SMEM = G_STAGES * (G_A_BYTES + G_B_BYTES) + 4 * G_C_BYTES + 256 + 1024;  // + barriers + align slack

__device__ __forceinline__ float act_apply(float t, int act) {
  if (act == 1) return 0.5f * t * (1.f + erff(t * 0.70710678118654752440f));
  if (act == 2) {
    const float k = 0.7978845608028654f;
    return 0.5f * t * (1.f + tanhf(k * (t + 0.044715f * t * t * t)));
  }
  return t;
}

__device__ __forceinline__ void tile_coords(int tile, int num_m, int num_n, int GM, int& mb, int& nb) {
  const int per_group = GM * num_n;
  const int g = tile / per_group;
  const int first_m = g * GM;
  const int gsz = min(num_m - first_m, GM);
  const int r = tile % per_group;
  mb = first_m + r % gsz;
  nb = r / gsz;
}

// A_MN / W_MN select the layout of each operand in global memory.  K-major (false): A[M][K] / W[N][K], one TMA box of
// 64 k-columns x 128 (256) rows per tile.  MN-major (true): A stored [K][M] / W stored [K][N] with the M / N index
// contiguous - the transposed operands of the backward products dX = dY W and dW = dY^T X - loaded as boxes of
// 64 contiguous M / N elements (128 B) x 64 k-rows, two per A tile and four per W tile, each 8 KB box holding 8-k-row
// groups of 1024 B; wgmma reads them with its transpose bit set.  Stage sizes, ring and barriers are the same.
//
// ACC selects the gradient-accumulation epilogue (lv_gemm_wgrad_acc_f32): accC[M, N] (fp32, row stride ldc) +=
// the fp32 accumulator, with no bias, activation or bf16 rounding; tmC, bias and act are unused.  Mainloop, ring,
// rasterisation and k-order are those of the bf16 epilogue, so the accumulator is the value whose bf16 rounding
// that epilogue stores.
template <bool A_MN, bool W_MN, bool ACC = false>
__global__ void __launch_bounds__(G_THREADS, 1)
    gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const __grid_constant__ CUtensorMap tmC, const __nv_bfloat16* __restrict__ bias, int M, int N,
                     int K, int act, int gm, float* accC, long long ldc) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + G_STAGES * G_A_BYTES;
  uint8_t* sC = sB + G_STAGES * G_B_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sC + 4 * G_C_BYTES);
  uint64_t* full = bars;                  // [G_STAGES]
  uint64_t* empty = bars + G_STAGES;      // [G_STAGES]: one arrival per consumer warpgroup

  const int wg = threadIdx.x >> 7;
  const int num_m = (M + G_BM - 1) / G_BM, num_n = (N + G_BN - 1) / G_BN;
  const int num_tiles = num_m * num_n;
  const int num_kb = (K + G_BK - 1) / G_BK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if constexpr (!ACC) tma_prefetch_desc(&tmC);
    for (int i = 0; i < G_STAGES; ++i) {
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
        tile_coords(tile, num_m, num_n, gm, mb, nb);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full[stage], G_A_BYTES + G_B_BYTES);
          if constexpr (A_MN) {
#pragma unroll
            for (int j = 0; j < G_BM / 64; ++j)
              tma_load_2d(sA + stage * G_A_BYTES + j * 8192, &tmA, &full[stage], mb * G_BM + j * 64, kb * G_BK, kEvictNormal);
          } else {
            tma_load_2d(sA + stage * G_A_BYTES, &tmA, &full[stage], kb * G_BK, mb * G_BM, kEvictNormal);
          }
          if constexpr (W_MN) {
#pragma unroll
            for (int j = 0; j < G_BN / 64; ++j)
              tma_load_2d(sB + stage * G_B_BYTES + j * 8192, &tmB, &full[stage], nb * G_BN + j * 64, kb * G_BK, kEvictNormal);
          } else {
            tma_load_2d(sB + stage * G_B_BYTES, &tmB, &full[stage], kb * G_BK, nb * G_BN, kEvictNormal);
          }
          if (++stage == G_STAGES) {
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
    uint8_t* stg_base = sC + cw * 2 * G_C_BYTES;
    // K-major: 128 B rows of 64 k, 8-row groups 1024 B apart, a k16 step is +32 B.  MN-major: 8-k-row groups 1024 B
    // apart, the next 64 M / N elements one 8 KB box (LBO) away, a k16 step is 16 rows = +2048 B.  A consumer's 64 rows
    // start 8 KB into the A tile in both layouts.
    constexpr uint32_t a_lbo = A_MN ? 8192 : 16, b_lbo = W_MN ? 8192 : 16;
    const uint64_t adesc0 = make_smem_desc(smem_u32(sA) + cw * 8192, a_lbo, 1024);
    const uint64_t bdesc0 = make_smem_desc(smem_u32(sB), b_lbo, 1024);
    constexpr int a_kstep = A_MN ? 2048 >> 4 : 32 >> 4, b_kstep = W_MN ? 2048 >> 4 : 32 >> 4;
    int stage = 0;
    uint32_t phase = 0;
    uint32_t chunk_counter = 0;
    float acc[128];
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      int mb, nb;
      tile_coords(tile, num_m, num_n, gm, mb, nb);
      int prev_stage = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        wgmma_fence();
        const uint64_t adesc = adesc0 + (uint64_t)((stage * G_A_BYTES) >> 4);
        const uint64_t bdesc = bdesc0 + (uint64_t)((stage * G_B_BYTES) >> 4);
#pragma unroll
        for (int kk = 0; kk < G_BK / 16; ++kk)
          wgmma_ss_n256<A_MN, W_MN>(acc, adesc + a_kstep * kk, bdesc + b_kstep * kk, (kb | kk) != 0 ? 1u : 0u);
        wgmma_commit();
        if constexpr (ACC) {
          // G_ACC_PREFETCH_KB k-blocks before the epilogue, pull this consumer's 64 x 256 fp32 block of accC into L2
          // (one 128-byte line per thread and step, 8 lines per 1 KB row): the epilogue's reads then hit L2 instead of
          // waiting on DRAM while the tensor cores idle
          if (kb == (num_kb > G_ACC_PREFETCH_KB ? num_kb - G_ACC_PREFETCH_KB : 0)) {
            const int prow = mb * G_BM + cw * 64 + (wg_tid >> 1);
#pragma unroll
            for (int l = 0; l < 4; ++l) {
              const int pcol = nb * G_BN + ((wg_tid & 1) * 4 + l) * 32;
              if (prow < M && pcol < N) asm volatile("prefetch.global.L2 [%0];" ::"l"(accC + prow * ldc + pcol));
            }
          }
        }
        // the k-block before this one has retired: its ring slot may be refilled
        wgmma_wait<1>();
        wgmma_keep(acc);
        if (prev_stage >= 0 && wg_tid == 0) mbar_arrive(&empty[prev_stage]);
        prev_stage = stage;
        if (++stage == G_STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
      wgmma_keep(acc);
      if (wg_tid == 0) mbar_arrive(&empty[prev_stage]);

      // ------------------------------- epilogue -----------------------------------
      if constexpr (ACC) {
        // accC += acc as a plain read-add-write from registers, not a TMA reduce-add: cp.reduce.async.bulk .add.f32
        // flushes subnormal inputs and results to zero, while add.rn.f32 (no .ftz) is one IEEE-754 round-to-nearest-
        // even add that keeps subnormals, so every element becomes exactly prior + acc, as torch computes it.  Each
        // element has one writer per launch (deterministic).  A quad's two-column pairs span 8 consecutive fp32 = one
        // full 32-byte sector per row, so the 8-byte accesses waste no DRAM traffic; the staging buffers are unused.
        // Per 64-column chunk, the 16 loads are issued before the adds and stores.
        const int row0 = mb * G_BM + cw * 64 + r_lo;
#pragma unroll
        for (int c = 0; c < G_BN / 64; ++c) {
          float2 prior[16];
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int col = nb * G_BN + 64 * c + 8 * jj + cq;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = row0 + 8 * h;
              prior[2 * jj + h] = make_float2(0.f, 0.f);
              if (row < M && col < N) prior[2 * jj + h] = *reinterpret_cast<const float2*>(accC + row * ldc + col);
            }
          }
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = c * 8 + jj;
            const int col = nb * G_BN + 64 * c + 8 * jj + cq;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int row = row0 + 8 * h;
              if (row < M && col < N) {
                float2 v = prior[2 * jj + h];
                asm("add.rn.f32 %0, %0, %1;" : "+f"(v.x) : "f"(acc[4 * j + 2 * h]));
                asm("add.rn.f32 %0, %0, %1;" : "+f"(v.y) : "f"(acc[4 * j + 2 * h + 1]));
                *reinterpret_cast<float2*>(accC + row * ldc + col) = v;
              }
            }
          }
        }
        continue;
      }
      // Output chunks of 64 x 64: staged (128-byte swizzle, the layout of the TMA map) and stored with TMA.  The
      // chunk loops are unrolled so that every accumulator index is a compile-time constant (registers, not stack).
      auto stage_begin = [&]() -> uint8_t* {
        uint8_t* stg = stg_base + (chunk_counter & 1) * G_C_BYTES;
        // the TMA store that last read this staging buffer (two chunks ago) must have drained
        if (wg_tid == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
        named_bar_sync(1 + cw, 128);
        return stg;
      };
      auto stage_end = [&](uint8_t* stg, int col0) {
        fence_proxy_async_smem();
        named_bar_sync(1 + cw, 128);
        if (wg_tid == 0) {
          tma_store_2d(&tmC, stg, col0, mb * G_BM + cw * 64);
          tma_store_commit();
        }
        ++chunk_counter;
      };
      if (act == 3) {
        // Fused SwiGLU: W rows are interleaved (gate_i, up_i), so accumulator columns (2i, 2i+1) - held by the same
        // thread - are gate_i and up_i; out[:, i] = bf16(silu(bf16 gate)) * bf16(up), the exact rounding sequence of
        // the un-fused GEMM + lv_swiglu pair.  Output chunk c covers 8-column groups 16c .. 16c + 15.
#pragma unroll
        for (int c = 0; c < G_BN / 128; ++c) {
          uint8_t* stg = stage_begin();
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
            const int j = c * 16 + jj;
            const int oc = 4 * jj + (lane & 3);           // output column inside the chunk
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const float g = __bfloat162float(__float2bfloat16_rn(acc[4 * j + 2 * h]));
              const float u = __bfloat162float(__float2bfloat16_rn(acc[4 * j + 2 * h + 1]));
              const float o = __bfloat162float(__float2bfloat16_rn(__fdividef(g, 1.f + __expf(-g)))) * u;
              const int row = r_lo + 8 * h;
              *reinterpret_cast<__nv_bfloat16*>(stg + row * 128 + (((oc >> 3) ^ (row & 7)) << 4) + (oc & 7) * 2) =
                  __float2bfloat16_rn(o);
            }
          }
          stage_end(stg, nb * (G_BN / 2) + c * 64);
        }
      } else {
#pragma unroll
        for (int c = 0; c < G_BN / 64; ++c) {
          uint8_t* stg = stage_begin();
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const int j = c * 8 + jj;
            const int col = nb * G_BN + 8 * j + cq;
            float b0 = 0.f, b1 = 0.f;
            if (bias != nullptr) {
              b0 = col < N ? __bfloat162float(bias[col]) : 0.f;
              b1 = col + 1 < N ? __bfloat162float(bias[col + 1]) : 0.f;
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float v0 = acc[4 * j + 2 * h] + b0, v1 = acc[4 * j + 2 * h + 1] + b1;
              if (act != 0) {
                // nn.Linear rounds its output to bf16 before the activation module sees it
                v0 = act_apply(__bfloat162float(__float2bfloat16_rn(v0)), act);
                v1 = act_apply(__bfloat162float(__float2bfloat16_rn(v1)), act);
              }
              const int row = r_lo + 8 * h;
              *reinterpret_cast<uint32_t*>(stg + row * 128 + ((jj ^ (row & 7)) << 4) + cq * 2) = pack_bf16(v0, v1);
            }
          }
          stage_end(stg, nb * G_BN + c * 64);
        }
      }
    }
    if (wg_tid == 0) tma_store_wait_all0();
  }
}

// ---------------------------------------------------------------------------------------------
// Patch embedding helpers: im2col of non-overlapping patches and the cls/pos epilogue.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) im2col_patch_kernel(const __nv_bfloat16* __restrict__ img,
                                                           __nv_bfloat16* __restrict__ col, int64_t n, int size, int ps,
                                                           int kpad) {
  const int g = size / ps;
  const int64_t patch = blockIdx.x;  // n * g * g
  const int64_t im = patch / (g * g);
  const int pr = (int)(patch % (g * g));
  const int py = pr / g, px = pr % g;
  const int kk = 3 * ps * ps;
  for (int e = threadIdx.x; e < kpad; e += blockDim.x) {
    __nv_bfloat16 v = __float2bfloat16_rn(0.f);
    if (e < kk) {
      const int c = e / (ps * ps), ky = (e / ps) % ps, kx = e % ps;
      v = img[((im * 3 + c) * size + (py * ps + ky)) * (int64_t)size + px * ps + kx];
    }
    col[patch * kpad + e] = v;
  }
}

// out[n, 0, :] = cls + pos[0]; out[n, 1+p, :] = tmp[n*P + p, :] + pos[1+p]   (bf16 adds)
__global__ void __launch_bounds__(128) add_cls_pos_kernel(const __nv_bfloat16* __restrict__ tmp,
                                                          const __nv_bfloat16* __restrict__ cls,
                                                          const __nv_bfloat16* __restrict__ pos,
                                                          __nv_bfloat16* __restrict__ out, int64_t n, int P, int C) {
  // cls == nullptr: no class token (SigLIP, siglip_vit_model.py:165-176): out[n, p] = tmp[n*P + p] + pos[p]
  const int hc = cls != nullptr ? 1 : 0;
  const int64_t tok = blockIdx.x;  // n * (P + hc)
  const int64_t im = tok / (P + hc);
  const int t = (int)(tok % (P + hc));
  const __nv_bfloat16* src = (hc && t == 0) ? cls : tmp + (im * P + (t - hc)) * (int64_t)C;
  for (int c = threadIdx.x; c < C; c += blockDim.x)
    out[tok * C + c] = __float2bfloat16_rn(__bfloat162float(src[c]) + __bfloat162float(pos[(int64_t)t * C + c]));
}

// ---------------------------------------------------------------------------------------------
// Small-M path (decode: M = 1 new token, up to 4): the product is a weight stream - every W row is read
// once, HBM-bound - and a 128x256 tensor-core tile would leave most SMs idle (N = 5120 -> 20 tiles).  One
// warp owns two adjacent output columns (W rows r, r+1: the (gate, up) pair of the fused SwiGLU layout),
// its lanes stride over K in 16-byte vectors with 4 loads in flight per row, fp32 accumulation, one
// shuffle reduction.  Same epilogue arithmetic (bias, bf16 rounding before the activation, SwiGLU on
// bf16-rounded gate / up) as the tensor-core kernel.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ld_stream_v4(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

__device__ __forceinline__ float dot8_bf16(const uint4& a, const uint4& b, float acc) {
  const uint32_t aw[4] = {a.x, a.y, a.z, a.w}, bw[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 af = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&aw[i]));
    const float2 bf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&bw[i]));
    acc = fmaf(af.x, bf.x, acc);
    acc = fmaf(af.y, bf.y, acc);
  }
  return acc;
}

constexpr int GV_WARPS = 8, GV_UNROLL = 4;

template <int MT>
__global__ void __launch_bounds__(GV_WARPS * 32)
    gemv_bf16_kernel(const __nv_bfloat16* __restrict__ A, const __nv_bfloat16* __restrict__ W,
                     const __nv_bfloat16* __restrict__ bias, __nv_bfloat16* __restrict__ C, int M, int N, int K,
                     long long lda, long long ldw, long long ldc, int act) {
  const int lane = threadIdx.x & 31;
  const long long r0 = 2ll * ((long long)blockIdx.x * GV_WARPS + (threadIdx.x >> 5));
  if (r0 >= N) return;
  const bool has1 = r0 + 1 < N;
  const __nv_bfloat16* w0 = W + r0 * ldw;
  const __nv_bfloat16* w1 = W + (has1 ? r0 + 1 : r0) * ldw;
  float acc0[MT], acc1[MT];
#pragma unroll
  for (int m = 0; m < MT; ++m) acc0[m] = acc1[m] = 0.f;
  for (int k0 = lane * 8; k0 < K; k0 += 256 * GV_UNROLL) {
    uint4 a[GV_UNROLL], b[GV_UNROLL];
#pragma unroll
    for (int u = 0; u < GV_UNROLL; ++u) {
      const int k = k0 + u * 256;
      if (k < K) {
        a[u] = ld_stream_v4(w0 + k);
        b[u] = ld_stream_v4(w1 + k);
      } else {
        a[u] = b[u] = make_uint4(0u, 0u, 0u, 0u);
      }
    }
#pragma unroll
    for (int u = 0; u < GV_UNROLL; ++u) {
      const int k = k0 + u * 256;
      if (k < K) {
#pragma unroll
        for (int m = 0; m < MT; ++m) {
          if (m < M) {
            const uint4 x = __ldg(reinterpret_cast<const uint4*>(A + m * lda + k));
            acc0[m] = dot8_bf16(a[u], x, acc0[m]);
            acc1[m] = dot8_bf16(b[u], x, acc1[m]);
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
  const float b0 = bias != nullptr ? __bfloat162float(bias[r0]) : 0.f;
  const float b1 = (bias != nullptr && has1) ? __bfloat162float(bias[r0 + 1]) : 0.f;
#pragma unroll
  for (int m = 0; m < MT; ++m) {
    if (m >= M) break;
    float v0 = acc0[m] + b0, v1 = acc1[m] + b1;
    if (act == 3) {   // (gate, up) pair -> one output column
      const float g = __bfloat162float(__float2bfloat16_rn(v0)), up = __bfloat162float(__float2bfloat16_rn(v1));
      C[m * ldc + r0 / 2] = __float2bfloat16_rn(__bfloat162float(__float2bfloat16_rn(__fdividef(g, 1.f + __expf(-g)))) * up);
      continue;
    }
    if (act != 0) {
      v0 = act_apply(__bfloat162float(__float2bfloat16_rn(v0)), act);
      v1 = act_apply(__bfloat162float(__float2bfloat16_rn(v1)), act);
    }
    C[m * ldc + r0] = __float2bfloat16_rn(v0);
    if (has1) C[m * ldc + r0 + 1] = __float2bfloat16_rn(v1);
  }
}

// LV_GEMV=0 sends small-M products through the tensor-core kernel as well (A/B switch).
static bool gemv_enabled() {
  static const bool on = [] {
    const char* e = getenv("LV_GEMV");
    return !(e != nullptr && e[0] == '0');
  }();
  return on;
}

static int launch_gemv(const void* A, const void* W, const void* bias, void* C, int64_t M, int64_t N, int64_t K,
                       int64_t lda, int64_t ldw, int64_t ldc, int act, cudaStream_t s) {
  const int64_t warps = (N + 1) / 2;
  const unsigned grid = (unsigned)((warps + GV_WARPS - 1) / GV_WARPS);
  const auto* a = reinterpret_cast<const __nv_bfloat16*>(A);
  const auto* w = reinterpret_cast<const __nv_bfloat16*>(W);
  const auto* b = reinterpret_cast<const __nv_bfloat16*>(bias);
  auto* c = reinterpret_cast<__nv_bfloat16*>(C);
  if (M == 1)
    gemv_bf16_kernel<1><<<grid, GV_WARPS * 32, 0, s>>>(a, w, b, c, (int)M, (int)N, (int)K, lda, ldw, ldc, act);
  else if (M == 2)
    gemv_bf16_kernel<2><<<grid, GV_WARPS * 32, 0, s>>>(a, w, b, c, (int)M, (int)N, (int)K, lda, ldw, ldc, act);
  else
    gemv_bf16_kernel<4><<<grid, GV_WARPS * 32, 0, s>>>(a, w, b, c, (int)M, (int)N, (int)K, lda, ldw, ldc, act);
  LV_CHECK_LAUNCH("gemv_bf16_kernel");
  return LV_OK;
}

// TMA map of one GEMM operand with `rows` M (or N) indices: K-major [rows][K] in boxes of 64 k x `rows_box`, MN-major
// [K][rows] in boxes of 64 rows x 64 k (see gemm_bf16_kernel).  Out-of-range rows and k are zero-filled.
static int encode_operand(CUtensorMap* m, const void* p, int64_t rows, int64_t K, int64_t ld, bool mn_major,
                          uint32_t rows_box) {
  const uint64_t dims[2] = {(uint64_t)(mn_major ? rows : K), (uint64_t)(mn_major ? K : rows)};
  const uint64_t str[2] = {2, (uint64_t)ld * 2};
  const uint32_t box[2] = {mn_major ? 64u : (uint32_t)G_BK, mn_major ? (uint32_t)G_BK : rows_box};
  return encode_tmap_bf16(m, p, 2, dims, str, box, true);
}

// ACC: C is fp32 and accumulated into (gemm_bf16_kernel); bias and act must be null / 0.
template <bool A_MN, bool W_MN, bool ACC = false>
static int launch_gemm(const void* A, const void* W, const void* bias, void* C, int64_t M, int64_t N, int64_t K,
                       int64_t lda, int64_t ldw, int64_t ldc, int act, cudaStream_t s) {
  CUtensorMap tmA, tmB, tmC;
  int r = encode_operand(&tmA, A, M, K, lda, A_MN, G_BM);
  if (r) return r;
  r = encode_operand(&tmB, W, N, K, ldw, W_MN, G_BN);
  if (r) return r;
  if constexpr (ACC) {
    memset(&tmC, 0, sizeof(tmC));
  } else {
    const uint64_t dims[2] = {(uint64_t)(act == 3 ? N / 2 : N), (uint64_t)M};
    const uint64_t str[2] = {2, (uint64_t)ldc * 2};
    const uint32_t box[2] = {64, 64};
    r = encode_tmap_bf16(&tmC, C, 2, dims, str, box, true);
    if (r) return r;
  }
  auto* const kernel = gemm_bf16_kernel<A_MN, W_MN, ACC>;
  static PerDeviceOnce attr_once;  // one per instantiation
  int attr_dev;
  if (attr_once.needed(&attr_dev)) {
    LV_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, G_SMEM));
    attr_once.done(attr_dev);
  }
  const int64_t tiles = ((M + G_BM - 1) / G_BM) * ((N + G_BN - 1) / G_BN);
  const int grid = (int)(tiles < sm_count() ? tiles : sm_count());
  // M-blocks per rasterisation group: the A panel of a group (gm x 128 rows x K) stays in L2 while its tiles sweep
  // the N-blocks, and W is re-read from HBM once per group, so DRAM traffic ~ A + C + (num_m / gm) * W.  The group is
  // sized so that the A panel takes ~16 MB of the 50 MB L2, but never fewer than 8 M-blocks.
  int gm = (int)((16ll << 20) / (256 * K));
  gm = gm < 8 ? 8 : (gm > 64 ? 64 : gm);
  kernel<<<grid, G_THREADS, G_SMEM, s>>>(tmA, tmB, tmC, reinterpret_cast<const __nv_bfloat16*>(bias), (int)M, (int)N,
                                         (int)K, act, gm, ACC ? reinterpret_cast<float*>(C) : nullptr,
                                         ACC ? (long long)ldc : 0ll);
  LV_CHECK_LAUNCH("gemm_bf16_kernel");
  return LV_OK;
}

}  // namespace lv

using namespace lv;

// The argument checks of the three GEMM entry points; `fn` names the entry point in lv_last_error.  a_mn / w_mn are the
// operand layouts (0, 0 for lv_gemm_bias_act); acc is the fp32 accumulation of lv_gemm_wgrad_acc_f32 (MN-major A and W
// only, K may be 0, N and ldc multiples of 4 fp32 elements, no bias or activation); `aligned` requires 16-byte aligned
// A, W and C (lv_gemm_bias_act does not: its GEMV path takes any C).
static int check_gemm_args(const char* fn, const void* A, const void* W, const void* bias, const void* C, int64_t M,
                           int64_t N, int64_t K, int64_t lda, int64_t ldw, int64_t ldc, int32_t a_mn, int32_t w_mn,
                           int32_t act, bool acc, bool aligned) {
  LV_CHECK_ARG(A && W && C, "%s: null pointer", fn);
  LV_CHECK_ARG((a_mn == 0 || a_mn == 1) && (w_mn == 0 || w_mn == 1), "%s: a_mn_major=%d and w_mn_major=%d must be 0 or 1",
               fn, a_mn, w_mn);
  LV_CHECK_ARG(!acc || (a_mn && w_mn), "%s: only MN-major A and W are built (dW = dY^T . X with dY and X read in place)",
               fn);
  LV_CHECK_ARG(M >= 0 && N > 0 && (acc ? K >= 0 : K > 0), "%s: bad shape M=%lld N=%lld K=%lld", fn, (long long)M,
               (long long)N, (long long)K);
  LV_CHECK_ARG(M < (1ll << 31) && N < (1ll << 31) && K < (1ll << 31), "%s: dimension too large", fn);
  const int nq = acc ? 4 : 8;  // N and ldc in elements of C: 16 bytes of fp32 or of bf16
  if (a_mn && w_mn)
    LV_CHECK_ARG(N % nq == 0, "%s: N=%lld must be a multiple of %d", fn, (long long)N, nq);
  else
    LV_CHECK_ARG(K % 8 == 0 && N % 8 == 0, "%s: K=%lld and N=%lld must be multiples of 8 while an operand is K-major", fn,
                 (long long)K, (long long)N);
  LV_CHECK_ARG(act >= 0 && act <= 3, "%s: unknown activation %d", fn, act);
  LV_CHECK_ARG(lda % 8 == 0 && lda >= (a_mn ? M : K), "%s: lda=%lld must be a multiple of 8 and >= %s=%lld", fn,
               (long long)lda, a_mn ? "M" : "K", (long long)(a_mn ? M : K));
  LV_CHECK_ARG(ldw % 8 == 0 && ldw >= (w_mn ? N : K), "%s: ldw=%lld must be a multiple of 8 and >= %s=%lld", fn,
               (long long)ldw, w_mn ? "N" : "K", (long long)(w_mn ? N : K));
  const int64_t row = act == 3 ? N / 2 : N;
  LV_CHECK_ARG(ldc % nq == 0 && ldc >= row, "%s: ldc=%lld must be a multiple of %d and >= the row length %lld", fn,
               (long long)ldc, nq, (long long)row);
  LV_CHECK_ARG(!aligned || ((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(W) |
                             reinterpret_cast<uintptr_t>(C)) & 15) == 0,
               "%s: A, W and C must be 16-byte aligned", fn);
  LV_CHECK_ARG(act != 3 || (N % 16 == 0 && bias == nullptr), "%s: fused SwiGLU needs N %% 16 == 0 and no bias", fn);
  return LV_OK;
}

extern "C" {

int lv_gemm_bias_act(const void* A, const void* W, const void* bias, void* C, int64_t M, int64_t N, int64_t K,
                     int64_t lda, int64_t ldw, int64_t ldc, int32_t act, lv_stream_t stream) {
  int r = check_gemm_args("lv_gemm_bias_act", A, W, bias, C, M, N, K, lda, ldw, ldc, 0, 0, act, false, false);
  if (r) return r;
  if (M == 0) return LV_OK;
  LV_BIND_DEVICE(A);
  // Weight-stream GEMV for decode-sized M - unless the tensor-core kernel already has a tile for every SM (the LM head:
  // 594 N-tiles)
  if (M <= 4 && gemv_enabled() && (N + G_BN - 1) / G_BN < sm_count() && (reinterpret_cast<uintptr_t>(A) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(W) & 15) == 0)
    return launch_gemv(A, W, bias, C, M, N, K, lda, ldw, ldc, act, (cudaStream_t)stream);
  return launch_gemm<false, false>(A, W, bias, C, M, N, K, lda, ldw, ldc, act, (cudaStream_t)stream);
}

int lv_gemm_ex(const void* A, const void* W, const void* bias, void* C, int64_t M, int64_t N, int64_t K, int64_t lda,
               int64_t ldw, int64_t ldc, int32_t a_mn_major, int32_t w_mn_major, int32_t act, lv_stream_t stream) {
  int r = check_gemm_args("lv_gemm_ex", A, W, bias, C, M, N, K, lda, ldw, ldc, a_mn_major, w_mn_major, act, false, true);
  if (r) return r;
  if (!a_mn_major && !w_mn_major) return lv_gemm_bias_act(A, W, bias, C, M, N, K, lda, ldw, ldc, act, stream);
  if (M == 0) return LV_OK;
  LV_BIND_DEVICE(A);
  // No GEMV for an MN-major operand: its rows are not contiguous along K; the tensor-core kernel is right for any M.
  const cudaStream_t s = (cudaStream_t)stream;
  if (a_mn_major && w_mn_major) return launch_gemm<true, true>(A, W, bias, C, M, N, K, lda, ldw, ldc, act, s);
  if (a_mn_major) return launch_gemm<true, false>(A, W, bias, C, M, N, K, lda, ldw, ldc, act, s);
  return launch_gemm<false, true>(A, W, bias, C, M, N, K, lda, ldw, ldc, act, s);
}

int lv_gemm_wgrad_acc_f32(const void* A, const void* W, float* C, int64_t M, int64_t N, int64_t K, int64_t lda,
                          int64_t ldw, int64_t ldc, int32_t a_mn_major, int32_t w_mn_major, lv_stream_t stream) {
  int r = check_gemm_args("lv_gemm_wgrad_acc_f32", A, W, nullptr, C, M, N, K, lda, ldw, ldc, a_mn_major, w_mn_major, 0,
                          true, true);
  if (r) return r;
  if (M == 0 || K == 0) return LV_OK;      // nothing to add
  LV_BIND_DEVICE(A);
  return launch_gemm<true, true, true>(A, W, nullptr, C, M, N, K, lda, ldw, ldc, 0, (cudaStream_t)stream);
}

int64_t lv_patch_embed_ws_bytes(int64_t n, int64_t img, int64_t ps, int64_t C) {
  const int64_t P = (img / ps) * (img / ps);
  const int64_t kpad = ((3 * ps * ps + 63) / 64) * 64;
  return n * P * (kpad + C) * 2;
}

int lv_patch_embed(const void* images, const void* W, const void* bias, const void* cls, const void* pos, void* out,
                   void* ws, int64_t n, int64_t img, int64_t ps, int64_t C, lv_stream_t stream) {
  LV_CHECK_ARG(images && W && pos && out && ws, "lv_patch_embed: null pointer");
  LV_CHECK_ARG(img > 0 && ps > 0 && img % ps == 0 && C % 8 == 0, "lv_patch_embed: bad geometry img=%lld ps=%lld C=%lld", (long long)img, (long long)ps, (long long)C);
  if (n == 0) return LV_OK;
  LV_BIND_DEVICE(images);
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t P = (img / ps) * (img / ps);
  const int64_t kpad = ((3 * ps * ps + 63) / 64) * 64;
  LV_CHECK_ARG(n * (P + 1) < (1ll << 31), "lv_patch_embed: too many tokens");
  __nv_bfloat16* col = reinterpret_cast<__nv_bfloat16*>(ws);
  __nv_bfloat16* tmp = col + n * P * kpad;
  im2col_patch_kernel<<<(unsigned)(n * P), 128, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(images), col, n, (int)img,
                                                       (int)ps, (int)kpad);
  LV_CHECK_LAUNCH("im2col_patch_kernel");
  int r = launch_gemm<false, false>(col, W, bias, tmp, n * P, C, kpad, kpad, kpad, C, 0, s);
  if (r) return r;
  add_cls_pos_kernel<<<(unsigned)(n * (P + (cls != nullptr ? 1 : 0))), 128, 0, s>>>(tmp, reinterpret_cast<const __nv_bfloat16*>(cls),
                                                           reinterpret_cast<const __nv_bfloat16*>(pos),
                                                           reinterpret_cast<__nv_bfloat16*>(out), n, (int)P, (int)C);
  LV_CHECK_LAUNCH("add_cls_pos_kernel");
  return LV_OK;
}

int lv_patch_im2col(const void* images, void* col, int64_t n, int64_t img, int64_t ps, int64_t kpad, lv_stream_t stream) {
  LV_CHECK_ARG(images && col, "lv_patch_im2col: null pointer");
  LV_CHECK_ARG(n >= 0 && img > 0 && ps > 0 && img % ps == 0, "lv_patch_im2col: bad geometry img=%lld ps=%lld", (long long)img, (long long)ps);
  LV_CHECK_ARG(kpad >= 3 * ps * ps && kpad % 8 == 0 && kpad < (1ll << 31), "lv_patch_im2col: kpad=%lld must be a multiple of 8 and >= 3*ps*ps", (long long)kpad);
  LV_CHECK_ARG((reinterpret_cast<uintptr_t>(images) & 15) == 0 && (reinterpret_cast<uintptr_t>(col) & 15) == 0,
               "lv_patch_im2col: pointers must be 16-byte aligned");
  if (n == 0) return LV_OK;
  const int64_t P = (img / ps) * (img / ps);
  LV_CHECK_ARG(n * P < (1ll << 31), "lv_patch_im2col: too many patches");
  LV_BIND_DEVICE(images);
  im2col_patch_kernel<<<(unsigned)(n * P), 128, 0, (cudaStream_t)stream>>>(reinterpret_cast<const __nv_bfloat16*>(images),
                                                                         reinterpret_cast<__nv_bfloat16*>(col), n, (int)img,
                                                                         (int)ps, (int)kpad);
  LV_CHECK_LAUNCH("im2col_patch_kernel");
  return LV_OK;
}

}  // extern "C"
