// FP8 (e4m3) attention forward for sm_90a, opt-in and lossy: causal softmax(scale * Q K^T) V with GQA and d = 128 on
// the FP8 tensor cores, the operand rule of csrc/attn_fp8_core.h.  Two kernels:
//   attn_fp8_quant_kv_kernel  bf16 K and V (strided views, V following K in a QKV or K|V buffer) -> K8, Vt8 and their
//                             per-block scales, one CTA per (128-key block, kv head, K or V), one HBM pass
//   attn_fwd_fp8_kernel       attn_fwd_kernel's structure and schedule (attn_fwd.cu, attn_sched.cuh): persistent, one
//                             TMA producer warp with a 2-deep K ring and V ring and the same mbarrier protocol, two
//                             consumer warpgroups of 64 query rows, the same work list and longest-first /
//                             boustrophedon order.  What differs is the arithmetic:
//     - each consumer quantises its 64 rows of the bf16 Q tile (one scale) into an e4m3 copy in shared memory;
//     - S = Q8 K8^T with wgmma m64n128k32 e4m3, scaled once per tile by s_q s_k scale log2(e);
//     - P = exp2(s - m) in fp32 feeds the row sum; e4m3(P * 2^8) is packed in registers straight into the A fragment
//       (the key permutation of the Vt8 layout makes the accumulator layout of S that fragment);
//     - promotion: P V accumulates in a fresh fp32 register set per key tile and O = alpha O + (s_v / 2^8) acc, so the
//       tensor cores' reduced-precision FP8 accumulation never spans more than one 128-key tile (gemm_fp8.cu does the
//       same per 128-deep k-block).
// Epilogue and LSE are those of attn_fwd_kernel.
#include <cuda_bf16.h>
#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "attn_fp8_core.h"
#include "attn_sched.cuh"
#include "common.cuh"
#include "ptx.cuh"

namespace lv {

constexpr int F8A_THREADS = 384;
constexpr int F8A_NS = 2;                          // K / V ring depth, as attn_fwd_kernel at d = 128
constexpr int F8A_TILE = 128 * 128;                // one 128-row e4m3 tile of K8 or Vt8: 16 KB
constexpr int F8A_SMEM_Q = 128 * 128 * 2;          // the bf16 Q tile (then the O staging)
constexpr int F8A_SMEM_Q8 = 128 * 128;             // its e4m3 copy, 64 rows per consumer warpgroup
constexpr int F8A_SMEM_TOTAL = F8A_SMEM_Q + F8A_SMEM_Q8 + 2 * F8A_NS * F8A_TILE + 256 + 1024;

struct Fp8KvParams {
  const float* k_scale;   // [b][hkv][nt]
  const float* v_scale;
  int nt;                 // key blocks per (b, kv head)
};

__device__ __forceinline__ void unpack_bf16x8(const uint4& v, float (&f)[8]) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 p = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&w[i]));
    f[2 * i] = p.x;
    f[2 * i + 1] = p.y;
  }
}

// four fp32 values (already scaled) -> four e4m3 bytes, a in the low byte
__device__ __forceinline__ uint32_t pack_e4m3x4(float a, float b, float c, float d) {
  return (uint32_t)lv_fp8_pack2(LV_FP8_E4M3, a, b) | ((uint32_t)lv_fp8_pack2(LV_FP8_E4M3, c, d) << 16);
}

// ---------------------------------------------------------------------------------------------------------------------
// K / V quantiser.  256 threads: thread t takes row t / 2 of the block and the 64 head-dim values (t % 2) * 64 .. + 63
// (eight 16-byte loads).  amax over the block (warp shuffles, then the 8 warps through shared memory; max is exact in
// any order), then the products x * inv as lv_fp8_quant_row computes them.  A K block goes straight out as 64-byte row
// pieces; a V block goes through shared memory and leaves transposed, byte kappa of a row holding key
// lv_attn8_key_of(kappa).  Rows at or past sk are read as zeros and written as zeros.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    attn_fp8_quant_kv_kernel(const __nv_bfloat16* __restrict__ k, const __nv_bfloat16* __restrict__ v, long long ks0,
                             long long ks1, long long ks2, long long vs0, long long vs1, long long vs2, int sk, int hkv,
                             int nt, uint8_t* __restrict__ k8, uint8_t* __restrict__ vt8, float* __restrict__ k_scale,
                             float* __restrict__ v_scale) {
  __shared__ float warp_max[8];
  __shared__ __align__(16) uint8_t tq[128 * 128];   // the quantised V block, [key][d]
  const int tile = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z >> 1, is_v = blockIdx.z & 1;
  const int r = threadIdx.x >> 1, h = threadIdx.x & 1;
  const int row = tile * 128 + r;
  uint4 x[8];
  if (row < sk) {
    const __nv_bfloat16* src = is_v ? v + b * vs0 + row * vs1 + kvh * vs2 : k + b * ks0 + row * ks1 + kvh * ks2;
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = *reinterpret_cast<const uint4*>(src + h * 64 + 8 * i);
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = make_uint4(0u, 0u, 0u, 0u);
  }
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float f[8];
    unpack_bf16x8(x[i], f);
#pragma unroll
    for (int e = 0; e < 8; ++e) amax = fmaxf(amax, fabsf(f[e]));
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, off));
  if ((threadIdx.x & 31) == 0) warp_max[threadIdx.x >> 5] = amax;
  __syncthreads();
#pragma unroll
  for (int w = 0; w < 8; ++w) amax = fmaxf(amax, warp_max[w]);
  const float inv = lv_fp8_inv(LV_FP8_E4M3, amax);
  const bool zero = lv_fp8_zero_row(inv);
  uint32_t q[16];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float f[8];
    unpack_bf16x8(x[i], f);
    q[2 * i] = zero ? 0u : pack_e4m3x4(__fmul_rn(f[0], inv), __fmul_rn(f[1], inv), __fmul_rn(f[2], inv), __fmul_rn(f[3], inv));
    q[2 * i + 1] = zero ? 0u : pack_e4m3x4(__fmul_rn(f[4], inv), __fmul_rn(f[5], inv), __fmul_rn(f[6], inv), __fmul_rn(f[7], inv));
  }
  const long long blk = (long long)(b * hkv + kvh) * nt + tile;
  const float scale = zero ? 0.f : lv_fp8_scale(LV_FP8_E4M3, amax);
  if (!is_v) {
    uint4* dst = reinterpret_cast<uint4*>(k8 + (blk * 128 + r) * 128 + h * 64);
#pragma unroll
    for (int j = 0; j < 4; ++j) dst[j] = make_uint4(q[4 * j], q[4 * j + 1], q[4 * j + 2], q[4 * j + 3]);
    if (threadIdx.x == 0) k_scale[blk] = scale;
    return;
  }
  uint4* st = reinterpret_cast<uint4*>(tq + r * 128 + h * 64);
#pragma unroll
  for (int j = 0; j < 4; ++j) st[j] = make_uint4(q[4 * j], q[4 * j + 1], q[4 * j + 2], q[4 * j + 3]);
  __syncthreads();
  // transposed: thread t writes head-dim row n = t / 2, bytes kappa = (t % 2) * 64 .. + 63
  const int n = r;
  uint32_t o[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    uint32_t word = 0;
#pragma unroll
    for (int e = 0; e < 4; ++e) word |= (uint32_t)tq[lv_attn8_key_of(h * 64 + 4 * j + e) * 128 + n] << (8 * e);
    o[j] = word;
  }
  uint4* dst = reinterpret_cast<uint4*>(vt8 + (blk * 128 + n) * 128 + h * 64);
#pragma unroll
  for (int j = 0; j < 4; ++j) dst[j] = make_uint4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
  if (threadIdx.x == 0) v_scale[blk] = scale;
}

// ---------------------------------------------------------------------------------------------------------------------
// Q of one consumer warpgroup: its 64 rows of the bf16 tile (two 128-byte-swizzled boxes of 64 columns) -> e4m3 rows of
// 128 bytes in its 8 KB of sQ8, 128-byte swizzled as TMA would write them.  Thread t takes row t / 2 and the columns
// (t % 2) * 64 .. + 63.  Returns the group's scale (0 for an all-zero group).
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float quant_q_rows(const uint8_t* sQ, uint8_t* sQ8, int c, int wg_tid, float* red) {
  const int rl = wg_tid >> 1, h = wg_tid & 1;
  const int r = c * 64 + rl;
  const uint8_t* src = sQ + h * 16384 + r * 128;
  uint4 x[8];
#pragma unroll
  for (int ch = 0; ch < 8; ++ch) x[ch] = *reinterpret_cast<const uint4*>(src + ((ch ^ (r & 7)) << 4));
  float amax = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float f[8];
    unpack_bf16x8(x[i], f);
#pragma unroll
    for (int e = 0; e < 8; ++e) amax = fmaxf(amax, fabsf(f[e]));
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, off));
  if ((wg_tid & 31) == 0) red[wg_tid >> 5] = amax;
  named_bar_sync(1 + c, 128);
  amax = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  const float inv = lv_fp8_inv(LV_FP8_E4M3, amax);
  const bool zero = lv_fp8_zero_row(inv);
  uint8_t* dst = sQ8 + c * 8192 + rl * 128;
#pragma unroll
  for (int j = 0; j < 4; ++j) {        // 16-byte chunk 4 h + j of the e4m3 row = bf16 chunks 2 j, 2 j + 1
    uint32_t w[4];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      float f[8];
      unpack_bf16x8(x[2 * j + u], f);
      w[2 * u] = zero ? 0u : pack_e4m3x4(__fmul_rn(f[0], inv), __fmul_rn(f[1], inv), __fmul_rn(f[2], inv), __fmul_rn(f[3], inv));
      w[2 * u + 1] = zero ? 0u : pack_e4m3x4(__fmul_rn(f[4], inv), __fmul_rn(f[5], inv), __fmul_rn(f[6], inv), __fmul_rn(f[7], inv));
    }
    *reinterpret_cast<uint4*>(dst + (((4 * h + j) ^ (rl & 7)) << 4)) = make_uint4(w[0], w[1], w[2], w[3]);
  }
  fence_proxy_async_smem();           // the generic stores above are read by wgmma (async proxy)
  named_bar_sync(1 + c, 128);
  return zero ? 0.f : lv_fp8_scale(LV_FP8_E4M3, amax);
}

__global__ void __launch_bounds__(F8A_THREADS, 1)
    attn_fwd_fp8_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmO,
                        const AttnKParams p, const Fp8KvParams f) {
  constexpr int NS = F8A_NS;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sQ8 = sQ + F8A_SMEM_Q;
  uint8_t* sK = sQ8 + F8A_SMEM_Q8;
  uint8_t* sV = sK + NS * F8A_TILE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + NS * F8A_TILE);
  uint64_t* q_full = bars;            // [1]
  uint64_t* q_empty = bars + 1;       // [1]: both consumer warpgroups have stored their O half out of the Q tile
  uint64_t* k_full = bars + 2;        // [NS]
  uint64_t* k_empty = bars + 2 + NS;  // [NS]
  uint64_t* v_full = bars + 2 + 2 * NS;
  uint64_t* v_empty = bars + 2 + 3 * NS;
  float* red = reinterpret_cast<float*>(bars + 16);   // [2][4]: the Q amax of each consumer's four warps

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    tma_prefetch_desc(&tmO);
    mbar_init(q_full, 1);
    mbar_init(q_empty, 2);
    for (int i = 0; i < NS; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 2);
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
    if (warp == 0 && lane == 0) {
      // =========================== TMA producer (attn_fwd_kernel's, over the e4m3 tiles) ===========================
      uint32_t item_cnt = 0, kcnt = 0, vcnt = 0;
      for (int round = 0, item; (item = sched_item(round, p.n_items, p.serpentine)) >= 0; ++round, ++item_cnt) {
        const WorkItem w = decode_item<false>(p, item);
        const int row_base = (w.b * p.hkv + w.kvh) * f.nt * A_BN;   // row of key block 0 in the K8 / Vt8 maps
        const int pre = min(NS, w.n);
        auto load_tile = [&](int j) {
          {
            const int st = kcnt % NS;
            mbar_wait(&k_empty[st], ((kcnt / NS) & 1) ^ 1);
            mbar_arrive_expect_tx(&k_full[st], F8A_TILE);
            tma_load_2d(sK + st * F8A_TILE, &tmK, &k_full[st], 0, row_base + j * A_BN, kEvictLast);
            ++kcnt;
          }
          {
            const int st = vcnt % NS;
            mbar_wait(&v_empty[st], ((vcnt / NS) & 1) ^ 1);
            mbar_arrive_expect_tx(&v_full[st], F8A_TILE);
            tma_load_2d(sV + st * F8A_TILE, &tmV, &v_full[st], 0, row_base + j * A_BN, kEvictLast);
            ++vcnt;
          }
        };
        for (int j = 0; j < pre; ++j) load_tile(j);
        mbar_wait(q_empty, (item_cnt & 1) ^ 1);
        mbar_arrive_expect_tx(q_full, F8A_SMEM_Q);
        for (int bx = 0; bx < 2; ++bx) tma_load_4d(sQ + bx * 16384, &tmQ, q_full, bx * 64, w.row0, w.h, w.b, kEvictFirst);
        for (int j = pre; j < w.n; ++j) load_tile(j);
      }
    }
  } else {
    // =========================== consumer warpgroups ===========================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
    const int c = (warp >> 2) - 1;                // 64-row half of the query tile
    const int wg_tid = threadIdx.x & 127;
    const int r_lo = ((wg_tid >> 5) << 4) + (lane >> 2);   // this thread's rows: r_lo and r_lo + 8 (of 64)
    const int cq = 2 * (lane & 3);                         // its first column in every 8-column group
    // K-major operands: 128-byte rows (128 e4m3), 8-row groups 1024 B apart, a k32 step is +32 B (+2 in the descriptor)
    const uint64_t qdesc = make_smem_desc(smem_u32(sQ8) + c * 8192, 16, 1024);
    const uint64_t kdesc0 = make_smem_desc(smem_u32(sK), 16, 1024);
    const uint64_t vdesc0 = make_smem_desc(smem_u32(sV), 16, 1024);
    const int n_kv_tiles = (p.sk + A_BN - 1) / A_BN;
    const int j_ragged = (p.sk % A_BN) ? n_kv_tiles - 1 : 0x7fffffff;
    uint32_t item_cnt = 0, kcnt = 0, vcnt = 0;

    for (int round = 0, item; (item = sched_item(round, p.n_items, p.serpentine)) >= 0; ++round, ++item_cnt) {
      const WorkItem w = decode_item<false>(p, item);
      const int n = w.n;
      const long long qpos0 = w.qpos + c * 64 + r_lo, qpos1 = qpos0 + 8;
      // first key tile that needs a mask: the diagonal ones and the ragged last one
      int j_mask = j_ragged;
      if (p.causal) {
        const long long dd = w.qpos + c * 64 - p.kv_pos0 - (A_BN - 1);
        const long long jd = dd < 0 ? 0 : dd / A_BN + 1;
        if (jd < j_mask) j_mask = (int)jd;
      }
      const float* ks = f.k_scale + (long long)(w.b * p.hkv + w.kvh) * f.nt;
      const float* vs = f.v_scale + (long long)(w.b * p.hkv + w.kvh) * f.nt;
      float o[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) o[i] = 0.f;
      float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // running max (log2 domain) and sum per row
      mbar_wait(q_full, item_cnt & 1);
      const float qs_log2 = quant_q_rows(sQ, sQ8, c, wg_tid, red + 4 * c) * p.scale_log2;
      for (int j = 0; j < n; ++j) {
        const float sk_j = __ldg(ks + j), sv_j = __ldg(vs + j) * (1.f / 256.f);
        const int kst = kcnt % NS;
        mbar_wait(&k_full[kst], (kcnt / NS) & 1);
        ++kcnt;
        float s[64];
        wgmma_fence();
        {
          const uint64_t kdesc = kdesc0 + (uint64_t)((kst * F8A_TILE) >> 4);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) wgmma_ss_n128_e4m3(s, qdesc + 2 * kk, kdesc + 2 * kk, kk != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_keep(s);
        if (wg_tid == 0) mbar_arrive(&k_empty[kst]);
        // log2-domain logit = s * cs.  A zero scale (an all-zero Q group or K block, whose products are exact zeros)
        // becomes the smallest normal float, so that a masked -inf stays -inf instead of becoming -inf * 0 = NaN.
        const float cs = fmaxf(qs_log2 * sk_j, FLT_MIN);

        // ---- mask (only diagonal tiles and the ragged last key tile) ----
        if (j >= j_mask) {
          const long long kidx0 = (long long)j * A_BN;
          long long lim0 = p.sk - kidx0, lim1 = lim0;                 // first invalid column of each row
          if (p.causal) {
            lim0 = min(lim0, qpos0 - p.kv_pos0 - kidx0 + 1);
            lim1 = min(lim1, qpos1 - p.kv_pos0 - kidx0 + 1);
          }
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = 8 * jj + cq + e;
              if (col >= lim0) s[4 * jj + e] = -INFINITY;
              if (col >= lim1) s[4 * jj + 2 + e] = -INFINITY;
            }
          }
        }

        // ---- online softmax: row max over the quad of threads that holds a row ----
        float mx0 = s[0], mx1 = s[2];
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          mx0 = fmaxf(mx0, fmaxf(s[4 * jj], s[4 * jj + 1]));
          mx1 = fmaxf(mx1, fmaxf(s[4 * jj + 2], s[4 * jj + 3]));
        }
#pragma unroll
        for (int off = 1; off <= 2; off <<= 1) {
          mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, off));
          mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, off));
        }
        const float mn0 = fmaxf(m0, mx0 * cs), mn1 = fmaxf(m1, mx1 * cs);
        // a row that has seen only masked keys keeps max -inf: subtract 0 instead (its P and alpha are 0)
        const float ms0 = mn0 == -INFINITY ? 0.f : mn0, ms1 = mn1 == -INFINITY ? 0.f : mn1;
        const float alpha0 = ex2(m0 - ms0), alpha1 = ex2(m1 - ms1);
        m0 = mn0;
        m1 = mn1;
        l0 *= alpha0;
        l1 *= alpha1;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          s[4 * jj] = ex2(fmaf(s[4 * jj], cs, -ms0));
          s[4 * jj + 1] = ex2(fmaf(s[4 * jj + 1], cs, -ms0));
          s[4 * jj + 2] = ex2(fmaf(s[4 * jj + 2], cs, -ms1));
          s[4 * jj + 3] = ex2(fmaf(s[4 * jj + 3], cs, -ms1));
          l0 += s[4 * jj] + s[4 * jj + 1];
          l1 += s[4 * jj + 2] + s[4 * jj + 3];
        }
        // e4m3(p * 2^8) in the A fragment of k-step kc (32 keys): register 0 = row r_lo, keys 8 (4 kc) + cq + 0..1 and
        // 8 (4 kc + 1) + cq + 0..1; register 1 = the same keys of row r_lo + 8; registers 2 / 3 = 8-column groups
        // 4 kc + 2 and 4 kc + 3 (attn_fp8_core.h: lv_attn8_key_of)
        uint32_t pk[16];
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            const float* g = s + 16 * kc + 8 * u;   // 8-column groups 4 kc + 2 u and 4 kc + 2 u + 1
            pk[4 * kc + 2 * u] = pack_e4m3x4(g[0] * 256.f, g[1] * 256.f, g[4] * 256.f, g[5] * 256.f);
            pk[4 * kc + 2 * u + 1] = pack_e4m3x4(g[2] * 256.f, g[3] * 256.f, g[6] * 256.f, g[7] * 256.f);
          }
        }

        // ---- acc = P8 V8 (fresh per tile), then O = alpha O + s_v acc ----
        const int vst = vcnt % NS;
        mbar_wait(&v_full[vst], (vcnt / NS) & 1);
        ++vcnt;
        float acc[64];
        wgmma_fence();
        {
          const uint64_t vdesc = vdesc0 + (uint64_t)((vst * F8A_TILE) >> 4);
#pragma unroll
          for (int kc = 0; kc < 4; ++kc) {
            const uint32_t a[4] = {pk[4 * kc], pk[4 * kc + 1], pk[4 * kc + 2], pk[4 * kc + 3]};
            wgmma_rs_n128_e4m3(acc, a, vdesc + 2 * kc, kc != 0 ? 1u : 0u);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_keep(acc);
        if (wg_tid == 0) mbar_arrive(&v_empty[vst]);
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          o[4 * jj] = fmaf(alpha0, o[4 * jj], sv_j * acc[4 * jj]);
          o[4 * jj + 1] = fmaf(alpha0, o[4 * jj + 1], sv_j * acc[4 * jj + 1]);
          o[4 * jj + 2] = fmaf(alpha1, o[4 * jj + 2], sv_j * acc[4 * jj + 2]);
          o[4 * jj + 3] = fmaf(alpha1, o[4 * jj + 3], sv_j * acc[4 * jj + 3]);
        }
      }

      // ---------------- epilogue (attn_fwd_kernel's): O / l -> bf16 -> smem (this half of the Q tile) -> TMA; LSE -------
#pragma unroll
      for (int off = 1; off <= 2; off <<= 1) {
        l0 += __shfl_xor_sync(0xffffffffu, l0, off);
        l1 += __shfl_xor_sync(0xffffffffu, l1, off);
      }
      const float inv0 = l0 > 0.f ? 1.f / l0 : 0.f, inv1 = l1 > 0.f ? 1.f / l1 : 0.f;
      uint8_t* stage = sQ + c * 8192;
      named_bar_sync(1 + c, 128);    // every thread of this warpgroup is done reading its Q rows
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        uint8_t* box = stage + (jj >> 3) * 16384;
        const int ch = jj & 7;       // 16-byte chunk of the 128-byte row
        *reinterpret_cast<uint32_t*>(box + r_lo * 128 + ((ch ^ (r_lo & 7)) << 4) + cq * 2) =
            pack_bf16(o[4 * jj] * inv0, o[4 * jj + 1] * inv0);
        const int r1 = r_lo + 8;
        *reinterpret_cast<uint32_t*>(box + r1 * 128 + ((ch ^ (r1 & 7)) << 4) + cq * 2) =
            pack_bf16(o[4 * jj + 2] * inv1, o[4 * jj + 3] * inv1);
      }
      if (p.lse != nullptr && (lane & 3) == 0) {
        const int row = w.row0 + c * 64 + r_lo;
        float* dst = p.lse + ((long long)w.b * p.hq + w.h) * p.sq;
        if (row < p.sq) dst[row] = l0 > 0.f ? (m0 + log2f(l0)) * 0.69314718055994530942f : -INFINITY;
        if (row + 8 < p.sq) dst[row + 8] = l1 > 0.f ? (m1 + log2f(l1)) * 0.69314718055994530942f : -INFINITY;
      }
      fence_proxy_async_smem();
      named_bar_sync(1 + c, 128);
      if (wg_tid == 0) {
        if (w.row0 + c * 64 < p.sq) {
          for (int bx = 0; bx < 2; ++bx) tma_store_4d(&tmO, stage + bx * 16384, bx * 64, w.row0 + c * 64, w.h, w.b);
          tma_store_commit();
          tma_store_wait_read0();
        }
        mbar_arrive(q_empty);   // this half of the Q / staging tile may be overwritten by a later item's Q load
      }
    }
    if (wg_tid == 0) tma_store_wait_all0();
  }
}

// TMA map of the K8 or Vt8 rows [rows][128 bytes], encoded as bf16 [rows][64] (csrc/gemm_fp8.cu: encode_fp8_operand):
// one box is a whole 128-row tile, 128-byte swizzled.
static int encode_fp8_tiles(CUtensorMap* m, const void* base, int64_t rows) {
  const uint64_t dims[2] = {64, (uint64_t)rows};
  const uint64_t str[2] = {2, 128};
  const uint32_t box[2] = {64, 128};
  return encode_tmap_bf16(m, base, 2, dims, str, box, true);
}

static int launch_attn_fp8(const lv_attn_params* a, const lv_attn_fp8_kv* kv, cudaStream_t s) {
  const int64_t nt = lv_attn8_blocks(a->sk);
  CUtensorMap tmQ, tmK, tmV, tmO;
  {
    const uint32_t box[4] = {64, 128, 1, 1};
    const uint32_t obox[4] = {64, 64, 1, 1};    // each consumer warpgroup stores its own 64 rows
    const uint64_t dims[4] = {128, (uint64_t)a->sq, (uint64_t)a->hq, (uint64_t)a->batch};
    const uint64_t str[4] = {2, (uint64_t)a->q_strides[1] * 2, (uint64_t)a->q_strides[2] * 2, (uint64_t)a->q_strides[0] * 2};
    int r = encode_tmap_bf16(&tmQ, a->q, 4, dims, str, box, true);
    if (r) return r;
    const uint64_t ostr[4] = {2, (uint64_t)a->o_strides[1] * 2, (uint64_t)a->o_strides[2] * 2, (uint64_t)a->o_strides[0] * 2};
    r = encode_tmap_bf16(&tmO, a->out, 4, dims, ostr, obox, true);
    if (r) return r;
  }
  int r = encode_fp8_tiles(&tmK, kv->k8, a->batch * a->hkv * nt * 128);
  if (r) return r;
  r = encode_fp8_tiles(&tmV, kv->vt8, a->batch * a->hkv * nt * 128);
  if (r) return r;
  AttnKParams p;
  attn_sched_params(a, p);
  p.lse = a->lse;
  p.docs = DocsKParams{nullptr, 0};
  const Fp8KvParams f{kv->k_scale, kv->v_scale, (int)nt};
  static PerDeviceOnce attr_once;
  int attr_dev;
  if (attr_once.needed(&attr_dev)) {
    LV_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd_fp8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, F8A_SMEM_TOTAL));
    attr_once.done(attr_dev);
  }
  const int grid = p.n_items < sm_count() ? p.n_items : sm_count();
  attn_fwd_fp8_kernel<<<grid, F8A_THREADS, F8A_SMEM_TOTAL, s>>>(tmQ, tmK, tmV, tmO, p, f);
  LV_CHECK_LAUNCH("attn_fwd_fp8_kernel");
  return LV_OK;
}

}  // namespace lv

using namespace lv;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

static int check_fp8_kv(const lv_attn_params* a, const lv_attn_fp8_kv* kv, const char* who) {
  LV_CHECK_ARG(a != nullptr && kv != nullptr, "%s: null params", who);
  LV_CHECK_ARG(kv->k8 && kv->vt8 && kv->k_scale && kv->v_scale, "%s: null K8 / Vt8 / scale pointer", who);
  LV_CHECK_ARG(aligned16(kv->k8) && aligned16(kv->vt8), "%s: K8 and Vt8 must be 16-byte aligned", who);
  LV_CHECK_ARG(a->d == 128, "%s: head_dim %lld not supported (128 only)", who, (long long)a->d);
  LV_CHECK_ARG(a->batch > 0 && a->sk > 0 && a->hkv > 0, "%s: empty shape", who);
  LV_CHECK_ARG(a->sk < (1ll << 30), "%s: sequence too long", who);
  // rows of the K8 / Vt8 maps and the int coordinates of the kernels
  LV_CHECK_ARG(a->batch * a->hkv * lv_attn8_blocks(a->sk) * 128 < (1ll << 31), "%s: too many key rows", who);
  return LV_OK;
}

extern "C" int lv_attn_fp8_quant_kv(const lv_attn_params* a, const lv_attn_fp8_kv* kv, lv_stream_t stream) {
  int rc = check_fp8_kv(a, kv, "lv_attn_fp8_quant_kv");
  if (rc) return rc;
  LV_CHECK_ARG(a->k && a->v, "lv_attn_fp8_quant_kv: null k / v");
  LV_CHECK_ARG(aligned16(a->k) && aligned16(a->v), "lv_attn_fp8_quant_kv: k and v must be 16-byte aligned");
  for (int i = 0; i < 3; ++i)
    LV_CHECK_ARG(a->k_strides[i] % 8 == 0 && a->v_strides[i] % 8 == 0,
                 "lv_attn_fp8_quant_kv: strides must be multiples of 8 elements (16 bytes)");
  LV_CHECK_ARG(a->batch <= 32767 && a->hkv <= 65535, "lv_attn_fp8_quant_kv: batch / hkv out of range");
  LV_BIND_DEVICE(a->k);
  const int64_t nt = lv_attn8_blocks(a->sk);
  const dim3 grid((unsigned)nt, (unsigned)a->hkv, (unsigned)(2 * a->batch));
  attn_fp8_quant_kv_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(a->k), reinterpret_cast<const __nv_bfloat16*>(a->v), a->k_strides[0],
      a->k_strides[1], a->k_strides[2], a->v_strides[0], a->v_strides[1], a->v_strides[2], (int)a->sk, (int)a->hkv,
      (int)nt, reinterpret_cast<uint8_t*>(kv->k8), reinterpret_cast<uint8_t*>(kv->vt8), kv->k_scale, kv->v_scale);
  LV_CHECK_LAUNCH("attn_fp8_quant_kv_kernel");
  return LV_OK;
}

extern "C" int lv_attn_fwd_fp8(const lv_attn_params* a, const lv_attn_fp8_kv* kv, lv_stream_t stream) {
  int rc = check_fp8_kv(a, kv, "lv_attn_fwd_fp8");
  if (rc) return rc;
  LV_CHECK_ARG(a->q && a->out, "lv_attn_fwd_fp8: null q / out");
  LV_CHECK_ARG(a->sq > 0 && a->hq > 0, "lv_attn_fwd_fp8: empty shape");
  LV_CHECK_ARG(a->hq % a->hkv == 0, "lv_attn_fwd_fp8: hq=%lld is not a multiple of hkv=%lld", (long long)a->hq,
               (long long)a->hkv);
  LV_CHECK_ARG(a->scale > 0.f && isfinite(a->scale), "lv_attn_fwd_fp8: scale %g must be finite and > 0", (double)a->scale);
  LV_CHECK_ARG(a->batch * a->hq * ((a->sq + 127) / 128) < (1ll << 31), "lv_attn_fwd_fp8: too many work items");
  LV_CHECK_ARG(a->causal == 1 && a->sq <= a->sk && a->q_seg_len == a->sq && a->q_seg_pos[0] == a->sk - a->sq &&
                   a->q_seg_pos[1] == 0 && a->kv_pos0 == 0,
               "lv_attn_fwd_fp8: only causal attention with sq <= sk, the mask aligned to the last key, is built (no "
               "query segments, no kv_pos0)");
  for (int i = 0; i < 3; ++i)
    LV_CHECK_ARG(a->q_strides[i] % 8 == 0 && a->o_strides[i] % 8 == 0,
                 "lv_attn_fwd_fp8: strides must be multiples of 8 elements (16 bytes)");
  LV_BIND_DEVICE(a->q);
  return launch_attn_fp8(a, kv, (cudaStream_t)stream);
}
