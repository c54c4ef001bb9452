// Attention backward for sm_90a (wgmma / TMA), deterministic two-pass formulation:
//
//   prep   : delta[b,h,i] = sum_d dO[b,i,h,d] * O[b,i,h,d]                         (HBM-bound)
//   pass A : dK, dV.  One CTA owns a 128-row K/V tile (resident in shared memory) and streams the
//            Q / dO tiles of every query head of its GQA group that can see it.
//   pass B : dQ.  One CTA owns a 128-row Q / dO tile and streams the K / V tiles it can see.
//
// Recomputing S in both passes costs 7 GEMM-units instead of the minimal 5, but needs no atomics
// (bit-reproducible dQ) and no dQ transposes.
//
// Document mode (DOCS, lv_attn_docs_bwd; see docs.cuh): pass B's key steps start at the 64-key tile holding the
// document start of the query tile's first row; pass A streams a 64-row query tile only if it starts before the end of
// the document of the key tile's last key.  Per element, a key is visible iff it is not after the query and lies in
// its document: kpos >= doc_start(qpos) in pass B (queries are rows), qpos < doc_end(kpos) in pass A (keys are rows) -
// the same predicate for kpos <= qpos, evaluated on the row side so it costs one lookup per row and item.
//
// Replaces flash-attn 2's backward, reached in the reference through autograd of
// flash_attn_func / TE AttnFuncWithCP (dot_product_attention.py:318-326, 374-390).
#include <cuda_bf16.h>
#include <math.h>
#include <string.h>

#include <stdlib.h>

#include "common.cuh"
#include "docs.cuh"
#include "ptx.cuh"

namespace lv {

struct BwdKParams {
  int batch, sq, sk, hq, hkv;
  int causal;
  float scale, scale_log2;
  int q_seg_len;
  long long q_seg_pos0, q_seg_pos1, kv_pos0;
  int n_qt, n_kt;       // 128-row tiles along q / kv
  int n_items;
  const float* lse;     // [b, hq, sq] natural log
  const float* delta;   // [b, hq, sq]
  DocsKParams docs;     // document mode only
};

// delta = rowsum(dO * O)
__global__ void __launch_bounds__(256) attn_bwd_prep_kernel(const __nv_bfloat16* __restrict__ o,
                                                            const __nv_bfloat16* __restrict__ d_o, float* __restrict__ delta,
                                                            int batch, int sq, int hq, int d, long long os_b, long long os_s,
                                                            long long os_h, long long ds_b, long long ds_s, long long ds_h) {
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long total = (long long)batch * sq * hq;
  if (warp >= total) return;
  const int h = (int)(warp % hq);
  const int i = (int)((warp / hq) % sq);
  const int b = (int)(warp / ((long long)hq * sq));
  const __nv_bfloat16* po = o + b * os_b + i * os_s + h * os_h;
  const __nv_bfloat16* pd = d_o + b * ds_b + i * ds_s + h * ds_h;
  float acc = 0.f;
  for (int c = lane * 2; c < d; c += 64) {
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(po + c));
    const float2 g = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(pd + c));
    acc += a.x * g.x + a.y * g.y;
  }
#pragma unroll
  for (int o2 = 16; o2 > 0; o2 >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o2);
  if (lane == 0) delta[((long long)b * hq + h) * sq + i] = acc;
}

// MODE 0: dK/dV pass (resident = 128-row K, V tile; streamed = 64-row Q, dO tiles of every query head of the group).
// MODE 1: dQ pass (resident = 128-row Q, dO tile; streamed = 64-row K, V tiles).
// One persistent CTA per SM, 3 warpgroups: warp 0 is the TMA producer (resident tiles per item, streamed tiles in a
// BW_STAGES ring); warpgroups 1-2 own 64 rows each of the resident tile and run, per streamed tile,
//   MODE 0:  S^T = K Q^T, dP^T = V dO^T (wgmma, both operands in shared memory),
//            P^T = exp2(S^T * scale_log2 - lse2[q]), dS^T = P^T * (dP^T - delta[q]) * scale,
//            dV += P^T dO, dK += dS^T Q (wgmma with P^T / dS^T from registers, dO / Q as MN-major operands)
//   MODE 1:  S = Q K^T, dP = dO V^T, dS = P * (dP - delta[i]) * scale, dQ += dS K
// with the accumulators in registers; the epilogue stages the bf16 result in the warpgroup's half of the resident
// tile and stores it with TMA.
constexpr int BW_THREADS = 384;
constexpr int BW_STAGES = 3;

template <int D>
struct BwdCfg {
  static constexpr int RES_TILE = 128 * D * 2;   // resident 128-row tile (64-column boxes of 16 KB)
  static constexpr int STR_TILE = 64 * D * 2;    // streamed 64-row tile (64-column boxes of 8 KB)
  // + barriers (128 B) + per-warpgroup column statistics of pass A (2 x 2 x 128 floats) + align slack
  static constexpr int SMEM = 2 * RES_TILE + 2 * BW_STAGES * STR_TILE + 128 + 2048 + 1024;
};

__device__ __forceinline__ long long q_row_pos(const BwdKParams& p, int row0) {
  const int seg = row0 / p.q_seg_len;
  return (seg == 0 ? p.q_seg_pos0 : p.q_seg_pos1) + (row0 - seg * p.q_seg_len);
}

// MODE 0: does the 64-row query tile qt see any key of [key0, key0 + nkeys)?  (64-row tiles never straddle segments)
__device__ __forceinline__ bool q_sees(const BwdKParams& p, int qt, long long key0) {
  return !p.causal || p.kv_pos0 + key0 <= q_row_pos(p, qt * 64) + 63;
}

// X[64 x 64] = A[64 rows of a resident tile] . B[64-row streamed tile]^T over the head dimension
template <int D>
__device__ __forceinline__ void mma_rows(float (&x)[32], uint64_t adesc, uint64_t bdesc) {
#pragma unroll
  for (int kk = 0; kk < D / 16; ++kk)
    wgmma_ss_n64(x, adesc + (((kk / 4) * 16384 + (kk % 4) * 32) >> 4), bdesc + (((kk / 4) * 8192 + (kk % 4) * 32) >> 4),
                 kk != 0 ? 1u : 0u);
}

// acc[64 x D] += X[64 x 64] (bf16 pairs in the accumulator layout) . B[64-row streamed tile] (MN-major)
template <int D>
__device__ __forceinline__ void mma_acc(float (&acc)[D / 2], const uint32_t (&xk)[16], uint64_t bdesc) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint32_t a[4] = {xk[4 * kk], xk[4 * kk + 1], xk[4 * kk + 2], xk[4 * kk + 3]};
    if constexpr (D == 128)
      wgmma_rs_n128(acc, a, bdesc + (uint64_t)(kk * 128), 1u);
    else
      wgmma_rs_n64(acc, a, bdesc + (uint64_t)(kk * 128), 1u);
  }
}

// Stage a 64 x D fp32 accumulator as bf16 into 64 rows of a 128-row resident tile (128-byte swizzle).
template <int D>
__device__ __forceinline__ void stage_rows(uint8_t* half, const float (&acc)[D / 2], int r_lo, int cq) {
#pragma unroll
  for (int jj = 0; jj < D / 8; ++jj) {
    uint8_t* box = half + (jj >> 3) * 16384;
    const int ch = jj & 7;
    const int r1 = r_lo + 8;
    *reinterpret_cast<uint32_t*>(box + r_lo * 128 + ((ch ^ (r_lo & 7)) << 4) + cq * 2) = pack_bf16(acc[4 * jj], acc[4 * jj + 1]);
    *reinterpret_cast<uint32_t*>(box + r1 * 128 + ((ch ^ (r1 & 7)) << 4) + cq * 2) = pack_bf16(acc[4 * jj + 2], acc[4 * jj + 3]);
  }
}

// Resident tile of a work item.  Causal dQ items run longest-first (the last query tiles see the most keys), which
// balances the static round-robin over the CTAs.
template <int MODE>
__device__ __forceinline__ int item_tile(const BwdKParams& p, int item) {
  const int n = MODE == 0 ? p.n_kt : p.n_qt;
  const int r = item % n;
  return (MODE == 1 && p.causal) ? n - 1 - r : r;
}

template <int D, int MODE, bool DOCS>
__global__ void __launch_bounds__(BW_THREADS, 1)
    attn_bwd_kernel(const __grid_constant__ CUtensorMap tmR0, const __grid_constant__ CUtensorMap tmR1,
                    const __grid_constant__ CUtensorMap tmS0, const __grid_constant__ CUtensorMap tmS1,
                    const __grid_constant__ CUtensorMap tmOut0, const __grid_constant__ CUtensorMap tmOut1,
                    const BwdKParams p) {
  using Cfg = BwdCfg<D>;
  constexpr int NS = BW_STAGES;
  constexpr int BOXES = D / 64;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sR0 = smem;                        // resident operand 0 (K or Q); later the staging tile of output 1
  uint8_t* sR1 = sR0 + Cfg::RES_TILE;         // resident operand 1 (V or dO); later the staging tile of output 0
  uint8_t* sS0 = sR1 + Cfg::RES_TILE;         // streamed operand 0 (Q or K), NS stages
  uint8_t* sS1 = sS0 + NS * Cfg::STR_TILE;    // streamed operand 1 (dO or V), NS stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(sS1 + NS * Cfg::STR_TILE);
  uint64_t* res_full = bars;
  uint64_t* res_empty = bars + 1;             // both warpgroups have stored their outputs out of the resident tiles
  uint64_t* str_full = bars + 2;              // [NS]
  uint64_t* str_empty = bars + 2 + NS;        // [NS]
  float* s_stat = reinterpret_cast<float*>(bars + 16);   // MODE 0: [warpgroup][2 buffers][lse2 x 64 | delta x 64]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int G = p.hq / p.hkv;
  const int n_q64 = (p.sq + 63) / 64;
  const int n_k64 = (p.sk + 63) / 64;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmR0);
    tma_prefetch_desc(&tmR1);
    tma_prefetch_desc(&tmS0);
    tma_prefetch_desc(&tmS1);
    mbar_init(res_full, 1);
    mbar_init(res_empty, 2);
    for (int i = 0; i < NS; ++i) {
      mbar_init(&str_full[i], 1);
      mbar_init(&str_empty[i], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  // Item decoding shared by all roles.  MODE 0: (b, kv head, 128-key tile); MODE 1: (b, head, 128-row query tile).
  // Streamed step list: MODE 0 - every (head of the group, 64-row query tile) that sees the key tile; MODE 1 - the
  // 64-key tiles [0, n) the query tile sees.
  auto n_k_steps = [&](int t) -> int {   // MODE 1: 64-key tiles visible to 128-row query tile t
    if (!p.causal) return n_k64;
    const long long hi = q_row_pos(p, t * 128) + 127 - p.kv_pos0;
    if (hi < 0) return 0;
    return (int)min((long long)n_k64, hi / 64 + 1);
  };
  // MODE 1, document mode: first 64-key tile visible to 128-row query tile t (query row == position there)
  auto k_first = [&](int t) -> int { return DOCS ? doc_start(p.docs, t * 128) / 64 : 0; };
  // MODE 0, document mode: one past the last query row that can see a key of [key0, key0 + 128) - the end of the
  // document holding the last key (< sk) of the range
  auto q_end = [&](int key0) -> int { return DOCS ? doc_end(p.docs, min(key0 + 127, p.sk - 1), p.sk) : 0x7fffffff; };

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (threadIdx.x == 0) {
      // =========================== TMA producer ===========================
      uint32_t item_cnt = 0, scnt = 0;
      auto load_str = [&](int row64, int head, int b) {
        const int st = scnt % NS;
        mbar_wait(&str_empty[st], ((scnt / NS) & 1) ^ 1);
        mbar_arrive_expect_tx(&str_full[st], 2 * Cfg::STR_TILE);
        for (int bx = 0; bx < BOXES; ++bx) {
          tma_load_4d(sS0 + st * Cfg::STR_TILE + bx * 8192, &tmS0, &str_full[st], bx * 64, row64 * 64, head, b, kEvictLast);
          tma_load_4d(sS1 + st * Cfg::STR_TILE + bx * 8192, &tmS1, &str_full[st], bx * 64, row64 * 64, head, b, kEvictLast);
        }
        ++scnt;
      };
      for (int item = blockIdx.x; item < p.n_items; item += gridDim.x, ++item_cnt) {
        const int t = item_tile<MODE>(p, item);
        const int bh = item / (MODE == 0 ? p.n_kt : p.n_qt);   // b * heads + head
        const int heads = MODE == 0 ? p.hkv : p.hq;
        const int b = bh / heads, head = bh % heads;
        mbar_wait(res_empty, (item_cnt & 1) ^ 1);
        mbar_arrive_expect_tx(res_full, 2 * Cfg::RES_TILE);
        for (int bx = 0; bx < BOXES; ++bx) {
          tma_load_4d(sR0 + bx * 16384, &tmR0, res_full, bx * 64, t * 128, head, b, kEvictFirst);
          tma_load_4d(sR1 + bx * 16384, &tmR1, res_full, bx * 64, t * 128, head, b, kEvictFirst);
        }
        if (MODE == 0) {
          const int qend = q_end(t * 128);
          for (int g = 0; g < G; ++g)
            for (int qt = 0; qt < n_q64; ++qt)
              if (q_sees(p, qt, (long long)t * 128) && qt * 64 < qend) load_str(qt, head * G + g, b);
        } else {
          const int n = n_k_steps(t);
          for (int kt = k_first(t); kt < n; ++kt) load_str(kt, head / G, b);
        }
      }
    }
  } else {
    // =========================== consumer warpgroups ===========================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int c = (warp >> 2) - 1;                         // 64-row half of the resident tile
    const int wg_tid = threadIdx.x & 127;
    const int r_lo = ((wg_tid >> 5) << 4) + (lane >> 2);   // this thread's rows: r_lo and r_lo + 8 (of 64)
    const int cq = 2 * (lane & 3);                         // its first column in every 8-column group
    const uint64_t r0desc = make_smem_desc(smem_u32(sR0) + c * 8192, 16, 1024);
    const uint64_t r1desc = make_smem_desc(smem_u32(sR1) + c * 8192, 16, 1024);
    const uint64_t s0desc = make_smem_desc(smem_u32(sS0), 16, 1024);
    const uint64_t s1desc = make_smem_desc(smem_u32(sS1), 16, 1024);
    const uint64_t s0mn = make_smem_desc(smem_u32(sS0), 8192, 1024);   // streamed operand 0 as an MN-major B
    const uint64_t s1mn = make_smem_desc(smem_u32(sS1), 8192, 1024);
    const float scale = p.scale, scale_log2 = p.scale_log2;
    constexpr float LOG2E = 1.4426950408889634f;
    uint32_t item_cnt = 0, scnt = 0, act_cnt = 0;
    for (int item = blockIdx.x; item < p.n_items; item += gridDim.x, ++item_cnt) {
      const int t = item_tile<MODE>(p, item);
      const int bh = item / (MODE == 0 ? p.n_kt : p.n_qt);
      const int heads = MODE == 0 ? p.hkv : p.hq;
      const int b = bh / heads, head = bh % heads;
      float acc0[D / 2], acc1[D / 2];    // MODE 0: dV, dK;  MODE 1: dQ, (unused)
#pragma unroll
      for (int i = 0; i < D / 2; ++i) acc0[i] = acc1[i] = 0.f;
      const int rrow0 = t * 128 + c * 64;                  // first resident row of this warpgroup
      // document mode, per resident row r of this thread: MODE 0 (rows = keys) the number of queries that see key r -
      // they are r .. doc_end(r) - 1 (0 for a row past the end) -, MODE 1 (rows = queries) the start of r's document
      int drow0 = 0, drow1 = 0;
      if (DOCS) {
        const int r0 = rrow0 + r_lo, r1 = r0 + 8;
        if (MODE == 0) {
          drow0 = r0 < p.sk ? doc_end(p.docs, r0, p.sk) - r0 : 0;
          drow1 = r1 < p.sk ? doc_end(p.docs, r1, p.sk) - r1 : 0;
        } else {
          drow0 = doc_start(p.docs, min(r0, p.sq - 1));
          drow1 = doc_start(p.docs, min(r1, p.sq - 1));
        }
      }
      mbar_wait(res_full, item_cnt & 1);

      // one streamed tile: rows / columns -> masking, P, dS, the two accumulating products
      auto step = [&](int row64, int hq_idx, bool active) {
        const int st = scnt % NS;
        mbar_wait(&str_full[st], (scnt / NS) & 1);
        ++scnt;
        if (active) {
          const uint64_t so = (uint64_t)((st * Cfg::STR_TILE) >> 4);
          float x[32], dp[32];
          wgmma_fence();
          mma_rows<D>(x, r0desc, s0desc + so);      // S^T = K Q^T  |  S = Q K^T
          mma_rows<D>(dp, r1desc, s1desc + so);     // dP^T = V dO^T  |  dP = dO V^T
          wgmma_commit();
          const long long stat = ((long long)b * p.hq + hq_idx) * p.sq;
          // MODE 0: the 64 query columns' lse2 and delta, loaded once per tile by the warpgroup while the MMAs run.
          // Two buffers alternate, so a buffer is rewritten only after every thread passed the next step's barrier.
          const float* st_buf = s_stat + (c * 2 + (act_cnt & 1)) * 128;
          if (MODE == 0) {
            const int qi = row64 * 64 + (wg_tid & 63);
            float v = 0.f;
            if (qi < p.sq) v = wg_tid < 64 ? p.lse[stat + qi] * LOG2E : p.delta[stat + qi];
            const_cast<float*>(st_buf)[wg_tid] = v;
            named_bar_sync(1 + c, 128);
          }
          ++act_cnt;
          wgmma_wait<0>();
          wgmma_keep(x);
          wgmma_keep(dp);
          uint32_t pk[16], dsk[16];
          if (MODE == 0) {
            // rows = keys rrow0 + r, columns = queries row64 * 64 + col
            const long long kpos0 = p.kv_pos0 + rrow0 + r_lo, kpos1 = kpos0 + 8;
            const bool kv0 = rrow0 + r_lo < p.sk, kv1 = rrow0 + r_lo + 8 < p.sk;
            const long long qp = q_row_pos(p, row64 * 64);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              float pr[4], ds[4];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int qi = row64 * 64 + 8 * jj + cq + e;
                const bool qv = qi < p.sq;
                const float lse2 = st_buf[8 * jj + cq + e];
                const float dl = st_buf[64 + 8 * jj + cq + e];
                const long long qpos = qp + 8 * jj + cq + e;
                bool vis0, vis1;
                if (DOCS) {   // query qi sees key k iff k <= qi < doc_end(k)
                  vis0 = (unsigned)(qi - (rrow0 + r_lo)) < (unsigned)drow0;
                  vis1 = (unsigned)(qi - (rrow0 + r_lo + 8)) < (unsigned)drow1;
                } else {
                  vis0 = qv && kv0 && (!p.causal || kpos0 <= qpos);
                  vis1 = qv && kv1 && (!p.causal || kpos1 <= qpos);
                }
                pr[e] = vis0 ? ex2(fmaf(x[4 * jj + e], scale_log2, -lse2)) : 0.f;
                pr[2 + e] = vis1 ? ex2(fmaf(x[4 * jj + 2 + e], scale_log2, -lse2)) : 0.f;
                ds[e] = pr[e] * (dp[4 * jj + e] - dl) * scale;
                ds[2 + e] = pr[2 + e] * (dp[4 * jj + 2 + e] - dl) * scale;
              }
              pk[2 * jj] = pack_bf16(pr[0], pr[1]);
              pk[2 * jj + 1] = pack_bf16(pr[2], pr[3]);
              dsk[2 * jj] = pack_bf16(ds[0], ds[1]);
              dsk[2 * jj + 1] = pack_bf16(ds[2], ds[3]);
            }
          } else {
            // rows = queries rrow0 + r, columns = keys row64 * 64 + col
            const int qi0 = rrow0 + r_lo, qi1 = qi0 + 8;
            const bool qv0 = qi0 < p.sq, qv1 = qi1 < p.sq;
            const float lse0 = qv0 ? p.lse[stat + qi0] * LOG2E : 0.f, lse1 = qv1 ? p.lse[stat + qi1] * LOG2E : 0.f;
            const float dl0 = qv0 ? p.delta[stat + qi0] : 0.f, dl1 = qv1 ? p.delta[stat + qi1] : 0.f;
            const long long qpos0 = q_row_pos(p, rrow0) + r_lo, qpos1 = qpos0 + 8;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              float pr[4], ds[4];
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int ki = row64 * 64 + 8 * jj + cq + e;
                const long long kpos = p.kv_pos0 + ki;
                const bool kv = ki < p.sk;
                const bool vis0 = qv0 && kv && (!p.causal || kpos <= qpos0) && (!DOCS || kpos >= drow0);
                const bool vis1 = qv1 && kv && (!p.causal || kpos <= qpos1) && (!DOCS || kpos >= drow1);
                pr[e] = vis0 ? ex2(fmaf(x[4 * jj + e], scale_log2, -lse0)) : 0.f;
                pr[2 + e] = vis1 ? ex2(fmaf(x[4 * jj + 2 + e], scale_log2, -lse1)) : 0.f;
                ds[e] = pr[e] * (dp[4 * jj + e] - dl0) * scale;
                ds[2 + e] = pr[2 + e] * (dp[4 * jj + 2 + e] - dl1) * scale;
              }
              dsk[2 * jj] = pack_bf16(ds[0], ds[1]);
              dsk[2 * jj + 1] = pack_bf16(ds[2], ds[3]);
              pk[2 * jj] = pk[2 * jj + 1] = 0u;
            }
          }
          wgmma_fence();
          if (MODE == 0) {
            mma_acc<D>(acc0, pk, s1mn + so);         // dV += P^T dO
            mma_acc<D>(acc1, dsk, s0mn + so);        // dK += dS^T Q
          } else {
            mma_acc<D>(acc0, dsk, s0mn + so);        // dQ += dS K
          }
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_keep(acc0);
          wgmma_keep(acc1);
        }
        if (wg_tid == 0) mbar_arrive(&str_empty[st]);
      };

      if (MODE == 0) {
        // document mode: a streamed tile this warpgroup's keys cannot see (all its queries past the document of the
        // keys) is masked element-wise; only the 128-key tile's range is skipped
        const int qend = q_end(t * 128);
        for (int g = 0; g < G; ++g)
          for (int qt = 0; qt < n_q64; ++qt)
            if (q_sees(p, qt, (long long)t * 128) && qt * 64 < qend) step(qt, head * G + g, q_sees(p, qt, (long long)rrow0));
      } else {
        const int n = n_k_steps(t);
        const long long my_last = q_row_pos(p, rrow0) + 63 - p.kv_pos0;   // last key index this half sees
        // document mode: the first key this half sees is the document start of its first row
        const int my_first = DOCS ? doc_start(p.docs, min(rrow0, p.sq - 1)) : 0;
        for (int kt = k_first(t); kt < n; ++kt)
          step(kt, head, (!p.causal || (long long)kt * 64 <= my_last) && (!DOCS || kt * 64 + 63 >= my_first));
      }

      // ---------------- epilogue: bf16 outputs staged in this warpgroup's half of the resident tiles -> TMA ----------
      named_bar_sync(1 + c, 128);    // every MMA of this warpgroup that read the resident rows has completed
      stage_rows<D>(sR1 + c * 8192, acc0, r_lo, cq);                  // dV | dQ
      if (MODE == 0) stage_rows<D>(sR0 + c * 8192, acc1, r_lo, cq);   // dK
      fence_proxy_async_smem();
      named_bar_sync(1 + c, 128);
      if (wg_tid == 0) {
        const int nrow = MODE == 0 ? p.sk : p.sq;
        if (rrow0 < nrow) {
          for (int bx = 0; bx < BOXES; ++bx) {
            tma_store_4d(&tmOut0, sR1 + c * 8192 + bx * 16384, bx * 64, rrow0, head, b);
            if (MODE == 0) tma_store_4d(&tmOut1, sR0 + c * 8192 + bx * 16384, bx * 64, rrow0, head, b);
          }
          tma_store_commit();
          tma_store_wait_read0();
        }
        mbar_arrive(res_empty);
      }
    }
    if (wg_tid == 0) tma_store_wait_all0();
  }
}

static int make_map(CUtensorMap* m, const void* ptr, int64_t D, int64_t s, int64_t h, int64_t b, const int64_t* str,
                    uint32_t rows) {
  const uint32_t box[4] = {64, rows, 1, 1};
  const uint64_t dims[4] = {(uint64_t)D, (uint64_t)s, (uint64_t)h, (uint64_t)b};
  const uint64_t st[4] = {2, (uint64_t)str[1] * 2, (uint64_t)str[2] * 2, (uint64_t)str[0] * 2};
  return encode_tmap_bf16(m, ptr, 4, dims, st, box, true);
}

template <int D, bool DOCS = false>
static int launch_bwd(const lv_attn_bwd_params* a, cudaStream_t s, const DocsKParams* docs = nullptr) {
  const lv_attn_params* f = &a->fwd;
  constexpr int SMEM = BwdCfg<D>::SMEM;
  // resident operands: 128-row boxes; streamed operands and outputs: 64-row boxes
  CUtensorMap tmQr, tmdOr, tmKr, tmVr, tmQs, tmdOs, tmKs, tmVs, tmdQ, tmdK, tmdV;
  int r;
  if ((r = make_map(&tmQr, f->q, D, f->sq, f->hq, f->batch, f->q_strides, 128))) return r;
  if ((r = make_map(&tmdOr, a->d_out, D, f->sq, f->hq, f->batch, a->do_strides, 128))) return r;
  if ((r = make_map(&tmKr, f->k, D, f->sk, f->hkv, f->batch, f->k_strides, 128))) return r;
  if ((r = make_map(&tmVr, f->v, D, f->sk, f->hkv, f->batch, f->v_strides, 128))) return r;
  if ((r = make_map(&tmQs, f->q, D, f->sq, f->hq, f->batch, f->q_strides, 64))) return r;
  if ((r = make_map(&tmdOs, a->d_out, D, f->sq, f->hq, f->batch, a->do_strides, 64))) return r;
  if ((r = make_map(&tmKs, f->k, D, f->sk, f->hkv, f->batch, f->k_strides, 64))) return r;
  if ((r = make_map(&tmVs, f->v, D, f->sk, f->hkv, f->batch, f->v_strides, 64))) return r;
  if ((r = make_map(&tmdQ, a->dq, D, f->sq, f->hq, f->batch, a->dq_strides, 64))) return r;
  if ((r = make_map(&tmdK, a->dk, D, f->sk, f->hkv, f->batch, a->dk_strides, 64))) return r;
  if ((r = make_map(&tmdV, a->dv, D, f->sk, f->hkv, f->batch, a->dv_strides, 64))) return r;
  // delta = rowsum(dO * O)
  {
    const long long warps = (long long)f->batch * f->sq * f->hq;
    const long long blocks = (warps * 32 + 255) / 256;
    attn_bwd_prep_kernel<<<(unsigned)blocks, 256, 0, s>>>(
        reinterpret_cast<const __nv_bfloat16*>(f->out), reinterpret_cast<const __nv_bfloat16*>(a->d_out), a->delta_ws,
        (int)f->batch, (int)f->sq, (int)f->hq, D, f->o_strides[0], f->o_strides[1], f->o_strides[2], a->do_strides[0],
        a->do_strides[1], a->do_strides[2]);
    LV_CHECK_LAUNCH("attn_bwd_prep_kernel");
  }
  BwdKParams p;
  p.batch = (int)f->batch;
  p.sq = (int)f->sq;
  p.sk = (int)f->sk;
  p.hq = (int)f->hq;
  p.hkv = (int)f->hkv;
  p.causal = f->causal ? 1 : 0;
  p.scale = f->scale;
  p.scale_log2 = f->scale * 1.4426950408889634f;
  p.q_seg_len = (int)f->q_seg_len;
  p.q_seg_pos0 = f->q_seg_pos[0];
  p.q_seg_pos1 = f->q_seg_pos[1];
  p.kv_pos0 = f->kv_pos0;
  p.n_qt = (int)((f->sq + 127) / 128);
  p.n_kt = (int)((f->sk + 127) / 128);
  p.lse = f->lse;
  p.delta = a->delta_ws;
  p.docs = DOCS ? *docs : DocsKParams{nullptr, 0};
  static PerDeviceOnce attr_once;
  int attr_dev;
  if (attr_once.needed(&attr_dev)) {
    LV_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<D, 0, DOCS>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    LV_CHECK_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<D, 1, DOCS>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    attr_once.done(attr_dev);
  }
  {
    p.n_items = p.batch * p.hkv * p.n_kt;
    const int grid = p.n_items < sm_count() ? p.n_items : sm_count();
    attn_bwd_kernel<D, 0, DOCS><<<grid, BW_THREADS, SMEM, s>>>(tmKr, tmVr, tmQs, tmdOs, tmdV, tmdK, p);
    LV_CHECK_LAUNCH("attn_bwd_kernel<dKdV>");
  }
  {
    p.n_items = p.batch * p.hq * p.n_qt;
    const int grid = p.n_items < sm_count() ? p.n_items : sm_count();
    attn_bwd_kernel<D, 1, DOCS><<<grid, BW_THREADS, SMEM, s>>>(tmQr, tmdOr, tmKs, tmVs, tmdQ, tmdQ, p);
    LV_CHECK_LAUNCH("attn_bwd_kernel<dQ>");
  }
  return LV_OK;
}

}  // namespace lv

using namespace lv;

extern "C" int64_t lv_attn_bwd_ws_bytes(int64_t batch, int64_t hq, int64_t sq) { return batch * hq * sq * (int64_t)sizeof(float); }

static int check_bwd_params(const lv_attn_bwd_params* a) {
  LV_CHECK_ARG(a != nullptr, "lv_attn_bwd: null params");
  const lv_attn_params* f = &a->fwd;
  LV_CHECK_ARG(f->q && f->k && f->v && f->out && f->lse, "lv_attn_bwd: q, k, v, out and lse of the forward pass are required");
  LV_CHECK_ARG(a->d_out && a->dq && a->dk && a->dv && a->delta_ws, "lv_attn_bwd: null gradient / workspace pointer");
  LV_CHECK_ARG(f->d == 64 || f->d == 128, "lv_attn_bwd: head_dim %lld not supported (64, 128)", (long long)f->d);
  LV_CHECK_ARG(f->batch > 0 && f->sq > 0 && f->sk > 0 && f->hq > 0 && f->hkv > 0 && f->hq % f->hkv == 0, "lv_attn_bwd: bad shape");
  LV_CHECK_ARG(f->scale > 0.f && isfinite(f->scale), "lv_attn_bwd: scale %g must be finite and > 0", (double)f->scale);
  // launch_bwd hands sizes, row indices and work-item counts to the kernels as int
  LV_CHECK_ARG(f->sq < (1ll << 30) && f->sk < (1ll << 30), "lv_attn_bwd: sequence too long");
  LV_CHECK_ARG(f->batch * f->hq * ((f->sq + 127) / 128) < (1ll << 31) && f->batch * f->hkv * ((f->sk + 127) / 128) < (1ll << 31),
               "lv_attn_bwd: too many work items");
  LV_CHECK_ARG(f->q_seg_len > 0 && f->q_seg_len <= f->sq && (f->q_seg_len == f->sq || (f->q_seg_len % 128 == 0 && f->sq <= 2 * f->q_seg_len)),
               "lv_attn_bwd: bad query segmentation");
  for (int i = 0; i < 3; ++i)
    LV_CHECK_ARG(f->q_strides[i] % 8 == 0 && f->k_strides[i] % 8 == 0 && f->v_strides[i] % 8 == 0 && f->o_strides[i] % 2 == 0 &&
                     a->do_strides[i] % 8 == 0 && a->dq_strides[i] % 8 == 0 && a->dk_strides[i] % 8 == 0 && a->dv_strides[i] % 8 == 0,
                 "lv_attn_bwd: strides must be multiples of 8 elements (16 bytes)");
  return LV_OK;
}

extern "C" int lv_attn_bwd(const lv_attn_bwd_params* a, lv_stream_t stream) {
  int rc = check_bwd_params(a);
  if (rc) return rc;
  const lv_attn_params* f = &a->fwd;
  LV_BIND_DEVICE(f->q);
  cudaStream_t s = (cudaStream_t)stream;
  if (f->d == 128) return launch_bwd<128>(a, s);
  return launch_bwd<64>(a, s);
}

extern "C" int lv_attn_docs_bwd(const lv_attn_bwd_params* a, const lv_attn_docs* docs, lv_stream_t stream) {
  int rc = check_bwd_params(a);
  if (rc) return rc;
  const lv_attn_params* f = &a->fwd;
  rc = check_docs_params(f, docs, "lv_attn_docs_bwd");
  if (rc) return rc;
  LV_BIND_DEVICE(f->q);
  const DocsKParams dk{docs->cu_seqlens, (int)docs->n_docs};
  cudaStream_t s = (cudaStream_t)stream;
  if (f->d == 128) return launch_bwd<128, true>(a, s, &dk);
  return launch_bwd<64, true>(a, s, &dk);
}
