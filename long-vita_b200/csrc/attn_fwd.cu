// Fused attention forward for sm_90a: softmax(scale * Q K^T + mask) V with online softmax, GQA,
// causal / zig-zag-causal / document-causal (packed samples) / no mask, LSE output.
//
// One persistent CTA per SM, 3 warpgroups, warp-specialised:
//   warp 0          TMA producer: one 128-row Q tile per work item and a K ring + V ring of 128-row
//                   tiles, 128-byte swizzle, mbarrier completion
//   warps 2-3       idle in this kernel (the context-parallel variant uses them to pull remote K/V)
//   warpgroups 1-2  consumers, 64 query rows each: S = Q K^T with wgmma (both operands from shared memory,
//                   accumulators in registers), online softmax in registers, then O += P V with P fed to
//                   wgmma from registers (the S accumulator layout is the A-operand layout) and V read from
//                   shared memory as an MN-major operand.  The two warpgroups share the K/V tiles but are
//                   not synchronised with each other beyond the ring barriers, so the warp schedulers can
//                   overlap one's softmax with the other's MMAs; nothing enforces that order.  At the end O is
//                   normalised, staged in the warpgroup's half of the (now free) Q tile and stored with TMA.
//
// Document mode (DOCS, lv_attn_docs_fwd): the query tile's key walk starts at the tile holding the document start of
// its first row instead of tile 0; tiles wholly before that document are never loaded.  Masks apply on the diagonal
// tiles, the ragged last tile and on tiles below the document start of the warpgroup's last row, where every row gets
// its own lower bound doc_start(row).
//
// Reference call sites replaced: flash_attn_func / _flash_attention_forward in
// long_vita_megatron/core/transformer/dot_product_attention.py:318-326, 374-390 and
// long_vita/models/long_vita_qwen2_intern/flash_attention.py:52-74.
#include <cuda_bf16.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "common.cuh"
#include "attn_sched.cuh"
#include "docs.cuh"
#include "ptx.cuh"

namespace lv {

constexpr int A_THREADS = 384;

// Context-parallel extension (zig-zag layout, training/utils.py:329-341).  Every rank keeps its own
// K/V rows inside a peer-mapped ("symmetric") buffer; the copier warps of this kernel pull the
// chunks this rank's queries can see from the owning GPUs over NVLink into a local staging copy in
// global sequence order, 128-token block by block, and publish a per-block flag the TMA producer
// polls - so the K/V exchange is part of the attention kernel and overlaps its math.
struct CpKParams {
  int rank, cp;
  int chunk;                 // tokens per zig-zag chunk: S / (2 cp)
  int nblk_needed;           // 128-token key blocks this rank's queries can see
  uint32_t epoch1;           // epoch + 1 (flags are monotonic, never reset)
  int kv_row_elems;          // hkv * d
  long long peer_tok_stride; // elements between consecutive tokens in a peer's K|V rows
  const __nv_bfloat16* peer_kv[8];   // peer p: address of K of its local token 0 (V follows K in the row)
  uint32_t* peer_ready[8];           // peer p: its ready[parity][my rank] word
  const uint32_t* my_ready;          // ready[parity][0..cp)
  __nv_bfloat16* k_full;             // staging [S, hkv*d]
  __nv_bfloat16* v_full;
  uint32_t* blk_flags;               // [S / 128]
  uint32_t* fault;                   // sticky fault word (0 = healthy); set when a peer wait times out
  unsigned long long timeout_ns;     // bound of one wait on another GPU's progress
  unsigned long long order;          // chunk visiting order of this rank, 4 bits per entry (2 cp entries): its own two
                                     // chunks first, then the peers' by ring distance (rank - 1, rank - 2, ...)
  int tiles_per_chunk;               // chunk / 128
};

// Visiting order of the key tiles under context parallelism.  Online softmax does not care in which order the key
// tiles of a query row arrive, so every rank starts on the K/V rows it owns (no waiting at all) and then walks the
// peers in ring order - rank r reads from r-1 first, r-2 next ... - which staggers the ranks over the NVSwitch ports
// instead of all of them pulling chunk 0 from rank 0 at once (the "ring" schedule of TE / ring-flash-attn, SURVEY.md
// 8e).  A query tile sees the key tiles [0, n); they are visited in chunk-priority order.
struct KvWalk {
  int n, li, g, gend;
  __device__ __forceinline__ void begin(int n_tiles) {
    n = n_tiles;
    li = -1;
    g = gend = 0;
  }
  // global index of the next key tile (call exactly n times per item)
  __device__ __forceinline__ int next(const CpKParams& c) {
    for (;;) {
      if (g < gend) return g++;
      const int ch = (int)((c.order >> (4 * ++li)) & 15ull);
      g = ch * c.tiles_per_chunk;
      gend = min(n, (ch + 1) * c.tiles_per_chunk);
    }
  }
};

// Waits on ANOTHER GPU's progress are bounded: a rank whose peer died (or never launched this layer) would otherwise
// spin forever and, because every other rank waits for it in turn, hang the whole node with no message.  After
// `timeout_ns` the waiter records a code in the sticky fault word and STOPS WAITING - the kernel finishes (its output
// is garbage), later waits of this and of the following launches return at once, and the host turns the word into
// LV_ESTATE at its next check (lv_cp_check_fault).  The clock is read every 1024 polls only.
constexpr uint32_t CP_FAULT_READY = 1u, CP_FAULT_BLOCK = 2u, CP_FAULT_EXIT = 4u;

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

struct PeerWait {
  unsigned long long t0 = 0;
  uint32_t polls = 0;
  // true: give up (fault already set by someone, or this wait timed out and sets it)
  __device__ __forceinline__ bool expired(const CpKParams& c, uint32_t code) {
    if ((++polls & 1023u) != 0) return false;
    if (*reinterpret_cast<volatile uint32_t*>(c.fault) != 0) return true;
    const unsigned long long now = global_ns();
    if (t0 == 0) {
      t0 = now;
      return false;
    }
    if (now - t0 > c.timeout_ns) {
      atomicOr(c.fault, code);
      return true;
    }
    return false;
  }
};

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint4 ld_peer_v4(const void* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}

__device__ __forceinline__ void red_release_gpu_add(uint32_t* p, uint32_t v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// Staging granularity: a 128-token key block is pulled as CP_SUB units of 32 tokens by different copier
// warps, and blk_flags[b] COUNTS completed units (it reaches CP_SUB * (epoch + 1) when block b of this
// epoch is whole).  With one unit per warp-visit and 8 x 16 B loads in flight per lane, a rank with few
// blocks (short sequences) still keeps every copier warp of the grid and ~1.2 MB of NVLink reads in
// flight; the first version moved one whole block per warp with 4 loads in flight and needed ~0.5 ms per
// layer at 18K tokens / 8 ranks, all of it exposed.
constexpr int CP_SUB = 4;
constexpr int CP_UNIT_ROWS = A_BN / CP_SUB;

__device__ __forceinline__ void cp_copier(const CpKParams& cpp, int warp, int lane) {
      const int cw = blockIdx.x * 2 + (warp - 2);          // copier index
      const int ncw = gridDim.x * 2;
      if (cw == 0) {
        // tell every peer that this rank's K/V rows for this epoch are complete (they were written
        // by earlier kernels on this stream; the fence orders them before the flag at system scope)
        __threadfence_system();
        if (lane < cpp.cp && lane != cpp.rank) st_release_sys(cpp.peer_ready[lane], cpp.epoch1);
      }
      uint32_t seen = 1u << cpp.rank;                      // peers whose ready flag has been observed
      const int vec_per_row = cpp.kv_row_elems / 4;        // 16-byte vectors in one K|V row pair
      const int vec_per_half = cpp.kv_row_elems / 8;
      const int n_units = cpp.nblk_needed * CP_SUB;
      for (int u = cw; u < n_units; u += ncw) {
        // the i-th block in this rank's chunk-priority order (own chunks, then peers by ring distance): the order in
        // which the query tiles consume them (KvWalk)
        int b = u / CP_SUB;
        {
          int i = b;
          for (int li = 0; li < 2 * cpp.cp; ++li) {
            const int ch = (int)((cpp.order >> (4 * li)) & 15ull);
            const int cnt = min(max(cpp.nblk_needed - ch * cpp.tiles_per_chunk, 0), cpp.tiles_per_chunk);
            if (i < cnt) {
              b = ch * cpp.tiles_per_chunk + i;
              break;
            }
            i -= cnt;
          }
        }
        const int tok0 = b * A_BN + (u % CP_SUB) * CP_UNIT_ROWS;
        const int chunk = tok0 / cpp.chunk;
        const int owner = chunk < cpp.cp ? chunk : 2 * cpp.cp - 1 - chunk;
        const int lrow0 = (chunk < cpp.cp ? 0 : cpp.chunk) + (tok0 - chunk * cpp.chunk);
        if (!(seen & (1u << owner))) {
          if (lane == 0)
            {
              [[maybe_unused]] uint32_t spins = 0;
              PeerWait pw;
              while (ld_acquire_sys(cpp.my_ready + owner) < cpp.epoch1) {
                LV_SPIN_GUARD(spins, "peer ready word", cpp.my_ready + owner, cpp.epoch1)
                if (pw.expired(cpp, CP_FAULT_READY)) break;
              }
            }
          __syncwarp();
          seen |= 1u << owner;
        }
        const __nv_bfloat16* src = cpp.peer_kv[owner] + (long long)lrow0 * cpp.peer_tok_stride;
        if (vec_per_row == 256) {
          // K|V row pair = 4 KB (8 kv heads x 128): one row per warp pass, 8 loads in flight per lane,
          // vectors 0..127 of the row are K, 128..255 are V
          const __nv_bfloat16* s_lane = src + lane * 8;
          __nv_bfloat16* dk = cpp.k_full + (long long)tok0 * cpp.kv_row_elems + lane * 8;
          __nv_bfloat16* dv = cpp.v_full + (long long)tok0 * cpp.kv_row_elems + lane * 8;
#pragma unroll 1
          for (int row = 0; row < CP_UNIT_ROWS; ++row) {
            uint4 v[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) v[i] = ld_peer_v4(s_lane + i * 256);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              *reinterpret_cast<uint4*>(dk + i * 256) = v[i];
              *reinterpret_cast<uint4*>(dv + i * 256) = v[4 + i];
            }
            s_lane += cpp.peer_tok_stride;
            dk += cpp.kv_row_elems;
            dv += cpp.kv_row_elems;
          }
        } else {
          const int total = CP_UNIT_ROWS * vec_per_row;
          for (int i0 = 0; i0 < total; i0 += 32 * 4) {
            uint4 v[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const int i = i0 + k * 32 + lane;
              const int row = i / vec_per_row, col = i - row * vec_per_row;
              if (i < total) v[k] = ld_peer_v4(src + (long long)row * cpp.peer_tok_stride + col * 8);
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const int i = i0 + k * 32 + lane;
              const int row = i / vec_per_row, col = i - row * vec_per_row;
              if (i < total) {
                __nv_bfloat16* dst = col < vec_per_half
                                         ? cpp.k_full + (long long)(tok0 + row) * cpp.kv_row_elems + col * 8
                                         : cpp.v_full + (long long)(tok0 + row) * cpp.kv_row_elems + (col - vec_per_half) * 8;
                *reinterpret_cast<uint4*>(dst) = v[k];
              }
            }
          }
        }
        // the staged rows are read by TMA (async proxy): order this lane's generic-proxy stores before the
        // async proxy on the writer side as well (the producer fences again after its acquire)
        fence_proxy_async_all();
        __threadfence();
        __syncwarp();
        if (lane == 0) red_release_gpu_add(cpp.blk_flags + b, 1u);
      }
      if (cw == 0) {
        // do not retire before every peer has entered this epoch: a peer's flag for epoch e+1 then
        // proves it finished reading our epoch e-1 rows (buffer parity reuse, see DESIGN.md)
        if (lane < cpp.cp && lane != cpp.rank)
        {
          [[maybe_unused]] uint32_t spins = 0;
          PeerWait pw;
          while (ld_acquire_sys(cpp.my_ready + lane) < cpp.epoch1) {
            LV_SPIN_GUARD(spins, "peer epoch word (exit)", cpp.my_ready + lane, cpp.epoch1)
            if (pw.expired(cpp, CP_FAULT_EXIT)) break;
          }
        }
        __syncwarp();
      }
}

template <int D>
struct AttnCfg {
  static constexpr int KV_STAGES = (D == 128) ? 2 : 4;
  static constexpr int TILE_BYTES = 128 * D * 2;           // one 128-row tile of Q / K / V
  static constexpr int BOXES = D / 64;                     // 64-column (128-byte) TMA boxes per row
  static constexpr int SMEM_Q = TILE_BYTES;
  static constexpr int SMEM_K = KV_STAGES * TILE_BYTES;
  static constexpr int SMEM_V = KV_STAGES * TILE_BYTES;
  static constexpr int SMEM_BAR = 256;
  static constexpr int SMEM_TOTAL = SMEM_Q + SMEM_K + SMEM_V + SMEM_BAR + 1024;
};

// S = Q K^T for one 64-row half of the query tile against one 128-key tile (fp32 accumulators, m64n128k16 steps).
template <int D>
__device__ __forceinline__ void mma_qk(float (&s)[64], uint64_t qdesc, uint64_t kdesc) {
#pragma unroll
  for (int kk = 0; kk < D / 16; ++kk) {
    // K-steps of 16 columns: four per 128-byte row, the next 64 head-dim columns one 16 KB box further
    const uint32_t qoff = ((kk / 4) * 16384 + (kk % 4) * 32) >> 4;
    wgmma_ss_n128(s, qdesc + qoff, kdesc + qoff, kk != 0 ? 1u : 0u);
  }
}

// O += P V: P (bf16, packed in the accumulator layout of S) from registers, V tile MN-major from shared memory,
// 16 key rows (2 KB) per k-step.
template <int D>
__device__ __forceinline__ void mma_pv(float (&o)[D / 2], const uint32_t (&pk)[32], uint64_t vdesc) {
#pragma unroll
  for (int kk = 0; kk < A_BN / 16; ++kk) {
    const uint32_t a[4] = {pk[4 * kk], pk[4 * kk + 1], pk[4 * kk + 2], pk[4 * kk + 3]};
    if constexpr (D == 128)
      wgmma_rs_n128(o, a, vdesc + (uint64_t)(kk * 128), 1u);
    else
      wgmma_rs_n64(o, a, vdesc + (uint64_t)(kk * 128), 1u);
  }
}

template <int D, bool CP, bool DOCS>
__global__ void __launch_bounds__(A_THREADS, 1)
    attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmO,
                    const AttnKParams p, const CpKParams cpp) {
  using Cfg = AttnCfg<D>;
  constexpr int NS = Cfg::KV_STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Cfg::SMEM_Q;
  uint8_t* sV = sK + Cfg::SMEM_K;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + Cfg::SMEM_V);
  uint64_t* q_full = bars;            // [1]
  uint64_t* q_empty = bars + 1;       // [1]: both consumer warpgroups have stored their O half out of the Q tile
  uint64_t* k_full = bars + 2;        // [NS]
  uint64_t* k_empty = bars + 2 + NS;  // [NS]
  uint64_t* v_full = bars + 2 + 2 * NS;
  uint64_t* v_empty = bars + 2 + 3 * NS;

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
    if (warp == 0) {
      // =========================== TMA producer ===========================
      if (lane == 0) {
        uint32_t item_cnt = 0, kcnt = 0, vcnt = 0;
        KvWalk walk;
        for (int round = 0, item; (item = sched_item(round, p.n_items, p.serpentine)) >= 0; ++round, ++item_cnt) {
          const WorkItem w = decode_item<DOCS>(p, item);
          if (CP) walk.begin(w.n);
          const int pre = min(NS, w.n - w.j0);
          auto load_tile = [&](int j) {
            int g = j;            // global key tile visited in step j
            if (CP) {
              g = walk.next(cpp);
              // staged by the copier warps of this GPU (any CTA)?  One L2 poll per tile; the K / V rings keep the
              // producer a step ahead of the tensor cores, so the poll latency is off the critical path.
              {
                [[maybe_unused]] uint32_t spins = 0;
                PeerWait pw;
                while (ld_acquire_gpu(cpp.blk_flags + g) < cpp.epoch1 * CP_SUB) {
                  LV_SPIN_GUARD(spins, "staged block flag", cpp.blk_flags + g, cpp.epoch1 * CP_SUB)
                  if (pw.expired(cpp, CP_FAULT_BLOCK)) break;
                }
              }
              fence_proxy_async_all();   // copier warps wrote the staging rows through the generic proxy
            }
            {
              const int st = kcnt % NS;
              mbar_wait(&k_empty[st], ((kcnt / NS) & 1) ^ 1);
              mbar_arrive_expect_tx(&k_full[st], Cfg::TILE_BYTES);
              for (int bx = 0; bx < Cfg::BOXES; ++bx)
                tma_load_4d(sK + st * Cfg::TILE_BYTES + bx * 16384, &tmK, &k_full[st], bx * 64, g * A_BN, w.kvh, w.b,
                            kEvictLast);
              ++kcnt;
            }
            {
              const int st = vcnt % NS;
              mbar_wait(&v_empty[st], ((vcnt / NS) & 1) ^ 1);
              mbar_arrive_expect_tx(&v_full[st], Cfg::TILE_BYTES);
              for (int bx = 0; bx < Cfg::BOXES; ++bx)
                tma_load_4d(sV + st * Cfg::TILE_BYTES + bx * 16384, &tmV, &v_full[st], bx * 64, g * A_BN, w.kvh, w.b,
                            kEvictLast);
              ++vcnt;
            }
          };
          // The Q load of this item waits for the previous item's epilogue (O is staged in the Q tile); its first key
          // tiles do not (their ring slots free up as the previous item's last MMAs retire), so they are requested first.
          for (int j = w.j0; j < w.j0 + pre; ++j) load_tile(j);
          mbar_wait(q_empty, (item_cnt & 1) ^ 1);
          mbar_arrive_expect_tx(q_full, Cfg::TILE_BYTES);
          for (int bx = 0; bx < Cfg::BOXES; ++bx)
            tma_load_4d(sQ + bx * 16384, &tmQ, q_full, bx * 64, w.row0, w.h, w.b, kEvictFirst);
          for (int j = w.j0 + pre; j < w.n; ++j) load_tile(j);
        }
      }
    } else if (warp >= 2) {
      // =========================== warps 2-3: context-parallel K/V copier ===========================
      if (CP) cp_copier(cpp, warp, lane);
    }
  } else {
    // =========================== consumer warpgroups ===========================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 224;");
    const int c = (warp >> 2) - 1;                // 64-row half of the query tile
    const int wg_tid = threadIdx.x & 127;
    const int r_lo = ((wg_tid >> 5) << 4) + (lane >> 2);   // this thread's rows: r_lo and r_lo + 8 (of 64)
    const int cq = 2 * (lane & 3);                         // its first column in every 8-column group
    const uint64_t qdesc = make_smem_desc(smem_u32(sQ) + c * 8192, 16, 1024);
    const uint64_t kdesc0 = make_smem_desc(smem_u32(sK), 16, 1024);
    const uint64_t vdesc0 = make_smem_desc(smem_u32(sV), 16384, 1024);
    const float scale_log2 = p.scale_log2;
    const int n_kv_tiles = (p.sk + A_BN - 1) / A_BN;
    const int j_ragged = (p.sk % A_BN) ? n_kv_tiles - 1 : 0x7fffffff;
    uint32_t item_cnt = 0, kcnt = 0, vcnt = 0;

    for (int round = 0, item; (item = sched_item(round, p.n_items, p.serpentine)) >= 0; ++round, ++item_cnt) {
      const WorkItem w = decode_item<DOCS>(p, item);
      const int n = w.n;
      // global positions of this thread's two query rows
      const long long qpos0 = w.qpos + c * 64 + r_lo, qpos1 = qpos0 + 8;
      KvWalk walk;
      if (CP) walk.begin(n);
      // first key tile (GLOBAL index) that needs a mask: the diagonal ones and the ragged last one
      int j_mask = j_ragged;
      if (p.causal) {
        const long long dd = w.qpos + c * 64 - p.kv_pos0 - (A_BN - 1);
        const long long jd = dd < 0 ? 0 : dd / A_BN + 1;
        if (jd < j_mask) j_mask = (int)jd;
      }
      // document mode: the first visible key of each of this thread's rows, and of the warpgroup's last row (tiles
      // below it hold keys of an earlier document for some row and need the mask)
      int ds0 = 0, ds1 = 0, ds_last = 0;
      if (DOCS) {
        ds0 = doc_start(p.docs, min((int)qpos0, p.sq - 1));
        ds1 = doc_start(p.docs, min((int)qpos1, p.sq - 1));
        ds_last = doc_start(p.docs, min((int)w.qpos + c * 64 + 63, p.sq - 1));
      }
      float o[D / 2];
#pragma unroll
      for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
      float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // running max (log2 domain) and sum per row
      mbar_wait(q_full, item_cnt & 1);
      for (int j = w.j0; j < n; ++j) {
        int g = j;         // global key tile of this step (context parallelism visits them out of order)
        if (CP) g = walk.next(cpp);
        const int kst = kcnt % NS;
        mbar_wait(&k_full[kst], (kcnt / NS) & 1);
        ++kcnt;
        float s[64];
        wgmma_fence();
        mma_qk<D>(s, qdesc, kdesc0 + (uint64_t)((kst * Cfg::TILE_BYTES) >> 4));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_keep(s);
        if (wg_tid == 0) mbar_arrive(&k_empty[kst]);

        // ---- mask (only diagonal tiles and the ragged last key tile; document mode: also tiles below a row's
        //      document start) ----
        if (g >= j_mask || (DOCS && g * A_BN < ds_last)) {
          const long long kidx0 = (long long)g * A_BN;
          long long lim0 = p.sk - kidx0, lim1 = lim0;                 // first invalid column of each row
          if (p.causal) {
            lim0 = min(lim0, qpos0 - p.kv_pos0 - kidx0 + 1);
            lim1 = min(lim1, qpos1 - p.kv_pos0 - kidx0 + 1);
          }
          const int lo0 = ds0 - (int)kidx0, lo1 = ds1 - (int)kidx0;   // first visible column (document mode)
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = 8 * jj + cq + e;
              if (col >= lim0) s[4 * jj + e] = -INFINITY;
              if (col >= lim1) s[4 * jj + 2 + e] = -INFINITY;
              if (DOCS && col < lo0) s[4 * jj + e] = -INFINITY;
              if (DOCS && col < lo1) s[4 * jj + 2 + e] = -INFINITY;
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
        const float mn0 = fmaxf(m0, mx0 * scale_log2), mn1 = fmaxf(m1, mx1 * scale_log2);
        // a row that has seen only masked keys keeps max -inf: subtract 0 instead (its P and alpha are 0)
        const float ms0 = mn0 == -INFINITY ? 0.f : mn0, ms1 = mn1 == -INFINITY ? 0.f : mn1;
        const float alpha0 = ex2(m0 - ms0), alpha1 = ex2(m1 - ms1);
        m0 = mn0;
        m1 = mn1;
        l0 *= alpha0;
        l1 *= alpha1;
#pragma unroll
        for (int jj = 0; jj < D / 8; ++jj) {
          o[4 * jj] *= alpha0;
          o[4 * jj + 1] *= alpha0;
          o[4 * jj + 2] *= alpha1;
          o[4 * jj + 3] *= alpha1;
        }
        uint32_t pk[32];
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const float p0 = ex2(fmaf(s[4 * jj], scale_log2, -ms0)), p1 = ex2(fmaf(s[4 * jj + 1], scale_log2, -ms0));
          const float p2 = ex2(fmaf(s[4 * jj + 2], scale_log2, -ms1)), p3 = ex2(fmaf(s[4 * jj + 3], scale_log2, -ms1));
          l0 += p0 + p1;
          l1 += p2 + p3;
          pk[2 * jj] = pack_bf16(p0, p1);
          pk[2 * jj + 1] = pack_bf16(p2, p3);
        }

        // ---- O += P V ----
        const int vst = vcnt % NS;
        mbar_wait(&v_full[vst], (vcnt / NS) & 1);
        ++vcnt;
        wgmma_fence();
        mma_pv<D>(o, pk, vdesc0 + (uint64_t)((vst * Cfg::TILE_BYTES) >> 4));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_keep(o);
        if (wg_tid == 0) mbar_arrive(&v_empty[vst]);
      }

      // ---------------- epilogue: O / l -> bf16 -> smem (swizzled, this half of the Q tile) -> TMA store; LSE -------
#pragma unroll
      for (int off = 1; off <= 2; off <<= 1) {
        l0 += __shfl_xor_sync(0xffffffffu, l0, off);
        l1 += __shfl_xor_sync(0xffffffffu, l1, off);
      }
      const float inv0 = l0 > 0.f ? 1.f / l0 : 0.f, inv1 = l1 > 0.f ? 1.f / l1 : 0.f;
      uint8_t* stage = sQ + c * 8192;
      named_bar_sync(1 + c, 128);    // every thread of this warpgroup is done reading its Q rows
#pragma unroll
      for (int jj = 0; jj < D / 8; ++jj) {
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
          for (int bx = 0; bx < Cfg::BOXES; ++bx)
            tma_store_4d(&tmO, stage + bx * 16384, bx * 64, w.row0 + c * 64, w.h, w.b);
          tma_store_commit();
          tma_store_wait_read0();
        }
        mbar_arrive(q_empty);   // this half of the Q / staging tile may be overwritten by a later item's Q load
      }
    }
    if (wg_tid == 0) tma_store_wait_all0();
  }
}

template <int D, bool CP, bool DOCS = false>
static int launch_attn(const lv_attn_params* a, const CpKParams* cp, cudaStream_t s, const DocsKParams* docs = nullptr) {
  using Cfg = AttnCfg<D>;
  CUtensorMap tmQ, tmK, tmV, tmO;
  const uint32_t box[4] = {64, 128, 1, 1};
  const uint32_t obox[4] = {64, 64, 1, 1};    // each consumer warpgroup stores its own 64 rows
  {
    const uint64_t dims[4] = {(uint64_t)D, (uint64_t)a->sq, (uint64_t)a->hq, (uint64_t)a->batch};
    const uint64_t str[4] = {2, (uint64_t)a->q_strides[1] * 2, (uint64_t)a->q_strides[2] * 2, (uint64_t)a->q_strides[0] * 2};
    int r = encode_tmap_bf16(&tmQ, a->q, 4, dims, str, box, true);
    if (r) return r;
    const uint64_t ostr[4] = {2, (uint64_t)a->o_strides[1] * 2, (uint64_t)a->o_strides[2] * 2, (uint64_t)a->o_strides[0] * 2};
    r = encode_tmap_bf16(&tmO, a->out, 4, dims, ostr, obox, true);
    if (r) return r;
  }
  {
    const uint64_t dims[4] = {(uint64_t)D, (uint64_t)a->sk, (uint64_t)a->hkv, (uint64_t)a->batch};
    const uint64_t kstr[4] = {2, (uint64_t)a->k_strides[1] * 2, (uint64_t)a->k_strides[2] * 2, (uint64_t)a->k_strides[0] * 2};
    const uint64_t vstr[4] = {2, (uint64_t)a->v_strides[1] * 2, (uint64_t)a->v_strides[2] * 2, (uint64_t)a->v_strides[0] * 2};
    int r = encode_tmap_bf16(&tmK, a->k, 4, dims, kstr, box, true);
    if (r) return r;
    r = encode_tmap_bf16(&tmV, a->v, 4, dims, vstr, box, true);
    if (r) return r;
  }
  AttnKParams p;
  attn_sched_params(a, p);
  p.lse = a->lse;
  p.docs = DOCS ? *docs : DocsKParams{nullptr, 0};
  static PerDeviceOnce attr_once;   // one per template instantiation
  int attr_dev;
  if (attr_once.needed(&attr_dev)) {
    LV_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<D, CP, DOCS>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_TOTAL));
    attr_once.done(attr_dev);
  }
  int grid = p.n_items < sm_count() ? p.n_items : sm_count();
  CpKParams cpp;
  memset(&cpp, 0, sizeof(cpp));
  if (CP) {
    cpp = *cp;
    grid = sm_count();   // every copier warp takes part, also when there are fewer work items than SMs
  }
  attn_fwd_kernel<D, CP, DOCS><<<grid, A_THREADS, Cfg::SMEM_TOTAL, s>>>(tmQ, tmK, tmV, tmO, p, cpp);
  LV_CHECK_LAUNCH("attn_fwd_kernel");
  return LV_OK;
}

}  // namespace lv

using namespace lv;

static int check_attn_params(const lv_attn_params* a) {
  LV_CHECK_ARG(a != nullptr, "lv_attn_fwd: null params");
  LV_CHECK_ARG(a->q && a->k && a->v && a->out, "lv_attn_fwd: null tensor pointer");
  LV_CHECK_ARG(a->d == 64 || a->d == 128, "lv_attn_fwd: head_dim %lld not supported (64, 128)", (long long)a->d);
  LV_CHECK_ARG(a->batch > 0 && a->sq > 0 && a->sk > 0 && a->hq > 0 && a->hkv > 0, "lv_attn_fwd: empty shape");
  LV_CHECK_ARG(a->hq % a->hkv == 0, "lv_attn_fwd: hq=%lld is not a multiple of hkv=%lld", (long long)a->hq, (long long)a->hkv);
  // masked scores are -inf before s * scale_log2 - m: a zero scale makes them NaN, a negative one gives them p = +inf
  LV_CHECK_ARG(a->scale > 0.f && isfinite(a->scale), "lv_attn_fwd: scale %g must be finite and > 0", (double)a->scale);
  LV_CHECK_ARG(a->sq < (1ll << 30) && a->sk < (1ll << 30), "lv_attn_fwd: sequence too long");
  LV_CHECK_ARG(a->batch * a->hq * ((a->sq + 127) / 128) < (1ll << 31), "lv_attn_fwd: too many work items");
  LV_CHECK_ARG(a->q_seg_len > 0 && a->q_seg_len <= a->sq, "lv_attn_fwd: q_seg_len=%lld out of range", (long long)a->q_seg_len);
  if (a->q_seg_len < a->sq) {
    LV_CHECK_ARG(a->q_seg_len % 128 == 0 && a->sq <= 2 * a->q_seg_len, "lv_attn_fwd: segmented queries need q_seg_len %% 128 == 0 (a 128-row query tile never straddles segments) and at most two segments");
  }
  for (int i = 0; i < 3; ++i)
    LV_CHECK_ARG(a->q_strides[i] % 8 == 0 && a->k_strides[i] % 8 == 0 && a->v_strides[i] % 8 == 0 && a->o_strides[i] % 8 == 0,
                 "lv_attn_fwd: strides must be multiples of 8 elements (16 bytes)");
  return LV_OK;
}

extern "C" int lv_attn_fwd(const lv_attn_params* a, lv_stream_t stream) {
  int rc = check_attn_params(a);
  if (rc) return rc;
  LV_BIND_DEVICE(a->q);
  cudaStream_t s = (cudaStream_t)stream;
  if (a->d == 128) return launch_attn<128, false>(a, nullptr, s);
  return launch_attn<64, false>(a, nullptr, s);
}

extern "C" int lv_attn_docs_fwd(const lv_attn_params* a, const lv_attn_docs* docs, lv_stream_t stream) {
  int rc = check_attn_params(a);
  if (rc) return rc;
  rc = check_docs_params(a, docs, "lv_attn_docs_fwd");
  if (rc) return rc;
  LV_BIND_DEVICE(a->q);
  const DocsKParams dk{docs->cu_seqlens, (int)docs->n_docs};
  cudaStream_t s = (cudaStream_t)stream;
  if (a->d == 128) return launch_attn<128, false, true>(a, nullptr, s, &dk);
  return launch_attn<64, false, true>(a, nullptr, s, &dk);
}

extern "C" int lv_attn_cp_fwd(const lv_attn_params* a, const lv_cp_params* c, lv_stream_t stream) {
  int rc = check_attn_params(a);
  if (rc) return rc;
  LV_CHECK_ARG(c != nullptr, "lv_attn_cp_fwd: null cp params");
  LV_CHECK_ARG(c->cp >= 2 && c->cp <= 8 && c->rank >= 0 && c->rank < c->cp, "lv_attn_cp_fwd: bad rank %d / cp %d", c->rank, c->cp);
  LV_CHECK_ARG(a->batch == 1 && a->causal, "lv_attn_cp_fwd: batch 1, causal only");
  LV_CHECK_ARG(a->d == 128, "lv_attn_cp_fwd: head_dim 128 only");
  const int64_t S = c->seq_total;
  LV_CHECK_ARG(S % (2 * c->cp) == 0, "lv_attn_cp_fwd: seq_total %lld not divisible by 2*cp", (long long)S);
  const int64_t chunk = S / (2 * c->cp);
  LV_CHECK_ARG(chunk % 128 == 0, "lv_attn_cp_fwd: chunk %lld must be a multiple of 128 tokens", (long long)chunk);
  LV_CHECK_ARG(a->sq == 2 * chunk && a->sk == S && a->q_seg_len == chunk && a->kv_pos0 == 0,
               "lv_attn_cp_fwd: expects sq = 2*chunk local queries against the S-row staging buffers");
  LV_CHECK_ARG(a->q_seg_pos[0] == c->rank * chunk && a->q_seg_pos[1] == (2 * c->cp - 1 - c->rank) * chunk,
               "lv_attn_cp_fwd: q_seg_pos does not match the zig-zag layout of rank %d", c->rank);
  LV_CHECK_ARG(a->k == c->k_full && a->v == c->v_full, "lv_attn_cp_fwd: k / v must be the staging buffers");
  LV_CHECK_ARG(c->my_ready && c->blk_flags && c->k_full && c->v_full, "lv_attn_cp_fwd: null cp buffer");
  CpKParams k;
  memset(&k, 0, sizeof(k));
  k.rank = c->rank;
  k.cp = c->cp;
  k.chunk = (int)chunk;
  k.nblk_needed = (int)((2 * c->cp - c->rank) * chunk / A_BN);
  k.epoch1 = c->epoch + 1;
  k.kv_row_elems = (int)(a->hkv * a->d);
  k.peer_tok_stride = c->peer_tok_stride;
  const int parity = (int)(c->epoch & 1);
  for (int p = 0; p < c->cp; ++p) {
    LV_CHECK_ARG(c->peer_kv[p] != nullptr && c->peer_ready[p] != nullptr, "lv_attn_cp_fwd: null peer pointer for rank %d", p);
    k.peer_kv[p] = reinterpret_cast<const __nv_bfloat16*>(c->peer_kv[p]);
    k.peer_ready[p] = reinterpret_cast<uint32_t*>(c->peer_ready[p]) + parity * 8 + c->rank;
  }
  LV_BIND_DEVICE(a->q);     // after every argument check, so that bad arguments are reported without touching CUDA
  k.my_ready = reinterpret_cast<const uint32_t*>(c->my_ready) + parity * 8;
  k.k_full = reinterpret_cast<__nv_bfloat16*>(c->k_full);
  k.v_full = reinterpret_cast<__nv_bfloat16*>(c->v_full);
  k.blk_flags = reinterpret_cast<uint32_t*>(c->blk_flags);
  LV_CHECK_ARG(c->fault != nullptr, "lv_attn_cp_fwd: null fault word");
  k.fault = reinterpret_cast<uint32_t*>(c->fault);
  static const unsigned long long timeout_ms = [] {
    const char* e = getenv("LV_CP_TIMEOUT_MS");
    const long long v = e ? atoll(e) : 0;
    return (unsigned long long)(v > 0 ? v : 120000);      // 2 minutes: far beyond any rank skew of a healthy job
  }();
  k.timeout_ns = timeout_ms * 1000000ull;
  // Chunk visiting order.  Default: plain global order - the result is then BIT-IDENTICAL to the single-device kernel
  // on the gathered K/V (same key order, same rounding sequence), which is what bench.py's in-run parity check
  // asserts.  LV_CP_ORDER=1: own chunks first, then the peers' by ring distance; measured on 8 GPUs at 18K tokens:
  // 107.46 ms per prefill against 107.48 ms in global order (the exchange is not what bounds that configuration), and
  // the output then differs from the single-device kernel by the rounding of a different summation order (3.1e-3
  // relative between the two bf16 results; both within the test bound against the fp32 oracle).
  k.tiles_per_chunk = (int)(chunk / A_BN);
  static const int ring_order = [] {
    const char* e = getenv("LV_CP_ORDER");
    return (e != nullptr && e[0] == '1') ? 1 : 0;
  }();
  k.order = 0;
  for (int i = 0; i < c->cp; ++i) {
    const int peer = ring_order ? (c->rank - i + c->cp) % c->cp : i;
    const unsigned long long first = ring_order ? (unsigned long long)peer : (unsigned long long)(2 * i);
    const unsigned long long second = ring_order ? (unsigned long long)(2 * c->cp - 1 - peer) : (unsigned long long)(2 * i + 1);
    k.order |= first << (4 * (2 * i));
    k.order |= second << (4 * (2 * i + 1));
  }
  return launch_attn<128, true>(a, &k, (cudaStream_t)stream);
}

// Peer-mappable ("symmetric") allocations for the context-parallel K/V exchange: plain cudaMalloc
// memory exported / imported with CUDA IPC handles (64 opaque bytes the host exchanges over
// torch.distributed).
extern "C" int lv_ipc_alloc(int64_t bytes, void** ptr) {
  LV_CHECK_ARG(ptr != nullptr && bytes > 0, "lv_ipc_alloc: bad arguments");
  LV_CHECK_CUDA(cudaMalloc(ptr, (size_t)bytes));
  LV_CHECK_CUDA(cudaMemset(*ptr, 0, (size_t)bytes));
  return LV_OK;
}
extern "C" int lv_ipc_free(void* ptr) {
  if (ptr) LV_CHECK_CUDA(cudaFree(ptr));
  return LV_OK;
}
extern "C" int lv_ipc_get_handle(void* ptr, void* handle64) {
  LV_CHECK_ARG(ptr && handle64, "lv_ipc_get_handle: null pointer");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
  cudaIpcMemHandle_t h;
  LV_CHECK_CUDA(cudaIpcGetMemHandle(&h, ptr));
  memcpy(handle64, &h, 64);
  return LV_OK;
}
extern "C" int lv_ipc_open_handle(const void* handle64, void** ptr) {
  LV_CHECK_ARG(ptr && handle64, "lv_ipc_open_handle: null pointer");
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  LV_CHECK_CUDA(cudaIpcOpenMemHandle(ptr, h, cudaIpcMemLazyEnablePeerAccess));
  return LV_OK;
}
// Read (and keep) the sticky fault word of a context-parallel context: LV_OK when healthy, LV_ESTATE with a message
// naming what timed out otherwise.  Synchronises `stream` (the word is written by kernels on it).
extern "C" int lv_cp_check_fault(const void* fault, lv_stream_t stream) {
  LV_CHECK_ARG(fault != nullptr, "lv_cp_check_fault: null pointer");
  LV_BIND_DEVICE(fault);
  uint32_t w = 0;
  LV_CHECK_CUDA(cudaMemcpyAsync(&w, fault, 4, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  LV_CHECK_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  if (w == 0) return LV_OK;
  lv::set_error("context-parallel exchange timed out (fault word 0x%x:%s%s%s): a peer rank did not publish its K/V rows "
                "for this layer in time - it died, hung, or is not running the same sequence of attention calls",
                w, (w & CP_FAULT_READY) ? " peer-ready" : "", (w & CP_FAULT_BLOCK) ? " staged-block" : "",
                (w & CP_FAULT_EXIT) ? " exit-handshake" : "");
  return LV_ESTATE;
}

extern "C" int lv_ipc_close_handle(void* ptr) {
  if (ptr) LV_CHECK_CUDA(cudaIpcCloseMemHandle(ptr));
  return LV_OK;
}
