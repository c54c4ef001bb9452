// Work list of the persistent attention forward kernels (attn_fwd.cu: attn_fwd_kernel; attn_fwd_fp8.cu:
// attn_fwd_fp8_kernel): the kernel parameters, the 128-row query work items, their longest-first order and the
// boustrophedon sweep of the CTAs over them.  Both kernels evaluate the same sequence in every warp role.
#pragma once
#include <stdint.h>
#include <stdlib.h>

#include "docs.cuh"

namespace lv {

constexpr int A_BM = 128;   // query rows per tile
constexpr int A_BN = 128;   // key rows per tile

struct AttnKParams {
  int batch, sq, sk, hq, hkv;
  int causal;
  float scale_log2;
  int q_seg_len;
  long long q_seg_pos0, q_seg_pos1, kv_pos0;
  int n_qblk;      // ceil(sq / 128)
  int n_items;     // batch * hq * n_qblk
  int block_major; // 1: order work items (q-block, kv-head, head) - global longest-first; 0: (kv-head, q-block, head)
  int serpentine;  // 1: odd rounds sweep the item list backwards (default); LV_ATTN_SCHED=0 turns it off for A/B runs
  float* lse;
  DocsKParams docs;  // document mode only
};

// Static work assignment: the item list is sorted longest-first; CTAs sweep it boustrophedon (round r
// forwards, round r+1 backwards) so every CTA receives a near-equal share of causal work without a
// global atomic.  All warp roles of a CTA evaluate the same sequence.
__device__ __forceinline__ int sched_item(int round, int n_items, int serpentine) {
  const int base = round * (int)gridDim.x;
  if (base >= n_items) return -1;
  const int item = base + ((serpentine && (round & 1)) ? ((int)gridDim.x - 1 - (int)blockIdx.x) : (int)blockIdx.x);
  return item < n_items ? item : -1;
}

// (b, kv head, q-block rank, head-in-group) of a work item.  Head-major order keeps one kv head's K/V
// hot in L2 when all heads do not fit; block-major order is globally longest-first (better balance).
__device__ __forceinline__ void split_item(const AttnKParams& p, int item, int& b, int& kvh, int& rank, int& g) {
  const int G = p.hq / p.hkv;
  g = item % G;
  int r = item / G;
  if (p.block_major) {
    kvh = r % p.hkv;
    r /= p.hkv;
    rank = r % p.n_qblk;
    b = r / p.n_qblk;
  } else {
    rank = r % p.n_qblk;
    r /= p.n_qblk;
    kvh = r % p.hkv;
    b = r / p.hkv;
  }
}

struct WorkItem {
  int b, h, kvh;
  int j0;            // first kv tile the query tile attends to (document mode; 0 otherwise)
  int n;             // one past the last kv tile the query tile attends to (0: nothing to do)
  long long qpos;    // global position of row 0 of the query tile
  int row0;          // local row index of row 0 of the query tile
};

template <bool DOCS>
__device__ __forceinline__ WorkItem decode_item(const AttnKParams& p, int item) {
  WorkItem w;
  const int G = p.hq / p.hkv;
  int g, rank;
  split_item(p, item, w.b, w.kvh, rank, g);
  w.h = w.kvh * G + g;
  const int qblk = p.causal ? (p.n_qblk - 1 - rank) : rank;   // heaviest causal blocks first
  const int n_kv_tiles = (p.sk + A_BN - 1) / A_BN;
  w.row0 = qblk * A_BM;
  const int seg = w.row0 / p.q_seg_len;
  w.qpos = (seg == 0 ? p.q_seg_pos0 : p.q_seg_pos1) + (w.row0 - seg * p.q_seg_len);
  int n = n_kv_tiles;
  if (p.causal) {
    const long long hi = w.qpos + (A_BM - 1) - p.kv_pos0;  // last visible key index for the tile
    if (hi < 0)
      n = 0;
    else {
      const long long lim = hi / A_BN + 1;
      if (lim < n) n = (int)lim;
    }
  }
  w.n = n;
  // document mode (qpos == row0, kv_pos0 == 0): start at the tile that holds the document start of the first row;
  // doc_start(row0) <= row0 < (the diagonal tile + 1) * 128, so every query tile keeps at least its diagonal
  w.j0 = DOCS ? doc_start(p.docs, w.row0) / A_BN : 0;
  return w;
}

// Work-list fields of AttnKParams for a call (the caller sets lse and docs): the order rule and the LV_ATTN_ORDER /
// LV_ATTN_SCHED switches for A/B runs.
inline void attn_sched_params(const lv_attn_params* a, AttnKParams& p) {
  p.batch = (int)a->batch;
  p.sq = (int)a->sq;
  p.sk = (int)a->sk;
  p.hq = (int)a->hq;
  p.hkv = (int)a->hkv;
  p.causal = a->causal ? 1 : 0;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.q_seg_len = (int)a->q_seg_len;
  p.q_seg_pos0 = a->q_seg_pos[0];
  p.q_seg_pos1 = a->q_seg_pos[1];
  p.kv_pos0 = a->kv_pos0;
  p.n_qblk = (int)((a->sq + A_BM - 1) / A_BM);
  p.n_items = (int)(a->batch * a->hq * p.n_qblk);
  // all kv heads' K and V fit comfortably in the 50 MB L2 -> global longest-first order
  p.block_major = (a->causal && a->sk * a->hkv * a->d * 4 <= (24ll << 20)) ? 1 : 0;
  static const int order_env = [] {   // LV_ATTN_ORDER=0 / 1 forces head-major / block-major order (A/B runs)
    const char* e = getenv("LV_ATTN_ORDER");
    return (e != nullptr && (e[0] == '0' || e[0] == '1')) ? (e[0] - '0') : -1;
  }();
  if (order_env >= 0 && a->causal) p.block_major = order_env;
  static const int serp = [] {
    const char* e = getenv("LV_ATTN_SCHED");
    return (e != nullptr && e[0] == '0') ? 0 : 1;
  }();
  p.serpentine = serp;
}

}  // namespace lv
