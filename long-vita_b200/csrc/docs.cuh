// Document mode of the attention kernels (packed training samples, `--reset-attention-mask`): one packed row of
// S tokens holds n documents with boundaries cu[0] = 0 < cu[1] < ... < cu[n] = S, and key j is visible to query i
// iff both lie in the same document and j <= i.
//
// The kernels look a document up by a binary search of cu (n + 1 int32 values, L1/L2-resident) once per work item
// and thread, never per tile.  A malformed table must not make a kernel read or write out of range, so every index
// into cu stays in [0, n] and the results are clamped to the position asked about: doc_start(x) is in [0, x] and
// doc_end(x) in [x + 1, S].  (The ops layer validates the table on the host; the clamps only keep the kernels
// memory-safe when a caller of the C ABI does not.)
#pragma once
#include <stdint.h>

#include "common.cuh"

namespace lv {

struct DocsKParams {
  const int32_t* cu;   // device, [n + 1]; nullptr outside document mode
  int n;               // number of documents (>= 1)
};

// index of the document holding position x: the largest i in [0, n - 1] with cu[i] <= x (0 if there is none)
__device__ __forceinline__ int doc_index(const DocsKParams& d, int x) {
  int lo = 0, hi = d.n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (__ldg(d.cu + mid) <= x)
      lo = mid;
    else
      hi = mid - 1;
  }
  return lo;
}

// first position of the document holding x
__device__ __forceinline__ int doc_start(const DocsKParams& d, int x) {
  const int s = __ldg(d.cu + doc_index(d, x));
  return s < 0 ? 0 : (s > x ? x : s);
}

// one past the last position of the document holding x (S = the sequence length)
__device__ __forceinline__ int doc_end(const DocsKParams& d, int x, int S) {
  const int e = __ldg(d.cu + doc_index(d, x) + 1);
  return e > S ? S : (e <= x ? x + 1 : e);
}

// Host-side argument check shared by lv_attn_docs_fwd / lv_attn_docs_bwd: one packed self-attention row, causal,
// without query segments or position offsets.  Runs before any CUDA call (bad arguments are reported without a GPU).
inline int check_docs_params(const lv_attn_params* a, const lv_attn_docs* docs, const char* who) {
  LV_CHECK_ARG(docs != nullptr, "%s: null docs", who);
  LV_CHECK_ARG(docs->cu_seqlens != nullptr, "%s: null cu_seqlens", who);
  LV_CHECK_ARG(docs->n_docs >= 1 && docs->n_docs <= a->sk, "%s: n_docs=%lld out of range [1, sk=%lld]", who,
               (long long)docs->n_docs, (long long)a->sk);
  LV_CHECK_ARG(a->batch == 1, "%s: packed documents need batch 1 (got %lld)", who, (long long)a->batch);
  LV_CHECK_ARG(a->sq == a->sk, "%s: packed documents need sq == sk (self-attention), got %lld / %lld", who,
               (long long)a->sq, (long long)a->sk);
  LV_CHECK_ARG(a->causal != 0, "%s: packed documents need causal = 1", who);
  LV_CHECK_ARG(a->q_seg_len == a->sq, "%s: packed documents need q_seg_len == sq (one query segment)", who);
  LV_CHECK_ARG(a->kv_pos0 == 0 && a->q_seg_pos[0] == 0 && a->q_seg_pos[1] == 0,
               "%s: packed documents need kv_pos0 = 0 and q_seg_pos = {0, 0}", who);
  return LV_OK;
}

}  // namespace lv
