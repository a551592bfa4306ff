// Device functions shared by the fused sampler (sampler.cu) and the beam-search step (beam.cu): the logits processors that read a
// sequence's generated-token history and the exact top-k threshold over one vocabulary row held in shared memory.  Both kernels run
// one CTA of NT threads per row.
#pragma once
#include "common.cuh"

namespace vcla {

__device__ __forceinline__ uint32_t order_key(float x) {   // monotone: a < b  <=>  key(a) < key(b)  (NaN sorts below everything)
  if (x != x) return 0u;
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ int block_count(int local, int* s_cnt) {
  const int w = __reduce_add_sync(0xffffffffu, local);
  __syncthreads();
  if (threadIdx.x == 0) *s_cnt = 0;
  __syncthreads();
  if ((threadIdx.x & 31) == 0 && w) atomicAdd(s_cnt, w);
  __syncthreads();
  return *s_cnt;
}

// HF's history processors on s_row, in HF's order (HF:generation/logits_process.py), for column b of the history [L][B]:
//   RepetitionPenaltyLogitsProcessor  x<0 ? x*p : x/p on every token of the generated history, once per distinct token
//   NoRepeatNGramLogitsProcessor      ban every token that would complete an n-gram already present in the history
//   (min_new_tokens)                  EOS ids masked while fewer than min_new_tokens tokens exist
// s_seen (vpad / 32 words) must be zero on entry.  Ends with a barrier.
template <int NT>
__device__ __forceinline__ void history_processors(float* s_row, uint32_t* s_seen, int V, const int32_t* __restrict__ history, int B, int b,
                                                   int L, float rep_penalty, int n, int n_eos, const int* eos, int min_new_tokens) {
  const int tid = threadIdx.x;
  const float NEG_INF = -INFINITY;
  // ---- repetition penalty: once per distinct token of the history
  if (rep_penalty != 1.0f) {
    for (int i = tid; i < L; i += NT) {
      const int t = history[(size_t)i * B + b];
      if (t >= 0 && t < V) {
        const uint32_t bit = 1u << (t & 31);
        const uint32_t old = atomicOr(&s_seen[t >> 5], bit);
        if (!(old & bit)) {
          const float x = s_row[t];
          s_row[t] = x < 0.f ? x * rep_penalty : __fdiv_rn(x, rep_penalty);
        }
      }
    }
    __syncthreads();
  }
  // ---- no-repeat-ngram: windows [i, i+n) of the history whose first n-1 tokens equal the last n-1 tokens ban their last token
  if (n > 0 && L + 1 >= n) {
    for (int i = tid; i + n <= L; i += NT) {
      bool same = true;
      for (int j = 0; j < n - 1 && same; ++j) same = history[(size_t)(i + j) * B + b] == history[(size_t)(L - n + 1 + j) * B + b];
      if (same) {
        const int t = history[(size_t)(i + n - 1) * B + b];
        if (t >= 0 && t < V) s_row[t] = NEG_INF;
      }
    }
    __syncthreads();
  }
  if (tid < n_eos && L < min_new_tokens) { const int e = eos[tid]; if (e >= 0 && e < V) s_row[e] = NEG_INF; }
  __syncthreads();
}

// The key of the k-th largest element of s_row[0, V) (k <= V).  Two levels instead of 32 counting passes over the whole row:
//  (1) T1 = the k-th largest of the NT per-thread maxima (bit search with __syncthreads_count: one barrier per bit).  At least
//      k elements are >= T1, so the k-th largest element of the row is >= T1: every top-k element survives the pre-filter.
//  (2) the (few) elements >= T1 are collected and the exact k-th largest is found among them.
// If the pre-filter keeps more than the candidate buffer holds (MAXKEEP, a row full of ties), the exact bit search over the row runs.
// On entry *s_n == 0 and *s_thr == 0xFFFFFFFF; on exit *s_n == 0.  s_val / s_idx: MAXKEEP scratch entries.
template <int NT, int MAXKEEP>
__device__ __forceinline__ uint32_t topk_threshold(const float* s_row, int V, int k, float* s_val, int* s_idx, int* s_cnt, int* s_n,
                                                   unsigned int* s_thr) {
  const int tid = threadIdx.x;
  uint32_t my_max = 0u;
  for (int v = tid; v < V; v += NT) { const uint32_t key = order_key(s_row[v]); my_max = key > my_max ? key : my_max; }
  uint32_t T = 0u;
  if (k <= NT) {
    for (int bit = 31; bit >= 0; --bit) {
      const uint32_t cand = T | (1u << bit);
      if (__syncthreads_count(my_max >= cand) >= k) T = cand;
    }
    int c1 = 0;
    for (int v = tid; v < V; v += NT) c1 += order_key(s_row[v]) >= T;
    const int n1 = block_count(c1, s_cnt);
    if (n1 <= MAXKEEP) {
      // exact k-th largest among the n1 pre-filtered elements (rank by counting)
      for (int v = tid; v < V; v += NT) {
        const float x = s_row[v];
        if (order_key(x) >= T) { const int pos = atomicAdd(s_n, 1); s_val[pos] = x; s_idx[pos] = v; }
      }
      __syncthreads();
      if (tid < n1) {
        const uint32_t kx = order_key(s_val[tid]);
        int greater = 0;
        for (int j = 0; j < n1; ++j) greater += order_key(s_val[j]) > kx;
        // the k-th largest value is the smallest key that still has fewer than k strictly greater elements
        if (greater < k) atomicMin(s_thr, kx);
      }
      __syncthreads();
      T = *s_thr;
      __syncthreads();
      if (tid == 0) { *s_n = 0; }
      __syncthreads();
    } else {
      T = 0u;
    }
  }
  if (T == 0u) {
    // exact bit search over the whole row: largest T with count(key >= T) >= k
    for (int bit = 31; bit >= 0; --bit) {
      const uint32_t cand = T | (1u << bit);
      int c = 0;
      for (int v = tid; v < V; v += NT) c += order_key(s_row[v]) >= cand;
      if (block_count(c, s_cnt) >= k) T = cand;
    }
  }
  return T;
}

}  // namespace vcla
