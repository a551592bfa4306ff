// Beam search without sampling (HF:generation/utils.py:2876-3395, the vectorised _beam_search of transformers 5.5), as two kernels
// per decode step inside the captured CUDA graph, right after the lm_head reduction:
//   dec_beam_step_kernel    one CTA per beam row: log_softmax, the history processors on that beam's own history, + the beam's
//                           running score, exact top-M of the row (M = max(2, 1 + n_eos) * K candidates)
//   dec_beam_select_kernel  one CTA per batch item: the global top-M of the item's K * M row candidates (it lies inside their union),
//                           stopping-criteria hits, the next K running beams, the finished-hypothesis store, the early-stop heuristic
// With inputs_embeds the prompt is not part of input_ids: decoder_prompt_len = 0, the processors see the generated tokens only and the
// length penalty divides by the generated length.  The K/V of the chosen beams are rearranged afterwards through the page table
// (kv_beam_reorder, elementwise.cu).
#include "kernels.h"
#include "logits_chain.cuh"

namespace vcla {

constexpr int kBeamThreads = 1024;
constexpr int kBeamMaxKeep = 1024;   // pre-filter candidate buffer of the top-M threshold search
constexpr int kSelThreads = 512;
constexpr float kBeamNeg = -1.0e9f;  // HF's "very large negative value" (exactly representable in fp32)

__device__ __forceinline__ float block_reduce_max(float v, float* red) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
  for (int w = 1; w < (int)(blockDim.x >> 5); ++w) r = fmaxf(r, red[w]);
  return r;
}
__device__ __forceinline__ float block_reduce_sum(float v, float* red) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) r += red[w];
  return r;
}

// history: [t][rows] (column r = this beam's generated tokens); run_score: [rows] or null (the first step: every row scores 0)
__global__ void __launch_bounds__(kBeamThreads, 1)
dec_beam_step_kernel(const float* __restrict__ logits, int ld, int V, int rows, const int32_t* __restrict__ history, const int32_t* __restrict__ step_idx,
                     const BeamParams* __restrict__ pp, const float* __restrict__ run_score, float* __restrict__ cand_val, int32_t* __restrict__ cand_tok) {
  extern __shared__ __align__(16) uint8_t s_raw[];
  float* s_row = reinterpret_cast<float*>(s_raw);
  const int vpad = (V + 31) & ~31;
  uint32_t* s_seen = reinterpret_cast<uint32_t*>(s_row + vpad);
  float* s_val = reinterpret_cast<float*>(s_seen + vpad / 32);
  int* s_idx = reinterpret_cast<int*>(s_val + kBeamMaxKeep);
  __shared__ int s_cnt, s_n;
  __shared__ unsigned int s_thr;
  __shared__ float s_red[32];
  __shared__ float s_cv[kBeamMaxCand];
  __shared__ int s_ci[kBeamMaxCand];

  TraceScope trace(15);
  trace.dep();
  const int r = blockIdx.x, tid = threadIdx.x;
  const BeamParams p = *pp;
  const int L = *step_idx;
  const int M = p.M;

  float mx = -INFINITY;
  for (int v = tid; v < V; v += kBeamThreads) { const float x = logits[(size_t)r * ld + v]; s_row[v] = x; mx = fmaxf(mx, x); }
  for (int i = tid; i < vpad / 32; i += kBeamThreads) s_seen[i] = 0u;
  if (tid == 0) { s_n = 0; s_thr = 0xFFFFFFFFu; }
  // ---- log_softmax (HF:generation/utils.py:3256): x - max - log(sum(exp(x - max)))
  mx = block_reduce_max(mx, s_red);
  float sum = 0.f;
  for (int v = tid; v < V; v += kBeamThreads) sum += expf(s_row[v] - mx);
  sum = block_reduce_sum(sum, s_red);
  const float lse = logf(sum);
  for (int v = tid; v < V; v += kBeamThreads) s_row[v] = (s_row[v] - mx) - lse;
  __syncthreads();
  // ---- processors on the log-probabilities (:3257), then + the running score (:3287)
  history_processors<kBeamThreads>(s_row, s_seen, V, history, rows, r, L, p.rep_penalty, p.no_repeat_ngram, p.n_eos, p.eos, p.min_new_tokens);
  const float rs = run_score ? run_score[r] : 0.f;
  for (int v = tid; v < V; v += kBeamThreads) s_row[v] = s_row[v] + rs;
  __syncthreads();
  // ---- exact top-M of the row, ordered by (score desc, token asc)
  const uint32_t T = topk_threshold<kBeamThreads, kBeamMaxKeep>(s_row, V, M, s_val, s_idx, &s_cnt, &s_n, &s_thr);
  for (int v = tid; v < V; v += kBeamThreads) {
    const float x = s_row[v];
    if (order_key(x) >= T) { const int pos = atomicAdd(&s_n, 1); if (pos < kBeamMaxKeep) { s_val[pos] = x; s_idx[pos] = v; } }
  }
  __syncthreads();
  const int c = s_n < kBeamMaxKeep ? s_n : kBeamMaxKeep;
  for (int i = tid; i < c; i += kBeamThreads) {
    const float xv = s_val[i]; const int xi = s_idx[i];
    int rk = 0;
    for (int j = 0; j < c; ++j) { const float y = s_val[j]; rk += (y > xv) || (y == xv && s_idx[j] < xi); }
    if (rk < M) { s_cv[rk] = xv; s_ci[rk] = xi; }
  }
  __syncthreads();
  if (tid < M) { cand_val[(size_t)r * M + tid] = s_cv[tid]; cand_tok[(size_t)r * M + tid] = s_ci[tid]; }
  trace.done();
}

// One CTA per batch item b; R = rows per item (1 at the first step, where every beam is still the prompt, else K).  Candidates of
// item b: cand_*[(b * R + k) * M + i].  Writes the next running beams j = 0..K-1 of the item (slot b * K + j): parent_row (the global
// row it continues), tok, run_score; updates the store hyp_* [b][K] (scores, lengths, finished flags, token rows of hyp_cap
// tokens) and item_state [b][2] = {early-stop heuristic unsatisfied, done}.  cand_out (nullable, operator tests): the item's global
// top-M as [b][M][2] = {flat index k * V + v, hit}.
__global__ void __launch_bounds__(kSelThreads)
dec_beam_select_kernel(const BeamParams* __restrict__ pp, int R, int V, const int32_t* __restrict__ step_idx, const float* __restrict__ cand_val,
                       const int32_t* __restrict__ cand_tok, const int32_t* __restrict__ history, float* __restrict__ run_score,
                       int32_t* __restrict__ parent_row, int32_t* __restrict__ tok, float* __restrict__ hyp_score, int32_t* __restrict__ hyp_len,
                       int32_t* __restrict__ hyp_fin, int32_t* __restrict__ hyp_tok, int32_t* __restrict__ hyp_tmp, int hyp_cap,
                       int32_t* __restrict__ item_state, int32_t* __restrict__ cand_out) {
  __shared__ float s_v[kBeamMaxCand * kBeamMaxK];
  __shared__ int s_f[kBeamMaxCand * kBeamMaxK];
  __shared__ float s_sv[kBeamMaxCand];
  __shared__ int s_sf[kBeamMaxCand];
  __shared__ int s_src[kBeamMaxK];      // new store slot s <- old slot (< K) or candidate K + i
  TraceScope trace(16);
  trace.dep();
  const int b = blockIdx.x, tid = threadIdx.x;
  const BeamParams p = *pp;
  const int K = p.K, M = p.M, n = R * M;
  const int t = *step_idx;                    // tokens generated before this step's pick
  const int hist_rows = gridDim.x * R;

  for (int i = tid; i < n; i += kSelThreads) {
    const int k = i / M;
    s_v[i] = cand_val[(size_t)(b * R) * M + i];
    s_f[i] = k * V + cand_tok[(size_t)(b * R) * M + i];
  }
  __syncthreads();
  // global top-M of the item: rank by (score desc, flat index asc) -- torch.topk over K * V (:2981) with ties to the lower index
  for (int i = tid; i < n; i += kSelThreads) {
    const float xv = s_v[i]; const int xf = s_f[i];
    int rk = 0;
    for (int j = 0; j < n; ++j) { const float y = s_v[j]; rk += (y > xv) || (y == xv && s_f[j] < xf); }
    if (rk < M) { s_sv[rk] = xv; s_sf[rk] = xf; }
  }
  __syncthreads();

  if (tid == 0) {
    float* hs = hyp_score + (size_t)b * K;
    int32_t* hl = hyp_len + (size_t)b * K;
    int32_t* hf = hyp_fin + (size_t)b * K;
    int32_t* st = item_state + (size_t)b * 2;
    if (t == 0) {                             // HF:3197-3208: empty store, heuristic unsatisfied
      for (int s = 0; s < K; ++s) { hs[s] = kBeamNeg; hl[s] = 0; hf[s] = 0; }
      st[0] = 1; st[1] = 0;
    }
    // stopping criteria on each candidate (:3306): EOS, or max_new_tokens reached (MaxLengthCriteria)
    bool hit[kBeamMaxCand];
    bool all_hit = true;
    for (int i = 0; i < M; ++i) {
      const int v = s_sf[i] % V;
      bool h = t + 1 >= p.max_new;
      for (int e = 0; e < p.n_eos; ++e) h |= v == p.eos[e];
      hit[i] = h; all_hit &= h;
    }
    // next running beams (:3013-3018): top K of score - 1e9 * hit
    float run[kBeamMaxCand];
    bool used[kBeamMaxCand];
    for (int i = 0; i < M; ++i) { run[i] = s_sv[i] + (hit[i] ? kBeamNeg : -0.0f); used[i] = false; }
    float best_run = 0.f;
    for (int s = 0; s < K; ++s) {
      int bi = -1;
      for (int i = 0; i < M; ++i) if (!used[i] && (bi < 0 || run[i] > run[bi])) bi = i;
      used[bi] = true;
      const int j = b * K + s;
      parent_row[j] = b * R + s_sf[bi] / V;
      tok[j] = s_sf[bi] % V;
      run_score[j] = run[bi];
      if (s == 0) best_run = run[bi];
    }
    // finished hypotheses (:3046-3071)
    bool all_fin = true;
    for (int s = 0; s < K; ++s) all_fin &= hf[s] != 0;
    const bool full = all_fin && p.early_stopping == 1;
    const bool unsat = st[0] != 0;
    const float den = (float)pow((double)(t + 1), (double)p.length_penalty);
    float ns[kBeamMaxCand];
    for (int i = 0; i < M; ++i) {
      const bool did = hit[i] && i < K;
      float x = __fdiv_rn(s_sv[i], den);
      x = x + (full ? kBeamNeg : -0.0f);
      x = x + (unsat ? -0.0f : kBeamNeg);
      x = x + (did ? -0.0f : kBeamNeg);
      ns[i] = x;
    }
    // merge [old K | new M] and keep the top K (torch.cat + topk order, ties to the lower index)
    bool taken[kBeamMaxK + kBeamMaxCand];
    for (int i = 0; i < K + M; ++i) taken[i] = false;
    float nsc[kBeamMaxK]; int nlen[kBeamMaxK], nfin[kBeamMaxK];
    for (int s = 0; s < K; ++s) {
      int bi = -1; float bv = 0.f;
      for (int i = 0; i < K + M; ++i) {
        if (taken[i]) continue;
        const float v = i < K ? hs[i] : ns[i - K];
        if (bi < 0 || v > bv) { bi = i; bv = v; }
      }
      taken[bi] = true;
      s_src[s] = bi;
      nsc[s] = bv;
      nlen[s] = bi < K ? hl[bi] : t + 1;
      nfin[s] = bi < K ? hf[bi] : ((hit[bi - K] && bi - K < K) ? 1 : 0);
    }
    bool fin_now = true; float mn = 0.f;
    for (int s = 0; s < K; ++s) {
      hs[s] = nsc[s]; hl[s] = nlen[s]; hf[s] = nfin[s];
      fin_now &= nfin[s] != 0;
      mn = s == 0 ? nsc[s] : fminf(mn, nsc[s]);
    }
    // early-stop heuristic (:2912-2920) at cur_len = t + 1, and this item's share of the loop condition (:2933-2943)
    const int hyp = (p.early_stopping == 2 && p.length_penalty > 0.f) ? p.max_new : t + 1;
    const float bp = __fdiv_rn(best_run, (float)pow((double)hyp, (double)p.length_penalty));
    bool any = false;
    for (int s = 0; s < K; ++s) any |= bp > (nfin[s] ? mn : kBeamNeg);
    const bool unsat_new = unsat && any;
    st[0] = unsat_new ? 1 : 0;
    st[1] = (st[1] || !unsat_new || (fin_now && p.early_stopping == 1) || all_hit) ? 1 : 0;
    if (cand_out) for (int i = 0; i < M; ++i) { cand_out[((size_t)b * M + i) * 2] = s_sf[i]; cand_out[((size_t)b * M + i) * 2 + 1] = hit[i] ? 1 : 0; }
  }
  __syncthreads();
  // token rows of the new store: an old hypothesis keeps its row, a new one is its beam's history + the candidate token
  const int len = t + 1;
  for (int e = tid; e < K * len; e += kSelThreads) {
    const int s = e / len, pos = e % len, src = s_src[s];
    int v;
    if (src < K) v = hyp_tok[((size_t)b * K + src) * hyp_cap + pos];
    else {
      const int f = s_sf[src - K];
      v = pos < t ? history[(size_t)pos * hist_rows + b * R + f / V] : f % V;
    }
    hyp_tmp[((size_t)b * K + s) * hyp_cap + pos] = v;
  }
  __syncthreads();
  for (int e = tid; e < K * len; e += kSelThreads) {
    const int s = e / len, pos = e % len;
    hyp_tok[((size_t)b * K + s) * hyp_cap + pos] = hyp_tmp[((size_t)b * K + s) * hyp_cap + pos];
  }
  trace.done();
}

size_t beam_step_smem_bytes(int V) {
  const size_t vpad = (size_t)((V + 31) & ~31);
  return vpad * 4 + vpad / 8 + (size_t)kBeamMaxKeep * 8;
}

int beam_init() {
  static bool done = false;
  if (done) return 0;
  done = true;
  VCLA_CUDA_OK(cudaFuncSetAttribute(dec_beam_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024 - 1024 - 4096)));
  return 0;
}

int beam_supported(int V) { return beam_step_smem_bytes(V) <= 227u * 1024u - 1024u - 4096u ? 1 : 0; }

int dec_beam_step(const float* logits, int ld, int V, int rows, const int32_t* history, const int32_t* step_idx, const BeamParams* params_dev,
                  const float* run_score, float* cand_val, int32_t* cand_tok, cudaStream_t st) {
  if (!beam_supported(V)) { set_error("beam search: vocabulary %d does not fit one CTA's shared memory", V); return -1; }
  if (rows < 1 || rows > 64) { set_error("beam search: %d rows", rows); return -1; }
  dec_beam_step_kernel<<<rows, kBeamThreads, beam_step_smem_bytes(V), st>>>(logits, ld, V, rows, history, step_idx, params_dev, run_score, cand_val, cand_tok);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

int dec_beam_select(const BeamParams* params_dev, int items, int R, int V, const int32_t* step_idx, const float* cand_val, const int32_t* cand_tok,
                    const int32_t* history, float* run_score, int32_t* parent_row, int32_t* tok, float* hyp_score, int32_t* hyp_len, int32_t* hyp_fin,
                    int32_t* hyp_tok, int32_t* hyp_tmp, int hyp_cap, int32_t* item_state, int32_t* cand_out, cudaStream_t st) {
  if (items < 1 || items > 32) { set_error("beam search: %d items", items); return -1; }
  dec_beam_select_kernel<<<items, kSelThreads, 0, st>>>(params_dev, R, V, step_idx, cand_val, cand_tok, history, run_score, parent_row, tok, hyp_score,
                                                         hyp_len, hyp_fin, hyp_tok, hyp_tmp, hyp_cap, item_state, cand_out);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

VCLA_DEFINE_TRACE_SETTER(trace_set_beam)

}  // namespace vcla
