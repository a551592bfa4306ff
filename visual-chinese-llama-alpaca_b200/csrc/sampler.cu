// Device-side sampling stack (SURVEY 8f-1): the logits-processor chain HF's generate() builds for the reference's
// DEFAULT_GENERATION_CONFIG (models/visualcla/modeling_utils.py:36-47) -- repetition penalty, no-repeat-ngram, temperature, top-k,
// top-p -- plus the multinomial draw, fused into ONE kernel per decode step that runs inside the captured CUDA graph right after
// the lm_head reduction.  One CTA per sequence; the sequence's logits row lives in shared memory for the whole chain.
//
// Semantics follow transformers' processors (HF:generation/logits_process.py), in HF's order:
//   RepetitionPenaltyLogitsProcessor  x<0 ? x*p : x/p on every token of the generated history, once per distinct token
//   NoRepeatNGramLogitsProcessor      ban every token that would complete an n-gram already present in the history
//   (min_new_tokens)                  EOS ids masked while fewer than min_new_tokens tokens exist
//   TemperatureLogitsWarper           x / T
//   TopKLogitsWarper                  keep x >= (k-th largest x)  (ties at the k-th value are all kept, as HF does)
//   TopPLogitsWarper                  ascending cumulative softmax <= 1 - top_p removed; the largest is always kept
//   multinomial                       inverse-CDF draw with a Philox4x32-10 uniform keyed by (seed, step, sequence)
// With inputs_embeds the processors only ever see the NEW tokens (HF starts input_ids empty), i.e. the device token history.
#include "kernels.h"
#include "logits_chain.cuh"

namespace vcla {

constexpr int kSampThreads = 1024;
constexpr int kSampMaxKeep = 1024;   // candidates surviving top-k (k plus ties at the k-th value)

// Philox4x32-10 (Salmon et al. 2011), counter = (step, sequence, 0, 0), key = seed
__device__ __forceinline__ float philox_uniform(unsigned long long seed, uint32_t c0, uint32_t c1) {
  uint32_t ctr[4] = {c0, c1, 0u, 0u};
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr[0]), lo0 = 0xD2511F53u * ctr[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr[2]), lo1 = 0xCD9E8D57u * ctr[2];
    const uint32_t n0 = hi1 ^ ctr[1] ^ k0, n2 = hi0 ^ ctr[3] ^ k1;
    ctr[0] = n0; ctr[1] = lo1; ctr[2] = n2; ctr[3] = lo0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return (float)(ctr[0] >> 8) * (1.0f / 16777216.0f);   // [0, 1)
}

// LOOKUP (prompt lookup verification, B = 1): CTA r scores query row r, whose history is column 0 with length *step_idx + r (the drafts
// being verified sit provisionally at rows *step_idx ..), and draws with counter (*step_idx + r, 0): exactly the draw one-token decoding
// makes at that length.  finished is neither read nor written (the accept kernel owns it); tok[r] receives the pick.
// fanout (not LOOKUP): sequence b reads logits row b / fanout -- the prefill's pick of N replies per prompt, where the B = prompts x N
// rows forked from one prompt share its last logits row and differ in their draw counters (L, b).  1 everywhere else.
template <bool LOOKUP = false>
__global__ void __launch_bounds__(kSampThreads, 1)
dec_sample_kernel(const float* __restrict__ logits, int ld, int V, int B, const int32_t* __restrict__ history, const int32_t* __restrict__ step_idx,
                  const SamplerParams* __restrict__ pp, int32_t* __restrict__ tok, int32_t* __restrict__ history_out, int32_t* __restrict__ dp_send,
                  int32_t* __restrict__ finished, float* __restrict__ scores_out, int fanout) {
  extern __shared__ __align__(16) uint8_t s_raw[];
  float* s_row = reinterpret_cast<float*>(s_raw);
  const int vpad = (V + 31) & ~31;
  uint32_t* s_seen = reinterpret_cast<uint32_t*>(s_row + vpad);            // vpad / 32 words
  float* s_val = reinterpret_cast<float*>(s_seen + vpad / 32);
  int* s_idx = reinterpret_cast<int*>(s_val + kSampMaxKeep);
  float* s_sval = reinterpret_cast<float*>(s_idx + kSampMaxKeep);
  int* s_sidx = reinterpret_cast<int*>(s_sval + kSampMaxKeep);
  __shared__ int s_cnt, s_n, s_choice, s_keep;
  __shared__ unsigned int s_thr;
  __shared__ float s_bv[32];
  __shared__ int s_bi[32];

  TraceScope trace(14);
  pdl_launch_dependents();
  pdl_wait();
  trace.dep();
  const int b = LOOKUP ? 0 : blockIdx.x, tid = threadIdx.x;
  const int row = blockIdx.x, lrow = LOOKUP ? row : row / fanout;
  const SamplerParams p = *pp;
  const int L = *step_idx + (LOOKUP ? row : 0);     // tokens generated so far = rows of the history
  const float NEG_INF = -INFINITY;

  for (int v = tid; v < V; v += kSampThreads) s_row[v] = logits[(size_t)lrow * ld + v];
  for (int i = tid; i < vpad / 32; i += kSampThreads) s_seen[i] = 0u;
  if (tid == 0) { s_n = 0; s_choice = 0; s_keep = 0; s_thr = 0xFFFFFFFFu; }
  __syncthreads();

  history_processors<kSampThreads>(s_row, s_seen, V, history, LOOKUP ? 1 : B, b, L, p.rep_penalty, p.no_repeat_ngram, p.n_eos, p.eos, p.min_new_tokens);

  int chosen = 0;
  if (!p.do_sample) {
    // greedy over the processed scores (first maximum wins, like torch.argmax)
    float best = NEG_INF; int bi = 0x7fffffff;
    for (int v = tid; v < V; v += kSampThreads) { const float x = s_row[v]; if (x > best || (x == best && v < bi)) { best = x; bi = v; } }
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if ((tid & 31) == 0) { s_bv[tid >> 5] = best; s_bi[tid >> 5] = bi; }
    __syncthreads();
    if (tid < 32) {
      best = s_bv[tid]; bi = s_bi[tid];
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o); const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
      }
      if (tid == 0) s_choice = (bi == 0x7fffffff) ? 0 : bi;
    }
    __syncthreads();
    if (scores_out) for (int v = tid; v < V; v += kSampThreads) scores_out[(size_t)row * V + v] = s_row[v];
    chosen = s_choice;
  } else {
    // ---- temperature
    if (p.temperature != 1.0f) {
      for (int v = tid; v < V; v += kSampThreads) s_row[v] = __fdiv_rn(s_row[v], p.temperature);
      __syncthreads();
    }
    // ---- top-k threshold = the k-th largest key
    const int k = p.top_k < V ? p.top_k : V;
    const uint32_t T = topk_threshold<kSampThreads, kSampMaxKeep>(s_row, V, k, s_val, s_idx, &s_cnt, &s_n, &s_thr);
    // ---- candidates (k plus ties), sorted by (value desc, index asc)
    for (int v = tid; v < V; v += kSampThreads) {
      const float x = s_row[v];
      if (order_key(x) >= T) { const int pos = atomicAdd(&s_n, 1); if (pos < kSampMaxKeep) { s_val[pos] = x; s_idx[pos] = v; } }
    }
    __syncthreads();
    const int c = s_n < kSampMaxKeep ? s_n : kSampMaxKeep;
    if (tid < c) {
      const float xv = s_val[tid]; const int xi = s_idx[tid];
      int r = 0;
      for (int j = 0; j < c; ++j) { const float y = s_val[j]; r += (y > xv) || (y == xv && s_idx[j] < xi); }
      s_sval[r] = xv; s_sidx[r] = xi;
    }
    __syncthreads();
    // ---- top-p + draw (sequential: c is ~k; the order of the sums is the order of a CPU cumsum)
    if (tid == 0) {
      const float m = s_sval[0];
      float sum = 0.f;
      for (int r = 0; r < c; ++r) sum += expf(s_sval[r] - m);
      int keep = c;
      if (p.top_p < 1.0f) {
        float cum = 0.f;                                        // ascending cumulative probability, smallest first
        for (int r = c - 1; r >= 1; --r) {
          cum += expf(s_sval[r] - m) / sum;
          if (cum <= p.one_minus_top_p) keep = r; else break;
        }
      }
      if (keep < 1) keep = 1;
      float tot = 0.f;
      for (int r = 0; r < keep; ++r) tot += expf(s_sval[r] - m);
      const float u = philox_uniform(p.seed, (uint32_t)L, (uint32_t)b) * tot;
      float acc = 0.f; int pick = keep - 1;
      for (int r = 0; r < keep; ++r) { acc += expf(s_sval[r] - m); if (acc > u) { pick = r; break; } }
      s_choice = s_sidx[pick];
      s_keep = keep;
    }
    __syncthreads();
    if (scores_out) {
      for (int v = tid; v < V; v += kSampThreads) scores_out[(size_t)row * V + v] = NEG_INF;
      __syncthreads();
      if (tid < s_keep) scores_out[(size_t)row * V + s_sidx[tid]] = s_sval[tid];
    }
    chosen = s_choice;
  }
  if (LOOKUP) {
    if (tid == 0) tok[row] = chosen;
    return;
  }
  if (tid == 0) {
    int t = chosen;
    if (finished) {
      if (finished[b]) t = p.pad_id;
      else for (int e = 0; e < p.n_eos; ++e) if (t == p.eos[e]) finished[b] = 1;
    }
    if (tok) tok[b] = t;
    if (history_out) history_out[(size_t)L * B + b] = t;
    if (dp_send) dp_send[b] = t;
  }
}

size_t sampler_smem_bytes(int V) {
  const size_t vpad = (size_t)((V + 31) & ~31);
  return vpad * 4 + vpad / 8 + (size_t)kSampMaxKeep * 16;
}

int sampler_supported(int V) { return sampler_smem_bytes(V) <= 227u * 1024u - 1024u ? 1 : 0; }

int dec_sample(const float* logits, int ld, int V, int B, const int32_t* history, const int32_t* step_idx, const SamplerParams* params_dev,
               int32_t* tok, int32_t* history_out, int32_t* dp_send, int32_t* finished, float* scores_out, cudaStream_t st, int fanout) {
  if (!sampler_supported(V)) { set_error("device sampler: vocabulary %d does not fit one CTA's shared memory", V); return -1; }
  if (fanout < 1 || B % fanout != 0) { set_error("device sampler: %d rows are not a fan-out of %d per logits row", B, fanout); return -1; }
  const size_t smem = sampler_smem_bytes(V);      // the opt-in for this much dynamic shared memory is done by sampler_init()
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(B); cfg.blockDim = dim3(kSampThreads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (pdl_enabled()) { attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[na].val.programmaticStreamSerializationAllowed = 1; ++na; }
  cfg.attrs = attr; cfg.numAttrs = na;
  VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, dec_sample_kernel<false>, logits, ld, V, B, history, step_idx, params_dev, tok, history_out, dp_send, finished, scores_out, fanout));
  return 0;
}

int dec_sample_lookup(const float* logits, int ld, int V, int R, const int32_t* history, const int32_t* step_idx, const SamplerParams* params_dev,
                      int32_t* tok, cudaStream_t st) {
  if (!sampler_supported(V)) { set_error("device sampler: vocabulary %d does not fit one CTA's shared memory", V); return -1; }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(R); cfg.blockDim = dim3(kSampThreads); cfg.dynamicSmemBytes = sampler_smem_bytes(V); cfg.stream = st;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (pdl_enabled()) { attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[na].val.programmaticStreamSerializationAllowed = 1; ++na; }
  cfg.attrs = attr; cfg.numAttrs = na;
  VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, dec_sample_kernel<true>, logits, ld, V, 1, history, step_idx, params_dev, tok, (int32_t*)nullptr,
                                  (int32_t*)nullptr, (int32_t*)nullptr, (float*)nullptr, 1));
  return 0;
}

int sampler_init() {
  // opt in to the dynamic shared memory once per process, outside any graph capture
  static bool done = false;
  if (done) return 0;
  done = true;
  VCLA_CUDA_OK(cudaFuncSetAttribute(dec_sample_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024 - 1024)));
  VCLA_CUDA_OK(cudaFuncSetAttribute(dec_sample_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(227 * 1024 - 1024)));
  return 0;
}

VCLA_DEFINE_TRACE_SETTER(trace_set_sampler)

}  // namespace vcla
