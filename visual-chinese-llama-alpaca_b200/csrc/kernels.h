// Host-side launch API of every CUDA kernel on the VisualCLA path (internal to libvcla.so).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stddef.h>
#include <stdint.h>

namespace vcla {

typedef __nv_bfloat16 bf16;

void set_error(const char* fmt, ...);
const char* get_error();
int num_sms();
bool pdl_enabled();
void set_pdl(bool on);

#define VCLA_CUDA_OK(expr)                                                                   \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      vcla::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      (void)cudaGetLastError();                                                              \
      return -1;                                                                             \
    }                                                                                        \
  } while (0)

// ------------------------------------------------------------------------------------------
// wgmma GEMM:  D[M,N] = A[M,K] * B[N,K]^T   (both operands K-major bf16, fp32 accumulate in registers)
// ------------------------------------------------------------------------------------------
enum GemmMode {
  GEMM_STORE_BF16 = 0,   // out_bf16[orow, col] = act(acc + bias[col])
  GEMM_ADD_F32 = 1,      // out_f32[orow, col]  = (accumulate ? old : 0) + acc + bias[col] + rowtab[(row % period), col]
  GEMM_SWIGLU_BF16 = 2,  // B rows interleaved [32 gate | 32 up]: out_bf16[orow, col/2] = silu(g) * u
  GEMM_PARTIAL_F32 = 3,  // swap-AB split-K partials: ws[(split*ws_rows + col) * ldo + row] = acc   (row = A row)
};
enum Act { ACT_NONE = 0, ACT_QUICK_GELU = 1, ACT_GELU_ERF = 2 };

// ---- paged KV cache ------------------------------------------------------------------------------------------------------
// One view of a layer's cache: its page pool and the page table.  The pool holds [total_pages][K|V][heads][page_tokens][128] bf16, so
// every (page, K|V, head) plane is page_tokens contiguous 128-wide rows.  Sequence b's i-th page is table[b][i]: its token t sits in
// slot t % page_tokens of page table[b][t / page_tokens].  This struct is the only place that knows the layout.  It is a field of the
// decode and prefill attention parameter blocks: keep it at 32 bytes, larger blocks change how those kernels are compiled.
//
// The int8 format (KV_INT8, kv_cache_dtype="int8") keeps the same page geometry: `pages` points at the layer's int8 rows
// [total_pages][K|V][heads][page_tokens][128] (row(...) * 128 bytes in), followed by one fp32 scale per row in the same order, so a
// (page, K|V, head) plane is page_tokens x 128 contiguous bytes and its scales page_tokens x 4 contiguous bytes (16 B aligned for
// page_tokens % 8 == 0).  A row holds q = clamp(rint(x * (127 / a)), -127, 127) and s = a / 127 with a = max |x| (the load_in_8bit
// quantiser); attention reads q * s.  The format is a template parameter of the kernels that read the pool, never a field: the
// scale region is derived from total_pages, and a bf16 kernel compiles exactly as it does without the int8 format.
enum KvFormat { KV_BF16 = 0, KV_INT8 = 1 };
constexpr int kKvQ8RowBytes = 128 + 4;   // int8 row + its fp32 scale
struct KvPool {
  bf16* pages = nullptr;
  int32_t* table = nullptr;          // [sequences][pages_per_seq]
  int heads = 0, page_tokens = 0, pages_per_seq = 0, total_pages = 0;

  // 128-element row of (page, K|V, head, slot) from the start of the pool: I = int for TMA coordinates, size_t for addresses
  template <typename I = size_t>
  __host__ __device__ __forceinline__ I row(int page, int kv, int head, int slot = 0) const {
    return (((I)page * 2 + kv) * heads + head) * page_tokens + slot;
  }
  __host__ __device__ __forceinline__ bf16* at(int page, int kv, int head, int slot) const { return pages + row(page, kv, head, slot) * 128; }
  // KV_INT8: the int8 row and its scale
  __host__ __device__ __forceinline__ int8_t* q8_at(int page, int kv, int head, int slot) const {
    return reinterpret_cast<int8_t*>(pages) + row(page, kv, head, slot) * 128;
  }
  __host__ __device__ __forceinline__ float* q8_scale(int page, int kv, int head, int slot) const {
    return reinterpret_cast<float*>(reinterpret_cast<int8_t*>(pages) + row(total_pages, 0, 0) * 128) + row(page, kv, head, slot);
  }
  __host__ __device__ __forceinline__ int planes() const { return 2 * heads; }   // (K|V, head) planes of a page
  __host__ __device__ __forceinline__ int32_t* seq_pages(int b) const { return table + (size_t)b * pages_per_seq; }
  // pages that hold n tokens, clamped to a table row
  __host__ __device__ __forceinline__ int pages_for(int n) const {
    const int p = (n + page_tokens - 1) / page_tokens;
    return p > pages_per_seq ? pages_per_seq : p;
  }
};
// The cache of every layer (pages is layer 0; the layers share the table) with the state of the device page allocator
// (elementwise.cu), which hands pages to sequences as they grow.
struct KvCache : KvPool {
  int32_t* free_stack = nullptr;     // [total_pages] free physical pages; the top is free_stack[state[0] - 1]
  int32_t* state = nullptr;          // {free pages, exhausted flag}
  int32_t* npages = nullptr;         // [sequences] pages owned: table[b][0 .. npages[b])
  int layers = 1;
  size_t layer_elems = 0;            // layer stride in bf16 units: row(total_pages, 0, 0) * 128, or * 132 / 2 for KV_INT8
  __host__ __device__ __forceinline__ KvPool layer(int i) const { KvPool v = *this; v.pages += i * layer_elems; return v; }
};

// ---- prefill epilogue fusions (non-swap GEMMs) --------------------------------------------------------------------------
// Deferred RMSNorm: the A operand holds xw = bf16(resid * norm_w) (NOT normalised); the row scale rstd[row] =
// rsqrt(sum_slots ssq[row][slot] / dim + eps) commutes with the GEMM and is applied to the accumulator in the epilogue.
struct GemmRowScale {
  const float* ssq = nullptr;   // [M][slots] partial sums of squares of the fp32 residual rows (written by the producing GEMM)
  int slots = 0;
  float inv_dim = 0.f, eps = 0.f;
};
// GEMM_ADD_F32 + accumulate: besides resid += acc, emit the NEXT GEMM's operand and the row statistics:
//   xw[orow, col] = bf16(resid_new * norm_w[col]) ; ssq_out[orow][n_blk] = sum over this tile's columns of resid_new^2
struct GemmEmitNorm {
  const float* norm_w = nullptr;   // [N]
  bf16* xw = nullptr; int ldxw = 0;
  float* ssq_out = nullptr;        // [M][n_tiles]
};
// GEMM_STORE_BF16 on the fused QKV projection [M, 3T]: rotate q and k heads (HF rotate_half pairs d, d+64; fp32 tables
// [pos][64]) on the fp32 accumulator, store q|k|v rows (the prefill attention reads them) AND append k, v to the paged KV cache.
struct GemmRope {
  const float* cos = nullptr; const float* sin = nullptr;
  KvPool kv;                                   // the layer's view; kv.heads heads
  int S = 0, T = 0;                            // rows per sequence, hidden size (= kv.heads * 128)
  const int32_t* left_pad = nullptr; int pos_from_mask = 0;
  const int32_t* base_len = nullptr;           // [B] or null: row t of sequence b is token base_len[b] + t (position and cache slot)
};

struct GemmCall {
  const bf16* A = nullptr;   // [M, K], row pitch lda elements
  const bf16* B = nullptr;   // [N, K], row pitch ldb elements
  int M = 0, N = 0, K = 0;
  int lda = 0, ldb = 0;
  int mode = GEMM_STORE_BF16;
  void* out = nullptr;
  int ldo = 0;
  const float* bias = nullptr;
  int act = ACT_NONE;
  int accumulate = 0;
  const float* rowtab = nullptr;
  int rowtab_period = 1;
  // output row remap: orow = (row / rows_per_group) * group_stride + (row % rows_per_group) + row_offset
  int rows_per_group = 0;    // 0 = identity
  int group_stride = 0;
  int row_offset = 0;
  // split-K (GEMM_PARTIAL_F32 only)
  int splits = 1;
  int ws_rows = 0;           // padded batch rows in the partial workspace
  int weights_are_A = 0;     // cache-policy hint: A is the streamed-once operand (decode)
  int bn = 0;                // tile N override (0 = auto)
  int l2_prefetch_kb = 0;    // k-blocks of the weight operand each CTA prefetches into L2 while it waits for its dependency
  GemmRowScale rowscale;     // deferred RMSNorm scale of the A rows (STORE_BF16 / SWIGLU_BF16)
  GemmEmitNorm emit;         // ADD_F32 + accumulate: also write the next operand + row statistics
  GemmRope rope;             // STORE_BF16: RoPE + KV-cache append (runs on the 64 x 256 tile, N = 3T)
  const float* colscale = nullptr;   // [N] or null: acc[row, col] *= colscale[col] before every epilogue (per-row scales of int8 weights)
  int kv_format = KV_BF16;           // rope.kv's format: KV_INT8 quantises each k / v head row, caches q and s, and stores bf16(q * s)
};
int gemm_tc(const GemmCall& c, cudaStream_t st);
int gemm_pick_bn(int M, int N);   // tile width gemm_tc picks for a non-swap GEMM (= the number of ssq slots per row it emits: ceil(N / bn))
// correctness reference for the tests only (CUDA-core, one thread per output)
int gemm_naive(const GemmCall& c, cudaStream_t st);
int gemm_init();   // resolves cuTensorMapEncodeTiled, sets smem attributes

// ------------------------------------------------------------------------------------------
// decode GEMM with the split-K reduction inside a thread-block cluster (gemm_decode.cu)
//   out[b, n] = sum_k W[n, k] * X[b, k]   W [M = N_out, K] bf16 (streamed), X [B <= 32, K] bf16
// ------------------------------------------------------------------------------------------
enum CskMode {
  CSK_OUT_F32 = 0,   // out[b * ldo + n] = rstd[b] * acc
  CSK_RESID = 1,     // resid[b, n] += acc ; xw[b, n] = bf16(resid * norm_w[n]) ; ssq_out[b, n / 128] = sum over the tile of resid^2
  CSK_SWIGLU = 2,    // W rows interleaved [32 gate | 32 up]: h[b, j] = bf16(silu(rstd[b] * g) * (rstd[b] * u))
};
struct CskCall {
  const bf16* W = nullptr; const bf16* X = nullptr;
  const int8_t* Wq = nullptr; const float* wscale = nullptr;   // int8 weights instead of W (k in fragment order, quant.cu) + fp32 row scales
  int M = 0, B = 0, K = 0;
  int splits = 1;                       // CTAs per cluster = K slices (1..8, every slice non-empty)
  int mode = CSK_OUT_F32;
  float* out = nullptr; int ldo = 0;
  float* resid = nullptr; const float* norm_w = nullptr; bf16* xw = nullptr; float* ssq_out = nullptr;
  bf16* h = nullptr;
  const float* ssq_in = nullptr; int ssq_slots = 0; float inv_dim = 0.f, eps = 0.f;   // rstd[b] = rsqrt(sum_slots ssq_in[b][slot] * inv_dim + eps); null: 1
};
int gemm_csk(const CskCall& c, cudaStream_t st);
int gemm_csk_clusters(int B, int splits, bool q8 = false);   // clusters of `splits` CTAs that can be co-resident (occupancy query, cached)
int gemm_csk_ctas_per_sm(int B, bool q8 = false);            // resident CTAs per SM of the kernel batch B runs (occupancy query)
int trace_set_gemm(void* buf, unsigned long long cap);
int trace_set_attention(void* buf, unsigned long long cap);
int trace_set_gemm_decode(void* buf, unsigned long long cap);
int trace_set_sampler(void* buf, unsigned long long cap);
int trace_set_elementwise(void* buf, unsigned long long cap);

// ------------------------------------------------------------------------------------------
// attention
// ------------------------------------------------------------------------------------------
struct AttnCall {
  const bf16* q = nullptr; int q_stride = 0;            // q[(b*Sq + i)*q_stride + h*HD + d]
  const bf16* k0 = nullptr; const bf16* v0 = nullptr; int kv0_stride = 0; int n0 = 0;   // segment 0: n0 rows / batch
  const bf16* k1 = nullptr; const bf16* v1 = nullptr; int kv1_stride = 0; int n1 = 0;   // segment 1 (optional)
  bf16* out = nullptr; int o_stride = 0;
  int B = 0, H = 0, Sq = 0, HD = 0;
  float scale = 1.f;
  int causal = 0;
  const int32_t* kv_start = nullptr;   // [B] first visible kv index per sequence (left padding); null: 0
};
int attention_prefill(const AttnCall& c, cudaStream_t st);      // dispatches to the wgmma kernel (attention_tc.cu) unless switched off
int attention_prefill_tc(const AttnCall& c, cudaStream_t st);   // wgmma: QK^T and PV on the tensor cores, S / O in registers, Q / K / V by TMA
int attention_prefill_mma(const AttnCall& c, cudaStream_t st);  // mma.sync m16n8k16 fallback (attention.cu)
void attention_set_tc(int mode);                                 // 0: mma.sync everywhere, 1 (default): wgmma at head dim 128, 2: wgmma everywhere (VCLA_ATTN_TC)
int trace_set_attention_tc(void* buf, unsigned long long cap);

// Causal prefill of a chunk of T new rows per sequence over its cached prefix (head dim 128, wgmma kernel of attention_tc.cu):
// queries q[(b*T + t)*q_stride + h*128 + d]; keys / values = the first base_len[b] + T tokens of sequence b in the layer view kv
// (kv.total_pages pages, kv.heads heads), read with TMA; key j is visible to row t iff j <= base_len[b] + t.  max_kv (an upper bound of base_len + T) and the grid size choose the split-KV factor; a split launch
// needs part (attention_paged_partials() x 64 x 132 floats) and counters (attention_paged_partials() int32, zeroed once).
struct AttnPagedCall {
  const bf16* q = nullptr; int q_stride = 0;
  KvPool kv;
  const int32_t* base_len = nullptr;
  int max_kv = 0;
  bf16* out = nullptr; int o_stride = 0;
  int B = 0, T = 0;
  float scale = 1.f;
  float* part = nullptr; int32_t* counters = nullptr;
};
int attention_paged(const AttnPagedCall& c, cudaStream_t st, KvFormat fmt = KV_BF16);   // fmt: c.kv's format
int attention_paged_partials();   // (query tile, head, sequence, split) partials a split launch may need at most
constexpr int kAttnPartialFloats = 64 * 132;

struct DecodeAttnCall {
  const float* qkv_partial = nullptr;  // [splits][ws_rows][3*T] fp32 split-K partials of the fused QKV projection
  int splits = 1, ws_rows = 0;
  const int32_t* seq_len = nullptr;    // [B] tokens already in the cache (the new token is appended at this index)
  bf16* out = nullptr;                 // [ws_rows][T] attention output (bf16, GEMM operand of o_proj)
  float* scratch = nullptr;            // [B][H][kv_splits][HD+2]
  int32_t* counters = nullptr;         // [B][H]
  int B = 0, HD = 0, kv_splits = 1;
  float scale = 1.f, rope_theta = 10000.f;
  const float* rope_cos = nullptr;     // [max_pos][HD/2] fp32 tables owned by the context
  const float* rope_sin = nullptr;
  int persistent_mode = 1;             // VCLA_ATTN_PERSISTENT (read once per context)
  int persistent_grid = 0;             // VCLA_ATTN_PERSISTENT_GRID
  KvPool kv;                           // this layer's view (kv.heads heads of HD = 128)
};
int attention_decode(const DecodeAttnCall& c, cudaStream_t st, KvFormat fmt = KV_BF16);   // fmt: c.kv's format
// Prompt lookup verification over c.B <= 16 query rows of sequence 0 (row r at position seq_len[0] + r, qkv / out row r): two launches,
// the K/V append of every row, then each row's attention over keys [0, seq_len[0] + r] with the one-token kernel's arithmetic at that
// length (c.kv_splits must be the split count the one-token call of sequence 0 uses).  scratch / counters are indexed by row.
int attention_decode_lookup(const DecodeAttnCall& c, cudaStream_t st, KvFormat fmt = KV_BF16);
int attention_decode_ctas_per_sm(const DecodeAttnCall& c, KvFormat fmt = KV_BF16);     // resident CTAs per SM of the kernel attention_decode picks for c
int attention_init();          // sets the dynamic-smem attributes and reads the VCLA_ATTN_* switches once (call outside graph capture)

// ------------------------------------------------------------------------------------------
// normalisation / elementwise / data movement
// ------------------------------------------------------------------------------------------
// y_bf16 = LN(x) * w + b (fp32 statistics); optionally also writes the fp32 normalised row back (in place ok)
int layernorm(const float* x, int rows, int D, const float* w, const float* b, float eps, bf16* y_bf16, float* y_f32,
              cudaStream_t st);
int rmsnorm(const float* x, int rows, int D, const float* w, float eps, bf16* y_bf16, cudaStream_t st);
// head of the deferred-norm chain: xw = bf16(x * w) (not normalised), ssq[row][0] = sum x^2, ssq[row][1..slots) = 0
int prenorm_rows(const float* x, int rows, int D, const float* w, bf16* xw, float* ssq, int slots, cudaStream_t st);
// pixels (B,3,I,I) in f32/f16/bf16 -> im2col rows [B*g*g, Kpad] bf16 (k = c*P*P + ky*P + kx), zero padded
int im2col(const void* pixels, int dtype, int B, int image, int patch, int kpad, bf16* out, cudaStream_t st);
// hidden[b, 0, :] = cls + pos[0]
int vit_cls_rows(float* hidden, int B, int tokens, int D, const float* cls, const float* pos, cudaStream_t st);
int broadcast_rows(const float* src, int rows, int D, int B, float* dst_f32, bf16* dst_bf16, cudaStream_t st);
// text embedding gather into the fp32 residual stream: dst[b, dst_pos(t), :] = table[ids[b,t], :]
//   mode 0: dst_pos = t (text only / placeholder layout: image rows are overwritten afterwards by the projector GEMM)
//   mode 1: image at head: t<2 -> t ; t>=2 -> t + nq
int embed_tokens(const int64_t* ids, int B, int T, int S, int D, const bf16* table, int vocab, int mode, int nq,
                 float* dst, cudaStream_t st);
int embed_tokens_i32(const int32_t* ids, int B, int D, const bf16* table, int vocab, float* dst, cudaStream_t st);
// copy the projected image rows (B, nq, D) fp32 into the residual stream at per-sample row offsets
int scatter_image_rows(const float* img, int B, int nq, int D, const int32_t* row_start, int S, float* dst, cudaStream_t st);
int gather_last_rows(const float* hidden, int B, int S, int D, float* dst, cudaStream_t st);

// decode consumers of split-K partials
// resid[b,:] += sum_s partial[s][b][:]  (partial may be null) ; xn = rmsnorm(resid) -> bf16
int dec_resid_norm(const float* partial, int splits, int ws_rows, float* resid, int B, int D, const float* w, float eps,
                   bf16* xn, cudaStream_t st);
// h[b, j] = silu(sum_s p[s][b][g(j)]) * (sum_s p[s][b][u(j)])  with the [32 gate | 32 up] interleave
int dec_silu_mul(const float* partial, int splits, int ws_rows, int B, int F, bf16* h, cudaStream_t st);
// logits[b, :] = sum_s partial[s][b][:V] ; tok[b] = argmax (first max wins, like torch.argmax; a row that is -inf everywhere gives 0)
// cand_val / cand_idx: [B][kArgmaxChunks] scratch owned by the context
constexpr int kArgmaxChunks = 32;
int dec_logits_argmax(const float* partial, int splits, int ws_rows, int ldp, int B, int V, float* logits, int ld_logits,
                      int32_t* tok, int32_t* history, const int32_t* step_idx, float* cand_val,
                      int32_t* cand_idx, int32_t* dp_send, cudaStream_t st);
// stage 1 only: logits[b, :] = sum_s partial (the sampler consumes them)
int dec_logits_reduce(const float* partial, int splits, int ws_rows, int ldp, int B, int V, float* logits, int ld_logits,
                      float* cand_val, int32_t* cand_idx, cudaStream_t st);
// ---- device-side sampling (sampler.cu) ----------------------------------------------------------------------------------
struct SamplerParams {     // lives in device memory: graphs captured once serve every parameter set
  int do_sample;           // 0: argmax of the processed scores
  float rep_penalty;       // 1 = off
  int no_repeat_ngram;     // 0 = off
  float temperature;       // 1 = off
  int top_k;               // 1..1024 (required when do_sample)
  float top_p;             // 1 = off
  float one_minus_top_p;   // (float)(1.0 - (double)top_p): the constant HF compares the cumulative probabilities with
  int min_new_tokens, n_eos, pad_id;
  int eos[4];
  unsigned long long seed;
};
int sampler_supported(int V);
int sampler_init();
// history: [L][B] int32 with L = *step_idx; writes tok[b], history_out[L][b], dp_send[b]; finished[b] (nullable): sticky EOS flag.
// fanout > 1: B is a multiple of it and sequence b scores logits row b / fanout (the prefill's pick of N replies per prompt)
int dec_sample(const float* logits, int ld, int V, int B, const int32_t* history, const int32_t* step_idx, const SamplerParams* params_dev,
               int32_t* tok, int32_t* history_out, int32_t* dp_send, int32_t* finished, float* scores_out, cudaStream_t st, int fanout = 1);
// prompt lookup verification (B = 1): row r < R scores logits row r with the history column of length *step_idx + r and draws with
// counter (*step_idx + r, 0); tok[r] = pick.  No history, finished or send-buffer writes.
int dec_sample_lookup(const float* logits, int ld, int V, int R, const int32_t* history, const int32_t* step_idx, const SamplerParams* params_dev,
                      int32_t* tok, cudaStream_t st);
int dp_unpack(const int32_t* recv, int n, int32_t* hist, int32_t* dp_step, cudaStream_t st);
// ---- beam search (beam.cu; HF:generation/utils.py:2876-3395 with decoder_prompt_len = 0) ---------------------------------------
constexpr int kBeamMaxK = 16;
constexpr int kBeamMaxCand = 5 * kBeamMaxK;   // M = max(2, 1 + n_eos) * K candidates per item, n_eos <= 4
struct BeamParams {        // lives in device memory, like SamplerParams
  int K, M;                // beams per item, candidates kept per step
  int n_eos; int eos[4];
  float length_penalty;
  int early_stopping;      // 0: False, 1: True, 2: "never"
  int max_new;             // max_new_tokens (MaxLengthCriteria)
  float rep_penalty; int no_repeat_ngram; int min_new_tokens;
};
int beam_supported(int V);
int beam_init();
// rows beams: log_softmax + history processors + running score (null: 0) -> the row's top-M (score desc, token asc)
int dec_beam_step(const float* logits, int ld, int V, int rows, const int32_t* history, const int32_t* step_idx, const BeamParams* params_dev,
                  const float* run_score, float* cand_val, int32_t* cand_tok, cudaStream_t st);
// per item: global top-M of the R rows' candidates, next K running beams (parent_row / tok / run_score of slot b*K+j), store + flags
int dec_beam_select(const BeamParams* params_dev, int items, int R, int V, const int32_t* step_idx, const float* cand_val, const int32_t* cand_tok,
                    const int32_t* history, float* run_score, int32_t* parent_row, int32_t* tok, float* hyp_score, int32_t* hyp_len, int32_t* hyp_fin,
                    int32_t* hyp_tok, int32_t* hyp_tmp, int hyp_cap, int32_t* item_state, int32_t* cand_out, cudaStream_t st);
int trace_set_beam(void* buf, unsigned long long cap);
// decode step entry of the cluster split-K schedule: resid[b,:] = table[ids[b]] ; xw = bf16(resid * norm_w) ;
// ssq[b][0] = sum resid^2, ssq[b][1..slots) = 0 (head of the deferred-norm chain)
int dec_embed(const int32_t* ids, int B, int D, const bf16* table, int vocab, float* resid, const float* norm_w,
              bf16* xw, float* ssq, int slots, cudaStream_t st);
// ---- device-side KV page allocator over a KvCache (stream-ordered, graph-capturable; one thread walks the <= 64 sequences, so the
//      assignment is deterministic) ------------------------------------------------------------------------------
// every page back on the free stack (kv_order[0] popped first), no sequence of max_batch owns any
int kv_reset(const KvCache& kv, const int32_t* kv_order, int max_batch, cudaStream_t st);
// make sure sequence b owns pages for (S - left_pad[b]) tokens, b < B; pages are handed out round-robin over the sequences
// (base_len non-null: make sure sequence b owns pages for base_len[b] + S tokens -- a chunk appended to cached tokens)
int kv_reserve(const KvCache& kv, int B, int S, const int32_t* left_pad, cudaStream_t st, const int32_t* base_len = nullptr);
// seq_len[b] = min(seq_len[b], len[b]) for b < B <= 64 (the pages stay owned)
int kv_truncate(int32_t* seq_len, const int32_t* len_host, int B, cudaStream_t st);
// Token stream ring (vcla_stream_*): pinned, mapped host memory the device writes and the host polls.  tokens[L][b] = token of
// sequence b chosen at step L (row stride 64); published = steps whose tokens are final (written with a system-scope release).
struct StreamRing {
  int32_t published;
  int32_t epoch;
  int32_t rows;          // capacity in steps (= rows of the device token history)
  int32_t pad_[29];      // tokens start on their own 128-byte line
  int32_t tokens[1];     // [rows][64]
};
inline size_t stream_ring_bytes(int rows) { return offsetof(StreamRing, tokens) + (size_t)rows * 64 * sizeof(int32_t); }
// seq_len[b] += by - left_pad[b] ; *step_idx += 1 ; then reserve the page the NEXT token of every sequence will be appended to.
// ring (nullable, device view of the mapped ring): first publish step L = *step_idx -- history row L ([L][B]) into ring row L, a
// system-scope fence per writer, then ring->published = L + 1 with st.release.sys.  ring == nullptr executes none of it.
// publish_rows (<= 64; 0: B): the width of history row L and of the published step -- a fan-out prefill publishes its B * N picks
// while it advances the B prompts.
int advance_seq(int32_t* seq_len, int B, int by, const int32_t* left_pad, int32_t* step_idx, const KvCache& kv, cudaStream_t st,
                StreamRing* ring = nullptr, const int32_t* history = nullptr, int publish_rows = 0);
// Fan-out (vcla_set_fanout): parent[r] = r / n for the rows = B * n rows forked from B prompts (the parent map of kv_beam_reorder).
// tok != nullptr: tok[0..B) holds one pick per prompt (the argmax); it is expanded in place to tok[r] = tok[r / n], which also becomes
// history row 0 ([0][rows]).  With the device sampler the picks are already per row (tok = nullptr).  One CTA.
int fanout_rows(int n, int rows, int32_t* parent, int32_t* tok, int32_t* history, cudaStream_t st);
// ---- prompt lookup decoding (one sequence): a verification step runs R = k + 1 rows -- the last emitted token and k drafts -- through
// the decode step; lookup_accept then replaces advance_seq.  Restates HF:generation/utils.py:3603-3620 (_assisted_decoding, greedy
// and sampled without an assistant: n_matches = leading drafts equal to the model's picks, valid_tokens = picks[: n_matches + 1],
// streamer.put(valid_tokens)) and HF:generation/candidate_generator.py:1057-1149 (PromptLookupCandidateGenerator.get_candidates, the
// draft rule, without its forbidden-token and EOS cropping).
struct LookupState {          // device memory: graphs captured once serve every call
  int32_t nd;                 // drafts in rows 1..nd of the current step
  int32_t n, max_new, prompt_len;   // largest n-gram, max_new_tokens (history rows), prompt ids searched
  unsigned long long steps, drafted, accepted;   // verification steps that advanced, drafts offered, drafts emitted
};
struct LookupCall {
  int R = 0;                                    // rows
  const int64_t* prompt = nullptr;
  int32_t* tok = nullptr;                       // [R] inputs of the next step: row 0 = last emitted token, rows 1..R-1 drafts
  const int32_t* pick = nullptr;                // [R] pick of each row of the step that just ran
  int32_t* history = nullptr; int32_t* step_idx = nullptr; int32_t* seq_len = nullptr; int32_t* finished = nullptr;
  const SamplerParams* samp = nullptr;          // nullable: the EOS ids
  LookupState* state = nullptr;
  KvCache kv;                                   // pages for the next step's rows
  StreamRing* ring = nullptr;                   // nullable: publish the emitted tokens (as advance_seq does)
};
// prime != 0: no acceptance (right after the prefill): reserve pages for R rows and draft the first step.  Otherwise, unless the row is
// finished or max_new tokens exist: accept the leading matching drafts, emit the picks up to and including the first mismatch (stopping
// after an EOS id, clamped to max_new) into the history, advance seq_len and the step counter by the emitted count, publish them to the
// ring (tokens, a system-scope fence, then the count with st.release.sys).  Then reserve pages for the next R rows and write the next
// step's inputs (drafts also provisionally into the history after the emitted tokens).
int lookup_accept(const LookupCall& c, int prime, cudaStream_t st);
// Beam reorder, after advance_seq (so every old row's write position seq_len and its page exist).  New row j (< rows_new) continues
// old row parent_row[j] (< rows_old): its table row, page count and length are the parent's.  Pages no new row references go back on
// the free stack; when several rows continue one parent, every one but the first gets a fresh page for the write position plus a
// copy-list entry {src page, dst page, rows [0, seq_len % page_tokens)} (copy_list[0] = count, then 3 ints per entry).  The token
// history [t][rows_old] (t = *step_idx - 1) is gathered into [t][rows_new] and new_tok is appended as its row t.  One CTA; the stack
// operations are serial, so the result is deterministic.  Scratch: table_tmp [rows_old][pages_per_seq], mark (total_pages / 32 words
// of dynamic shared memory).  cow_bytes (nullable) accumulates the bytes of the copied rows over every layer.
int kv_beam_reorder(int rows_old, int rows_new, const int32_t* parent_row, const int32_t* new_tok, int32_t* seq_len, const KvCache& kv,
                    int32_t* table_tmp, int32_t* history, const int32_t* step_idx, int32_t* copy_list, unsigned long long* cow_bytes,
                    cudaStream_t st, KvFormat fmt = KV_BF16);
// copies the copy list's rows of every layer (K and V, every head) from src to dst page; fixed grid (max_entries x layers)
int kv_page_copy(const KvCache& kv, const int32_t* copy_list, int max_entries, cudaStream_t st, KvFormat fmt = KV_BF16);
// fp32 RoPE tables [max_pos][head_dim/2], computed on the host the way HF does and uploaded to cos_dev / sin_dev
int rope_fill_tables(int max_pos, int head_dim, float theta, float* cos_dev, float* sin_dev);

// weights
int fill_hash_normal(bf16* dst_bf16, float* dst_f32, int64_t n, uint32_t seed, float mul, float offset, cudaStream_t st);
int convert_to_bf16(const void* src, int dtype, int64_t n, bf16* dst, cudaStream_t st);
int convert_to_f32(const void* src, int dtype, int64_t n, float* dst, cudaStream_t st);
// dst rows [r0, r0+rows) of a [*, ld] bf16 matrix <- src [rows, cols] (zero pad cols..ld)
int copy_rows_bf16(const bf16* src, int rows, int cols, bf16* dst, int ld, cudaStream_t st);
// interleave gate/up rows in blocks of 32: dst[(j/32)*64 + which*32 + j%32, :] = src[j, :]
int interleave_rows32(const bf16* src, int rows, int cols, int which, bf16* dst, cudaStream_t st);

// ---- weight-only int8 (quant.cu): one fp32 scale per row, q = clamp(rint(w * (127 / absmax)), -127, 127), s = absmax / 127 ---------
// Stored rows keep the k of each 64-column block in the decode kernel's fragment order (gemm_decode.cu); `which` >= 0 places logical row
// r at the gate/up interleave row (r / 32) * 64 + which * 32 + r % 32, -1 at row r.
int quantize_rows_q8(const void* src, int dtype, int rows, int cols, int which, int8_t* q, float* scale, cudaStream_t st);
// caller's logical int8 rows + scales -> stored rows
int place_rows_q8(const int8_t* q_src, const float* s_src, int rows, int cols, int which, int8_t* q, float* scale, cudaStream_t st);
// stored rows -> logical order: int8 + scales, and/or fp32 q * s (any output may be null)
int read_rows_q8(const int8_t* q, const float* scale, int rows, int cols, int which, int8_t* q_out, float* s_out, float* f32_out, cudaStream_t st);
// bf16(q) of `rows` rows with k in logical order (permuted != 0: stored fragment order, else already logical): the prefill GEMM operand
int expand_rows_q8(const int8_t* q, int rows, int cols, int permuted, bf16* out, cudaStream_t st);

}  // namespace vcla
