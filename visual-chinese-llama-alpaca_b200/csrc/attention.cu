// Attention kernels of the VisualCLA path.
//
//  attention_prefill : flash-style fused softmax(QK^T)V for ViT (non-causal, S=257, hd 64), the Resampler
//                      (64 queries over [64 query-rows ; 257 image rows] = two KV segments, hd 64) and LLaMA prefill
//                      (causal, hd 128).  Attention is <3 % of the path's FLOPs (SURVEY section 8a), so this uses the
//                      register-fragment tensor path (mma.sync m16n8k16) with fp32 online softmax; the dense
//                      contractions that dominate run on wgmma (gemm.cu).
//  attention_decode  : one new token per sequence against the paged KV cache.  HBM-bound.  Fuses: split-K
//                      reduction of the QKV projection partials, RoPE, KV-cache append, split-KV attention and the
//                      final cross-split combine (last-arriving CTA, fixed order => deterministic).
#include "common.cuh"
#include "kernels.h"

#include <mutex>
#include <stdlib.h>

namespace vcla {

// =================================================================================================
// prefill
// =================================================================================================
template <int HD>
__device__ __forceinline__ uint32_t swz(int row, int chunk) {  // byte offset of 16 B chunk in a [rows][HD] bf16 tile
  return (uint32_t)(row * (HD * 2) + ((chunk ^ (row & 7)) << 4));
}

template <int HD>
__global__ void __launch_bounds__(128) attn_prefill_kernel(const AttnCall c) {
  constexpr int BQ = 64, BKV = 64, CHUNKS = HD / 8;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sQ = smem_u32(smem), sKV0 = sQ + BQ * HD * 2;   // then 2 x {K tile, V tile} (double buffered)
  constexpr uint32_t kTileBytes = BKV * HD * 2;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int q0 = blockIdx.x * BQ, h = blockIdx.y, b = blockIdx.z;
  const int Sk = c.n0 + c.n1;
  const int off = Sk - c.Sq;  // causal: kv j visible to query i iff j <= i + off
  TraceScope trace(3);
  const int kv0 = c.kv_start ? __ldg(c.kv_start + b) : 0;   // left padding: keys before kv0 are invisible

  pdl_launch_dependents();   // dependents may become resident early; they block in their own griddepcontrol.wait
  pdl_wait();
  trace.dep();

  // ---- Q tile -> smem
  for (int i = tid; i < BQ * CHUNKS; i += 128) {
    int r = i / CHUNKS, ch = i % CHUNKS;
    int qi = q0 + r;
    bool ok = qi < c.Sq;
    const bf16* src = c.q + ((size_t)(b * c.Sq + (ok ? qi : 0)) * c.q_stride + h * HD + ch * 8);
    cp_async_16(sQ + swz<HD>(r, ch), src, ok);
  }
  cp_async_commit();

  float o_acc[HD / 8][4];
#pragma unroll
  for (int i = 0; i < HD / 8; ++i) { o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f; }
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const float sl2 = c.scale * 1.4426950408889634f;

  int kv_end = Sk;
  if (c.causal) kv_end = min(Sk, q0 + BQ + off);
  const int r0 = q0 + warp * 16 + (lane >> 2), r1 = r0 + 8;  // the two query rows this thread owns

  auto load_kv_tile = [&](int j0, int buf) {
    const uint32_t sKb = sKV0 + (uint32_t)buf * 2u * kTileBytes, sVb = sKb + kTileBytes;
    for (int i = tid; i < BKV * CHUNKS; i += 128) {
      int r = i / CHUNKS, ch = i % CHUNKS;
      int j = j0 + r;
      bool ok = j < Sk;
      const bf16 *ks, *vs;
      if (j < c.n0 || !ok) {
        int jj = ok ? j : 0;
        size_t ro = (size_t)(b * c.n0 + jj) * c.kv0_stride + h * HD + ch * 8;
        ks = c.k0 + ro; vs = c.v0 + ro;
      } else {
        size_t ro = (size_t)(b * c.n1 + (j - c.n0)) * c.kv1_stride + h * HD + ch * 8;
        ks = c.k1 + ro; vs = c.v1 + ro;
      }
      cp_async_16(sKb + swz<HD>(r, ch), ks, ok);
      cp_async_16(sVb + swz<HD>(r, ch), vs, ok);
    }
    cp_async_commit();
  };
  const int j_first = (kv0 / BKV) * BKV;
  if (j_first < kv_end) load_kv_tile(j_first, 0);
  int buf = 0;
  for (int j0 = j_first; j0 < kv_end; j0 += BKV, buf ^= 1) {
    // prefetch the next K/V tile into the other buffer while this one is consumed
    const bool has_next = (j0 + BKV) < kv_end;
    if (has_next) load_kv_tile(j0 + BKV, buf ^ 1);
    if (has_next) cp_async_wait<1>(); else cp_async_wait<0>();
    __syncthreads();
    const uint32_t sK = sKV0 + (uint32_t)buf * 2u * kTileBytes, sV = sK + kTileBytes;

    // ---- S = Q K^T  (16 x 64 per warp)
    float s[BKV / 8][4];
#pragma unroll
    for (int i = 0; i < BKV / 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) {
      uint32_t a[4];
      ldmatrix_x4(a, sQ + swz<HD>(warp * 16 + (lane & 15), ks * 2 + (lane >> 4)));
#pragma unroll
      for (int nt = 0; nt < BKV / 8; nt += 2) {
        uint32_t kb[4];
        const int m = lane >> 3;
        ldmatrix_x4(kb, sK + swz<HD>((nt + (m >> 1)) * 8 + (lane & 7), ks * 2 + (m & 1)));
        uint32_t b0[2] = {kb[0], kb[1]}, b1[2] = {kb[2], kb[3]};
        mma_bf16_16816(s[nt], a, b0);
        mma_bf16_16816(s[nt + 1], a, b1);
      }
    }
    // ---- mask + online softmax (fp32)
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < BKV / 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        int j = j0 + nt * 8 + (lane & 3) * 2 + (e & 1);
        int qi = (e < 2) ? r0 : r1;
        bool vis = (j < Sk) && (j >= kv0) && (!c.causal || j <= qi + off);
        float v = vis ? s[nt][e] * sl2 : -INFINITY;
        s[nt][e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
      }
    }
    float corr[2], msafe[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      float mnew = fmaxf(m_run[r], mx[r]);
      msafe[r] = (mnew == -INFINITY) ? 0.f : mnew;
      corr[r] = exp2f(m_run[r] - msafe[r]);
      m_run[r] = mnew;
      l_run[r] *= corr[r];
    }
    float ls[2] = {0.f, 0.f};
#pragma unroll
    for (int nt = 0; nt < BKV / 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float pv = exp2f(s[nt][e] - msafe[e >> 1]);
        s[nt][e] = pv;
        ls[e >> 1] += pv;
      }
    }
    l_run[0] += ls[0];
    l_run[1] += ls[1];
#pragma unroll
    for (int i = 0; i < HD / 8; ++i) {
      o_acc[i][0] *= corr[0]; o_acc[i][1] *= corr[0];
      o_acc[i][2] *= corr[1]; o_acc[i][3] *= corr[1];
    }
    // ---- O += P V
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      uint32_t a[4];
      a[0] = pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
      a[1] = pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
      a[2] = pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      a[3] = pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int nd = 0; nd < HD / 8; nd += 2) {
        uint32_t vb[4];
        const int m = lane >> 3;
        ldmatrix_x4_trans(vb, sV + swz<HD>(kk * 16 + (m & 1) * 8 + (lane & 7), nd + (m >> 1)));
        uint32_t b0[2] = {vb[0], vb[1]}, b1[2] = {vb[2], vb[3]};
        mma_bf16_16816(o_acc[nd], a, b0);
        mma_bf16_16816(o_acc[nd + 1], a, b1);
      }
    }
    __syncthreads();   // all warps are done with this buffer before the next iteration's prefetch overwrites it
  }
  // ---- finalise: O / l  (l summed over the 4 lanes that share a row)
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
    l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
  }
  const float inv0 = l_run[0] > 0.f ? 1.f / l_run[0] : 0.f;
  const float inv1 = l_run[1] > 0.f ? 1.f / l_run[1] : 0.f;
#pragma unroll
  for (int nd = 0; nd < HD / 8; ++nd) {
    const int d = nd * 8 + (lane & 3) * 2;
    if (r0 < c.Sq) {
      uint32_t* dst = reinterpret_cast<uint32_t*>(c.out + (size_t)(b * c.Sq + r0) * c.o_stride + h * HD + d);
      *dst = pack_bf16x2(o_acc[nd][0] * inv0, o_acc[nd][1] * inv0);
    }
    if (r1 < c.Sq) {
      uint32_t* dst = reinterpret_cast<uint32_t*>(c.out + (size_t)(b * c.Sq + r1) * c.o_stride + h * HD + d);
      *dst = pack_bf16x2(o_acc[nd][2] * inv1, o_acc[nd][3] * inv1);
    }
  }
}

// 0 = mma.sync kernel for everything, 1 (default) = wgmma kernel at head dim 128 (LLaMA prefill), mma.sync at head dim 64 (ViT,
// Resampler: short sequences, few KV tiles per CTA), 2 = wgmma kernel for everything it can describe (tests).
static int g_attn_tc = -1;
void attention_set_tc(int mode) { g_attn_tc = mode < 0 ? 0 : (mode > 2 ? 2 : mode); }
int attention_prefill(const AttnCall& c, cudaStream_t st) {
  if (g_attn_tc < 0) { const char* e = getenv("VCLA_ATTN_TC"); g_attn_tc = (e != nullptr) ? atoi(e) : 1; if (g_attn_tc < 0 || g_attn_tc > 2) g_attn_tc = 1; }
  // the wgmma kernel needs TMA-describable operands (16 B aligned, 16 B-multiple pitches) and one KV segment when causal
  const bool tma_ok = (c.q_stride % 8) == 0 && (c.kv0_stride % 8) == 0 && (c.n1 == 0 || (c.kv1_stride % 8) == 0) && (c.o_stride % 8) == 0 &&
                      !(c.causal && c.n1 > 0);
  const bool want_tc = g_attn_tc == 2 || (g_attn_tc == 1 && c.HD == 128);
  if (want_tc && tma_ok) return attention_prefill_tc(c, st);
  return attention_prefill_mma(c, st);
}

int attention_prefill_mma(const AttnCall& c, cudaStream_t st) {
  if (c.HD != 64 && c.HD != 128) { set_error("attention_prefill: head dim %d unsupported (64/128)", c.HD); return -1; }
  if ((c.q_stride % 8) || (c.kv0_stride % 8) || (c.n1 > 0 && (c.kv1_stride % 8)) || (c.o_stride % 2)) {
    set_error("attention_prefill: strides must keep 16 B alignment");
    return -1;
  }
  dim3 grid((c.Sq + 63) / 64, c.H, c.B);
  const size_t smem = 5 * 64 * c.HD * 2;     // Q + 2 x (K, V) tiles
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = dim3(128); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (pdl_enabled()) { attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[na].val.programmaticStreamSerializationAllowed = 1; ++na; }
  cfg.attrs = attr; cfg.numAttrs = na;
  if (attention_init()) return -1;
  if (c.HD == 64) {
    VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_prefill_kernel<64>, c));
  } else {
    VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_prefill_kernel<128>, c));
  }
  return 0;
}

// =================================================================================================
// decode (hd = 128): grid (kv_splits, H, B), 128 threads
// =================================================================================================
constexpr int kDecWarps = 8;        // 256 threads
// KV pages in flight per CTA (32 KB each at 64 tokens/page).  3 stages -> 2 CTAs per SM: the persistent kernel, and the one-shot kernel
// when its grid needs more than one wave at two CTAs per SM (2 stages with 3 CTAs per SM measured slower at B=32 on B200, 37 vs 34 us
// per layer, with the grid filling all three slots).  A one-shot grid of at most two CTAs per SM (small batches: B = 1..8 at 32 heads)
// runs 2 stages, so a third CTA fits per SM; that free slot is where the O-projection GEMM becomes resident and starts streaming
// weights while attention drains.
constexpr int kDecStages = 3;
constexpr int kDecStagesSmallBatch = 2;
constexpr int kDecMaxPT = 64;       // page_tokens supported by the smem ring

// One CTA per (kv split, head, sequence).  The cached K/V rows of a head are contiguous per page (page_tokens x 128 bf16 =
// 16 KB), so whole pages are streamed with TMA bulk copies (cp.async.bulk, mbarrier completion) into a 2- or 3-stage shared-memory
// ring and the dot products / PV accumulation run out of shared memory: the kernel is bandwidth- instead of latency-bound
// (the register-prefetch version had one DRAM round trip per 32 tokens per CTA).
//
// Prompt lookup verification (MODE != kDecPlain): blockIdx.z is query row r of sequence 0, the token at position seq_len[0] + r.  Row r
// runs exactly the arithmetic of the one-token kernel at length seq_len[0] + r + 1.  Rows read keys that lower rows append, and CTAs
// of one launch cannot rely on each other's stores, so a verification step launches this kernel twice: kDecAppend (grid (1, H, R), no
// KV stream) writes the RoPE'd K and V of all R rows, then kDecAttend attends without writing the cache.
//
// FMT = KV_INT8 reads a pool of int8 rows + fp32 row scales (kernels.h): a stage holds the page's K rows, V rows, K scales and V
// scales (PT x 264 B, 16.5 KB at 64 tokens); a score is s_k * sum q k and the accumulator takes (p s_v) v.  The new row is quantised
// (absmax over its 128 dims), stored, and attended through the same arithmetic as a cached row.  Stage counts and occupancy are the
// bf16 kernel's (the register budget, not shared memory, bounds the CTAs per SM), so the kv_splits choice stays format-independent.
constexpr int kDecPlain = 0, kDecAttend = 1, kDecAppend = 2;
constexpr int kDecQ8Extra = 16 * 4;   // KV_INT8: floats after the ring: per-warp k / v absmax [0, 8), the new row's s_k, s_v [8, 10)
__host__ __device__ constexpr uint32_t dec_stage_bytes(int fmt, int pt) { return fmt == KV_INT8 ? (uint32_t)pt * (128 * 2 + 4 * 2) : (uint32_t)pt * 128 * 2 * 2; }
static size_t dec_smem_bytes(int fmt, int stages, int pt) { return (size_t)stages * dec_stage_bytes(fmt, pt) + (fmt == KV_INT8 ? kDecQ8Extra : 0); }
// KV_INT8: attend over ntok cached rows of one ring stage {K rows, V rows, K scales, V scales}; the token / lane split of the bf16 loop
// (lane `sub` of a token group owns dims [8 sub, 8 sub + 8) and [64 + 8 sub, 64 + 8 sub + 8): two 8 B loads per row)
__device__ __forceinline__ void dec_page_q8(const uint8_t* stage, int PT, int ntok, int warp, int grp, int sub, uint32_t gmask,
                                            const float (&qreg)[16], float& m, float& l, float (&acc)[16]) {
  constexpr int HD = 128;
  const uint8_t* vbase = stage + (size_t)PT * HD;
  const float* ksc = reinterpret_cast<const float*>(stage + (size_t)PT * HD * 2);
  const float* vsc = ksc + PT;
  for (int tk = warp * 4 + grp; tk < ntok; tk += kDecWarps * 4) {
    const uint2 k0 = *reinterpret_cast<const uint2*>(stage + (size_t)tk * HD + sub * 8);
    const uint2 k1 = *reinterpret_cast<const uint2*>(stage + (size_t)tk * HD + 64 + sub * 8);
    const uint2 v0 = *reinterpret_cast<const uint2*>(vbase + (size_t)tk * HD + sub * 8);
    const uint2 v1 = *reinterpret_cast<const uint2*>(vbase + (size_t)tk * HD + 64 + sub * 8);
    const uint32_t kw[4] = {k0.x, k0.y, k1.x, k1.y};
    const uint32_t vw[4] = {v0.x, v0.y, v1.x, v1.y};
    float sc = 0.f;
#pragma unroll
    for (int j = 0; j < 16; ++j) sc += qreg[j] * q8_lane(kw[j >> 2], j & 3);
    sc += __shfl_xor_sync(gmask, sc, 1);
    sc += __shfl_xor_sync(gmask, sc, 2);
    sc += __shfl_xor_sync(gmask, sc, 4);
    sc *= ksc[tk];
    const float mn = fmaxf(m, sc);
    const float cr = __expf(m - mn), p = __expf(sc - mn);
    m = mn;
    l = l * cr + p;
    const float pv = p * vsc[tk];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = acc[j] * cr + pv * q8_lane(vw[j >> 2], j & 3);
  }
}

template <int STAGES, int MODE = kDecPlain, int FMT = KV_BF16>
__global__ void __launch_bounds__(kDecWarps * 32, STAGES == 2 ? 3 : 2) attn_decode_kernel(const DecodeAttnCall c, const float* __restrict__ rope_cos,
                                                                                  const float* __restrict__ rope_sin) {
  constexpr int HD = 128;
  constexpr bool Q8 = FMT == KV_INT8;
  extern __shared__ __align__(128) uint8_t dsm[];      // [STAGES][2][PT][HD] bf16 (KV_INT8: [STAGES]{K rows, V rows, K scales, V scales}, then kDecQ8Extra)
  __shared__ __align__(8) uint64_t s_bar[STAGES];
  __shared__ float s_q[HD];
  __shared__ float s_k[HD];
  __shared__ float s_v[HD];
  __shared__ float s_acc[kDecWarps][HD];
  __shared__ float s_m[kDecWarps], s_l[kDecWarps];
  __shared__ int s_last;

  const int split = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int T = c.kv.heads * HD, PT = c.kv.page_tokens;
  const uint32_t stage_bytes = Q8 ? dec_stage_bytes(KV_INT8, PT) : (uint32_t)PT * HD * 2 * 2;      // K page + V page
  TraceScope trace(MODE == kDecAppend ? 19 : 4);
  const int sb = MODE == kDecPlain ? b : 0;   // the sequence whose pages and length this CTA reads

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) mbar_init(smem_u32(&s_bar[s]), 1);
    fence_barrier_init();
  }
  pdl_launch_dependents();
  pdl_wait();
  trace.dep();
  __syncthreads();

  const int L = c.seq_len[sb] + (MODE == kDecPlain ? 0 : b);   // tokens already cached; the new token gets index L
  const int n = L + 1;
  int chunk = (n + c.kv_splits - 1) / c.kv_splits;
  chunk = (chunk + PT - 1) / PT * PT;                 // splits own whole pages
  const int t_begin = split * chunk;
  const int t_end = min(n, t_begin + chunk);
  const bool owns_new = MODE == kDecAppend || ((t_begin <= L) && (L < t_end));
  const int c_end = min(t_end, L);                    // cached tokens of this CTA: [t_begin, c_end)
  const int p0 = t_begin / PT;
  const int npages = (MODE != kDecAppend && c_end > t_begin) ? (c_end - t_begin + PT - 1) / PT : 0;

  auto issue_page = [&](int i) {                      // thread 0: request page i of this CTA into stage i % STAGES
    const int stage = i % STAGES;
    const int page = __ldg(c.kv.seq_pages(sb) + p0 + i);
    const int ntok = min(PT, c_end - (t_begin + i * PT));
    const uint32_t bytes = (uint32_t)ntok * HD * 2;
    const uint32_t bar = smem_u32(&s_bar[stage]);
    const uint32_t dst = smem_u32(dsm) + stage * stage_bytes;
    if constexpr (Q8) {
      const uint32_t rbytes = (uint32_t)ntok * HD, sbytes = (uint32_t)((ntok + 3) & ~3) * 4;   // scales in whole 16 B (inside the plane)
      mbar_arrive_expect_tx(bar, 2 * (rbytes + sbytes));
      bulk_load_1d(dst, c.kv.q8_at(page, 0, h, 0), rbytes, bar);
      bulk_load_1d(dst + (uint32_t)PT * HD, c.kv.q8_at(page, 1, h, 0), rbytes, bar);
      bulk_load_1d(dst + (uint32_t)PT * HD * 2, c.kv.q8_scale(page, 0, h, 0), sbytes, bar);
      bulk_load_1d(dst + (uint32_t)PT * (HD * 2 + 4), c.kv.q8_scale(page, 1, h, 0), sbytes, bar);
    } else {
    const bf16* ksrc = c.kv.at(page, 0, h, 0);
    const bf16* vsrc = c.kv.at(page, 1, h, 0);
    mbar_arrive_expect_tx(bar, 2 * bytes);
    bulk_load_1d(dst, ksrc, bytes, bar);
    bulk_load_1d(dst + (uint32_t)PT * HD * 2, vsrc, bytes, bar);
    }
  };
  if (tid == 0) {
    for (int i = 0; i < npages && i < STAGES; ++i) issue_page(i);   // the KV stream starts before the q reduction below
  }

  // ---- reduce the split-K partials of this head's q (and k, v if this CTA owns the new token); RoPE
  {
    const int d = tid & (HD - 1);
    float qv = 0.f, kv = 0.f, vv = 0.f;
    if (tid < HD) {
      for (int s = 0; s < c.splits; ++s) {
        const float* row = c.qkv_partial + ((size_t)s * c.ws_rows + b) * (size_t)(3 * T);
        qv += __ldcg(row + h * HD + d);
        if (owns_new) { kv += __ldcg(row + T + h * HD + d); vv += __ldcg(row + 2 * T + h * HD + d); }
      }
      s_q[d] = qv; s_k[d] = kv; s_v[d] = vv;
    }
    __syncthreads();
    float qr = 0.f, kr = 0.f;
    if (tid < HD) {
      const float cs = rope_cos[(size_t)L * (HD / 2) + (d & 63)], sn = rope_sin[(size_t)L * (HD / 2) + (d & 63)];
      const float qp = (d < 64) ? -s_q[d + 64] : s_q[d - 64];
      const float kp = (d < 64) ? -s_k[d + 64] : s_k[d - 64];
      qr = (qv * cs + qp * sn) * c.scale;
      kr = kv * cs + kp * sn;
    }
    __syncthreads();
    if constexpr (Q8) {
      // the cache holds q and s: quantise both rows (block absmax over the 128 dims of warps 0..3), keep q in s_k / s_v and the
      // scales in q8x[8..9], so the new row is attended with the arithmetic every later step applies to it
      float* q8x = reinterpret_cast<float*>(dsm + (MODE == kDecAppend ? 0 : (size_t)STAGES * stage_bytes));   // the append streams no pages
      if (owns_new) {
        const float ka = warp_max(tid < HD ? fabsf(kr) : 0.f), va = warp_max(tid < HD ? fabsf(vv) : 0.f);
        if (tid < HD && lane == 0) { q8x[warp] = ka; q8x[4 + warp] = va; }
      }
      __syncthreads();
      if (tid < HD) {
        s_q[d] = qr;
        if (owns_new) {
          const float ka = fmaxf(fmaxf(q8x[0], q8x[1]), fmaxf(q8x[2], q8x[3])), va = fmaxf(fmaxf(q8x[4], q8x[5]), fmaxf(q8x[6], q8x[7]));
          const int kq = q8_quant(kr, q8_inv(ka)), vq = q8_quant(vv, q8_inv(va));
          s_k[d] = (float)kq;
          s_v[d] = (float)vq;
          if (tid == 0) { q8x[8] = q8_step(ka); q8x[9] = q8_step(va); }
          if (MODE != kDecAttend) {
            const int page = c.kv.seq_pages(sb)[L / PT];
            const int slot = L % PT;
            c.kv.q8_at(page, 0, h, slot)[d] = (int8_t)kq;
            c.kv.q8_at(page, 1, h, slot)[d] = (int8_t)vq;
            if (tid == 0) { *c.kv.q8_scale(page, 0, h, slot) = q8_step(ka); *c.kv.q8_scale(page, 1, h, slot) = q8_step(va); }
          }
        }
      }
    } else {
    if (tid < HD) {
      s_q[d] = qr;
      if (owns_new) {
        // the cache holds bf16; attend over the same rounded values every later step will read
        const bf16 kb = __float2bfloat16(kr), vb = __float2bfloat16(vv);
        s_k[d] = __bfloat162float(kb);
        s_v[d] = __bfloat162float(vb);
        if (MODE != kDecAttend) {
          const int page = c.kv.seq_pages(sb)[L / PT];
          const int slot = L % PT;
          bf16* kdst = c.kv.at(page, 0, h, slot);
          bf16* vdst = c.kv.at(page, 1, h, slot);
          kdst[d] = kb;
          vdst[d] = vb;
        }
      }
    }
    }
    __syncthreads();
  }
  if constexpr (MODE == kDecAppend) { trace.done(); return; }

  // ---- attention over the cached tokens, page by page out of shared memory.  8 lanes per token; lane `sub` owns the 16 B
  //      chunks `sub` and `sub + 8` of a 256 B row (dims [8 sub, 8 sub + 8) and [64 + 8 sub, 64 + 8 sub + 8)): a quarter warp
  //      then touches 128 contiguous bytes -> conflict-free LDS.128.
  const int grp = lane >> 3, sub = lane & 7;
  const uint32_t gmask = 0xffu << (grp * 8);
  float qreg[16];
#pragma unroll
  for (int i = 0; i < 8; ++i) { qreg[i] = s_q[sub * 8 + i]; qreg[8 + i] = s_q[64 + sub * 8 + i]; }
  float m = -INFINITY, l = 0.f, acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = 0.f;

  for (int i = 0; i < npages; ++i) {
    const int stage = i % STAGES;
    const uint32_t parity = (uint32_t)((i / STAGES) & 1);
    mbar_wait(smem_u32(&s_bar[stage]), parity);
    const int ntok = min(PT, c_end - (t_begin + i * PT));
    const uint8_t* kbase = dsm + (size_t)stage * stage_bytes;
    if constexpr (Q8) {
      dec_page_q8(kbase, PT, ntok, warp, grp, sub, gmask, qreg, m, l, acc);
    } else {
    const uint8_t* vbase = kbase + (size_t)PT * HD * 2;
    for (int tk = warp * 4 + grp; tk < ntok; tk += kDecWarps * 4) {
      const uint4 k0 = *reinterpret_cast<const uint4*>(kbase + (size_t)tk * HD * 2 + sub * 16);
      const uint4 k1 = *reinterpret_cast<const uint4*>(kbase + (size_t)tk * HD * 2 + 128 + sub * 16);
      const uint4 v0 = *reinterpret_cast<const uint4*>(vbase + (size_t)tk * HD * 2 + sub * 16);
      const uint4 v1 = *reinterpret_cast<const uint4*>(vbase + (size_t)tk * HD * 2 + 128 + sub * 16);
      const uint32_t kw[8] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z, k1.w};
      const uint32_t vw[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
      float sc = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 kf = unpack_bf16x2(kw[j]);
        sc += qreg[2 * j] * kf.x + qreg[2 * j + 1] * kf.y;
      }
      // token groups of a warp may run different trip counts: reduce with the group's own 8-lane mask
      sc += __shfl_xor_sync(gmask, sc, 1);
      sc += __shfl_xor_sync(gmask, sc, 2);
      sc += __shfl_xor_sync(gmask, sc, 4);
      const float mn = fmaxf(m, sc);
      const float cr = __expf(m - mn), p = __expf(sc - mn);
      m = mn;
      l = l * cr + p;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float2 vf = unpack_bf16x2(vw[j]);
        acc[2 * j] = acc[2 * j] * cr + p * vf.x;
        acc[2 * j + 1] = acc[2 * j + 1] * cr + p * vf.y;
      }
    }
    }
    __syncthreads();                                   // every warp is done with this stage
    if (tid == 0 && i + STAGES < npages) issue_page(i + STAGES);
  }
  __syncwarp();
  // the new token (from smem), handled by warp 0 group 0 of the owning CTA
  if (owns_new && warp == 0 && grp == 0) {
    float sc = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) sc += qreg[i] * s_k[sub * 8 + i] + qreg[8 + i] * s_k[64 + sub * 8 + i];
    sc += __shfl_xor_sync(0x000000ffu, sc, 1);
    sc += __shfl_xor_sync(0x000000ffu, sc, 2);
    sc += __shfl_xor_sync(0x000000ffu, sc, 4);
    float pv_scale = 1.f;
    if constexpr (Q8) {
      const float* q8x = reinterpret_cast<const float*>(dsm + (size_t)STAGES * stage_bytes);
      sc *= q8x[8];
      pv_scale = q8x[9];
    }
    const float mn = fmaxf(m, sc);
    const float cr = __expf(m - mn), p = __expf(sc - mn);
    m = mn;
    l = l * cr + p;
    const float pv = Q8 ? p * pv_scale : p;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      acc[i] = acc[i] * cr + pv * s_v[sub * 8 + i];
      acc[8 + i] = acc[8 + i] * cr + pv * s_v[64 + sub * 8 + i];
    }
  }
  __syncwarp();
  // ---- merge the 4 token groups of a warp (lanes with equal `sub` hold the same dims)
#pragma unroll
  for (int o = 8; o <= 16; o <<= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), l2 = __shfl_xor_sync(0xffffffffu, l, o);
    const float mn = fmaxf(m, m2);
    const float c1 = (m == -INFINITY) ? 0.f : __expf(m - mn), c2 = (m2 == -INFINITY) ? 0.f : __expf(m2 - mn);
    l = l * c1 + l2 * c2;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const float a2 = __shfl_xor_sync(0xffffffffu, acc[i], o);
      acc[i] = acc[i] * c1 + a2 * c2;
    }
    m = mn;
  }
  if (grp == 0) {
#pragma unroll
    for (int i = 0; i < 8; ++i) { s_acc[warp][sub * 8 + i] = acc[i]; s_acc[warp][64 + sub * 8 + i] = acc[8 + i]; }
    if (sub == 0) { s_m[warp] = m; s_l[warp] = l; }
  }
  __syncthreads();
  // ---- merge the warps: thread d (< 128) owns output dim d
  float M = -INFINITY;
#pragma unroll
  for (int w = 0; w < kDecWarps; ++w) M = fmaxf(M, s_m[w]);
  float Lsum = 0.f, O = 0.f;
  if (tid < HD) {
#pragma unroll
    for (int w = 0; w < kDecWarps; ++w) {
      const float cw = (s_m[w] == -INFINITY) ? 0.f : __expf(s_m[w] - M);
      Lsum += s_l[w] * cw;
      O += s_acc[w][tid] * cw;
    }
  }
  if (c.kv_splits == 1) {
    if (tid < HD) c.out[(size_t)b * T + h * HD + tid] = __float2bfloat16(O / Lsum);
    trace.done();
    return;
  }
  // ---- cross-CTA combine: publish partial, last arriver reduces in fixed split order
  float* sp = c.scratch + (((size_t)b * c.kv.heads + h) * c.kv_splits + split) * (HD + 2);
  if (tid < HD) sp[tid] = O;
  if (tid == 0) { sp[HD] = M; sp[HD + 1] = Lsum; }
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const int old = atomicAdd(c.counters + b * c.kv.heads + h, 1);
    s_last = (old == c.kv_splits - 1);
  }
  __syncthreads();
  if (!s_last) { trace.done(); return; }
  __threadfence();
  if (tid < HD) {
    const float* base = c.scratch + ((size_t)b * c.kv.heads + h) * c.kv_splits * (HD + 2);
    float Mg = -INFINITY;
    for (int s = 0; s < c.kv_splits; ++s) Mg = fmaxf(Mg, __ldcg(base + (size_t)s * (HD + 2) + HD));
    float Lg = 0.f, Og = 0.f;
    for (int s = 0; s < c.kv_splits; ++s) {
      const float ms = __ldcg(base + (size_t)s * (HD + 2) + HD);
      const float cw = (ms == -INFINITY) ? 0.f : __expf(ms - Mg);
      Lg += __ldcg(base + (size_t)s * (HD + 2) + HD + 1) * cw;
      Og += __ldcg(base + (size_t)s * (HD + 2) + tid) * cw;
    }
    c.out[(size_t)b * T + h * HD + tid] = __float2bfloat16(Og / Lg);
  }
  if (tid == 0) c.counters[b * c.kv.heads + h] = 0;  // ready for the next step / graph replay
  trace.done();
}

// ------------------------------------------------------------------------------------------------------------------------
// Persistent variant for large batches (more (sequence, head) items than resident CTAs, kv_splits == 1): each CTA loops over
// items; a dedicated producer warp streams the KV pages of item i+1 into the ring while the 8 consumer warps are still in the
// reduction / epilogue of item i, so the fixed per-item latency chain (seq_len -> page table -> TMA -> q reduce -> combine)
// is paid once per CTA instead of once per wave (B=32: 3.5 waves of one-shot CTAs).
// ------------------------------------------------------------------------------------------------------------------------
template <int FMT = KV_BF16>
__global__ void __launch_bounds__((kDecWarps + 2) * 32, 2) attn_decode_persistent_kernel(const DecodeAttnCall c, const float* __restrict__ rope_cos,
                                                                                       const float* __restrict__ rope_sin, int n_items) {
  // warps 0..7: consumers; warp 8: KV page producer (TMA bulk copies); warp 9: q/k/v producer (split-K reduce, deferred norm
  // scale, RoPE, cache append) -- both producers run ahead of the consumers (KV ring / 2-slot q buffer), so no global-memory
  // round trip is left on the consumers' per-item critical path.
  constexpr int HD = 128;
  constexpr int NC = kDecWarps * 32;                    // consumer threads
  constexpr bool Q8 = FMT == KV_INT8;
  extern __shared__ __align__(128) uint8_t dsm[];      // [kDecStages][2][PT][HD] bf16 (KV_INT8: as attn_decode_kernel, then s_k, s_v of both q slots)
  __shared__ __align__(8) uint64_t s_full[kDecStages];
  __shared__ __align__(8) uint64_t s_empty[kDecStages];
  __shared__ __align__(8) uint64_t s_qfull[2];
  __shared__ __align__(8) uint64_t s_qempty[2];
  __shared__ __align__(16) float s_q[2][HD];
  __shared__ __align__(16) float s_k[2][HD];
  __shared__ __align__(16) float s_v[2][HD];
  __shared__ float s_acc[kDecWarps][HD];
  __shared__ float s_m[kDecWarps], s_l[kDecWarps];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int T = c.kv.heads * HD, PT = c.kv.page_tokens;
  const uint32_t stage_bytes = Q8 ? dec_stage_bytes(KV_INT8, PT) : (uint32_t)PT * HD * 2 * 2;
  TraceScope trace(4);
  if (tid == 0) {
    for (int s = 0; s < kDecStages; ++s) { mbar_init(smem_u32(&s_full[s]), 1); mbar_init(smem_u32(&s_empty[s]), kDecWarps); }
    for (int s = 0; s < 2; ++s) { mbar_init(smem_u32(&s_qfull[s]), 1); mbar_init(smem_u32(&s_qempty[s]), kDecWarps); }
    fence_barrier_init();
  }
  pdl_launch_dependents();
  pdl_wait();
  trace.dep();
  __syncthreads();

  if (warp == kDecWarps) {
    // ===================== KV page producer =====================
    if (lane == 0) {
      uint32_t n = 0;                                   // pages issued so far (ring position)
      for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int b = item / c.kv.heads, h = item % c.kv.heads;
        const int L = c.seq_len[b];
        const int npages = (L + PT - 1) / PT;
        for (int i = 0; i < npages; ++i, ++n) {
          const int stage = n % kDecStages;
          mbar_wait(smem_u32(&s_empty[stage]), ((n / kDecStages) & 1u) ^ 1u);
          const int page = __ldg(c.kv.seq_pages(b) + i);
          const int ntok = min(PT, L - i * PT);
          const uint32_t bytes = (uint32_t)ntok * HD * 2;
          const uint32_t bar = smem_u32(&s_full[stage]);
          const uint32_t dst = smem_u32(dsm) + stage * stage_bytes;
          if constexpr (Q8) {
            const uint32_t rbytes = (uint32_t)ntok * HD, sbytes = (uint32_t)((ntok + 3) & ~3) * 4;
            mbar_arrive_expect_tx(bar, 2 * (rbytes + sbytes));
            bulk_load_1d(dst, c.kv.q8_at(page, 0, h, 0), rbytes, bar);
            bulk_load_1d(dst + (uint32_t)PT * HD, c.kv.q8_at(page, 1, h, 0), rbytes, bar);
            bulk_load_1d(dst + (uint32_t)PT * HD * 2, c.kv.q8_scale(page, 0, h, 0), sbytes, bar);
            bulk_load_1d(dst + (uint32_t)PT * (HD * 2 + 4), c.kv.q8_scale(page, 1, h, 0), sbytes, bar);
          } else {
          const bf16* ksrc = c.kv.at(page, 0, h, 0);
          const bf16* vsrc = c.kv.at(page, 1, h, 0);
          mbar_arrive_expect_tx(bar, 2 * bytes);
          bulk_load_1d(dst, ksrc, bytes, bar);
          bulk_load_1d(dst + (uint32_t)PT * HD * 2, vsrc, bytes, bar);
          }
        }
      }
    }
    return;
  }
  if (warp == kDecWarps + 1) {
    // ===================== q/k/v producer: lane l owns dims [4l, 4l+4) =====================
    uint32_t qi = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++qi) {
      const int slot = qi & 1;
      mbar_wait(smem_u32(&s_qempty[slot]), ((qi >> 1) & 1u) ^ 1u);
      const int b = item / c.kv.heads, h = item % c.kv.heads;
      const int L = c.seq_len[b];
      float q4[4] = {0.f, 0.f, 0.f, 0.f}, k4[4] = {0.f, 0.f, 0.f, 0.f}, v4[4] = {0.f, 0.f, 0.f, 0.f};
      for (int s0 = 0; s0 < c.splits; s0 += 2) {          // two splits (6 x 16 B loads) in flight
        float4 t[2][3];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const int sp = s0 + u;
          const float* row = c.qkv_partial + ((size_t)(sp < c.splits ? sp : 0) * c.ws_rows + b) * (size_t)(3 * T) + h * HD + 4 * lane;
          const bool ok = sp < c.splits;
          t[u][0] = ok ? __ldcg(reinterpret_cast<const float4*>(row)) : make_float4(0.f, 0.f, 0.f, 0.f);
          t[u][1] = ok ? __ldcg(reinterpret_cast<const float4*>(row + T)) : make_float4(0.f, 0.f, 0.f, 0.f);
          t[u][2] = ok ? __ldcg(reinterpret_cast<const float4*>(row + 2 * T)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < 2; ++u) {                     // fixed split order
          q4[0] += t[u][0].x; q4[1] += t[u][0].y; q4[2] += t[u][0].z; q4[3] += t[u][0].w;
          k4[0] += t[u][1].x; k4[1] += t[u][1].y; k4[2] += t[u][1].z; k4[3] += t[u][1].w;
          v4[0] += t[u][2].x; v4[1] += t[u][2].y; v4[2] += t[u][2].z; v4[3] += t[u][2].w;
        }
      }
      const float4 cs4 = *reinterpret_cast<const float4*>(rope_cos + (size_t)L * (HD / 2) + ((4 * lane) & 63));
      const float4 sn4 = *reinterpret_cast<const float4*>(rope_sin + (size_t)L * (HD / 2) + ((4 * lane) & 63));
      const float cs[4] = {cs4.x, cs4.y, cs4.z, cs4.w}, sn[4] = {sn4.x, sn4.y, sn4.z, sn4.w};
      float qo[4], ko[4], vo[4];
      uint32_t kpk[2], vpk[2];
      if constexpr (Q8) {
        // quantise the new k / v rows (warp absmax: lane l holds dims [4l, 4l+4)); s_k / s_v take q, the scales go after the ring
        float kr[4], ka = 0.f, va = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float kp = __shfl_xor_sync(0xffffffffu, k4[j], 16), qp = __shfl_xor_sync(0xffffffffu, q4[j], 16);
          const float sgn = (lane < 16) ? -1.f : 1.f;
          qo[j] = (q4[j] * cs[j] + sgn * qp * sn[j]) * c.scale;
          kr[j] = k4[j] * cs[j] + sgn * kp * sn[j];
          ka = fmaxf(ka, fabsf(kr[j])); va = fmaxf(va, fabsf(v4[j]));
        }
        ka = warp_max(ka); va = warp_max(va);
        const float kinv = q8_inv(ka), vinv = q8_inv(va);
        uint32_t kq = 0, vq = 0;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int a = q8_quant(kr[j], kinv), v = q8_quant(v4[j], vinv);
          ko[j] = (float)a; vo[j] = (float)v;
          kq |= (uint32_t)(a & 0xff) << (8 * j); vq |= (uint32_t)(v & 0xff) << (8 * j);
        }
        float* q8x = reinterpret_cast<float*>(dsm + (size_t)kDecStages * stage_bytes);
        *reinterpret_cast<float4*>(&s_q[slot][4 * lane]) = make_float4(qo[0], qo[1], qo[2], qo[3]);
        *reinterpret_cast<float4*>(&s_k[slot][4 * lane]) = make_float4(ko[0], ko[1], ko[2], ko[3]);
        *reinterpret_cast<float4*>(&s_v[slot][4 * lane]) = make_float4(vo[0], vo[1], vo[2], vo[3]);
        if (lane == 0) { q8x[2 * slot] = q8_step(ka); q8x[2 * slot + 1] = q8_step(va); }
        const int page = __ldg(c.kv.seq_pages(b) + L / PT);
        const int cslot = L % PT;
        *reinterpret_cast<uint32_t*>(c.kv.q8_at(page, 0, h, cslot) + 4 * lane) = kq;
        *reinterpret_cast<uint32_t*>(c.kv.q8_at(page, 1, h, cslot) + 4 * lane) = vq;
        if (lane == 0) { *c.kv.q8_scale(page, 0, h, cslot) = q8_step(ka); *c.kv.q8_scale(page, 1, h, cslot) = q8_step(va); }
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&s_qfull[slot]));
        continue;
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float qv = q4[j], kv = k4[j], vv = v4[j];
        const float qp = __shfl_xor_sync(0xffffffffu, qv, 16), kp = __shfl_xor_sync(0xffffffffu, kv, 16);   // dims d +- 64
        const float sgn = (lane < 16) ? -1.f : 1.f;
        qo[j] = (qv * cs[j] + sgn * qp * sn[j]) * c.scale;
        ko[j] = __bfloat162float(__float2bfloat16(kv * cs[j] + sgn * kp * sn[j]));     // the cache holds bf16: attend over the rounded values
        vo[j] = __bfloat162float(__float2bfloat16(vv));
      }
      kpk[0] = pack_bf16x2(ko[0], ko[1]); kpk[1] = pack_bf16x2(ko[2], ko[3]);
      vpk[0] = pack_bf16x2(vo[0], vo[1]); vpk[1] = pack_bf16x2(vo[2], vo[3]);
      *reinterpret_cast<float4*>(&s_q[slot][4 * lane]) = make_float4(qo[0], qo[1], qo[2], qo[3]);
      *reinterpret_cast<float4*>(&s_k[slot][4 * lane]) = make_float4(ko[0], ko[1], ko[2], ko[3]);
      *reinterpret_cast<float4*>(&s_v[slot][4 * lane]) = make_float4(vo[0], vo[1], vo[2], vo[3]);
      const int page = __ldg(c.kv.seq_pages(b) + L / PT);
      const int cslot = L % PT;
      *reinterpret_cast<uint2*>(c.kv.at(page, 0, h, cslot) + 4 * lane) = make_uint2(kpk[0], kpk[1]);
      *reinterpret_cast<uint2*>(c.kv.at(page, 1, h, cslot) + 4 * lane) = make_uint2(vpk[0], vpk[1]);
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&s_qfull[slot]));
    }
    return;
  }

  // ===================== consumer warps (named barrier 1, NC threads) =====================
  const int grp = lane >> 3, sub = lane & 7;
  const uint32_t gmask = 0xffu << (grp * 8);
  uint32_t n = 0, qi = 0;
  for (int item = blockIdx.x; item < n_items; item += gridDim.x, ++qi) {
    const int b = item / c.kv.heads, h = item % c.kv.heads;
    const int L = c.seq_len[b];
    const int npages = (L + PT - 1) / PT;
    const int slot = qi & 1;
    mbar_wait(smem_u32(&s_qfull[slot]), (qi >> 1) & 1u);
    float qreg[16];
#pragma unroll
    for (int i = 0; i < 8; ++i) { qreg[i] = s_q[slot][sub * 8 + i]; qreg[8 + i] = s_q[slot][64 + sub * 8 + i]; }
    float m = -INFINITY, l = 0.f, acc[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = 0.f;
    for (int i = 0; i < npages; ++i, ++n) {
      const int stage = n % kDecStages;
      mbar_wait(smem_u32(&s_full[stage]), (n / kDecStages) & 1u);
      const int ntok = min(PT, L - i * PT);
      const uint8_t* kbase = dsm + (size_t)stage * stage_bytes;
      if constexpr (Q8) {
        dec_page_q8(kbase, PT, ntok, warp, grp, sub, gmask, qreg, m, l, acc);
      } else {
      const uint8_t* vbase = kbase + (size_t)PT * HD * 2;
      for (int tk = warp * 4 + grp; tk < ntok; tk += kDecWarps * 4) {
        const uint4 k0 = *reinterpret_cast<const uint4*>(kbase + (size_t)tk * HD * 2 + sub * 16);
        const uint4 k1 = *reinterpret_cast<const uint4*>(kbase + (size_t)tk * HD * 2 + 128 + sub * 16);
        const uint4 v0 = *reinterpret_cast<const uint4*>(vbase + (size_t)tk * HD * 2 + sub * 16);
        const uint4 v1 = *reinterpret_cast<const uint4*>(vbase + (size_t)tk * HD * 2 + 128 + sub * 16);
        const uint32_t kw[8] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z, k1.w};
        const uint32_t vw[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
        float sc = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) { const float2 kf = unpack_bf16x2(kw[j]); sc += qreg[2 * j] * kf.x + qreg[2 * j + 1] * kf.y; }
        sc += __shfl_xor_sync(gmask, sc, 1);
        sc += __shfl_xor_sync(gmask, sc, 2);
        sc += __shfl_xor_sync(gmask, sc, 4);
        const float mn = fmaxf(m, sc);
        const float cr = __expf(m - mn), p = __expf(sc - mn);
        m = mn;
        l = l * cr + p;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float2 vf = unpack_bf16x2(vw[j]);
          acc[2 * j] = acc[2 * j] * cr + p * vf.x;
          acc[2 * j + 1] = acc[2 * j + 1] * cr + p * vf.y;
        }
      }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&s_empty[stage]));     // this warp is done with the stage
    }
    __syncwarp();
    if (warp == 0 && grp == 0) {                                  // the new token, from the q/k/v producer's slot
      float sc = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) sc += qreg[i] * s_k[slot][sub * 8 + i] + qreg[8 + i] * s_k[slot][64 + sub * 8 + i];
      sc += __shfl_xor_sync(0x000000ffu, sc, 1);
      sc += __shfl_xor_sync(0x000000ffu, sc, 2);
      sc += __shfl_xor_sync(0x000000ffu, sc, 4);
      float pv_scale = 1.f;
      if constexpr (Q8) {
        const float* q8x = reinterpret_cast<const float*>(dsm + (size_t)kDecStages * stage_bytes);
        sc *= q8x[2 * slot];
        pv_scale = q8x[2 * slot + 1];
      }
      const float mn = fmaxf(m, sc);
      const float cr = __expf(m - mn), p = __expf(sc - mn);
      m = mn;
      l = l * cr + p;
      const float pv = Q8 ? p * pv_scale : p;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        acc[i] = acc[i] * cr + pv * s_v[slot][sub * 8 + i];
        acc[8 + i] = acc[8 + i] * cr + pv * s_v[slot][64 + sub * 8 + i];
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(&s_qempty[slot]));         // this warp no longer needs the slot
#pragma unroll
    for (int o = 8; o <= 16; o <<= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, m, o), l2 = __shfl_xor_sync(0xffffffffu, l, o);
      const float mn = fmaxf(m, m2);
      const float c1 = (m == -INFINITY) ? 0.f : __expf(m - mn), c2 = (m2 == -INFINITY) ? 0.f : __expf(m2 - mn);
      l = l * c1 + l2 * c2;
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        const float a2 = __shfl_xor_sync(0xffffffffu, acc[i], o);
        acc[i] = acc[i] * c1 + a2 * c2;
      }
      m = mn;
    }
    if (grp == 0) {
#pragma unroll
      for (int i = 0; i < 8; ++i) { s_acc[warp][sub * 8 + i] = acc[i]; s_acc[warp][64 + sub * 8 + i] = acc[8 + i]; }
      if (sub == 0) { s_m[warp] = m; s_l[warp] = l; }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(NC) : "memory");
    if (tid < HD) {
      float M = -INFINITY;
#pragma unroll
      for (int w = 0; w < kDecWarps; ++w) M = fmaxf(M, s_m[w]);
      float Lsum = 0.f, O = 0.f;
#pragma unroll
      for (int w = 0; w < kDecWarps; ++w) {
        const float cw = (s_m[w] == -INFINITY) ? 0.f : __expf(s_m[w] - M);
        Lsum += s_l[w] * cw;
        O += s_acc[w][tid] * cw;
      }
      c.out[(size_t)b * T + h * HD + tid] = __float2bfloat16(O / Lsum);
    }
    asm volatile("bar.sync 1, %0;" ::"n"(NC) : "memory");          // s_acc is reused by the next item
  }
  trace.done();
}

VCLA_DEFINE_TRACE_SETTER(trace_set_attention)

int attention_init() {
  // dynamic shared-memory opt-ins of every attention kernel; called once per process from vcla_create (never during capture)
  static std::once_flag once;
  static int rc = 0;
  std::call_once(once, [] {
    auto set = [](const void* fn, int bytes) { return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) == cudaSuccess ? 0 : -1; };
    rc |= set((const void*)attn_decode_kernel<kDecStages>, kDecStages * kDecMaxPT * 128 * 2 * 2);
    rc |= set((const void*)attn_decode_kernel<kDecStagesSmallBatch>, kDecStagesSmallBatch * kDecMaxPT * 128 * 2 * 2);
    rc |= set((const void*)attn_decode_persistent_kernel<KV_BF16>, kDecStages * kDecMaxPT * 128 * 2 * 2);
    rc |= set((const void*)attn_decode_kernel<kDecStages, kDecAttend>, kDecStages * kDecMaxPT * 128 * 2 * 2);
    rc |= set((const void*)attn_decode_kernel<kDecStagesSmallBatch, kDecAttend>, kDecStagesSmallBatch * kDecMaxPT * 128 * 2 * 2);
    rc |= set((const void*)attn_prefill_kernel<128>, 5 * 64 * 128 * 2);
    rc |= set((const void*)attn_prefill_kernel<64>, 5 * 64 * 64 * 2);
    const int q8_3 = (int)dec_smem_bytes(KV_INT8, kDecStages, kDecMaxPT), q8_2 = (int)dec_smem_bytes(KV_INT8, kDecStagesSmallBatch, kDecMaxPT);
    rc |= set((const void*)attn_decode_kernel<kDecStages, kDecPlain, KV_INT8>, q8_3);
    rc |= set((const void*)attn_decode_kernel<kDecStagesSmallBatch, kDecPlain, KV_INT8>, q8_2);
    rc |= set((const void*)attn_decode_persistent_kernel<KV_INT8>, q8_3);
    rc |= set((const void*)attn_decode_kernel<kDecStages, kDecAttend, KV_INT8>, q8_3);
    rc |= set((const void*)attn_decode_kernel<kDecStagesSmallBatch, kDecAttend, KV_INT8>, q8_2);
    if (rc) set_error("attention_init: cudaFuncSetAttribute failed: %s", cudaGetErrorString(cudaGetLastError()));
  });
  return rc;
}

// The decode kernel attention_decode launches for c: the persistent kernel (-> its grid in *persistent_ctas) or the one-shot kernel with
// a 2- or 3-stage ring.  The choice does not depend on the cache format.
enum DecodeKernel { kDecPersistent, kDecOneShot2, kDecOneShot3 };
static DecodeKernel decode_kernel_pick(const DecodeAttnCall& c, int* persistent_ctas) {
  const int n_items = c.B * c.kv.heads;
  int slots = 2 * num_sms();
  // persistent_mode: 0 = never, 1 (default) = when items outnumber the resident CTAs, 2 = whenever kv_splits == 1 (tests);
  // persistent_grid caps the persistent grid (tests: several items per CTA on small problems).  Both are read from the
  // environment once per context (vcla_create), not per launch.
  if (c.persistent_grid > 0 && c.persistent_grid < slots) slots = c.persistent_grid;
  if (c.kv_splits == 1 && ((c.persistent_mode == 1 && n_items > slots) || c.persistent_mode == 2)) {
    *persistent_ctas = n_items < slots ? n_items : slots;   // more (sequence, head) items than resident CTAs
    return kDecPersistent;
  }
  // one wave at two CTAs per SM: the small ring leaves a third slot free
  return c.kv_splits * n_items <= 2 * num_sms() ? kDecOneShot2 : kDecOneShot3;
}

static int decode_check(const char* who, const DecodeAttnCall& c, KvFormat fmt) {
  if (c.HD != 128) { set_error("%s: head dim %d unsupported (128)", who, c.HD); return -1; }
  if (c.kv.page_tokens < 8 || c.kv.page_tokens > kDecMaxPT || c.kv.page_tokens % 8 != 0) { set_error("%s: page_tokens %d unsupported (8..%d, multiple of 8)", who, c.kv.page_tokens, kDecMaxPT); return -1; }
  if (c.rope_cos == nullptr || c.rope_sin == nullptr) { set_error("%s: rope table not initialised", who); return -1; }
  if (fmt != KV_BF16 && fmt != KV_INT8) { set_error("%s: KV cache format %d unsupported", who, (int)fmt); return -1; }
  return attention_init();
}

template <int FMT>
static int decode_launch(const DecodeAttnCall& c, cudaStream_t st) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(c.kv_splits, c.kv.heads, c.B); cfg.blockDim = dim3(kDecWarps * 32);
  cfg.dynamicSmemBytes = dec_smem_bytes(FMT, kDecStages, c.kv.page_tokens); cfg.stream = st;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (pdl_enabled()) { attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[na].val.programmaticStreamSerializationAllowed = 1; ++na; }
  cfg.attrs = attr; cfg.numAttrs = na;
  int persistent_ctas = 0;
  switch (decode_kernel_pick(c, &persistent_ctas)) {
    case kDecPersistent:
      cfg.gridDim = dim3(persistent_ctas);
      cfg.blockDim = dim3((kDecWarps + 2) * 32);
      VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_decode_persistent_kernel<FMT>, c, c.rope_cos, c.rope_sin, c.B * c.kv.heads));
      break;
    case kDecOneShot2:
      cfg.dynamicSmemBytes = dec_smem_bytes(FMT, kDecStagesSmallBatch, c.kv.page_tokens);
      VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_decode_kernel<kDecStagesSmallBatch, kDecPlain, FMT>, c, c.rope_cos, c.rope_sin));
      break;
    case kDecOneShot3:
      VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_decode_kernel<kDecStages, kDecPlain, FMT>, c, c.rope_cos, c.rope_sin));
      break;
  }
  return 0;
}

int attention_decode(const DecodeAttnCall& c, cudaStream_t st, KvFormat fmt) {
  if (decode_check("attention_decode", c, fmt)) return -1;
  return fmt == KV_INT8 ? decode_launch<KV_INT8>(c, st) : decode_launch<KV_BF16>(c, st);
}

template <int FMT>
static int decode_lookup_launch(const DecodeAttnCall& c, cudaStream_t st) {
  cudaLaunchConfig_t cfg = {};
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (pdl_enabled()) { attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[na].val.programmaticStreamSerializationAllowed = 1; ++na; }
  cfg.attrs = attr; cfg.numAttrs = na; cfg.stream = st; cfg.blockDim = dim3(kDecWarps * 32);
  // the append launch streams no pages: no ring; the int8 rows need only the absmax scratch
  cfg.gridDim = dim3(1, c.kv.heads, c.B); cfg.dynamicSmemBytes = FMT == KV_INT8 ? kDecQ8Extra : 0;
  VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_decode_kernel<kDecStagesSmallBatch, kDecAppend, FMT>, c, c.rope_cos, c.rope_sin));
  // the ring depth changes no arithmetic; the one-token rule picks it from the grid size
  cfg.gridDim = dim3(c.kv_splits, c.kv.heads, c.B);
  if (c.kv_splits * c.B * c.kv.heads <= 2 * num_sms()) {
    cfg.dynamicSmemBytes = dec_smem_bytes(FMT, kDecStagesSmallBatch, c.kv.page_tokens);
    VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_decode_kernel<kDecStagesSmallBatch, kDecAttend, FMT>, c, c.rope_cos, c.rope_sin));
  } else {
    cfg.dynamicSmemBytes = dec_smem_bytes(FMT, kDecStages, c.kv.page_tokens);
    VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_decode_kernel<kDecStages, kDecAttend, FMT>, c, c.rope_cos, c.rope_sin));
  }
  return 0;
}

int attention_decode_lookup(const DecodeAttnCall& c, cudaStream_t st, KvFormat fmt) {
  if (c.kv_splits < 1 || c.kv_splits > 8 || c.B < 1 || c.B > 16) { set_error("attention_decode_lookup: %d rows x %d KV splits unsupported", c.B, c.kv_splits); return -1; }
  if (decode_check("attention_decode_lookup", c, fmt)) return -1;
  return fmt == KV_INT8 ? decode_lookup_launch<KV_INT8>(c, st) : decode_lookup_launch<KV_BF16>(c, st);
}

template <int FMT>
static int decode_ctas_per_sm(const DecodeAttnCall& c) {
  int persistent_ctas = 0, n = 0;
  cudaError_t e = cudaSuccess;
  switch (decode_kernel_pick(c, &persistent_ctas)) {
    case kDecPersistent:
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, attn_decode_persistent_kernel<FMT>, (kDecWarps + 2) * 32, dec_smem_bytes(FMT, kDecStages, c.kv.page_tokens));
      break;
    case kDecOneShot2:
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, attn_decode_kernel<kDecStagesSmallBatch, kDecPlain, FMT>, kDecWarps * 32, dec_smem_bytes(FMT, kDecStagesSmallBatch, c.kv.page_tokens));
      break;
    case kDecOneShot3:
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, attn_decode_kernel<kDecStages, kDecPlain, FMT>, kDecWarps * 32, dec_smem_bytes(FMT, kDecStages, c.kv.page_tokens));
      break;
  }
  if (e != cudaSuccess) { set_error("attention_decode_ctas_per_sm: %s", cudaGetErrorString(e)); (void)cudaGetLastError(); return -1; }
  return n;
}

int attention_decode_ctas_per_sm(const DecodeAttnCall& c, KvFormat fmt) {
  if (attention_init()) return -1;
  return fmt == KV_INT8 ? decode_ctas_per_sm<KV_INT8>(c) : decode_ctas_per_sm<KV_BF16>(c);
}

}  // namespace vcla
