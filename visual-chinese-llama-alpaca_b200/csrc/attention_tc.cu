// wgmma flash attention for the prefill side of the path (sm_90a): LLaMA's causal prefill (hd 128) by default; it also covers
// ViT self-attention (257 tokens, hd 64) and the Resampler's 64 queries over [their own 64 rows ; 257 image rows] (two KV segments,
// hd 64), which the default dispatch leaves on the mma.sync kernel (attention.cu: attention_prefill; VCLA_ATTN_TC=2 forces this
// kernel everywhere, and the tests run it on every shape).
//
// One CTA per (64 query rows, head, sequence); one warpgroup computes, one warp loads.  Both contractions run on wgmma:
//   S = Q K^T   m64n64k16 x HD/16   A = Q tile, B = K tile, both K-major [64-element k-blocks][64 rows][128 B] staged by TMA
//               (128 B swizzle); fp32 scores in registers
//   O += P V    m64nHDk16 x 4       A = P from registers (the score fragment rounded to bf16 IS the A fragment layout), B = V tile
//               exactly as TMA delivers it ([head-dim block][kv rows][64 head dims] = an MN-major operand: transpose bit + a
//               descriptor with SBO = 8 kv rows, LBO = the next 64 head dims)
// O accumulates in registers; the online-softmax rescale (O *= exp2(m_old - m_new)) is a multiply of the thread's fragment rows.
// K/V tiles are double buffered, two CTAs share an SM.  Masks: keys past a segment's end, causal (key <= query + Sk - Sq), left
// padding (kv_start).  Fully masked rows produce zeros, like the mma.sync kernel (csrc/attention.cu).
//
// PAGED = true is the prefill of a chunk of new tokens over a cached prefix (vcla_prefill_extend): the queries are the Sq new rows
// of sequence b, the keys / values are its first base_len[b] + Sq cached tokens, read straight from the layer's page pool (the
// chunk's own K/V were appended by the QKV GEMM epilogue).  Key j is visible to chunk row t iff j <= base_len[b] + t.  The pool
// [pages][K|V][H][page_tokens][128] is one 2D tensor of 128-column rows (256 B pitch); a 64-key tile is 64 / page_tokens boxes of
// page_tokens rows (a multiple of 8 rows = whole 128 B-swizzle atoms, so the boxes stack into the same smem image a 64-row box
// gives) times two 64-column halves, each box addressed through the page table.  When the grid would leave SMs idle the key tiles
// are split over kv_splits CTAs; each writes its unnormalised (O, m, l) and the last one to arrive combines them in split order.
#include "common.cuh"
#include "kernels.h"

#include <algorithm>
#include <mutex>
#include <stdlib.h>
#include <string.h>

namespace vcla {

constexpr int kAtThreads = 160;                 // warps 0..3 = the wgmma warpgroup, warp 4 = TMA producer
constexpr int kAtBQ = 64, kAtBKV = 64;
constexpr int kAtStages = 2;
constexpr int kAtMaxKvSplits = 16;

struct AttnTcParams {
  int Sq, n0, n1, H;
  float sl2;                       // softmax scale * log2(e)
  int causal;
  const int32_t* kv_start;         // [B] or null
  bf16* out; int o_stride;
  // PAGED only
  const int32_t* base_len;         // [B] cached tokens before the chunk
  int kv_splits;                   // CTAs per (query tile, head, sequence); blockIdx.z = b * kv_splits + split
  float* part;                     // kv_splits > 1: [tile][split][64 rows][HD + 4] = unnormalised O, running max, row sum, pad
  int32_t* counters;               // [tile] arrivals, back to 0 after the combine
  KvPool kv;                       // the layer's pages
};

template <int HD>
struct AttnTcCfg {
  static constexpr int KB = HD / 64;                         // 64-element k-blocks of the head dimension
  static constexpr int Q_BYTES = KB * kAtBQ * 128;           // [KB][64 rows][128 B]
  static constexpr int K_BYTES = KB * kAtBKV * 128;
  static constexpr int V_BYTES = KB * kAtBKV * 128;          // [KB (head-dim blocks)][64 kv rows][128 B]
  static constexpr int KV_OFF = Q_BYTES;
  static constexpr int BAR_OFF = KV_OFF + kAtStages * (K_BYTES + V_BYTES);
  static constexpr int SMEM_BYTES = BAR_OFF + 256 + 1024;
  static constexpr int PART_LD = HD + 4;                      // split-KV partial row: O[HD], m, l, 2 pad floats (16 B rows)
};

// MN-major operand, 128 B swizzle: rows (the contraction index) of 128 B = 64 contiguous MN elements, 8-row atoms 1024 B apart
// (stride byte offset), the next 64 MN elements `lbo_bytes` away (leading byte offset)
__device__ __forceinline__ uint64_t make_desc_mn_sw128(uint32_t smem_addr, uint32_t lbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

template <int HD>
__device__ __forceinline__ void wgmma_pv(float (&o)[HD / 2], const uint32_t (&a)[4], uint64_t bdesc) {
  if constexpr (HD == 64) wgmma_bf16_rs_tb_n64(o, a, bdesc, 1);
  else wgmma_bf16_rs_tb_n128(o, a, bdesc, 1);
}

// FMT = KV_INT8 (PAGED only): the pool holds int8 rows + fp32 row scales (kernels.h).  TMA brings each page's int8 rows (a UINT8 map
// over the 128-byte rows) into the upper half of the stage's K / V tiles and a bulk copy its scales; the warpgroup converts the rows
// to bf16 in the 128 B-swizzled image the descriptors read (exact: |q| <= 127), multiplies S by s_k, scales P's columns by s_v before
// P is rounded to bf16, and keeps the row sum on the unscaled p.
constexpr int kAtQ8ScaleBytes = 2 * kAtBKV * 4;   // per stage: K scales, V scales of the tile's 64 keys
template <int HD, bool PAGED, int FMT = KV_BF16>
__global__ void __launch_bounds__(kAtThreads, 2)
attn_prefill_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK0, const __grid_constant__ CUtensorMap tmV0,
                       const __grid_constant__ CUtensorMap tmK1, const __grid_constant__ CUtensorMap tmV1, const AttnTcParams p) {
  using C = AttnTcCfg<HD>;
  constexpr bool Q8 = FMT == KV_INT8;
  static_assert(!Q8 || (PAGED && HD == 128), "the int8 pool is read by the paged kernel only");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar0 = base + C::BAR_OFF;
  const uint32_t q_full = bar0;
  auto kv_full = [&](int s) { return bar0 + 8u * (1 + s); };
  auto kv_empty = [&](int s) { return bar0 + 8u * (1 + kAtStages + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kAtBQ, h = blockIdx.y;
  const int b = PAGED ? (int)blockIdx.z / p.kv_splits : (int)blockIdx.z;
  const int split = PAGED ? (int)blockIdx.z % p.kv_splits : 0;
  TraceScope trace(3);
  // PAGED: the keys are the sequence's cached tokens; their count is read after the kernels that wrote it have finished
  if constexpr (PAGED) pdl_wait();
  const int base_len = PAGED ? p.base_len[b] : 0;
  const int n0 = PAGED ? base_len + p.Sq : p.n0, n1 = PAGED ? 0 : p.n1;
  const int Sk = n0 + n1;
  const int off = Sk - p.Sq;                                   // causal: key j visible to query i iff j <= i + off
  const int kv0 = p.kv_start ? __ldg(p.kv_start + b) : 0;

  // KV tiles: segment 0 tiles first, then segment 1; causal launches have one segment and stop at the diagonal tile
  const int nt0 = (n0 + kAtBKV - 1) / kAtBKV, nt1 = (n1 + kAtBKV - 1) / kAtBKV;
  int nt = nt0 + nt1;
  if (p.causal) { const int kv_end = min(Sk, q0 + kAtBQ + off); nt = min(nt, (max(kv_end, 0) + kAtBKV - 1) / kAtBKV); }
  int jt0 = kv0 / kAtBKV;                                      // tiles entirely left of the padding boundary are skipped
  if (PAGED && p.kv_splits > 1) {                              // split-KV: this CTA's contiguous share of the key tiles
    const int per = (nt + p.kv_splits - 1) / p.kv_splits;
    jt0 = split * per;
    nt = min(nt, jt0 + per);
  }
  const int n_tiles = max(nt - jt0, 0);

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < kAtStages; ++s) { mbar_init(kv_full(s), 1); mbar_init(kv_empty(s), 1); }
    fence_barrier_init();
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK0); tma_prefetch_desc(&tmV0);
    if (n1 > 0) { tma_prefetch_desc(&tmK1); tma_prefetch_desc(&tmV1); }
  }
  __syncthreads();
  pdl_launch_dependents();

  if (warp == 4) {
    if (lane == 0 && n_tiles > 0) {
      // ===================== TMA producer =====================
      pdl_wait();                                             // q / k / v come from the previous kernel
      mbar_arrive_expect_tx(q_full, C::Q_BYTES);
      for (int kb = 0; kb < C::KB; ++kb) tma_load_2d(base + kb * kAtBQ * 128, &tmQ, h * HD + kb * 64, b * p.Sq + q0, q_full, kEvictNormal);
      for (int i = 0; i < n_tiles; ++i) {
        const int j = jt0 + i, stage = i % kAtStages;
        mbar_wait_mma(kv_empty(stage), (((uint32_t)(i / kAtStages)) & 1u) ^ 1u);
        const uint32_t sk = base + C::KV_OFF + stage * (C::K_BYTES + C::V_BYTES), sv = sk + C::K_BYTES;
        if constexpr (Q8) {
          // int8 rows into the second k-block of the K / V tiles (the warpgroup expands them in place), scales after the barriers
          mbar_arrive_expect_tx(kv_full(stage), 2 * kAtBKV * 128 + kAtQ8ScaleBytes);
          const uint32_t ssc = base + C::BAR_OFF + 256 + stage * kAtQ8ScaleBytes;
          const int pt = p.kv.page_tokens, last_page = (n0 - 1) / pt;
          const int32_t* prow = p.kv.seq_pages(b);
          for (int r = 0; r < kAtBKV; r += pt) {
            const int page = prow[min((j * kAtBKV + r) / pt, last_page)];
            tma_load_2d(sk + kAtBKV * 128 + r * 128, &tmK0, 0, p.kv.row<int>(page, 0, h), kv_full(stage), kEvictNormal);
            tma_load_2d(sv + kAtBKV * 128 + r * 128, &tmK0, 0, p.kv.row<int>(page, 1, h), kv_full(stage), kEvictNormal);
            bulk_load_1d(ssc + r * 4, p.kv.q8_scale(page, 0, h, 0), (uint32_t)pt * 4, kv_full(stage));
            bulk_load_1d(ssc + kAtBKV * 4 + r * 4, p.kv.q8_scale(page, 1, h, 0), (uint32_t)pt * 4, kv_full(stage));
          }
          continue;
        }
        mbar_arrive_expect_tx(kv_full(stage), C::K_BYTES + C::V_BYTES);
        if constexpr (PAGED) {
          // one box of page_tokens rows per page and 64-column half; boxes past the sequence's last page re-read that page
          // (only pages the sequence owns are touched; those rows are masked)
          const int pt = p.kv.page_tokens, last_page = (n0 - 1) / pt;
          const int32_t* prow = p.kv.seq_pages(b);
          for (int r = 0; r < kAtBKV; r += pt) {
            const int page = prow[min((j * kAtBKV + r) / pt, last_page)];
            const int krow = p.kv.row<int>(page, 0, h), vrow = p.kv.row<int>(page, 1, h);
            for (int kb = 0; kb < C::KB; ++kb) {
              tma_load_2d(sk + kb * kAtBKV * 128 + r * 128, &tmK0, kb * 64, krow, kv_full(stage), kEvictNormal);
              tma_load_2d(sv + kb * kAtBKV * 128 + r * 128, &tmK0, kb * 64, vrow, kv_full(stage), kEvictNormal);
            }
          }
        } else {
          const bool seg1 = j >= nt0;
          const CUtensorMap* mk = seg1 ? &tmK1 : &tmK0;
          const CUtensorMap* mv = seg1 ? &tmV1 : &tmV0;
          const int row = seg1 ? b * n1 + (j - nt0) * kAtBKV : b * n0 + j * kAtBKV;
          for (int kb = 0; kb < C::KB; ++kb) {
            tma_load_2d(sk + kb * kAtBKV * 128, mk, h * HD + kb * 64, row, kv_full(stage), kEvictNormal);
            tma_load_2d(sv + kb * kAtBKV * 128, mv, h * HD + kb * 64, row, kv_full(stage), kEvictNormal);
          }
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== wgmma warpgroup: S = Q K^T, online softmax, O += P V, epilogue =====================
    // Thread (warp w, lane l) holds query rows 16 w + l / 4 (+ 8) and columns 8 j + 2 (l % 4) (+ 1) of S and O; the 4 lanes of a
    // quad share a row.  l_run is this thread's partial row sum (alpha is uniform over the quad), reduced over the quad at the end.
    const int fr = warp * 16 + (lane >> 2), fc = 2 * (lane & 3);
    pdl_wait();
    trace.dep();                                               // (the trace slot belongs to thread 0, a thread of this warpgroup)
    float o[HD / 2];
#pragma unroll
    for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    if (n_tiles > 0) mbar_wait_mma(q_full, 0);
    for (int i = 0; i < n_tiles; ++i) {
      const int j = jt0 + i, stage = i % kAtStages;
      const bool seg1 = j >= nt0;
      const int kbase = seg1 ? n0 + (j - nt0) * kAtBKV : j * kAtBKV;         // global key index of the tile's first row
      const int kvalid = seg1 ? n1 - (j - nt0) * kAtBKV : n0 - j * kAtBKV;   // keys of this tile that exist in the segment
      const int lo = max(kv0 - kbase, 0);
      const uint32_t sk = base + C::KV_OFF + stage * (C::K_BYTES + C::V_BYTES), sv = sk + C::K_BYTES;
      mbar_wait_mma(kv_full(stage), ((uint32_t)(i / kAtStages)) & 1u);
      const float* ksc = nullptr;
      const float* vsc = nullptr;
      if constexpr (Q8) {
        // expand the int8 rows (upper k-block of each tile) to the bf16 swizzled image: thread t owns row t / 2, k-block t % 2.  All
        // reads finish before any write, since the bf16 image overwrites the int8 rows.
        const int r = threadIdx.x >> 1, kb = threadIdx.x & 1;
        uint4 kr[4], vr[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(kr[c].x), "=r"(kr[c].y), "=r"(kr[c].z), "=r"(kr[c].w)
                       : "r"(sk + kAtBKV * 128 + r * 128 + kb * 64 + c * 16));
          asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(vr[c].x), "=r"(vr[c].y), "=r"(vr[c].z), "=r"(vr[c].w)
                       : "r"(sv + kAtBKV * 128 + r * 128 + kb * 64 + c * 16));
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const uint32_t kw[4] = {kr[c].x, kr[c].y, kr[c].z, kr[c].w}, vw[4] = {vr[c].x, vr[c].y, vr[c].z, vr[c].w};
#pragma unroll
          for (int half = 0; half < 2; ++half) {             // 16 int8 -> two 16 B chunks of 8 bf16
            const int chunk = 2 * c + half;
            const uint32_t off = kb * kAtBKV * 128 + r * 128 + ((chunk ^ (r & 7)) << 4);
            uint32_t ko[4], vo[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const uint32_t kword = kw[2 * half + (e >> 1)], vword = vw[2 * half + (e >> 1)];
              const int lo = 2 * (e & 1);
              ko[e] = pack_bf16x2(q8_lane(kword, lo), q8_lane(kword, lo + 1));
              vo[e] = pack_bf16x2(q8_lane(vword, lo), q8_lane(vword, lo + 1));
            }
            asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(sk + off), "r"(ko[0]), "r"(ko[1]), "r"(ko[2]), "r"(ko[3]) : "memory");
            asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(sv + off), "r"(vo[0]), "r"(vo[1]), "r"(vo[2]), "r"(vo[3]) : "memory");
          }
        }
        fence_proxy_async();
        asm volatile("bar.sync 1, 128;" ::: "memory");
        ksc = reinterpret_cast<const float*>(smem_raw + (base - smem_u32(smem_raw)) + C::BAR_OFF + 256 + stage * kAtQ8ScaleBytes);
        vsc = ksc + kAtBKV;
      }
      if constexpr (PAGED) {
        // V rows past the sequence end are cache slots nobody wrote (any bits, NaN included) and P = 0 does not cancel a NaN
        // in the PV product: zero them (whole 128 B rows, so the swizzle does not matter) before the tensor core reads them
        if (kvalid < kAtBKV) {
          for (int idx = threadIdx.x; idx < C::KB * (kAtBKV - kvalid) * 8; idx += 128) {
            const int kb = idx / ((kAtBKV - kvalid) * 8), rem = idx % ((kAtBKV - kvalid) * 8);
            const uint32_t addr = sv + kb * kAtBKV * 128 + (kvalid + rem / 8) * 128 + (rem % 8) * 16;
            asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(addr), "r"(0u) : "memory");
          }
          fence_proxy_async();
          asm volatile("bar.sync 1, 128;" ::: "memory");
        }
      }
      float s[kAtBKV / 2];
      wgmma_fence();
#pragma unroll
      for (int kb = 0; kb < C::KB; ++kb) {
        const uint64_t adesc = make_desc_sw128(base + kb * kAtBQ * 128), bdesc = make_desc_sw128(sk + kb * kAtBKV * 128);
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_bf16<kAtBKV>(s, adesc + 2u * k, bdesc + 2u * k, (kb > 0 || k > 0) ? 1 : 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(s);
      if constexpr (Q8) {
#pragma unroll
        for (int jj = 0; jj < kAtBKV / 8; ++jj)
#pragma unroll
          for (int e = 0; e < 4; ++e) s[4 * jj + e] *= ksc[8 * jj + fc + (e & 1)];   // NaN scales of unwritten slots stay masked
      }
      uint32_t pa[kAtBKV / 16][4];                             // P as the A fragments of the 4 k-steps of P V
#pragma unroll
      for (int h2 = 0; h2 < 2; ++h2) {
        const int qi = q0 + fr + 8 * h2;
        int hi = min(kvalid, kAtBKV);
        if (p.causal) hi = min(hi, qi + off - kbase + 1);
        float mx = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < kAtBKV / 8; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * jj + fc + e;
            if (col >= lo && col < hi) mx = fmaxf(mx, s[4 * jj + 2 * h2 + e] * p.sl2);
          }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m_run[h2], mx);
        const float m_safe = (m_new == -INFINITY) ? 0.f : m_new;
        const float alpha = exp2f(m_run[h2] - m_safe);         // 0 when nothing was visible before
        m_run[h2] = m_new;
        float ls = 0.f;
#pragma unroll
        for (int jj = 0; jj < kAtBKV / 8; ++jj) {
          const int col = 8 * jj + fc;
          const float p0 = (col >= lo && col < hi) ? exp2f(s[4 * jj + 2 * h2] * p.sl2 - m_safe) : 0.f;
          const float p1 = (col + 1 >= lo && col + 1 < hi) ? exp2f(s[4 * jj + 2 * h2 + 1] * p.sl2 - m_safe) : 0.f;
          __nv_bfloat162 pb;
          if constexpr (Q8) {
            pb = __floats2bfloat162_rn(p0 > 0.f ? p0 * vsc[col] : 0.f, p1 > 0.f ? p1 * vsc[col + 1] : 0.f);
            ls += p0 + p1;                                        // the row sum of the unscaled p
          } else {
          pb = __floats2bfloat162_rn(p0, p1);
          ls += __bfloat162float(pb.x) + __bfloat162float(pb.y);   // the sum of what the tensor core will actually multiply
          }
          // k-step jj / 2: registers {row, cols 0-7 | row + 8, cols 0-7 | row, cols 8-15 | row + 8, cols 8-15}
          pa[jj >> 1][(jj & 1) * 2 + h2] = *reinterpret_cast<const uint32_t*>(&pb);
        }
        l_run[h2] = l_run[h2] * alpha + ls;
#pragma unroll
        for (int jj = 0; jj < HD / 8; ++jj) { o[4 * jj + 2 * h2] *= alpha; o[4 * jj + 2 * h2 + 1] *= alpha; }
      }
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < kAtBKV / 16; ++ks)                 // 16 kv rows per MMA: V rows +16 * 128 B
        wgmma_pv<HD>(o, pa[ks], make_desc_mn_sw128(sv + ks * 16 * 128, (uint32_t)(kAtBKV * 128)));
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(o);
      if (threadIdx.x == 0) mbar_arrive(kv_empty(stage));     // K/V stage reusable
    }
    // ---- epilogue: O / l -> bf16
#pragma unroll
    for (int h2 = 0; h2 < 2; ++h2) {
      float l = l_run[h2];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      if (PAGED && p.kv_splits > 1) {
        // this split's unnormalised rows: O, the running max (log2 domain, scaled) and the row sum
        float* prow = p.part + ((((size_t)(b * p.H + h) * gridDim.x + blockIdx.x) * p.kv_splits + split) * kAtBQ + fr + 8 * h2) * C::PART_LD;
#pragma unroll
        for (int jj = 0; jj < HD / 8; ++jj)
          *reinterpret_cast<float2*>(prow + 8 * jj + fc) = make_float2(o[4 * jj + 2 * h2], o[4 * jj + 2 * h2 + 1]);
        if ((lane & 3) == 0) *reinterpret_cast<float2*>(prow + HD) = make_float2(m_run[h2], l);
        continue;
      }
      const float inv = l > 0.f ? 1.f / l : 0.f;
      const int qi = q0 + fr + 8 * h2;
      if (qi < p.Sq) {
        bf16* orow = p.out + (size_t)(b * p.Sq + qi) * p.o_stride + h * HD;
#pragma unroll
        for (int jj = 0; jj < HD / 8; ++jj)
          *reinterpret_cast<uint32_t*>(orow + 8 * jj + fc) = pack_bf16x2(o[4 * jj + 2 * h2] * inv, o[4 * jj + 2 * h2 + 1] * inv);
      }
    }
  }

  if constexpr (PAGED) {
    if (p.kv_splits > 1) {
      // split-KV combine: the last CTA of this (query tile, head, sequence) to arrive merges every split's partial in split order,
      // so the result does not depend on which CTA that is (bit-deterministic)
      __shared__ int s_last;
      const size_t tile = (size_t)(b * p.H + h) * gridDim.x + blockIdx.x;
      __threadfence();
      __syncthreads();
      if (threadIdx.x == 0) s_last = atomicAdd(p.counters + tile, 1) == p.kv_splits - 1;
      __syncthreads();
      if (s_last) {
        __threadfence();
        const float* part = p.part + tile * p.kv_splits * kAtBQ * C::PART_LD;
        for (int idx = threadIdx.x; idx < kAtBQ * (HD / 4); idx += kAtThreads) {
          const int r = idx / (HD / 4), d = (idx % (HD / 4)) * 4;
          if (q0 + r >= p.Sq) continue;
          float mx = -INFINITY;
          for (int s = 0; s < p.kv_splits; ++s) mx = fmaxf(mx, __ldcg(part + ((size_t)s * kAtBQ + r) * C::PART_LD + HD));
          float l = 0.f;
          float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
          if (mx != -INFINITY) {
            for (int s = 0; s < p.kv_splits; ++s) {
              const float* prow = part + ((size_t)s * kAtBQ + r) * C::PART_LD;
              const float w = exp2f(__ldcg(prow + HD) - mx);      // 0 for a split that saw no visible key of this row
              l += __ldcg(prow + HD + 1) * w;
              const float4 v = __ldcg(reinterpret_cast<const float4*>(prow + d));
              acc.x += v.x * w; acc.y += v.y * w; acc.z += v.z * w; acc.w += v.w * w;
            }
          }
          const float inv = l > 0.f ? 1.f / l : 0.f;
          bf16* orow = p.out + (size_t)(b * p.Sq + q0 + r) * p.o_stride + h * HD + d;
          *reinterpret_cast<uint2*>(orow) = make_uint2(pack_bf16x2(acc.x * inv, acc.y * inv), pack_bf16x2(acc.z * inv, acc.w * inv));
        }
        if (threadIdx.x == 0) p.counters[tile] = 0;           // ready for the next launch
      }
    }
  }

  __syncthreads();
  trace.done();
}

VCLA_DEFINE_TRACE_SETTER(trace_set_attention_tc)

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled g_at_encode = nullptr;
static std::once_flag g_at_once;
static int g_at_rc = 0;

static int attn_tc_init() {
  std::call_once(g_at_once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || fn == nullptr) {
      set_error("cuTensorMapEncodeTiled not available"); g_at_rc = -1; return;
    }
    g_at_encode = reinterpret_cast<PFN_encodeTiled>(fn);
    if (cudaFuncSetAttribute(attn_prefill_tc_kernel<64, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnTcCfg<64>::SMEM_BYTES) != cudaSuccess ||
        cudaFuncSetAttribute(attn_prefill_tc_kernel<128, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnTcCfg<128>::SMEM_BYTES) != cudaSuccess ||
        cudaFuncSetAttribute(attn_prefill_tc_kernel<128, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnTcCfg<128>::SMEM_BYTES) != cudaSuccess ||
        cudaFuncSetAttribute(attn_prefill_tc_kernel<128, true, KV_INT8>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             AttnTcCfg<128>::SMEM_BYTES + kAtStages * kAtQ8ScaleBytes) != cudaSuccess) {
      set_error("attention_tc: cudaFuncSetAttribute failed: %s", cudaGetErrorString(cudaGetLastError())); g_at_rc = -1;
    }
  });
  return g_at_rc;
}

// rows x cols bf16 view with a row pitch of `ld` elements; boxes of `box_rows` (default 64) rows x 64 columns (128 B), 128 B swizzle
static int attn_tmap(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, int box_rows = kAtBQ) {
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (ld * 2) % 16 != 0) { set_error("attention_tc: operands must be 16 B aligned with a 16 B-multiple pitch"); return -1; }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_at_encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("attention_tc: cuTensorMapEncodeTiled failed (%d)", (int)r); return -1; }
  return 0;
}

// the int8 pool's rows as a [rows][128] uint8 tensor: boxes of box_rows whole rows, no swizzle (the kernel expands them)
static int attn_tmap_q8(CUtensorMap* m, const void* ptr, uint64_t rows, int box_rows) {
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0) { set_error("attention_tc: the int8 pool must be 16 B aligned"); return -1; }
  cuuint64_t dims[2] = {128, rows};
  cuuint64_t strides[1] = {128};
  cuuint32_t box[2] = {128, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_at_encode(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("attention_tc: cuTensorMapEncodeTiled (uint8) failed (%d)", (int)r); return -1; }
  return 0;
}

int attention_prefill_tc(const AttnCall& c, cudaStream_t st) {
  if (attn_tc_init()) return -1;
  if (c.HD != 64 && c.HD != 128) { set_error("attention_tc: head dim %d unsupported (64/128)", c.HD); return -1; }
  if (c.causal && c.n1 > 0) { set_error("attention_tc: causal attention takes one KV segment"); return -1; }
  if ((c.o_stride % 8) != 0) { set_error("attention_tc: output pitch must keep 16 B alignment"); return -1; }
  const uint64_t cols = (uint64_t)c.H * c.HD;
  CUtensorMap tq, tk0, tv0, tk1, tv1;
  if (attn_tmap(&tq, c.q, (uint64_t)c.B * c.Sq, cols, c.q_stride)) return -1;
  if (attn_tmap(&tk0, c.k0, (uint64_t)c.B * c.n0, cols, c.kv0_stride) || attn_tmap(&tv0, c.v0, (uint64_t)c.B * c.n0, cols, c.kv0_stride)) return -1;
  if (c.n1 > 0) {
    if (attn_tmap(&tk1, c.k1, (uint64_t)c.B * c.n1, cols, c.kv1_stride) || attn_tmap(&tv1, c.v1, (uint64_t)c.B * c.n1, cols, c.kv1_stride)) return -1;
  } else {
    tk1 = tk0; tv1 = tv0;
  }
  AttnTcParams p;
  memset(&p, 0, sizeof(p));
  p.Sq = c.Sq; p.n0 = c.n0; p.n1 = c.n1; p.H = c.H; p.sl2 = c.scale * 1.4426950408889634f; p.causal = c.causal; p.kv_start = c.kv_start;
  p.out = c.out; p.o_stride = c.o_stride;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((c.Sq + kAtBQ - 1) / kAtBQ, c.H, c.B); cfg.blockDim = dim3(kAtThreads); cfg.stream = st;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (pdl_enabled()) { attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[na].val.programmaticStreamSerializationAllowed = 1; ++na; }
  cfg.attrs = attr; cfg.numAttrs = na;
  if (c.HD == 64) {
    cfg.dynamicSmemBytes = AttnTcCfg<64>::SMEM_BYTES;
    VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_prefill_tc_kernel<64, false>, tq, tk0, tv0, tk1, tv1, p));
  } else {
    cfg.dynamicSmemBytes = AttnTcCfg<128>::SMEM_BYTES;
    VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_prefill_tc_kernel<128, false>, tq, tk0, tv0, tk1, tv1, p));
  }
  return 0;
}

int attention_paged_partials() { return 3 * num_sms(); }

// Split count of a paged launch: none once the grid covers the SMs; otherwise enough CTAs for two per SM, each with >= 2 key
// tiles of the longest possible sequence.  ctas * splits < 2 * SMs + ctas < attention_paged_partials().
static int paged_kv_splits(int ctas, int max_kv) {
  const int sms = num_sms();
  if (ctas >= sms) return 1;
  const int tiles = (max_kv + kAtBKV - 1) / kAtBKV;
  int s = std::min((2 * sms + ctas - 1) / ctas, (tiles + 1) / 2);
  return std::max(1, std::min(s, kAtMaxKvSplits));
}

int attention_paged(const AttnPagedCall& c, cudaStream_t st, KvFormat fmt) {
  if (attn_tc_init()) return -1;
  if (c.kv.page_tokens < 8 || c.kv.page_tokens > 64 || c.kv.page_tokens % 8 != 0) { set_error("attention_paged: page_tokens %d must be a multiple of 8 <= 64", c.kv.page_tokens); return -1; }
  if (c.B < 1 || c.kv.heads < 1 || c.T < 1 || c.kv.total_pages < 1) { set_error("attention_paged: empty launch"); return -1; }
  if ((c.o_stride % 8) != 0) { set_error("attention_paged: output pitch must keep 16 B alignment"); return -1; }
  if (fmt != KV_BF16 && fmt != KV_INT8) { set_error("attention_paged: KV cache format %d unsupported", (int)fmt); return -1; }
  CUtensorMap tq, tkv;
  if (attn_tmap(&tq, c.q, (uint64_t)c.B * c.T, (uint64_t)c.kv.heads * 128, c.q_stride)) return -1;
  if (fmt == KV_INT8) {
    if (attn_tmap_q8(&tkv, c.kv.pages, c.kv.row<uint64_t>(c.kv.total_pages, 0, 0), c.kv.page_tokens)) return -1;
  } else {
    if (attn_tmap(&tkv, c.kv.pages, c.kv.row<uint64_t>(c.kv.total_pages, 0, 0), 128, 128, c.kv.page_tokens)) return -1;
  }
  const int qt = (c.T + kAtBQ - 1) / kAtBQ, ctas = qt * c.kv.heads * c.B;
  const int splits = paged_kv_splits(ctas, c.max_kv);
  if (splits > 1 && (c.part == nullptr || c.counters == nullptr || (int64_t)ctas * splits > attention_paged_partials())) {
    set_error("attention_paged: split-KV scratch missing or too small"); return -1;
  }
  AttnTcParams p;
  memset(&p, 0, sizeof(p));
  p.Sq = c.T; p.H = c.kv.heads; p.sl2 = c.scale * 1.4426950408889634f; p.causal = 1; p.out = c.out; p.o_stride = c.o_stride;
  p.kv = c.kv; p.base_len = c.base_len;
  p.kv_splits = splits; p.part = c.part; p.counters = c.counters;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(qt, c.kv.heads, c.B * splits); cfg.blockDim = dim3(kAtThreads); cfg.stream = st;
  cfg.dynamicSmemBytes = AttnTcCfg<128>::SMEM_BYTES;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (pdl_enabled()) { attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[na].val.programmaticStreamSerializationAllowed = 1; ++na; }
  cfg.attrs = attr; cfg.numAttrs = na;
  if (fmt == KV_INT8) {
    cfg.dynamicSmemBytes = AttnTcCfg<128>::SMEM_BYTES + kAtStages * kAtQ8ScaleBytes;
    VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_prefill_tc_kernel<128, true, KV_INT8>, tq, tkv, tkv, tkv, tkv, p));
    return 0;
  }
  VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_prefill_tc_kernel<128, true>, tq, tkv, tkv, tkv, tkv, p));
  return 0;
}

}  // namespace vcla
