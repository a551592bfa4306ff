// Decode weight-streaming GEMM with the split-K reduction INSIDE a thread-block cluster (sm_90a).
//
//   out[b, n] = sum_k W[n, k] * x[b, k]        W = nn.Linear weight [N_out, K] (the 128-row wgmma M operand, streamed once from HBM
//                                              through TMA), x = the <= 32 activation rows of the batch (the wgmma N operand)
//
// gemm.cu's swap-AB kernel writes one fp32 partial per K split to an L2 workspace and leaves the reduction to the next kernel
// (dec_resid_norm / dec_silu_mul / the attention prologue): 3 extra kernel boundaries per layer and S x the output in L2 traffic.
// Here the S CTAs that share a 128-row tile form ONE CLUSTER (cluster dims (S,1,1), S <= 8): each CTA accumulates its K slice in
// registers, then the cluster reduce-scatters over the batch columns through distributed shared memory -- CTA r receives, from every
// peer, the columns it owns (st.shared::cluster into its buffer, one remote mbarrier arrive per peer) -- sums them in a fixed
// order (deterministic) and applies the consumer that used to be a kernel of its own:
//   CSK_OUT_F32 : out[b, n]  = rstd[b] * acc                                   (fused QKV projection, lm_head)
//   CSK_RESID   : resid[b,n] += acc ; xw[b,n] = bf16(resid * norm_w[n]) ; ssq[b, tile] = sum_n resid^2     (o_proj, down_proj)
//   CSK_SWIGLU  : h[b, j]    = bf16(silu(rstd[b] * gate) * (rstd[b] * up))      (fused gate/up, rows interleaved [32 gate | 32 up])
// RMSNorm is deferred: operands are xw = bf16(resid * norm_w), the row scale rstd[b] = rsqrt(sum_tiles ssq[b, tile] / D + eps)
// commutes with the GEMM and is applied by the consumer of the NEXT GEMM (a row scalar; bf16's relative rounding is scale free).
// A decode layer is then 5 kernels (QKV, attention, O, gate/up, down) instead of 8.
//
// Reduce buffering (template NBUF): 2 = double buffered (tile t+1's partials may arrive while tile t is being summed; the hand-shake
// is one remote arrive per peer and tile), 1 = one buffer + a second 'consumed' barrier, which frees shared memory for a deeper TMA
// ring.  The 16-column batch tile (B <= 16) runs 3 stages + one reduce buffer (66 KB), small enough for a THIRD CTA per SM: where the
// grid leaves a slot free (o_proj, down_proj: 32 tiles), the next kernel's first CTAs become resident there under PDL and start their
// weight TMAs while this kernel's last tiles reduce and exit; the larger GEMMs deal their tiles evenly over the clusters resident at
// three CTAs per SM (csk_launch).
//
// Per CTA (160 threads): warp 4 = TMA producer (weight tiles are requested BEFORE griddepcontrol.wait: they never depend on the
// previous kernel), warps 0..3 = one wgmma warpgroup: MMAs (2 x m64nBNk16 per k step) -> peers' smem -> reduce -> consumer.
#include "common.cuh"
#include "kernels.h"

#include <algorithm>
#include <mutex>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace vcla {

constexpr int kCskThreads = 160;
constexpr int kCskBlockM = 128;
constexpr int kCskBlockK = 64;
constexpr int kCskMaxSplits = 8;
constexpr int kCskGridSmem = 96 * 1024;   // shared memory per CTA the grid is sized with: two such CTAs fit an SM, three do not

struct CskParams {
  int M, B, K;                 // output features, batch rows, reduction length
  int m_tiles, splits, kb_per_split, kb_total, n_clusters;
  int mode;
  float* out; int ldo;         // OUT_F32: out[b * ldo + n]
  float* resid;                // RESID: [B, M] fp32
  const float* norm_w; bf16* xw; float* ssq_out;   // RESID: [M], [B, M], [B, m_tiles]
  bf16* h;                     // SWIGLU: [B, M / 2]
  const float* ssq_in; int ssq_slots; float inv_dim, eps;   // deferred scale of the operand rows (null: 1)
  uint64_t policy_w, policy_x;
  int cluster_fence;           // explicit fence.acq_rel.cluster before the remote arrive (VCLA_CSK_FENCE=1; the arrive itself is release.cluster)
  const float* wscale;         // Q8: per-row scale of the int8 weight rows
};

// Q8: the weight tile is int8 (64 B rows, no swizzle, k permuted into fragment order, see gemm_csk_kernel), the batch tile stays bf16.
template <int BN, int STAGES, int NBUF, bool Q8 = false>
struct CskCfg {
  static constexpr int A_BYTES = kCskBlockM * kCskBlockK * (Q8 ? 1 : 2);
  static constexpr int B_BYTES = BN * kCskBlockK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int RED_COLS = BN + 4;                                 // >= S * ceil(B / S) (checked at launch)
  static constexpr int RED_BYTES = RED_COLS * kCskBlockM * 4;             // one reduce buffer: [source][owned column][128 rows] fp32
  static constexpr int RED_OFF = STAGES * STAGE_BYTES;
  static constexpr int BAR_OFF = RED_OFF + NBUF * RED_BYTES;        // NBUF = 2: double-buffered reduce; 1: one buffer + a 'consumed' barrier
  static constexpr int MISC_OFF = BAR_OFF + 256;                          // rstd[BN], ssq warp partials [4][BN]
  static constexpr int MISC_BYTES = BN * 20 > 1024 ? BN * 20 : 1024;
  static constexpr int SMEM_BYTES = MISC_OFF + MISC_BYTES + 1024;        // + slack for the 1024 B alignment of the ring
  // CTAs per SM the shared memory allows (228 KB per SM, 1 KB of it reserved per CTA); the launch bound asks for registers to match
  static constexpr int CTAS_PER_SM = 3 * (SMEM_BYTES + 1024) <= 228 * 1024 ? 3 : 2;
  static_assert(STAGE_BYTES % 1024 == 0, "stage must keep 1024 B alignment for SWIZZLE_128B");
  static_assert(BN == 16 || BN == 32 || (Q8 && BN == 64), "decode batch tile");
};

__device__ __forceinline__ uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ uint32_t mapa_u32(uint32_t local, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster_f32(uint32_t addr, float v) { asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory"); }
__device__ __forceinline__ void mbar_arrive_remote(uint32_t cluster_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait_cluster(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait_cluster(bar, parity)) return;
  long long t0 = clock64();
  while (!mbar_try_wait_cluster(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();   // no printf: a call anywhere in the kernel serialises its wgmma
  }
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Two bytes of an int8 word -> bf16x2, exactly: byte + 128 is placed in the mantissa of 2^23 and the bias subtracted in fp32.
__device__ __forceinline__ uint32_t i8x2_to_bf16x2(uint32_t biased, uint32_t sel_lo, uint32_t sel_hi) {
  const float lo = __int_as_float((int)__byte_perm(biased, 0x4B000000u, sel_lo)) - 8388736.f;
  const float hi = __int_as_float((int)__byte_perm(biased, 0x4B000000u, sel_hi)) - 8388736.f;
  return pack_bf16x2(lo, hi);
}

// Q8 = true: W is int8 with one fp32 scale per row (weight-only int8).  Each 64-column k-block of a weight row is stored in fragment
// order: byte 16 q + 4 s + j holds column 16 s + 2 q + {0, 1, 8, 9}[j], so the 16 bytes at offset 16 (lane % 4) of a row are exactly the
// A-fragment elements the thread needs for the four k16 steps (one 16-byte shared-memory load per row).  They are converted to bf16 in
// registers (int8 is exact in bf16) and fed to register-A wgmma; the row scale commutes with the contraction and is applied after the
// cluster reduction.
template <int BN, int STAGES, int NBUF, bool Q8 = false>
__global__ void __launch_bounds__(kCskThreads, CskCfg<BN, STAGES, NBUF, Q8>::CTAS_PER_SM)
gemm_csk_kernel(const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmX, const CskParams p) {
  using C = CskCfg<BN, STAGES, NBUF, Q8>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t bar0 = base + C::BAR_OFF;
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (STAGES + s); };
  auto red_bar = [&](int b) { return bar0 + 8u * (2 * STAGES + b); };
  float* s_rstd = reinterpret_cast<float*>(base_ptr + C::MISC_OFF);                 // [BN]
  float* s_part = s_rstd + BN;                                                       // [4][BN] warp partial sums of squares

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int S = p.splits;
  const int rank = (int)cluster_ctarank();
  const int cluster_id = blockIdx.x / S;
  TraceScope trace(1);

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), 1); }
    for (int b = 0; b < 2; ++b) mbar_init(red_bar(b), (uint32_t)S);            // one arrive per source CTA (this one included)
    fence_barrier_init();
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmX);
  }
  __syncthreads();
  // Cluster rendezvous, split: everybody ARRIVES now (this CTA's barriers are initialised), only the MMA / epilogue warps WAIT, right
  // before their first remote access -- the TMA producer starts streaming weights without waiting for the peers to become resident.
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");

  pdl_launch_dependents();

  const int kb0 = rank * p.kb_per_split;
  const int kb1 = min(p.kb_total, kb0 + p.kb_per_split);

  if (warp == 4) {
    if (lane == 0) {
      // ===================== TMA producer =====================
      int stage = 0; uint32_t phase = 0;
      bool dep_ready = false;
      int npend = 0;
      uint32_t pend_dst[STAGES], pend_bar[STAGES]; int pend_c0[STAGES];
      auto flush_pending = [&]() {
        pdl_wait();
        for (int i = 0; i < npend; ++i) tma_load_2d(pend_dst[i], &tmX, pend_c0[i], 0, pend_bar[i], p.policy_x);
        npend = 0;
        dep_ready = true;
      };
      for (int t = cluster_id; t < p.m_tiles; t += p.n_clusters) {
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait_mma(empty_bar(stage), phase ^ 1u);
          mbar_arrive_expect_tx(full_bar(stage), C::STAGE_BYTES);
          const uint32_t sa = base + stage * C::STAGE_BYTES;
          tma_load_2d(sa, &tmW, kb * kCskBlockK, t * kCskBlockM, full_bar(stage), p.policy_w);          // weights: no dependency
          if (dep_ready) {
            tma_load_2d(sa + C::A_BYTES, &tmX, kb * kCskBlockK, 0, full_bar(stage), p.policy_x);
          } else {
            pend_dst[npend] = sa + C::A_BYTES; pend_bar[npend] = full_bar(stage); pend_c0[npend] = kb * kCskBlockK; ++npend;
            if (npend == STAGES) flush_pending();
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
      if (!dep_ready) flush_pending();
    }
    __syncwarp();
  } else {
    // ===================== wgmma warpgroup: MMAs -> reduce-scatter over the cluster -> consumer =====================
    const int q = warp;
    const int row_in_tile = q * 32 + lane;          // this thread's row in the reduce / consumer phase
    const int et = row_in_tile;                     // 0..127 inside the warpgroup
    const int fr = warp * 16 + (lane >> 2), fc = 2 * (lane & 3);   // accumulator fragment: rows fr (+8) of each 64-row block
    const int cols_per = (p.B + S - 1) / S;         // batch columns owned by one CTA
    const int my_c0 = rank * cols_per;
    const int my_nc = max(0, min(cols_per, p.B - my_c0));
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");   // every peer's reduce barriers exist from here on
    pdl_wait();                                     // everything below reads / writes buffers of the previous kernels
    trace.dep();                                    // (the trace slot belongs to thread 0, a thread of this warpgroup)
    // deferred RMSNorm scale of the operand rows
    for (int b = warp; b < BN; b += 4) {
      float v = 1.f;
      if (p.ssq_in != nullptr && b < p.B) {
        float ss = 0.f;
        for (int i = lane; i < p.ssq_slots; i += 32) ss += __ldcg(p.ssq_in + (size_t)b * p.ssq_slots + i);
        ss = warp_sum(ss);
        v = rsqrtf(ss * p.inv_dim + p.eps);
      }
      if (lane == 0) s_rstd[b] = v;
    }
    asm volatile("bar.sync 1, 128;" ::: "memory");

    int stage = 0; uint32_t phase = 0;
    int buf = 0; uint32_t redphase[2] = {0u, 0u};
    float acc[2][BN / 2];
    // NBUF == 1: red_bar(1) counts, per tile, the S destinations that have consumed what this CTA delivered ("your slot in my buffer
    // is free again"); the scatter of the next tile waits for it.  A deeper TMA ring fits in the shared memory this saves.
    uint32_t freephase = 0u; bool first_tile = true;
    for (int t = cluster_id; t < p.m_tiles; t += p.n_clusters) {
      const bool last_tile = t + p.n_clusters >= p.m_tiles;
      int prev = -1;
      if constexpr (Q8) {
        // One register set of A fragments: each k-block's MMAs are waited for before the next k-block is converted.  Two sets used
        // alternately with one MMA group in flight make ptxas serialise every wgmma (C7513: non-wgmma instructions define wgmma
        // input registers inside the pipeline stage), which is slower still.
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait_mma(full_bar(stage), phase);
          const uint32_t sa = base + stage * C::STAGE_BYTES;
          const uint64_t bdesc = make_desc_sw128(sa + C::A_BYTES);
          const uint8_t* tile = base_ptr + stage * C::STAGE_BYTES;
          uint32_t a[2][4][4];                        // [64-row block][k16 step][fragment register]
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int h2 = 0; h2 < 2; ++h2) {
              const uint4 v = *reinterpret_cast<const uint4*>(tile + (h * 64 + fr + 8 * h2) * kCskBlockK + 16 * (lane & 3));
              const uint32_t w[4] = {v.x ^ 0x80808080u, v.y ^ 0x80808080u, v.z ^ 0x80808080u, v.w ^ 0x80808080u};
#pragma unroll
              for (int s = 0; s < 4; ++s) {
                a[h][s][h2] = i8x2_to_bf16x2(w[s], 0x7540u, 0x7541u);
                a[h][s][2 + h2] = i8x2_to_bf16x2(w[s], 0x7542u, 0x7543u);
              }
            }
          }
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < kCskBlockK / 16; ++k) {
#pragma unroll
            for (int h = 0; h < 2; ++h) wgmma_bf16_rs<BN>(acc[h], a[h][k], bdesc + 2u * k, (kb > kb0 || k > 0) ? 1 : 0);
          }
          wgmma_commit();
          wgmma_wait<0>();                          // the A registers are rewritten by the next k-block
          fence_regs(acc[0]);
          fence_regs(acc[1]);
          if (threadIdx.x == 0) mbar_arrive(empty_bar(stage));
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      } else {
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait_mma(full_bar(stage), phase);
        const uint32_t sa = base + stage * C::STAGE_BYTES;
        const uint64_t bdesc = make_desc_sw128(sa + C::A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kCskBlockK / 16; ++k) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
            wgmma_bf16<BN>(acc[h], make_desc_sw128(sa + h * 64 * 128) + 2u * k, bdesc + 2u * k, (kb > kb0 || k > 0) ? 1 : 0);
        }
        wgmma_commit();
        wgmma_wait<1>();                            // the previous k-block's MMAs are done reading their stage
        if (prev >= 0 && threadIdx.x == 0) mbar_arrive(empty_bar(prev));
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      fence_regs(acc[0]);
      fence_regs(acc[1]);
      if (prev >= 0 && threadIdx.x == 0) mbar_arrive(empty_bar(prev));
      }
      if constexpr (NBUF == 1) {
        if (!first_tile) { mbar_wait_cluster(red_bar(1), freephase); freephase ^= 1u; }
        first_tile = false;
      }
      // scatter: column c of this partial goes to CTA c / cols_per, slot [source = rank][c % cols_per][row]
      const uint32_t red_local = base + C::RED_OFF + (uint32_t)buf * C::RED_BYTES;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
          const int r = h * 64 + fr + 8 * h2;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int c = 8 * j + fc + e;
              if (c < p.B) {
                const int dst = c / cols_per, cl = c - dst * cols_per;
                const uint32_t off = (uint32_t)(((rank * cols_per + cl) * kCskBlockM + r) * 4);
                st_cluster_f32(mapa_u32(red_local + off, (uint32_t)dst), acc[h][4 * j + 2 * h2 + e]);
              }
            }
          }
        }
      }
      if (p.cluster_fence) asm volatile("fence.acq_rel.cluster;" ::: "memory");
      asm volatile("bar.sync 1, 128;" ::: "memory");              // all 128 rows of this CTA's partial are written
      if (et < S) mbar_arrive_remote(mapa_u32(red_bar(buf), (uint32_t)et));   // release.cluster: publishes them to CTA `et`
      // gather: wait until all S sources have delivered the columns this CTA owns
      mbar_wait_cluster(red_bar(buf), redphase[buf]);
      redphase[buf] ^= 1u;
      const float* red = reinterpret_cast<const float*>(base_ptr + C::RED_OFF + (size_t)buf * C::RED_BYTES);
      const int row = t * kCskBlockM + row_in_tile;               // output feature
      const bool row_ok = row < p.M;

      if (p.mode == CSK_SWIGLU) {
        // tile rows = [32 gate | 32 up | 32 gate | 32 up]: reduce, park the sums in the (now consumed) source-0 slice, pair them up
        float* park = const_cast<float*>(red);                    // [cl][128] of source 0
        for (int cl = 0; cl < my_nc; ++cl) {
          float sum = 0.f;
          for (int s = 0; s < S; ++s) sum += red[(size_t)((s * cols_per + cl) * kCskBlockM) + row_in_tile];   // fixed order
          if constexpr (Q8) sum *= row_ok ? __ldg(p.wscale + row) : 0.f;
          park[(size_t)cl * kCskBlockM + row_in_tile] = sum;      // source 0's value of this element was read by this thread only
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (et < 64) {
          const int blk = et >> 5, gi = et & 31;
          const int grow = t * kCskBlockM + blk * 64 + gi;        // gate row; up row = grow + 32
          const int jout = t * 64 + blk * 32 + gi;                // output feature
          if (grow + 32 < p.M) {
            for (int cl = 0; cl < my_nc; ++cl) {
              const int b = my_c0 + cl;
              const float rs = s_rstd[b];
              const float g = park[(size_t)cl * kCskBlockM + blk * 64 + gi] * rs, u = park[(size_t)cl * kCskBlockM + blk * 64 + 32 + gi] * rs;
              p.h[(size_t)b * (p.M >> 1) + jout] = __float2bfloat16(g / (1.f + __expf(-g)) * u);
            }
          }
        }
        asm volatile("bar.sync 1, 128;" ::: "memory");            // park is part of the buffer the peers rewrite two tiles later
      } else {
        for (int cl = 0; cl < my_nc; ++cl) {
          const int b = my_c0 + cl;
          float sum = 0.f;
          for (int s = 0; s < S; ++s) sum += red[(size_t)((s * cols_per + cl) * kCskBlockM) + row_in_tile];   // fixed order
          if constexpr (Q8) sum *= row_ok ? __ldg(p.wscale + row) : 0.f;
          if (p.mode == CSK_OUT_F32) {
            if (row_ok) p.out[(size_t)b * p.ldo + row] = sum * s_rstd[b];
          } else {   // CSK_RESID
            float r = 0.f;
            if (row_ok) {
              r = p.resid[(size_t)b * p.M + row] + sum;
              p.resid[(size_t)b * p.M + row] = r;
              p.xw[(size_t)b * p.M + row] = __float2bfloat16(r * __ldg(p.norm_w + row));
            }
            const float q2 = warp_sum(r * r);
            if (lane == 0) s_part[q * BN + cl] = q2;
          }
        }
        if (p.mode == CSK_RESID) {
          asm volatile("bar.sync 1, 128;" ::: "memory");
          if (et < my_nc) p.ssq_out[(size_t)(my_c0 + et) * p.m_tiles + t] = s_part[et] + s_part[BN + et] + s_part[2 * BN + et] + s_part[3 * BN + et];
          asm volatile("bar.sync 1, 128;" ::: "memory");          // s_part is reused by the next tile
        }
      }
      if constexpr (NBUF == 1) {
        // every thread of this CTA is done reading the buffer: tell the S sources (never after the last tile: a peer may be gone)
        asm volatile("bar.sync 1, 128;" ::: "memory");
        if (!last_tile && et < S) mbar_arrive_remote(mapa_u32(red_bar(1), (uint32_t)et));
      } else {
        buf ^= 1;
      }
    }
  }

  // No closing cluster barrier: a CTA leaves its last reduce only after all S peers have delivered (and arrived on) its buffer, i.e.
  // nobody addresses its shared memory afterwards, and every peer it wrote to is still waiting for exactly that delivery.
  __syncthreads();
  trace.done();
}

VCLA_DEFINE_TRACE_SETTER(trace_set_gemm_decode)

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled g_csk_encode = nullptr;
static std::once_flag g_csk_once;
static int g_csk_rc = 0;

static int csk_init() {
  std::call_once(g_csk_once, [] {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess || fn == nullptr) {
      set_error("cuTensorMapEncodeTiled not available"); g_csk_rc = -1; return;
    }
    g_csk_encode = reinterpret_cast<PFN_encodeTiled>(fn);
    // two or three CTAs per SM need (almost) the whole 228 KB of an SM as shared memory: ask for the maximum carve-out explicitly (the
    // occupancy query for cluster launches otherwise assumes a carve-out that holds only one CTA).  The opt-in covers kCskGridSmem, the
    // footprint csk_max_clusters sizes the grid with.
    auto prep = [](const void* fn, int bytes) {
      return cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, std::max(bytes, kCskGridSmem)) == cudaSuccess &&
             cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared) == cudaSuccess;
    };
    if (!prep((const void*)gemm_csk_kernel<16, 3, 1>, CskCfg<16, 3, 1>::SMEM_BYTES) || !prep((const void*)gemm_csk_kernel<32, 3, 2>, CskCfg<32, 3, 2>::SMEM_BYTES) ||
        !prep((const void*)gemm_csk_kernel<32, 4, 1>, CskCfg<32, 4, 1>::SMEM_BYTES) ||
        !prep((const void*)gemm_csk_kernel<16, 8, 2, true>, CskCfg<16, 8, 2, true>::SMEM_BYTES) ||
        !prep((const void*)gemm_csk_kernel<32, 6, 2, true>, CskCfg<32, 6, 2, true>::SMEM_BYTES) ||
        !prep((const void*)gemm_csk_kernel<64, 4, 1, true>, CskCfg<64, 4, 1, true>::SMEM_BYTES)) {
      set_error("gemm_csk: cudaFuncSetAttribute failed: %s", cudaGetErrorString(cudaGetLastError())); g_csk_rc = -1;
    }
  });
  return g_csk_rc;
}

// int8 = true: a byte matrix in plain (unswizzled) 64 B rows, the layout the Q8 kernel's fragment loads expect
static int csk_tmap(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows, bool int8 = false) {
  const uint64_t esz = int8 ? 1 : 2;
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (ld * esz) % 16 != 0) { set_error("gemm_csk: TMA operand alignment"); return -1; }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * esz};
  cuuint32_t box[2] = {(cuuint32_t)kCskBlockK, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_csk_encode(m, int8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, int8 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("gemm_csk: cuTensorMapEncodeTiled failed (%d)", (int)r); return -1; }
  return 0;
}

// Upper bound on the clusters of S CTAs per launch, cached per (BN, S); csk_pick's split counts are chosen from it.  The query is asked
// about a CTA of at least kCskGridSmem bytes of shared memory, which admits two per SM, so a configuration small enough for a third CTA
// gets the bound (and hence the split counts, which fix the summation order) of the two-per-SM configurations.
template <int BN, int STAGES, int NBUF, bool Q8 = false>
static int csk_max_clusters(int S) {
  static int cache[kCskMaxSplits + 1] = {0};
  if (cache[S] != 0) return cache[S];
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(S * 64); cfg.blockDim = dim3(kCskThreads);
  cfg.dynamicSmemBytes = std::max(CskCfg<BN, STAGES, NBUF, Q8>::SMEM_BYTES, kCskGridSmem);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = S; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, gemm_csk_kernel<BN, STAGES, NBUF, Q8>, &cfg) != cudaSuccess || n <= 0) {
    (void)cudaGetLastError();
    n = (2 * num_sms()) / S * 3 / 4;                 // conservative fallback
    if (n < 1) n = 1;
  }
  // The cluster occupancy query counts ONE CTA per SM on this driver even when two fit (shared memory, registers and the plain
  // per-SM occupancy query all allow 2): scale by the per-SM block occupancy, capped at 2 (the launch bound).
  int per_sm = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gemm_csk_kernel<BN, STAGES, NBUF, Q8>, kCskThreads, CskCfg<BN, STAGES, NBUF, Q8>::SMEM_BYTES) != cudaSuccess) { (void)cudaGetLastError(); per_sm = 1; }
  if (per_sm > 2) per_sm = 2;
  // Both occupancy queries may answer 1 block per SM for this cluster launch while the kernel is sized for 2 CTAs per SM (launch
  // bound, <= 113 KB of shared memory each), so that is what the launch assumes; VCLA_CSK_OCC=1 restores the query's answer.
  int mult = 2;
  if (const char* e = getenv("VCLA_CSK_OCC")) { const int v = atoi(e); if (v >= 1 && v <= 2) mult = v; }
  if (getenv("VCLA_DEBUG")) fprintf(stderr, "[vcla] gemm_csk<%d,%d,%d%s> S=%d: cluster query %d, blocks/SM %d, using x%d\n", BN, STAGES, NBUF, Q8 ? ",q8" : "", S, n, per_sm, mult);
  n *= mult;
  cache[S] = n;
  return n;
}

// clusters of S CTAs the cluster occupancy query finds co-resident at the configuration's own shared memory, cached per (BN, S)
template <int BN, int STAGES, int NBUF, bool Q8 = false>
static int csk_resident_clusters(int S) {
  static int cache[kCskMaxSplits + 1] = {0};
  if (cache[S] != 0) return cache[S];
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(S * 64); cfg.blockDim = dim3(kCskThreads);
  cfg.dynamicSmemBytes = CskCfg<BN, STAGES, NBUF, Q8>::SMEM_BYTES;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = S; attr[0].val.clusterDim.y = 1; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  int n = 0;
  if (cudaOccupancyMaxActiveClusters(&n, gemm_csk_kernel<BN, STAGES, NBUF, Q8>, &cfg) != cudaSuccess || n <= 0) {
    (void)cudaGetLastError();
    n = (2 * num_sms()) / S;                         // two CTAs per SM
    if (n < 1) n = 1;
  }
  if (getenv("VCLA_DEBUG")) fprintf(stderr, "[vcla] gemm_csk<%d,%d,%d%s> S=%d: %d clusters resident\n", BN, STAGES, NBUF, Q8 ? ",q8" : "", S, n);
  cache[S] = n;
  return n;
}

template <int BN, int STAGES, int NBUF, bool Q8 = false>
static int csk_launch(const CskCall& c, CskParams p, cudaStream_t st) {
  CUtensorMap tw, tx;
  if (Q8 ? csk_tmap(&tw, c.Wq, c.M, c.K, c.K, kCskBlockM, true) : csk_tmap(&tw, c.W, c.M, c.K, c.K, kCskBlockM)) return -1;
  if (csk_tmap(&tx, c.X, c.B, c.K, c.K, BN)) return -1;
  int ncl = csk_max_clusters<BN, STAGES, NBUF, Q8>(p.splits);
  if (ncl > p.m_tiles) ncl = p.m_tiles;
  if constexpr (CskCfg<BN, STAGES, NBUF, Q8>::CTAS_PER_SM == 3) {
    // Tiles are dealt to clusters round-robin (t = cluster, cluster + n_clusters, ...), and clusters beyond those resident start only
    // when a resident one exits: with more clusters than fit at once, the late ones run their whole share in a tail of their own.
    // Deal the tiles evenly over the rounds the resident clusters need instead.  Which cluster reduces a tile changes no arithmetic.
    const int res = std::min(ncl, csk_resident_clusters<BN, STAGES, NBUF, Q8>(p.splits));
    const int rounds = (p.m_tiles + res - 1) / res;
    ncl = (p.m_tiles + rounds - 1) / rounds;
  }
  p.n_clusters = ncl;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(ncl * p.splits); cfg.blockDim = dim3(kCskThreads); cfg.dynamicSmemBytes = CskCfg<BN, STAGES, NBUF, Q8>::SMEM_BYTES; cfg.stream = st;
  cudaLaunchAttribute attr[2];
  int na = 0;
  attr[na].id = cudaLaunchAttributeClusterDimension;
  attr[na].val.clusterDim.x = p.splits; attr[na].val.clusterDim.y = 1; attr[na].val.clusterDim.z = 1;
  ++na;
  if (pdl_enabled()) { attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[na].val.programmaticStreamSerializationAllowed = 1; ++na; }
  cfg.attrs = attr; cfg.numAttrs = na;
  VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, gemm_csk_kernel<BN, STAGES, NBUF, Q8>, tw, tx, p));
  return 0;
}

// Configurations: batch <= 16 (16-column tile): 3 TMA stages + one reduce buffer (three CTAs fit per SM, see the top of this file);
// batch 17..32 (32-column tile): ONE buffer + 'consumed' barrier, which frees the shared memory for a 4th TMA stage, or with
// VCLA_CSK_NBUF = 2 a double-buffered reduce + 3 stages.
static bool csk_double_buffered_32() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("VCLA_CSK_NBUF"); v = e != nullptr ? atoi(e) : 0; }
  return v == 2;
}

// int8 weights: half the A stage, so every batch tile is double buffered with a deeper ring, and batches 33..64 get a 64-column tile
static int csk_q8_bn(int B) { return B <= 16 ? 16 : (B <= 32 ? 32 : 64); }

int gemm_csk_clusters(int B, int splits, bool q8) {
  if (csk_init()) return -1;
  if (splits < 1 || splits > kCskMaxSplits) return -1;
  if (q8) {
    const int bn = csk_q8_bn(B);
    return bn == 16 ? csk_max_clusters<16, 8, 2, true>(splits) : bn == 32 ? csk_max_clusters<32, 6, 2, true>(splits) : csk_max_clusters<64, 4, 1, true>(splits);
  }
  if (B <= 16) return csk_max_clusters<16, 3, 1>(splits);
  return csk_double_buffered_32() ? csk_max_clusters<32, 3, 2>(splits) : csk_max_clusters<32, 4, 1>(splits);
}

template <int BN, int STAGES, int NBUF, bool Q8 = false>
static int csk_ctas_per_sm() {
  int n = 0;
  const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, gemm_csk_kernel<BN, STAGES, NBUF, Q8>, kCskThreads, CskCfg<BN, STAGES, NBUF, Q8>::SMEM_BYTES);
  if (e != cudaSuccess) { set_error("gemm_csk_ctas_per_sm: %s", cudaGetErrorString(e)); (void)cudaGetLastError(); return -1; }
  return n;
}

int gemm_csk_ctas_per_sm(int B, bool q8) {
  if (csk_init()) return -1;
  if (q8) {
    const int bn = csk_q8_bn(B);
    return bn == 16 ? csk_ctas_per_sm<16, 8, 2, true>() : bn == 32 ? csk_ctas_per_sm<32, 6, 2, true>() : csk_ctas_per_sm<64, 4, 1, true>();
  }
  if (B <= 16) return csk_ctas_per_sm<16, 3, 1>();
  return csk_double_buffered_32() ? csk_ctas_per_sm<32, 3, 2>() : csk_ctas_per_sm<32, 4, 1>();
}

int gemm_csk(const CskCall& c, cudaStream_t st) {
  if (csk_init()) return -1;
  if (c.M <= 0 || c.B <= 0 || c.K <= 0 || c.K % 8 != 0) { set_error("gemm_csk: bad problem (M %d B %d K %d)", c.M, c.B, c.K); return -1; }
  const bool q8 = c.Wq != nullptr;
  if (q8 && (c.wscale == nullptr || c.K % kCskBlockK != 0)) { set_error("gemm_csk: int8 weights need row scales and K %% 64 == 0 (K %d)", c.K); return -1; }
  if (c.B > (q8 ? 64 : 32)) { set_error("gemm_csk: batch %d > %d (use the split-K workspace path)", c.B, q8 ? 64 : 32); return -1; }
  if (c.splits < 1 || c.splits > kCskMaxSplits) { set_error("gemm_csk: splits %d unsupported (1..%d)", c.splits, kCskMaxSplits); return -1; }
  CskParams p;
  memset(&p, 0, sizeof(p));
  p.M = c.M; p.B = c.B; p.K = c.K;
  p.m_tiles = (c.M + kCskBlockM - 1) / kCskBlockM;
  p.kb_total = (c.K + kCskBlockK - 1) / kCskBlockK;
  p.kb_per_split = (p.kb_total + c.splits - 1) / c.splits;
  p.splits = (p.kb_total + p.kb_per_split - 1) / p.kb_per_split;
  if (p.splits != c.splits) { set_error("gemm_csk: split count %d not realisable for %d k-blocks (use %d)", c.splits, p.kb_total, p.splits); return -1; }
  p.mode = c.mode; p.out = c.out; p.ldo = c.ldo; p.resid = c.resid; p.norm_w = c.norm_w; p.xw = c.xw; p.ssq_out = c.ssq_out; p.h = c.h;
  p.ssq_in = c.ssq_in; p.ssq_slots = c.ssq_slots; p.inv_dim = c.inv_dim; p.eps = c.eps;
  p.policy_w = kEvictFirst; p.policy_x = kEvictLast;
  { static int fence = -1; if (fence < 0) { const char* e = getenv("VCLA_CSK_FENCE"); fence = e ? atoi(e) : 0; } p.cluster_fence = fence; }
  p.wscale = c.wscale;
  if (c.mode == CSK_OUT_F32 && (!c.out || c.ldo < c.M)) { set_error("gemm_csk: OUT_F32 needs out / ldo"); return -1; }
  if (c.mode == CSK_RESID && (!c.resid || !c.norm_w || !c.xw || !c.ssq_out)) { set_error("gemm_csk: RESID needs resid / norm_w / xw / ssq_out"); return -1; }
  if (c.mode == CSK_SWIGLU && (!c.h || (c.M % 64) != 0)) { set_error("gemm_csk: SWIGLU needs h and rows %% 64 == 0"); return -1; }
  {
    const int cols_per = (c.B + p.splits - 1) / p.splits, bn = q8 ? csk_q8_bn(c.B) : (c.B <= 16 ? 16 : 32);
    if (cols_per * p.splits > bn + 4) { set_error("gemm_csk: %d splits of batch %d need %d reduce columns (max %d)", p.splits, c.B, cols_per * p.splits, bn + 4); return -1; }
  }
  if (q8) {
    const int bn = csk_q8_bn(c.B);
    return bn == 16 ? csk_launch<16, 8, 2, true>(c, p, st) : bn == 32 ? csk_launch<32, 6, 2, true>(c, p, st) : csk_launch<64, 4, 1, true>(c, p, st);
  }
  if (c.B <= 16) return csk_launch<16, 3, 1>(c, p, st);
  return csk_double_buffered_32() ? csk_launch<32, 3, 2>(c, p, st) : csk_launch<32, 4, 1>(c, p, st);
}

}  // namespace vcla
