// wgmma GEMM for sm_90a:  D[M,N] = A[M,K] * B[N,K]^T, bf16 operands, fp32 accumulation in registers.
//
// One kernel template serves the whole path:
//   * prefill / ViT / Resampler / projector: A = activations (tokens are the wgmma M dimension),
//     B = nn.Linear weight [N_out, K]; fused epilogues: bias, quick_gelu / erf-gelu, fp32 residual add
//     with output-row remap (+ position-embedding table), SwiGLU, deferred RMSNorm, RoPE + KV-cache append.
//   * decode ("swap-AB"): A = weight [N_out, K] (streamed once from HBM through TMA), B = the few
//     activation rows [batch_pad, K]; split-K partials are written to an fp32 workspace that the
//     next (fused consumer) kernel reduces in a fixed order, so results are deterministic.
//
// Structure (per CTA, 160 threads): warp 4 lane 0 = TMA producer, warps 0..3 = one wgmma warpgroup that issues the
// MMAs (BM / 64 blocks of m64nBNk16 per 16-wide k step) and then runs the epilogue straight from its accumulator registers.
// smem ring of STAGES x {A BMx64, B BNx64} tiles in the 128B-swizzled K-major layout that both TMA and the wgmma
// shared-memory descriptors understand; the producer keeps filling the ring for the next tile while the epilogue runs.
// Persistent: each CTA walks tiles blockIdx.x, +gridDim.x, ...
#include "common.cuh"
#include "kernels.h"

#include <mutex>
#include <stdarg.h>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>

namespace vcla {

// ------------------------------------------------------------------------------------------------
// error / device info plumbing shared by all translation units
// ------------------------------------------------------------------------------------------------
static thread_local char g_err[1024] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }
int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}
static bool g_pdl = false;
bool pdl_enabled() { return g_pdl; }
void set_pdl(bool on) { g_pdl = on; }

// ------------------------------------------------------------------------------------------------
// kernel
// ------------------------------------------------------------------------------------------------
struct GemmParams {
  int M, N, K;
  int m_tiles, n_tiles, splits, kb_per_split, kb_total, total_tiles;
  int mode, act, accumulate;
  void* out;
  int ldo;
  const float* bias;
  const float* rowtab;
  int rowtab_period;
  int rows_per_group, group_stride, row_offset;
  int ws_rows;
  int l2_prefetch_kb;
  uint64_t policy_a, policy_b;
  GemmRowScale rowscale;
  GemmEmitNorm emit;
  GemmRope rope;
  const float* colscale;
};

constexpr int kBlockK = 64;
constexpr int kGemmThreads = 160;   // warps 0..3 = the wgmma warpgroup (MMA + epilogue), warp 4 = TMA producer
constexpr int kSwapBlockM = 128;    // swap-AB tiles: 128 weight rows (the two 64-row wgmma blocks of one warpgroup)

// BM x BN tile, BM / 64 wgmma row blocks; the accumulators take BM * BN / 128 fp32 registers per thread (<= 128)
template <int BM, int BN, int STAGES>
struct GemmCfg {
  static constexpr int MH = BM / 64;
  static constexpr int A_BYTES = BM * kBlockK * 2;
  static constexpr int B_BYTES = BN * kBlockK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int BAR_OFF = STAGES * STAGE_BYTES;
  static constexpr int SMEM_BYTES = BAR_OFF + 256 + 1024;   // barriers, + slack for 1024 B alignment
  static_assert(STAGE_BYTES % 1024 == 0, "stage must keep 1024 B alignment for SWIZZLE_128B");
  static_assert(BM == 64 || BM == 128, "tile rows");
  static_assert(BN % 16 == 0 && BN >= 16 && BN <= 256 && BM * BN <= 64 * 256, "wgmma N constraint / accumulator registers");
};

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == ACT_QUICK_GELU) return x / (1.f + __expf(-1.702f * x));
  if (act == ACT_GELU_ERF) return 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
  return x;
}

// KVF = KV_INT8 (the fused QKV epilogue of an int8 KV cache only): every k / v head row is quantised (kernels.h: KvPool), its q and
// s go to the cache and bf16(q * s) to the k / v columns of the output, so the prefill attention reads what the cache holds.
template <int BM, int BN, int STAGES, bool SWAP, int KVF = KV_BF16>
__global__ void __launch_bounds__(kGemmThreads, SWAP ? 2 : 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  using C = GemmCfg<BM, BN, STAGES>;
  constexpr int MH = C::MH;
  static_assert(!SWAP || BM == kSwapBlockM, "swap-AB tiles are 128 weight rows");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar0 = base + C::BAR_OFF;
  auto full_bar = [&](int s) { return bar0 + 8u * s; };
  auto empty_bar = [&](int s) { return bar0 + 8u * (STAGES + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  TraceScope trace(SWAP ? 1 : 2);

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 1);
    }
    fence_barrier_init();
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
  }
  __syncthreads();

  // PDL: let the next kernel's CTAs become resident as soon as ours are (they only prefetch read-only weights and
  // then block in griddepcontrol.wait until this grid has completed), see the producer below.
  pdl_launch_dependents();

  auto tile_coords = [&](int t, int& m_blk, int& n_blk, int& kb0, int& kb1, int& ks) {
    m_blk = t % p.m_tiles;
    int r = t / p.m_tiles;
    n_blk = r % p.n_tiles;
    ks = r / p.n_tiles;
    kb0 = ks * p.kb_per_split;
    kb1 = min(p.kb_total, kb0 + p.kb_per_split);
  };

  if (warp == 4) {
    if (lane == 0) {
      // ===================== TMA producer =====================
      // The weight operand (A when swap-AB, else B) never depends on the previous kernel, so its tiles for the first
      // STAGES pipeline slots are requested BEFORE griddepcontrol.wait: weight streaming from HBM continues across
      // kernel boundaries.  The activation operand is loaded only after the dependency has resolved.
      int stage = 0;
      uint32_t phase = 0;
      bool dep_ready = false;
      int npend = 0;
      uint32_t pend_dst[STAGES], pend_bar[STAGES];
      int pend_c0[STAGES], pend_c1[STAGES];
      const CUtensorMap* act_map = SWAP ? &tmB : &tmA;
      const uint64_t act_policy = SWAP ? p.policy_b : p.policy_a;
      auto flush_pending = [&]() {
        pdl_wait();
        for (int i = 0; i < npend; ++i) tma_load_2d(pend_dst[i], act_map, pend_c0[i], pend_c1[i], pend_bar[i], act_policy);
        npend = 0;
        dep_ready = true;
      };
      for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
        int m_blk, n_blk, kb0, kb1, ks;
        tile_coords(t, m_blk, n_blk, kb0, kb1, ks);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait_mma(empty_bar(stage), phase ^ 1u);
          const uint32_t sa = base + stage * C::STAGE_BYTES;
          mbar_arrive_expect_tx(full_bar(stage), C::STAGE_BYTES);
          if constexpr (SWAP) {
            tma_load_2d(sa, &tmA, kb * kBlockK, m_blk * BM, full_bar(stage), p.policy_a);           // weights
            if (dep_ready) {
              tma_load_2d(sa + C::A_BYTES, &tmB, kb * kBlockK, n_blk * BN, full_bar(stage), p.policy_b);
            } else {
              pend_dst[npend] = sa + C::A_BYTES; pend_bar[npend] = full_bar(stage); pend_c0[npend] = kb * kBlockK; pend_c1[npend] = n_blk * BN; ++npend;
            }
          } else {
            tma_load_2d(sa + C::A_BYTES, &tmB, kb * kBlockK, n_blk * BN, full_bar(stage), p.policy_b);   // weights
            if (dep_ready) {
              tma_load_2d(sa, &tmA, kb * kBlockK, m_blk * BM, full_bar(stage), p.policy_a);
            } else {
              pend_dst[npend] = sa; pend_bar[npend] = full_bar(stage); pend_c0[npend] = kb * kBlockK; pend_c1[npend] = m_blk * BM; ++npend;
            }
          }
          if (!dep_ready && npend == STAGES) {
            // The smem ring is full and the dependency is (probably) still unresolved: HBM would idle while the small
            // consumer kernel in front of us runs.  Pull this CTA's NEXT weight tiles into L2 so the main loop
            // streams them from L2 afterwards.
            if (p.l2_prefetch_kb > 0) {
              int budget = p.l2_prefetch_kb;
              int kbn = kb + 1;
              for (int t2 = t; t2 < p.total_tiles && budget > 0; t2 += gridDim.x) {
                int m2, n2, k0, k1, s2;
                tile_coords(t2, m2, n2, k0, k1, s2);
                for (int kk = (t2 == t ? kbn : k0); kk < k1 && budget > 0; ++kk, --budget) {
                  if constexpr (SWAP) tma_prefetch_l2_2d(&tmA, kk * kBlockK, m2 * BM);
                  else tma_prefetch_l2_2d(&tmB, kk * kBlockK, n2 * BN);
                }
              }
            }
            flush_pending();
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
      if (!dep_ready) flush_pending();
    }
    __syncwarp();
  } else {
    // ===================== wgmma warpgroup: MMAs, then the epilogue from the register accumulators =====================
    // Thread (warp w, lane l) holds rows 16 w + l / 4 (+ 8) of every 64-row block and columns 8 j + 2 (l % 4) (+ 1).
    const int fr = warp * 16 + (lane >> 2);
    const int fc = 2 * (lane & 3);
    pdl_wait();                            // outputs / residual reads are ordered after the previous grid
    trace.dep();                           // (the trace slot belongs to thread 0, a thread of this warpgroup)
    int stage = 0;
    uint32_t phase = 0;
    float acc[MH][BN / 2];
    for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
      int m_blk, n_blk, kb0, kb1, ks;
      tile_coords(t, m_blk, n_blk, kb0, kb1, ks);
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait_mma(full_bar(stage), phase);
        const uint32_t sa = base + stage * C::STAGE_BYTES;
        const uint64_t bdesc = make_desc_sw128(sa + C::A_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / 16; ++k) {
#pragma unroll
          for (int h = 0; h < MH; ++h)
            wgmma_bf16<BN>(acc[h], make_desc_sw128(sa + h * 64 * 128) + 2u * k, bdesc + 2u * k, (kb > kb0 || k > 0) ? 1 : 0);
        }
        wgmma_commit();
        wgmma_wait<1>();                   // the previous k-block's MMAs are done reading their stage
        if (prev >= 0 && threadIdx.x == 0) mbar_arrive(empty_bar(prev));
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int h = 0; h < MH; ++h) fence_regs(acc[h]);
      if (prev >= 0 && threadIdx.x == 0) mbar_arrive(empty_bar(prev));

      if constexpr (SWAP) {
        // rows = weight rows (output features), columns = batch
        float* ws = reinterpret_cast<float*>(p.out);
#pragma unroll
        for (int h = 0; h < MH; ++h) {
#pragma unroll
          for (int h2 = 0; h2 < 2; ++h2) {
            const int row = m_blk * BM + h * 64 + fr + 8 * h2;
            if (row < p.M) {
#pragma unroll
              for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const int b = 8 * j + fc + e;
                  if (b < p.ws_rows) ws[((size_t)ks * p.ws_rows + b) * (size_t)p.ldo + row] = acc[h][4 * j + 2 * h2 + e];
                }
              }
            }
          }
        }
      } else {
        const int col_tile = n_blk * BN;
        if (p.colscale != nullptr) {
          // per-column scale of int8 weights (their row scales), ahead of every epilogue
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = col_tile + 8 * j + fc + e;
              const float cs = col < p.N ? __ldg(p.colscale + col) : 0.f;
#pragma unroll
              for (int h = 0; h < MH; ++h) {
                acc[h][4 * j + e] *= cs;
                acc[h][4 * j + 2 + e] *= cs;
              }
            }
          }
        }
#pragma unroll
        for (int h = 0; h < MH; ++h) {
#pragma unroll
          for (int h2 = 0; h2 < 2; ++h2) {
#define ACC(j, e) acc[h][4 * (j) + 2 * h2 + (e)]
            const int row = m_blk * BM + h * 64 + fr + 8 * h2;
            const bool row_ok = row < p.M;
            int orow = row;
            if (p.rows_per_group > 0) orow = (row / p.rows_per_group) * p.group_stride + (row % p.rows_per_group) + p.row_offset;
            // deferred RMSNorm: the operand rows were not normalised; their scale commutes with the GEMM and lands here
            float rs = 1.f;
            if (p.rowscale.ssq != nullptr && row_ok) {
              const float* sp = p.rowscale.ssq + (size_t)row * p.rowscale.slots;
              float ss = 0.f;
              for (int i = 0; i < p.rowscale.slots; ++i) ss += __ldg(sp + i);       // fixed order: deterministic
              rs = rsqrtf(ss * p.rowscale.inv_dim + p.rowscale.eps);
            }
            if (p.rope.cos != nullptr) {
              // ---- fused QKV epilogue: RoPE on q / k heads, store q|k|v rows, append k / v to the paged cache (whole heads per tile)
              if constexpr (BN % 128 == 0) {
                const GemmRope& R = p.rope;
                if (row_ok) {
                  const int bq = row / R.S, sq = row % R.S;
                  const int pad = (R.left_pad != nullptr) ? __ldg(R.left_pad + bq) : 0;
                  const int cbase = (R.base_len != nullptr) ? __ldg(R.base_len + bq) : 0;   // tokens cached before this chunk
                  const int cpos = cbase + sq - pad;                       // index inside the (compact) KV cache
                  const bool cached = cpos >= 0;                           // padding rows are neither rotated nor cached
                  const int pos = R.base_len != nullptr ? cpos : (R.pos_from_mask ? (cpos > 0 ? cpos : 0) : sq);
                  int page = 0, slot = 0;
                  if (cached) { page = __ldg(R.kv.seq_pages(bq) + cpos / R.kv.page_tokens); slot = cpos % R.kv.page_tokens; }
                  const float* ct = R.cos + (size_t)pos * 64;
                  const float* stb = R.sin + (size_t)pos * 64;
                  bf16* orow_ptr = reinterpret_cast<bf16*>(p.out) + (size_t)orow * p.ldo;
#pragma unroll
                  for (int hh = 0; hh < BN / 128; ++hh) {
                    const int hcol = col_tile + hh * 128;                  // first column of this head inside [q | k | v]
                    if (hcol < p.N) {
                      const int region = hcol / R.T, head = (hcol % R.T) / 128;
                      if constexpr (KVF == KV_INT8) {
                        if (region >= 1) {
                          // the 4 lanes of a quad hold the row's 128 dims: 32 values each, absmax in two quad shuffles
                          float x[32];
#pragma unroll
                          for (int jj = 0; jj < 8; ++jj) {
                            const int d = 8 * jj + fc;
                            float lo0 = ACC(hh * 16 + jj, 0) * rs, lo1 = ACC(hh * 16 + jj, 1) * rs;
                            float hi0 = ACC(hh * 16 + jj + 8, 0) * rs, hi1 = ACC(hh * 16 + jj + 8, 1) * rs;
                            if (region < 2 && cached) {
                              const float2 c2 = __ldg(reinterpret_cast<const float2*>(ct + d));
                              const float2 s2 = __ldg(reinterpret_cast<const float2*>(stb + d));
                              const float a0 = lo0, b0 = hi0, a1 = lo1, b1 = hi1;
                              lo0 = a0 * c2.x - b0 * s2.x; hi0 = b0 * c2.x + a0 * s2.x;
                              lo1 = a1 * c2.y - b1 * s2.y; hi1 = b1 * c2.y + a1 * s2.y;
                            }
                            x[4 * jj] = lo0; x[4 * jj + 1] = lo1; x[4 * jj + 2] = hi0; x[4 * jj + 3] = hi1;
                          }
                          float a = 0.f;
#pragma unroll
                          for (int i = 0; i < 32; ++i) a = fmaxf(a, fabsf(x[i]));
                          const unsigned qmask = 0xfu << (lane & 28);
                          a = fmaxf(a, __shfl_xor_sync(qmask, a, 1));
                          a = fmaxf(a, __shfl_xor_sync(qmask, a, 2));
                          const float inv = q8_inv(a), sc = q8_step(a);
                          int8_t* qdst = cached ? R.kv.q8_at(page, region - 1, head, slot) : nullptr;
#pragma unroll
                          for (int jj = 0; jj < 8; ++jj) {
                            const int d = 8 * jj + fc;
                            const int q0 = q8_quant(x[4 * jj], inv), q1 = q8_quant(x[4 * jj + 1], inv);
                            const int q2 = q8_quant(x[4 * jj + 2], inv), q3 = q8_quant(x[4 * jj + 3], inv);
                            *reinterpret_cast<uint32_t*>(orow_ptr + hcol + d) = pack_bf16x2(__fmul_rn((float)q0, sc), __fmul_rn((float)q1, sc));
                            *reinterpret_cast<uint32_t*>(orow_ptr + hcol + 64 + d) = pack_bf16x2(__fmul_rn((float)q2, sc), __fmul_rn((float)q3, sc));
                            if (qdst != nullptr) {
                              *reinterpret_cast<uint16_t*>(qdst + d) = (uint16_t)((q0 & 0xff) | ((q1 & 0xff) << 8));
                              *reinterpret_cast<uint16_t*>(qdst + 64 + d) = (uint16_t)((q2 & 0xff) | ((q3 & 0xff) << 8));
                            }
                          }
                          if (qdst != nullptr && (lane & 3) == 0) *R.kv.q8_scale(page, region - 1, head, slot) = sc;
                          continue;
                        }
                      }
                      bf16* cdst = (region >= 1 && cached) ? R.kv.at(page, region - 1, head, slot) : nullptr;
#pragma unroll
                      for (int jj = 0; jj < 8; ++jj) {                     // dims d = 8 jj + fc (+1) pair with d + 64 (HF rotate_half)
                        const int d = 8 * jj + fc;
                        float lo0 = ACC(hh * 16 + jj, 0) * rs, lo1 = ACC(hh * 16 + jj, 1) * rs;
                        float hi0 = ACC(hh * 16 + jj + 8, 0) * rs, hi1 = ACC(hh * 16 + jj + 8, 1) * rs;
                        if (region < 2 && cached) {
                          const float2 c2 = __ldg(reinterpret_cast<const float2*>(ct + d));
                          const float2 s2 = __ldg(reinterpret_cast<const float2*>(stb + d));
                          const float a0 = lo0, b0 = hi0, a1 = lo1, b1 = hi1;
                          lo0 = a0 * c2.x - b0 * s2.x; hi0 = b0 * c2.x + a0 * s2.x;
                          lo1 = a1 * c2.y - b1 * s2.y; hi1 = b1 * c2.y + a1 * s2.y;
                        }
                        const uint32_t plo = pack_bf16x2(lo0, lo1), phi = pack_bf16x2(hi0, hi1);
                        *reinterpret_cast<uint32_t*>(orow_ptr + hcol + d) = plo;
                        *reinterpret_cast<uint32_t*>(orow_ptr + hcol + 64 + d) = phi;
                        if (cdst != nullptr) {
                          *reinterpret_cast<uint32_t*>(cdst + d) = plo;
                          *reinterpret_cast<uint32_t*>(cdst + 64 + d) = phi;
                        }
                      }
                    }
                  }
                }
              }
            } else if (p.mode == GEMM_SWIGLU_BF16) {
              // columns interleaved [32 gate | 32 up]: gate column 8 jj + fc of a 64-block pairs with up column 8 (jj + 4) + fc
              if constexpr (BN % 64 == 0) {
                bf16* out = reinterpret_cast<bf16*>(p.out);
                if (row_ok) {
#pragma unroll
                  for (int c = 0; c < BN / 64; ++c) {
                    const int col0 = col_tile + c * 64;            // first gate column of this pair (in interleaved space)
                    if (col0 < p.N) {
#pragma unroll
                      for (int jj = 0; jj < 4; ++jj) {
                        const float g0 = ACC(8 * c + jj, 0) * rs, g1 = ACC(8 * c + jj, 1) * rs;
                        const float u0 = ACC(8 * c + jj + 4, 0) * rs, u1 = ACC(8 * c + jj + 4, 1) * rs;
                        const float h0 = g0 / (1.f + __expf(-g0)) * u0;
                        const float h1 = g1 / (1.f + __expf(-g1)) * u1;
                        bf16* dst = out + (size_t)orow * p.ldo + col0 / 2 + 8 * jj + fc;
                        if ((p.ldo & 1) == 0) *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(h0, h1);
                        else { dst[0] = __float2bfloat16(h0); dst[1] = __float2bfloat16(h1); }
                      }
                    }
                  }
                }
              }
            } else {
              float ssq_acc = 0.f;     // GemmEmitNorm: this thread's share of the row's sum of squares over the tile
              if (row_ok) {
#pragma unroll
                for (int j = 0; j < BN / 8; ++j) {
                  const int col = col_tile + 8 * j + fc;
                  if (col >= p.N) continue;
                  const bool two = col + 1 < p.N;
                  float x0 = ACC(j, 0) * rs, x1 = ACC(j, 1) * rs;
                  if (p.bias != nullptr) { x0 += __ldg(p.bias + col); if (two) x1 += __ldg(p.bias + col + 1); }
                  if (p.mode == GEMM_STORE_BF16) {
                    if (p.act != ACT_NONE) { x0 = apply_act(x0, p.act); x1 = apply_act(x1, p.act); }
                    bf16* out = reinterpret_cast<bf16*>(p.out) + (size_t)orow * p.ldo + col;
                    if (two && (p.ldo & 1) == 0) *reinterpret_cast<uint32_t*>(out) = pack_bf16x2(x0, x1);
                    else { out[0] = __float2bfloat16(x0); if (two) out[1] = __float2bfloat16(x1); }
                  } else {  // GEMM_ADD_F32
                    float* out = reinterpret_cast<float*>(p.out) + (size_t)orow * p.ldo + col;
                    if (p.rowtab) {
                      const float* rt = p.rowtab + (size_t)(row % p.rowtab_period) * p.N + col;
                      x0 += __ldg(rt); if (two) x1 += __ldg(rt + 1);
                    }
                    if (two && (p.ldo & 1) == 0) {
                      float2* o2 = reinterpret_cast<float2*>(out);
                      if (p.accumulate) { const float2 old = *o2; x0 += old.x; x1 += old.y; }
                      *o2 = make_float2(x0, x1);
                    } else {
                      if (p.accumulate) { x0 += out[0]; if (two) x1 += out[1]; }
                      out[0] = x0; if (two) out[1] = x1;
                    }
                    if (p.emit.xw != nullptr) {
                      bf16* xd = p.emit.xw + (size_t)orow * p.emit.ldxw + col;
                      const float y0 = x0 * __ldg(p.emit.norm_w + col);
                      ssq_acc += x0 * x0;
                      if (two) {
                        const float y1 = x1 * __ldg(p.emit.norm_w + col + 1);
                        ssq_acc += x1 * x1;
                        if ((p.emit.ldxw & 1) == 0) *reinterpret_cast<uint32_t*>(xd) = pack_bf16x2(y0, y1);
                        else { xd[0] = __float2bfloat16(y0); xd[1] = __float2bfloat16(y1); }
                      } else {
                        xd[0] = __float2bfloat16(y0);
                      }
                    }
                  }
                }
              }
              if (p.emit.ssq_out != nullptr) {
                // the 4 lanes of a quad hold one row
                ssq_acc += __shfl_xor_sync(0xffffffffu, ssq_acc, 1);
                ssq_acc += __shfl_xor_sync(0xffffffffu, ssq_acc, 2);
                if (row_ok && (lane & 3) == 0) p.emit.ssq_out[(size_t)orow * p.n_tiles + n_blk] = ssq_acc;
              }
            }
#undef ACC
          }
        }
      }
    }
  }

  __syncthreads();
  trace.done();
}

VCLA_DEFINE_TRACE_SETTER(trace_set_gemm)

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled g_encode = nullptr;
static std::once_flag g_gemm_once;
static int g_gemm_init_rc = 0;

template <int BM, int BN, int STAGES, bool SWAP, int KVF = KV_BF16>
static int set_attr() {
  using C = GemmCfg<BM, BN, STAGES>;
  VCLA_CUDA_OK(cudaFuncSetAttribute(gemm_tc_kernel<BM, BN, STAGES, SWAP, KVF>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
  return 0;
}

// tile configurations (BM x BN, STAGES): prefill 64x256x5 / 128x128x6 / 128x64x8 ; decode swap-AB 128 x {16x5, 32x5, 64x4}
// (two CTAs per SM).  Every configuration keeps <= 128 accumulator registers per thread of the single wgmma warpgroup.
static int gemm_init_impl() {
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || fn == nullptr || qres != cudaDriverEntryPointSuccess) {
    set_error("cuTensorMapEncodeTiled not available: %s", cudaGetErrorString(e));
    return -1;
  }
  g_encode = reinterpret_cast<PFN_encodeTiled>(fn);
  if (set_attr<64, 256, 5, false>()) return -1;
  if (set_attr<64, 256, 5, false, KV_INT8>()) return -1;
  if (set_attr<128, 128, 6, false>()) return -1;
  if (set_attr<128, 64, 8, false>()) return -1;
  if (set_attr<128, 16, 5, true>()) return -1;
  if (set_attr<128, 32, 5, true>()) return -1;
  if (set_attr<128, 64, 4, true>()) return -1;
  return 0;
}
int gemm_init() {
  std::call_once(g_gemm_once, [] { g_gemm_init_rc = gemm_init_impl(); });
  return g_gemm_init_rc;
}

static int make_tmap(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows) {
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (ld * 2) % 16 != 0) {
    set_error("TMA operand must be 16 B aligned with a 16 B-multiple row pitch (ptr %p ld %llu)", ptr, (unsigned long long)ld);
    return -1;
  }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)kBlockK, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) rows %llu cols %llu ld %llu box %u", (int)r, (unsigned long long)rows,
              (unsigned long long)cols, (unsigned long long)ld, box_rows);
    return -1;
  }
  return 0;
}

template <int BM, int BN, int STAGES, bool SWAP, int KVF = KV_BF16>
static int launch(const GemmCall& c, GemmParams p, cudaStream_t st) {
  using C = GemmCfg<BM, BN, STAGES>;
  CUtensorMap ta, tb;
  if (make_tmap(&ta, c.A, c.M, c.K, c.lda, BM)) return -1;
  if (make_tmap(&tb, c.B, c.N, c.K, c.ldb, BN)) return -1;
  p.m_tiles = (c.M + BM - 1) / BM;
  p.n_tiles = (c.N + BN - 1) / BN;
  p.total_tiles = p.m_tiles * p.n_tiles * p.splits;
  const int slots = num_sms() * (SWAP ? 2 : 1);
  const int grid = p.total_tiles < slots ? p.total_tiles : slots;
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kGemmThreads);
  cfg.dynamicSmemBytes = C::SMEM_BYTES;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  int nattr = 0;
  if (pdl_enabled()) {
    attr[nattr].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[nattr].val.programmaticStreamSerializationAllowed = 1;
    ++nattr;
  }
  cfg.attrs = attr;
  cfg.numAttrs = nattr;
  if (getenv("VCLA_DEBUG")) {
    static bool once = false;
    if (!once) {
      once = true;
      int per_sm = -1;
      cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gemm_tc_kernel<BM, BN, STAGES, SWAP, KVF>, kGemmThreads, C::SMEM_BYTES);
      fprintf(stderr, "[vcla] gemm_tc<%d,%d,%d,%d>: smem %d, occupancy query %d blocks/SM, grid %d\n", BM, BN, STAGES, (int)SWAP, C::SMEM_BYTES, per_sm, grid);
    }
  }
  VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, gemm_tc_kernel<BM, BN, STAGES, SWAP, KVF>, ta, tb, p));
  return 0;
}

// tile width of a non-swap GEMM with M rows and N output columns (the widest tile that still gives every SM work)
int gemm_pick_bn(int M, int N) {
  const long m_tiles = (M + 127) / 128;
  const long tiles256 = m_tiles * ((N + 255) / 256);
  const long tiles128 = m_tiles * ((N + 127) / 128);
  if (tiles256 >= num_sms() || N >= 4096) return 256;
  if (tiles128 >= num_sms() / 2 || N > 64) return 128;
  return 64;
}

int gemm_tc(const GemmCall& c, cudaStream_t st) {
  if (gemm_init()) return -1;
  if (c.M <= 0 || c.N <= 0 || c.K <= 0) { set_error("gemm: empty problem"); return -1; }
  if (c.K % 8 != 0) { set_error("gemm: K (%d) must be a multiple of 8", c.K); return -1; }
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = c.M; p.N = c.N; p.K = c.K;
  p.m_tiles = (c.M + kSwapBlockM - 1) / kSwapBlockM;
  p.kb_total = (c.K + kBlockK - 1) / kBlockK;
  p.mode = c.mode; p.act = c.act; p.accumulate = c.accumulate;
  p.out = c.out; p.ldo = c.ldo; p.bias = c.bias;
  p.rowtab = c.rowtab; p.rowtab_period = c.rowtab_period > 0 ? c.rowtab_period : 1;
  p.rows_per_group = c.rows_per_group; p.group_stride = c.group_stride; p.row_offset = c.row_offset;
  p.ws_rows = c.ws_rows;
  p.l2_prefetch_kb = c.l2_prefetch_kb;
  p.rowscale = c.rowscale; p.emit = c.emit; p.rope = c.rope; p.colscale = c.colscale;
  p.policy_a = c.weights_are_A ? kEvictFirst : kEvictLast;
  p.policy_b = c.weights_are_A ? kEvictLast : kEvictNormal;

  if (c.colscale != nullptr && c.mode == GEMM_PARTIAL_F32) { set_error("gemm: colscale is not defined for split-K partials"); return -1; }
  if (c.mode == GEMM_PARTIAL_F32) {
    int splits = c.splits > 0 ? c.splits : 1;
    if (splits > p.kb_total) splits = p.kb_total;
    p.kb_per_split = (p.kb_total + splits - 1) / splits;
    p.splits = (p.kb_total + p.kb_per_split - 1) / p.kb_per_split;   // every split non-empty
    if (p.splits != splits) { set_error("gemm: split count %d not realisable for %d k-blocks (use %d)", splits, p.kb_total, p.splits); return -1; }
    if (c.N > 64 || c.ws_rows < c.N) { set_error("gemm: swap-AB batch rows %d (ws_rows %d) unsupported", c.N, c.ws_rows); return -1; }
    if (c.N <= 16) return launch<128, 16, 5, true>(c, p, st);
    if (c.N <= 32) return launch<128, 32, 5, true>(c, p, st);
    return launch<128, 64, 4, true>(c, p, st);
  }
  p.splits = 1;
  p.kb_per_split = p.kb_total;
  if (c.mode == GEMM_SWIGLU_BF16 && (c.N % 64) != 0) { set_error("gemm: SwiGLU needs N %% 64 == 0 (N=%d)", c.N); return -1; }
  if (c.emit.xw != nullptr && !(c.mode == GEMM_ADD_F32 && c.accumulate && c.emit.norm_w && c.emit.ssq_out)) { set_error("gemm: emit-norm needs ADD_F32 + accumulate + norm_w + ssq_out"); return -1; }
  if (c.rope.cos != nullptr && !(c.mode == GEMM_STORE_BF16 && c.N == 3 * c.rope.T && c.rope.T % 128 == 0 && c.bias == nullptr && c.act == ACT_NONE && c.rows_per_group == 0 && (c.ldo % 8) == 0)) {
    set_error("gemm: the RoPE + KV-append epilogue needs the plain fused QKV projection (N = 3T, T %% 128 == 0)"); return -1;
  }
  if (c.kv_format != KV_BF16 && (c.rope.cos == nullptr || c.kv_format != KV_INT8)) { set_error("gemm: KV cache format %d needs the fused QKV epilogue", c.kv_format); return -1; }
  if (c.kv_format == KV_INT8) return launch<64, 256, 5, false, KV_INT8>(c, p, st);
  int bn = c.bn;
  if (c.rope.cos != nullptr) bn = 256;    // two whole heads per tile
  if (bn == 0) bn = gemm_pick_bn(c.M, c.N);
  if (bn == 256) return launch<64, 256, 5, false>(c, p, st);
  if (bn == 128) return launch<128, 128, 6, false>(c, p, st);
  if (bn == 64) return launch<128, 64, 8, false>(c, p, st);
  set_error("gemm: unsupported tile N %d", bn);
  return -1;
}

// ------------------------------------------------------------------------------------------------
// naive reference (tests only): one thread per output element, same epilogue semantics
// ------------------------------------------------------------------------------------------------
__global__ void gemm_naive_kernel(const bf16* A, const bf16* B, GemmParams p, int lda, int ldb) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  const int row = blockIdx.y;
  const int ncols = (p.mode == GEMM_SWIGLU_BF16) ? p.N / 2 : p.N;
  if (col >= ncols || row >= p.M) return;
  auto dot = [&](int n, int k0, int k1) {
    float s = 0.f;
    for (int k = k0; k < k1; ++k) s += __bfloat162float(A[(size_t)row * lda + k]) * __bfloat162float(B[(size_t)n * ldb + k]);
    return s;
  };
  int orow = row;
  if (p.rows_per_group > 0) orow = (row / p.rows_per_group) * p.group_stride + (row % p.rows_per_group) + p.row_offset;
  if (p.mode == GEMM_PARTIAL_F32) {
    float* ws = reinterpret_cast<float*>(p.out);
    for (int s = 0; s < p.splits; ++s) {
      int k0 = s * p.kb_per_split * kBlockK, k1 = min(p.K, (s + 1) * p.kb_per_split * kBlockK);
      ws[((size_t)s * p.ws_rows + col) * p.ldo + row] = dot(col, k0, k1);
    }
    return;
  }
  if (p.mode == GEMM_SWIGLU_BF16) {
    const int gcol = (col / 32) * 64 + (col % 32);
    float g = dot(gcol, 0, p.K), u = dot(gcol + 32, 0, p.K);
    reinterpret_cast<bf16*>(p.out)[(size_t)orow * p.ldo + col] = __float2bfloat16(g / (1.f + expf(-g)) * u);
    return;
  }
  float x = dot(col, 0, p.K);
  if (p.bias) x += p.bias[col];
  if (p.mode == GEMM_STORE_BF16) {
    if (p.act == ACT_QUICK_GELU) x = x / (1.f + expf(-1.702f * x));
    if (p.act == ACT_GELU_ERF) x = 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
    reinterpret_cast<bf16*>(p.out)[(size_t)orow * p.ldo + col] = __float2bfloat16(x);
  } else {
    float* o = reinterpret_cast<float*>(p.out) + (size_t)orow * p.ldo + col;
    if (p.rowtab) x += p.rowtab[(size_t)(row % p.rowtab_period) * p.N + col];
    if (p.accumulate) x += *o;
    *o = x;
  }
}

int gemm_naive(const GemmCall& c, cudaStream_t st) {
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = c.M; p.N = c.N; p.K = c.K;
  p.kb_total = (c.K + kBlockK - 1) / kBlockK;
  p.mode = c.mode; p.act = c.act; p.accumulate = c.accumulate;
  p.out = c.out; p.ldo = c.ldo; p.bias = c.bias;
  p.rowtab = c.rowtab; p.rowtab_period = c.rowtab_period > 0 ? c.rowtab_period : 1;
  p.rows_per_group = c.rows_per_group; p.group_stride = c.group_stride; p.row_offset = c.row_offset;
  p.ws_rows = c.ws_rows;
  p.splits = 1; p.kb_per_split = p.kb_total;
  if (c.mode == GEMM_PARTIAL_F32) {
    int splits = c.splits > 0 ? c.splits : 1;
    p.kb_per_split = (p.kb_total + splits - 1) / splits;
    p.splits = (p.kb_total + p.kb_per_split - 1) / p.kb_per_split;
  }
  const int ncols = (c.mode == GEMM_SWIGLU_BF16) ? c.N / 2 : c.N;
  dim3 grid((ncols + 127) / 128, c.M);
  gemm_naive_kernel<<<grid, 128, 0, st>>>(c.A, c.B, p, c.lda, c.ldb);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace vcla
