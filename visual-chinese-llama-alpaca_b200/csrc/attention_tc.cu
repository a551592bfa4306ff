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
#include "common.cuh"
#include "kernels.h"

#include <mutex>
#include <stdlib.h>
#include <string.h>

namespace vcla {

constexpr int kAtThreads = 160;                 // warps 0..3 = the wgmma warpgroup, warp 4 = TMA producer
constexpr int kAtBQ = 64, kAtBKV = 64;
constexpr int kAtStages = 2;

struct AttnTcParams {
  int Sq, n0, n1, H;
  float sl2;                       // softmax scale * log2(e)
  int causal;
  const int32_t* kv_start;         // [B] or null
  bf16* out; int o_stride;
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

template <int HD>
__global__ void __launch_bounds__(kAtThreads, 2)
attn_prefill_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK0, const __grid_constant__ CUtensorMap tmV0,
                       const __grid_constant__ CUtensorMap tmK1, const __grid_constant__ CUtensorMap tmV1, const AttnTcParams p) {
  using C = AttnTcCfg<HD>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar0 = base + C::BAR_OFF;
  const uint32_t q_full = bar0;
  auto kv_full = [&](int s) { return bar0 + 8u * (1 + s); };
  auto kv_empty = [&](int s) { return bar0 + 8u * (1 + kAtStages + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * kAtBQ, h = blockIdx.y, b = blockIdx.z;
  const int Sk = p.n0 + p.n1;
  const int off = Sk - p.Sq;                                   // causal: key j visible to query i iff j <= i + off
  const int kv0 = p.kv_start ? __ldg(p.kv_start + b) : 0;
  TraceScope trace(3);

  // KV tiles: segment 0 tiles first, then segment 1; causal launches have one segment and stop at the diagonal tile
  const int nt0 = (p.n0 + kAtBKV - 1) / kAtBKV, nt1 = (p.n1 + kAtBKV - 1) / kAtBKV;
  int nt = nt0 + nt1;
  if (p.causal) { const int kv_end = min(Sk, q0 + kAtBQ + off); nt = min(nt, (max(kv_end, 0) + kAtBKV - 1) / kAtBKV); }
  const int jt0 = kv0 / kAtBKV;                                // tiles entirely left of the padding boundary are skipped
  const int n_tiles = max(nt - jt0, 0);

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < kAtStages; ++s) { mbar_init(kv_full(s), 1); mbar_init(kv_empty(s), 1); }
    fence_barrier_init();
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK0); tma_prefetch_desc(&tmV0);
    if (p.n1 > 0) { tma_prefetch_desc(&tmK1); tma_prefetch_desc(&tmV1); }
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
        mbar_arrive_expect_tx(kv_full(stage), C::K_BYTES + C::V_BYTES);
        const uint32_t sk = base + C::KV_OFF + stage * (C::K_BYTES + C::V_BYTES), sv = sk + C::K_BYTES;
        const bool seg1 = j >= nt0;
        const CUtensorMap* mk = seg1 ? &tmK1 : &tmK0;
        const CUtensorMap* mv = seg1 ? &tmV1 : &tmV0;
        const int row = seg1 ? b * p.n1 + (j - nt0) * kAtBKV : b * p.n0 + j * kAtBKV;
        for (int kb = 0; kb < C::KB; ++kb) {
          tma_load_2d(sk + kb * kAtBKV * 128, mk, h * HD + kb * 64, row, kv_full(stage), kEvictNormal);
          tma_load_2d(sv + kb * kAtBKV * 128, mv, h * HD + kb * 64, row, kv_full(stage), kEvictNormal);
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
      const int kbase = seg1 ? p.n0 + (j - nt0) * kAtBKV : j * kAtBKV;       // global key index of the tile's first row
      const int kvalid = seg1 ? p.n1 - (j - nt0) * kAtBKV : p.n0 - j * kAtBKV; // keys of this tile that exist in the segment
      const int lo = max(kv0 - kbase, 0);
      const uint32_t sk = base + C::KV_OFF + stage * (C::K_BYTES + C::V_BYTES), sv = sk + C::K_BYTES;
      mbar_wait_mma(kv_full(stage), ((uint32_t)(i / kAtStages)) & 1u);
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
          const __nv_bfloat162 pb = __floats2bfloat162_rn(p0, p1);
          ls += __bfloat162float(pb.x) + __bfloat162float(pb.y);   // the sum of what the tensor core will actually multiply
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
    if (cudaFuncSetAttribute(attn_prefill_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnTcCfg<64>::SMEM_BYTES) != cudaSuccess ||
        cudaFuncSetAttribute(attn_prefill_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, AttnTcCfg<128>::SMEM_BYTES) != cudaSuccess) {
      set_error("attention_tc: cudaFuncSetAttribute failed: %s", cudaGetErrorString(cudaGetLastError())); g_at_rc = -1;
    }
  });
  return g_at_rc;
}

// rows x cols bf16 view with a row pitch of `ld` elements; boxes of 64 rows x 64 columns (128 B), 128 B swizzle
static int attn_tmap(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld) {
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) != 0 || (ld * 2) % 16 != 0) { set_error("attention_tc: operands must be 16 B aligned with a 16 B-multiple pitch"); return -1; }
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)kAtBQ};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_at_encode(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                           CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("attention_tc: cuTensorMapEncodeTiled failed (%d)", (int)r); return -1; }
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
    VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_prefill_tc_kernel<64>, tq, tk0, tv0, tk1, tv1, p));
  } else {
    cfg.dynamicSmemBytes = AttnTcCfg<128>::SMEM_BYTES;
    VCLA_CUDA_OK(cudaLaunchKernelEx(&cfg, attn_prefill_tc_kernel<128>, tq, tk0, tv0, tk1, tv1, p));
  }
  return 0;
}

}  // namespace vcla
