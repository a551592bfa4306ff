// HBM-bound kernels of the VisualCLA path: normalisation, embedding / splice, the decode
// consumers of the split-K partial sums, argmax, synthetic-weight generation and checkpoint repacking.
// All are simple streaming kernels: 128-bit coalesced accesses where layouts allow, fp32 statistics.
#include "common.cuh"
#include "kernels.h"

#include <cooperative_groups.h>
#include <math.h>
#include <vector>

namespace vcla {

static inline cudaLaunchConfig_t make_cfg(dim3 grid, dim3 block, size_t smem, cudaStream_t st, cudaLaunchAttribute* attr) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  int na = 0;
  if (pdl_enabled()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr; cfg.numAttrs = na;
  return cfg;
}
#define VCLA_LAUNCH(kernel, grid, block, smem, st, ...)                         \
  do {                                                                          \
    cudaLaunchAttribute _attr[1];                                               \
    cudaLaunchConfig_t _cfg = make_cfg(grid, block, smem, st, _attr);           \
    VCLA_CUDA_OK(cudaLaunchKernelEx(&_cfg, kernel, __VA_ARGS__));               \
  } while (0)

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = (lane < nw) ? red[lane] : 0.f;
  t = warp_sum(t);
  return t;
}

// ------------------------------------------------------------------------------------------------
// LayerNorm / RMSNorm: one CTA per row, row cached in smem, two-pass fp32 statistics
// ------------------------------------------------------------------------------------------------
__global__ void layernorm_kernel(const float* x, int D, const float* __restrict__ w, const float* __restrict__ b,
                                 float eps, bf16* __restrict__ y_bf16, float* y_f32) {
  extern __shared__ float rowbuf[];
  __shared__ float red[32];
  TraceScope trace(5);
  pdl_launch_dependents();   // dependents may become resident early; they block in their own griddepcontrol.wait
  pdl_wait();
  trace.dep();
  const size_t row = blockIdx.x;
  const float* xr = x + row * D;
  float s = 0.f;
  for (int i = threadIdx.x * 4; i < D; i += blockDim.x * 4) {
    float4 v = *reinterpret_cast<const float4*>(xr + i);
    *reinterpret_cast<float4*>(rowbuf + i) = v;
    s += v.x + v.y + v.z + v.w;
  }
  const float mean = block_sum(s, red) / D;
  float q = 0.f;
  for (int i = threadIdx.x * 4; i < D; i += blockDim.x * 4) {
    float4 v = *reinterpret_cast<float4*>(rowbuf + i);
    float a = v.x - mean, bb = v.y - mean, cc = v.z - mean, dd = v.w - mean;
    q += a * a + bb * bb + cc * cc + dd * dd;
  }
  const float rstd = rsqrtf(block_sum(q, red) / D + eps);
  for (int i = threadIdx.x * 4; i < D; i += blockDim.x * 4) {
    float4 v = *reinterpret_cast<float4*>(rowbuf + i);
    float4 wv = *reinterpret_cast<const float4*>(w + i), bv = *reinterpret_cast<const float4*>(b + i);
    float o0 = (v.x - mean) * rstd * wv.x + bv.x, o1 = (v.y - mean) * rstd * wv.y + bv.y;
    float o2 = (v.z - mean) * rstd * wv.z + bv.z, o3 = (v.w - mean) * rstd * wv.w + bv.w;
    if (y_bf16) *reinterpret_cast<uint2*>(y_bf16 + row * D + i) = make_uint2(pack_bf16x2(o0, o1), pack_bf16x2(o2, o3));
    if (y_f32) *reinterpret_cast<float4*>(y_f32 + row * D + i) = make_float4(o0, o1, o2, o3);
  }
}
int layernorm(const float* x, int rows, int D, const float* w, const float* b, float eps, bf16* y_bf16, float* y_f32, cudaStream_t st) {
  if (D % 4) { set_error("layernorm: D %% 4 != 0"); return -1; }
  if (rows == 0) return 0;
  VCLA_LAUNCH(layernorm_kernel, dim3(rows), dim3(D >= 2048 ? 256 : 128), (size_t)D * 4, st, x, D, w, b, eps, y_bf16, y_f32);
  return 0;
}

__global__ void rmsnorm_kernel(const float* __restrict__ x, int D, const float* __restrict__ w, float eps, bf16* __restrict__ y) {
  extern __shared__ float rowbuf[];
  __shared__ float red[32];
  TraceScope trace(6);
  pdl_launch_dependents();   // dependents may become resident early; they block in their own griddepcontrol.wait
  pdl_wait();
  trace.dep();
  const size_t row = blockIdx.x;
  const float* xr = x + row * D;
  float q = 0.f;
  for (int i = threadIdx.x * 4; i < D; i += blockDim.x * 4) {
    float4 v = *reinterpret_cast<const float4*>(xr + i);
    *reinterpret_cast<float4*>(rowbuf + i) = v;
    q += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  const float rstd = rsqrtf(block_sum(q, red) / D + eps);
  for (int i = threadIdx.x * 4; i < D; i += blockDim.x * 4) {
    float4 v = *reinterpret_cast<float4*>(rowbuf + i);
    float4 wv = *reinterpret_cast<const float4*>(w + i);
    *reinterpret_cast<uint2*>(y + row * D + i) =
        make_uint2(pack_bf16x2(v.x * rstd * wv.x, v.y * rstd * wv.y), pack_bf16x2(v.z * rstd * wv.z, v.w * rstd * wv.w));
  }
}
int rmsnorm(const float* x, int rows, int D, const float* w, float eps, bf16* y, cudaStream_t st) {
  if (D % 4) { set_error("rmsnorm: D %% 4 != 0"); return -1; }
  if (rows == 0) return 0;
  VCLA_LAUNCH(rmsnorm_kernel, dim3(rows), dim3(D >= 2048 ? 256 : 128), (size_t)D * 4, st, x, D, w, eps, y);
  return 0;
}

__global__ void prenorm_rows_kernel(const float* __restrict__ x, int D, const float* __restrict__ w, bf16* __restrict__ xw, float* __restrict__ ssq, int slots) {
  __shared__ float red[32];
  TraceScope trace(6);
  pdl_launch_dependents();
  pdl_wait();
  trace.dep();
  const size_t row = blockIdx.x;
  const float* xr = x + row * D;
  float q = 0.f;
  for (int i = threadIdx.x * 4; i < D; i += blockDim.x * 4) {
    const float4 v = *reinterpret_cast<const float4*>(xr + i);
    const float4 wv = *reinterpret_cast<const float4*>(w + i);
    q += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
    *reinterpret_cast<uint2*>(xw + row * D + i) = make_uint2(pack_bf16x2(v.x * wv.x, v.y * wv.y), pack_bf16x2(v.z * wv.z, v.w * wv.w));
  }
  q = block_sum(q, red);
  for (int sidx = threadIdx.x; sidx < slots; sidx += blockDim.x) ssq[row * slots + sidx] = sidx == 0 ? q : 0.f;
}
int prenorm_rows(const float* x, int rows, int D, const float* w, bf16* xw, float* ssq, int slots, cudaStream_t st) {
  if (D % 4) { set_error("prenorm_rows: D %% 4 != 0"); return -1; }
  if (rows == 0) return 0;
  VCLA_LAUNCH(prenorm_rows_kernel, dim3(rows), dim3(D >= 2048 ? 256 : 128), 0, st, x, D, w, xw, ssq, slots);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// ViT front end
// ------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_f32<bf16>(bf16 v) { return __bfloat162float(v); }

template <typename T>
__global__ void im2col_kernel(const T* __restrict__ px, int B, int image, int patch, int kpad, bf16* __restrict__ out) {
  // one CTA per patch row; k = c*P*P + ky*P + kx  (Conv2d weight (D,3,P,P) flattened)
  const int g = image / patch;
  const int prow = blockIdx.x;  // b*g*g + py*g + px
  const int b = prow / (g * g), pp = prow % (g * g), py = pp / g, pxi = pp % g;
  const int kreal = 3 * patch * patch;
  for (int k = threadIdx.x; k < kpad; k += blockDim.x) {
    float v = 0.f;
    if (k < kreal) {
      int c = k / (patch * patch), r = k % (patch * patch), ky = r / patch, kx = r % patch;
      v = to_f32<T>(px[(((size_t)b * 3 + c) * image + (py * patch + ky)) * image + (pxi * patch + kx)]);
    }
    out[(size_t)prow * kpad + k] = __float2bfloat16(v);
  }
}
int im2col(const void* pixels, int dtype, int B, int image, int patch, int kpad, bf16* out, cudaStream_t st) {
  const int g = image / patch;
  dim3 grid(B * g * g), block(128);
  if (dtype == 0) im2col_kernel<float><<<grid, block, 0, st>>>((const float*)pixels, B, image, patch, kpad, out);
  else if (dtype == 1) im2col_kernel<__half><<<grid, block, 0, st>>>((const __half*)pixels, B, image, patch, kpad, out);
  else if (dtype == 2) im2col_kernel<bf16><<<grid, block, 0, st>>>((const bf16*)pixels, B, image, patch, kpad, out);
  else { set_error("im2col: unknown pixel dtype %d", dtype); return -1; }
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

__global__ void vit_cls_rows_kernel(float* hidden, int tokens, int D, const float* cls, const float* pos) {
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < D; i += blockDim.x) hidden[(size_t)b * tokens * D + i] = cls[i] + pos[i];
}
int vit_cls_rows(float* hidden, int B, int tokens, int D, const float* cls, const float* pos, cudaStream_t st) {
  vit_cls_rows_kernel<<<B, 256, 0, st>>>(hidden, tokens, D, cls, pos);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

__global__ void broadcast_rows_kernel(const float* src, int rows, int D, float* dst_f32, bf16* dst_bf16) {
  const int r = blockIdx.x, b = blockIdx.y;
  for (int i = threadIdx.x; i < D; i += blockDim.x) {
    float v = src[(size_t)r * D + i];
    size_t o = ((size_t)b * rows + r) * D + i;
    if (dst_f32) dst_f32[o] = v;
    if (dst_bf16) dst_bf16[o] = __float2bfloat16(v);
  }
}
int broadcast_rows(const float* src, int rows, int D, int B, float* dst_f32, bf16* dst_bf16, cudaStream_t st) {
  broadcast_rows_kernel<<<dim3(rows, B), 256, 0, st>>>(src, rows, D, dst_f32, dst_bf16);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// embedding gather / image splice
// ------------------------------------------------------------------------------------------------
__global__ void embed_tokens_kernel(const int64_t* __restrict__ ids, int T, int S, int D, const bf16* __restrict__ table,
                                    int vocab, int mode, int nq, float* __restrict__ dst) {
  const int t = blockIdx.x, b = blockIdx.y;
  long long id = ids[(size_t)b * T + t];
  if (id < 0 || id >= vocab) id = 0;
  const int pos = (mode == 1 && t >= 2) ? t + nq : t;
  const bf16* src = table + (size_t)id * D;
  float* d = dst + ((size_t)b * S + pos) * D;
  for (int i = threadIdx.x * 8; i < D; i += blockDim.x * 8) {
    uint4 v = *reinterpret_cast<const uint4*>(src + i);
    float2 a = unpack_bf16x2(v.x), bb = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z), e = unpack_bf16x2(v.w);
    *reinterpret_cast<float4*>(d + i) = make_float4(a.x, a.y, bb.x, bb.y);
    *reinterpret_cast<float4*>(d + i + 4) = make_float4(c.x, c.y, e.x, e.y);
  }
}
int embed_tokens(const int64_t* ids, int B, int T, int S, int D, const bf16* table, int vocab, int mode, int nq, float* dst, cudaStream_t st) {
  if (D % 8) { set_error("embed: D %% 8 != 0"); return -1; }
  VCLA_LAUNCH(embed_tokens_kernel, dim3(T, B), dim3(128), 0, st, ids, T, S, D, table, vocab, mode, nq, dst);
  return 0;
}
__global__ void embed_tokens_i32_kernel(const int32_t* __restrict__ ids, int D, const bf16* __restrict__ table, int vocab, float* __restrict__ dst) {
  TraceScope trace(13);
  pdl_launch_dependents();   // dependents may become resident early; they block in their own griddepcontrol.wait
  pdl_wait();
  trace.dep();
  const int b = blockIdx.x;
  int id = ids[b];
  if (id < 0 || id >= vocab) id = 0;
  const bf16* src = table + (size_t)id * D;
  float* d = dst + (size_t)b * D;
  for (int i = threadIdx.x * 8; i < D; i += blockDim.x * 8) {
    uint4 v = *reinterpret_cast<const uint4*>(src + i);
    float2 a = unpack_bf16x2(v.x), bb = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z), e = unpack_bf16x2(v.w);
    *reinterpret_cast<float4*>(d + i) = make_float4(a.x, a.y, bb.x, bb.y);
    *reinterpret_cast<float4*>(d + i + 4) = make_float4(c.x, c.y, e.x, e.y);
  }
}
int embed_tokens_i32(const int32_t* ids, int B, int D, const bf16* table, int vocab, float* dst, cudaStream_t st) {
  VCLA_LAUNCH(embed_tokens_i32_kernel, dim3(B), dim3(256), 0, st, ids, D, table, vocab, dst);
  return 0;
}

// decode step entry (one CTA per sequence): embedding row -> fp32 residual, bf16 GEMM operand pre-multiplied by the first
// layer's RMSNorm weight, and the row's sum of squares (the consuming GEMM turns it into the deferred scale 1/rms)
__global__ void dec_embed_kernel(const int32_t* __restrict__ ids, int D, const bf16* __restrict__ table, int vocab, float* __restrict__ resid,
                                 const float* __restrict__ norm_w, bf16* __restrict__ xw, float* __restrict__ ssq, int slots) {
  __shared__ float red[32];
  TraceScope trace(13);
  pdl_launch_dependents();   // dependents may become resident early; they block in their own griddepcontrol.wait
  pdl_wait();
  trace.dep();
  const int b = blockIdx.x;
  int id = ids[b];
  if (id < 0 || id >= vocab) id = 0;
  const bf16* src = table + (size_t)id * D;
  float q = 0.f;
  for (int i = threadIdx.x * 8; i < D; i += blockDim.x * 8) {
    const uint4 v = *reinterpret_cast<const uint4*>(src + i);
    const uint32_t w4[4] = {v.x, v.y, v.z, v.w};
    float f[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) { const float2 t = unpack_bf16x2(w4[j]); f[2 * j] = t.x; f[2 * j + 1] = t.y; }
    *reinterpret_cast<float4*>(resid + (size_t)b * D + i) = make_float4(f[0], f[1], f[2], f[3]);
    *reinterpret_cast<float4*>(resid + (size_t)b * D + i + 4) = make_float4(f[4], f[5], f[6], f[7]);
    const float4 w0 = *reinterpret_cast<const float4*>(norm_w + i), w1 = *reinterpret_cast<const float4*>(norm_w + i + 4);
    *reinterpret_cast<uint4*>(xw + (size_t)b * D + i) = make_uint4(pack_bf16x2(f[0] * w0.x, f[1] * w0.y), pack_bf16x2(f[2] * w0.z, f[3] * w0.w),
                                                                    pack_bf16x2(f[4] * w1.x, f[5] * w1.y), pack_bf16x2(f[6] * w1.z, f[7] * w1.w));
#pragma unroll
    for (int j = 0; j < 8; ++j) q += f[j] * f[j];
  }
  q = block_sum(q, red);
  // deferred-norm chain head: the row's sum of squares in slot 0, the other slots empty
  for (int i = threadIdx.x; i < slots; i += blockDim.x) ssq[(size_t)b * slots + i] = i == 0 ? q : 0.f;
}
int dec_embed(const int32_t* ids, int B, int D, const bf16* table, int vocab, float* resid, const float* norm_w, bf16* xw,
              float* ssq, int slots, cudaStream_t st) {
  if (D % 8) { set_error("dec_embed: D %% 8 != 0"); return -1; }
  VCLA_LAUNCH(dec_embed_kernel, dim3(B), dim3(256), 0, st, ids, D, table, vocab, resid, norm_w, xw, ssq, slots);
  return 0;
}

__global__ void scatter_image_rows_kernel(const float* __restrict__ img, int nq, int D, const int32_t* __restrict__ row_start, int S, float* __restrict__ dst) {
  const int q = blockIdx.x, b = blockIdx.y;
  const int rs = row_start[b];
  if (rs < 0) return;  // this sample carries no image
  const float4* s = reinterpret_cast<const float4*>(img + ((size_t)b * nq + q) * D);
  float4* d = reinterpret_cast<float4*>(dst + ((size_t)b * S + rs + q) * D);
  for (int i = threadIdx.x; i < D / 4; i += blockDim.x) d[i] = s[i];
}
int scatter_image_rows(const float* img, int B, int nq, int D, const int32_t* row_start, int S, float* dst, cudaStream_t st) {
  scatter_image_rows_kernel<<<dim3(nq, B), 256, 0, st>>>(img, nq, D, row_start, S, dst);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

__global__ void gather_last_rows_kernel(const float* hidden, int S, int D, float* dst) {
  const int b = blockIdx.x;
  const float4* s = reinterpret_cast<const float4*>(hidden + ((size_t)b * S + (S - 1)) * D);
  float4* d = reinterpret_cast<float4*>(dst + (size_t)b * D);
  for (int i = threadIdx.x; i < D / 4; i += blockDim.x) d[i] = s[i];
}
int gather_last_rows(const float* hidden, int B, int S, int D, float* dst, cudaStream_t st) {
  gather_last_rows_kernel<<<B, 256, 0, st>>>(hidden, S, D, dst);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// RoPE tables (fp32, computed once on the host the way HF does: HF:models/llama/modeling_llama.py:98-141)
// ------------------------------------------------------------------------------------------------
int rope_fill_tables(int max_pos, int head_dim, float theta, float* cos_dev, float* sin_dev) {
  const int half = head_dim / 2;
  std::vector<float> hc((size_t)max_pos * half), hs((size_t)max_pos * half);
  for (int i = 0; i < half; ++i) {
    const float inv = 1.0f / powf(theta, (float)(2 * i) / (float)head_dim);
    for (int p = 0; p < max_pos; ++p) {
      const float f = (float)p * inv;
      hc[(size_t)p * half + i] = (float)cos((double)f);
      hs[(size_t)p * half + i] = (float)sin((double)f);
    }
  }
  VCLA_CUDA_OK(cudaMemcpy(cos_dev, hc.data(), hc.size() * 4, cudaMemcpyHostToDevice));
  VCLA_CUDA_OK(cudaMemcpy(sin_dev, hs.data(), hs.size() * 4, cudaMemcpyHostToDevice));
  return 0;
}

// ------------------------------------------------------------------------------------------------
// decode consumers of split-K partial sums
// ------------------------------------------------------------------------------------------------
// One 8-CTA thread-block cluster per batch row: each CTA reduces the split-K partials of D/8 columns into the fp32
// residual stream, the row's sum of squares is exchanged through distributed shared memory, then every CTA writes its
// slice of the normalised bf16 GEMM operand.  (One CTA per row was latency-bound: 12 us per launch, 65 launches/step.)
constexpr int kNormCluster = 8;
__global__ void __cluster_dims__(kNormCluster, 1, 1) __launch_bounds__(128)
dec_resid_norm_kernel(const float* __restrict__ partial, int splits, int ws_rows, float* __restrict__ resid, int D,
                      const float* __restrict__ w, float eps, bf16* __restrict__ xn) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  __shared__ float red[32];
  __shared__ float s_part;
  TraceScope trace(8);
  pdl_launch_dependents();   // dependents may become resident early; they block in their own griddepcontrol.wait
  pdl_wait();
  trace.dep();
  const int b = blockIdx.y;
  const int chunk = D / kNormCluster;
  const int c0 = blockIdx.x * chunk;
  constexpr int MAXV = 4;
  float4 vals[MAXV];
  float q = 0.f;
  int nv = 0;
  for (int i = threadIdx.x * 4; i < chunk; i += blockDim.x * 4, ++nv) {
    const int col = c0 + i;
    float4 v = *reinterpret_cast<const float4*>(resid + (size_t)b * D + col);
    if (partial) {
      // (issuing all <= 24 partial loads at once was measured slower in situ: 6.96 vs 5.40 us after o_proj)
#pragma unroll 4
      for (int s = 0; s < splits; ++s) {
        const float4 p = __ldcg(reinterpret_cast<const float4*>(partial + ((size_t)s * ws_rows + b) * D + col));
        v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
      }
      *reinterpret_cast<float4*>(resid + (size_t)b * D + col) = v;
    }
    vals[nv] = v;
    q += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  q = block_sum(q, red);
  if (threadIdx.x == 0) s_part = q;
  cluster.sync();
  float tot = 0.f;
#pragma unroll
  for (int r = 0; r < kNormCluster; ++r) tot += *cluster.map_shared_rank(&s_part, r);
  cluster.sync();            // nobody may exit while a peer still reads its shared memory
  const float rstd = rsqrtf(tot / D + eps);
  nv = 0;
  for (int i = threadIdx.x * 4; i < chunk; i += blockDim.x * 4, ++nv) {
    const int col = c0 + i;
    const float4 v = vals[nv];
    const float4 wv = *reinterpret_cast<const float4*>(w + col);
    *reinterpret_cast<uint2*>(xn + (size_t)b * D + col) =
        make_uint2(pack_bf16x2(v.x * rstd * wv.x, v.y * rstd * wv.y), pack_bf16x2(v.z * rstd * wv.z, v.w * rstd * wv.w));
  }
}
int dec_resid_norm(const float* partial, int splits, int ws_rows, float* resid, int B, int D, const float* w, float eps, bf16* xn, cudaStream_t st) {
  if (D % (kNormCluster * 4) != 0 || D / kNormCluster > 128 * 4 * 4) { set_error("dec_resid_norm: unsupported D %d", D); return -1; }
  VCLA_LAUNCH(dec_resid_norm_kernel, dim3(kNormCluster, B), dim3(128), 0, st, partial, splits, ws_rows, resid, D, w, eps, xn);
  return 0;
}

__global__ void dec_silu_mul_kernel(const float* __restrict__ partial, int splits, int ws_rows, int F, bf16* __restrict__ h) {
  TraceScope trace(9);
  pdl_launch_dependents();   // dependents may become resident early; they block in their own griddepcontrol.wait
  pdl_wait();
  trace.dep();
  const int b = blockIdx.y;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= F) return;
  const int gi = (j >> 5) * 64 + (j & 31);
  float g = 0.f, u = 0.f;
  for (int s = 0; s < splits; ++s) {
    const float* row = partial + ((size_t)s * ws_rows + b) * (size_t)(2 * F);
    g += row[gi];
    u += row[gi + 32];
  }
  h[(size_t)b * F + j] = __float2bfloat16(g / (1.f + __expf(-g)) * u);
}
int dec_silu_mul(const float* partial, int splits, int ws_rows, int B, int F, bf16* h, cudaStream_t st) {
  VCLA_LAUNCH(dec_silu_mul_kernel, dim3((F + 255) / 256, B), dim3(256), 0, st, partial, splits, ws_rows, F, h);
  return 0;
}

// logits + argmax: stage 1 per (vocab chunk, b) -> candidate ; stage 2 per b
constexpr int kArgChunks = kArgmaxChunks;
__global__ void dec_logits_stage1(const float* __restrict__ partial, int splits, int ws_rows, int ldp, int V, float* __restrict__ logits,
                                  int ld_logits, float* __restrict__ cand_val, int* __restrict__ cand_idx) {
  __shared__ float sv[32];
  __shared__ int si[32];
  TraceScope trace(10);
  pdl_launch_dependents();   // dependents may become resident early; they block in their own griddepcontrol.wait
  pdl_wait();
  trace.dep();
  const int b = blockIdx.y, ch = blockIdx.x;
  const int per = (V + kArgChunks - 1) / kArgChunks;
  const int v0 = ch * per, v1 = min(V, v0 + per);
  // a thread starts from its own first column, so a row that is -inf everywhere still yields a column of the row (index 0 after
  // the tie rule, as torch.argmax); threads and chunks without a column keep the sentinel and lose every tie
  float best = -INFINITY;
  int bi = (v0 + (int)threadIdx.x < v1) ? v0 + (int)threadIdx.x : 0x7fffffff;
  for (int v = v0 + threadIdx.x; v < v1; v += blockDim.x) {
    float x = 0.f;
    for (int s = 0; s < splits; ++s) x += __ldcg(partial + ((size_t)s * ws_rows + b) * (size_t)ldp + v);
    if (logits) logits[(size_t)b * ld_logits + v] = x;
    if (x > best) { best = x; bi = v; }   // strided order: smaller index kept on ties via the reduction below
  }
  // warp + block reduce, ties -> smallest index
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, best, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) { sv[warp] = best; si[warp] = bi; }
  __syncthreads();
  if (warp == 0) {
    const int nw = blockDim.x >> 5;
    best = lane < nw ? sv[lane] : -INFINITY;
    bi = lane < nw ? si[lane] : 0x7fffffff;
    for (int o = 16; o > 0; o >>= 1) {
      float ov = __shfl_xor_sync(0xffffffffu, best, o);
      int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (lane == 0) { cand_val[b * kArgChunks + ch] = best; cand_idx[b * kArgChunks + ch] = bi; }
  }
}
__global__ void dec_logits_stage2(const float* __restrict__ cand_val, const int* __restrict__ cand_idx, int32_t* __restrict__ tok,
                                  int32_t* __restrict__ history, const int32_t* __restrict__ step_idx, int32_t* __restrict__ dp_send) {
  TraceScope trace(11);
  pdl_launch_dependents();   // dependents may become resident early; they block in their own griddepcontrol.wait
  pdl_wait();
  trace.dep();
  const int b = blockIdx.x, lane = threadIdx.x;
  float best = cand_val[b * kArgChunks + lane];
  int bi = cand_idx[b * kArgChunks + lane];
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, best, o);
    int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  }
  if (lane == 0) {
    tok[b] = bi;
    if (history) history[(size_t)(*step_idx) * gridDim.x + b] = bi;   // [step][B] log of every chosen token since the prefill
    if (dp_send) dp_send[b] = bi;                                      // send buffer of the per-step token all-gather (data parallel)
  }
}
int dec_logits_argmax(const float* partial, int splits, int ws_rows, int ldp, int B, int V, float* logits, int ld_logits, int32_t* tok,
                      int32_t* history, const int32_t* step_idx, float* cand_val, int32_t* cand_idx, int32_t* dp_send, cudaStream_t st) {
  if (!cand_val || !cand_idx) { set_error("argmax scratch missing"); return -1; }
  VCLA_LAUNCH(dec_logits_stage1, dim3(kArgChunks, B), dim3(256), 0, st, partial, splits, ws_rows, ldp, V, logits, ld_logits, cand_val, (int*)cand_idx);
  VCLA_LAUNCH(dec_logits_stage2, dim3(B), dim3(32), 0, st, (const float*)cand_val, (const int*)cand_idx, tok, history, step_idx, dp_send);
  return 0;
}

int dec_logits_reduce(const float* partial, int splits, int ws_rows, int ldp, int B, int V, float* logits, int ld_logits,
                      float* cand_val, int32_t* cand_idx, cudaStream_t st) {
  if (!logits || !cand_val || !cand_idx) { set_error("dec_logits_reduce: missing buffers"); return -1; }
  VCLA_LAUNCH(dec_logits_stage1, dim3(kArgChunks, B), dim3(256), 0, st, partial, splits, ws_rows, ldp, V, logits, ld_logits, cand_val, (int*)cand_idx);
  return 0;
}

// data parallel: append the all-gathered tokens of this step to the global history [step][world * width]
__global__ void dp_unpack_kernel(const int32_t* __restrict__ recv, int n, int32_t* __restrict__ hist, int32_t* __restrict__ dp_step) {
  const int s = *dp_step;
  for (int i = threadIdx.x; i < n; i += blockDim.x) hist[(size_t)s * n + i] = recv[i];
  __syncthreads();
  if (threadIdx.x == 0) *dp_step = s + 1;
}
int dp_unpack(const int32_t* recv, int n, int32_t* hist, int32_t* dp_step, cudaStream_t st) {
  dp_unpack_kernel<<<1, 128, 0, st>>>(recv, n, hist, dp_step);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// device-side KV page allocator
// ------------------------------------------------------------------------------------------------
__global__ void kv_reset_kernel(const KvCache kv, const int32_t* __restrict__ kv_order, int max_batch) {
  // stack top is the END of the free stack: page kv_order[0] must be popped first
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < kv.total_pages; i += gridDim.x * blockDim.x) kv.free_stack[kv.total_pages - 1 - i] = kv_order[i];
  if (blockIdx.x == 0) {
    for (int b = threadIdx.x; b < max_batch; b += blockDim.x) kv.npages[b] = 0;
    if (threadIdx.x == 0) { kv.state[0] = kv.total_pages; kv.state[1] = 0; }
  }
}
int kv_reset(const KvCache& kv, const int32_t* kv_order, int max_batch, cudaStream_t st) {
  int blocks = (kv.total_pages + 255) / 256;
  if (blocks > 64) blocks = 64;
  if (blocks < 1) blocks = 1;
  kv_reset_kernel<<<blocks, 256, 0, st>>>(kv, kv_order, max_batch);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

// One thread: for page rank p = 0,1,..: every sequence that needs a p-th page and does not own one yet pops the stack.
// need[b] = pages for `tokens[b]` tokens, clamped to the table row.
__device__ void kv_reserve_serial(const KvCache& kv, int B, const int* s_tokens) {
  int top = kv.state[0];
  bool more = true;
  for (int p = 0; more && p < kv.pages_per_seq; ++p) {
    more = false;
    for (int b = 0; b < B; ++b) {
      const int need = kv.pages_for(s_tokens[b]);
      if (need > p + 1) more = true;
      if (need > p && kv.npages[b] == p) {
        if (top <= 0) { kv.state[1] = 1; continue; }          // pool exhausted (unreachable behind the host-side capacity check)
        kv.seq_pages(b)[p] = kv.free_stack[--top];
        kv.npages[b] = p + 1;
      }
    }
  }
  kv.state[0] = top;
}
__global__ void kv_reserve_kernel(const KvCache kv, int B, int S, const int32_t* __restrict__ left_pad, const int32_t* __restrict__ base_len) {
  __shared__ int s_tokens[64];
  if (threadIdx.x < B) s_tokens[threadIdx.x] = (base_len ? base_len[threadIdx.x] : 0) + S - (left_pad ? left_pad[threadIdx.x] : 0);
  __syncthreads();
  if (threadIdx.x == 0) kv_reserve_serial(kv, B, s_tokens);
}
int kv_reserve(const KvCache& kv, int B, int S, const int32_t* left_pad, cudaStream_t st, const int32_t* base_len) {
  if (B > 64) { set_error("kv_reserve: batch %d > 64", B); return -1; }
  kv_reserve_kernel<<<1, 64, 0, st>>>(kv, B, S, left_pad, base_len);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

struct KvLens { int32_t v[64]; };
__global__ void kv_truncate_kernel(int32_t* seq_len, int B, const KvLens len) {
  const int b = threadIdx.x;
  if (b < B) seq_len[b] = min(seq_len[b], len.v[b]);
}
int kv_truncate(int32_t* seq_len, const int32_t* len_host, int B, cudaStream_t st) {
  if (B < 1 || B > 64) { set_error("kv_truncate: batch %d not in 1..64", B); return -1; }
  KvLens len;
  for (int b = 0; b < 64; ++b) len.v[b] = b < B ? len_host[b] : 0;
  kv_truncate_kernel<<<1, 64, 0, st>>>(seq_len, B, len);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

__device__ __forceinline__ void st_release_sys(int32_t* p, int32_t v) {
  asm volatile("st.release.sys.global.b32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}

__global__ void advance_seq_kernel(int32_t* seq_len, int B, int by, const int32_t* __restrict__ left_pad, int32_t* step_idx, const KvCache kv,
                                   StreamRing* ring, const int32_t* __restrict__ history, int publish_rows) {
  __shared__ int s_tokens[64];
  __shared__ int s_step;
  TraceScope trace(12);
  pdl_launch_dependents();   // dependents may become resident early; they block in their own griddepcontrol.wait
  pdl_wait();
  trace.dep();
  const int b = threadIdx.x;
  if (b < B) {
    const int L = seq_len[b] + by - (left_pad ? left_pad[b] : 0);
    seq_len[b] = L;
    s_tokens[b] = L + 1;                 // the next token of this sequence is appended at index L
  }
  if (step_idx != nullptr && b == 0) {
    const int step = *step_idx;          // this step's tokens (history row `step`) are final: their kernel precedes this one
    if (ring != nullptr) s_step = step;
    *step_idx = step + 1;
  }
  __syncthreads();
  if (ring != nullptr) {
    // publish: tokens into the host ring, each writer's stores made visible system-wide, then one release store of the count.
    // The ring has as many rows as the history (max_seq + 2), so any step whose history row exists has a ring row.
    const int step = s_step;
    if (b < publish_rows) {
      ring->tokens[(size_t)step * 64 + b] = history[(size_t)step * publish_rows + b];
      __threadfence_system();
    }
    __syncthreads();
    if (b == 0) st_release_sys(&ring->published, step + 1);
  }
  if (threadIdx.x == 0) {
    // fast path (every step but one in page_tokens): nobody crosses a page boundary
    bool any = false;
    for (int i = 0; i < B; ++i) any |= kv.pages_for(s_tokens[i]) > kv.npages[i];
    if (any) kv_reserve_serial(kv, B, s_tokens);
  }
}
int advance_seq(int32_t* seq_len, int B, int by, const int32_t* left_pad, int32_t* step_idx, const KvCache& kv, cudaStream_t st,
                StreamRing* ring, const int32_t* history, int publish_rows) {
  if (publish_rows <= 0) publish_rows = B;
  if (B > 64 || publish_rows > 64) { set_error("advance_seq: batch %d (%d published) > 64", B, publish_rows); return -1; }
  if (ring != nullptr && (history == nullptr || step_idx == nullptr)) { set_error("advance_seq: publishing needs the token history"); return -1; }
  VCLA_LAUNCH(advance_seq_kernel, dim3(1), dim3(64), 0, st, seq_len, B, by, left_pad, step_idx, kv, ring, (const int32_t*)history, publish_rows);
  return 0;
}

// ---- fan-out: N replies per prompt forked from one prefill (vcla_set_fanout) ------------------------------------------------------
__global__ void fanout_rows_kernel(int n, int rows, int32_t* __restrict__ parent, int32_t* tok, int32_t* history) {
  TraceScope trace(21);
  trace.dep();
  const int r = threadIdx.x;
  int v = 0;
  if (tok != nullptr && r < rows) v = tok[r / n];
  __syncthreads();                     // every prompt pick is read before any row is rewritten in place
  if (r < rows) {
    parent[r] = r / n;
    if (tok != nullptr) { tok[r] = v; history[r] = v; }
  }
  trace.done();
}
int fanout_rows(int n, int rows, int32_t* parent, int32_t* tok, int32_t* history, cudaStream_t st) {
  if (n < 1 || rows < n || rows > 64 || rows % n != 0) { set_error("fanout_rows: %d rows are not a fan-out of %d", rows, n); return -1; }
  if (tok != nullptr && history == nullptr) { set_error("fanout_rows: expanding the picks needs the token history"); return -1; }
  fanout_rows_kernel<<<1, 64, 0, st>>>(n, rows, parent, tok, history);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ---- prompt lookup decoding: accept, advance and draft (one CTA, B = 1) ---------------------------------------------------------
__global__ void __launch_bounds__(256) lookup_accept_kernel(const LookupCall c, int prime) {
  __shared__ int s_done, s_prod, s_best;
  TraceScope trace(20);
  pdl_launch_dependents();
  pdl_wait();
  trace.dep();
  const int tid = threadIdx.x;
  const int max_new = c.state->max_new;
  if (tid == 0) {
    int produced = *c.step_idx;
    bool done = produced >= max_new || c.finished[0] != 0;
    if (!prime && !done) {
      // HF _assisted_decoding: n_matches = leading drafts equal to the model's picks; the picks of rows 0..n_matches are emitted
      const int nd = c.state->nd;
      int a = 0;
      while (a < nd && c.pick[a] == c.tok[a + 1]) ++a;
      int cnt = 0, fin = 0;
      for (int j = 0; j <= a && produced + cnt < max_new && !fin; ++j) {
        const int t = c.pick[j];
        c.history[produced + cnt] = t;
        ++cnt;
        if (c.samp) for (int e = 0; e < c.samp->n_eos; ++e) fin |= t == c.samp->eos[e];   // plain decoding stops at the EOS too
      }
      if (fin) c.finished[0] = 1;
      c.seq_len[0] += cnt;                    // row 0 and the accepted drafts before the last emitted token are cached now
      if (c.ring != nullptr) {
        // the ring has as many rows as the history (max_seq + 2): every emitted row has a ring row
        for (int j = 0; j < cnt; ++j) c.ring->tokens[(size_t)(produced + j) * 64] = c.history[produced + j];
        __threadfence_system();
        st_release_sys(&c.ring->published, produced + cnt);
      }
      produced += cnt;
      *c.step_idx = produced;
      c.state->steps += 1; c.state->drafted += nd; c.state->accepted += cnt - 1;
      done = produced >= max_new || fin;
    }
    // pages for the R rows the next step appends (idle steps after the end append there too, beyond seq_len)
    const int need = c.seq_len[0] + c.R;
    if (c.kv.pages_for(need) > c.kv.npages[0]) { int tokens[1] = {need}; kv_reserve_serial(c.kv, 1, tokens); }
    s_done = done; s_prod = produced; s_best = 0x7fffffff;
  }
  __syncthreads();
  if (s_done) { trace.done(); return; }
  // HF PromptLookupCandidateGenerator.get_candidates over text = prompt ids ++ emitted tokens: for g = min(n, N - 1) .. 1, the leftmost
  // earlier window equal to the last g tokens whose continuation is non-empty (every window but the tail itself); draft = up to R - 1
  // tokens of that continuation, clamped so that produced + drafts + 1 <= max_new
  const int produced = s_prod, P = c.state->prompt_len, N = P + produced;
  auto at = [&](int i) -> int { return i < P ? (int)c.prompt[i] : c.history[i - P]; };
  int start = -1;
  for (int g = min(c.state->n, N - 1); g >= 1; --g) {
    for (int i = tid; i < N - g; i += blockDim.x) {
      bool same = true;
      for (int j = 0; j < g && same; ++j) same = at(i + j) == at(N - g + j);
      if (same) atomicMin(&s_best, i);
    }
    __syncthreads();
    const int best = s_best;
    __syncthreads();                          // every thread has read s_best before the next n-gram size may lower it
    if (best != 0x7fffffff) { start = best + g; break; }
  }
  if (tid == 0) {
    int nd = 0;
    if (start >= 0) nd = min(min(c.R - 1, N - start), max_new - produced - 1);
    if (nd < 0) nd = 0;
    const int last = c.history[produced - 1];
    c.tok[0] = last;
    for (int j = 1; j < c.R; ++j) {
      const int t = j <= nd ? at(start + j - 1) : last;
      c.tok[j] = t;
      c.history[produced + j - 1] = t;        // provisional: row j's sampler reads the history extended by drafts 1..j-1
    }
    c.state->nd = nd;
  }
  trace.done();
}
int lookup_accept(const LookupCall& c, int prime, cudaStream_t st) {
  if (c.R < 2 || c.R > 16 || !c.prompt || !c.tok || !c.pick || !c.history || !c.step_idx || !c.seq_len ||
      !c.finished || !c.state) {
    set_error("lookup_accept: bad arguments"); return -1;
  }
  VCLA_LAUNCH(lookup_accept_kernel, dim3(1), dim3(256), 0, st, c, prime);
  return 0;
}

// ---- beam search: rows continue their parents' pages (shared through the page table, copy-on-write for the page written next) ----
// Pages are never shared across a row boundary of positions: a page covers positions [i * page_tokens, (i + 1) * page_tokens) and sits at
// index i of every row that references it.  Rows that share page i also share every page before it (a fork copies the parent's row;
// only pages created after it differ), so an old row's pages that no new row keeps are a suffix of its row.
constexpr int kReorderThreads = 1024;
template <int FMT = KV_BF16>   // the cache format sets the bytes a copied row counts
__global__ void __launch_bounds__(kReorderThreads, 1)
kv_beam_reorder_kernel(int rows_old, int rows_new, const int32_t* __restrict__ parent_row, const int32_t* __restrict__ new_tok, int32_t* seq_len,
                       const KvCache kv, int32_t* table_tmp, int32_t* history, const int32_t* __restrict__ step_idx, int32_t* copy_list,
                       unsigned long long* cow_bytes) {
  extern __shared__ uint32_t s_mark[];
  __shared__ int s_np[64], s_len[64], s_par[64];
  TraceScope trace(17);
  trace.dep();
  const int pps = kv.pages_per_seq, pt = kv.page_tokens;
  const int tid = threadIdx.x, words = (kv.total_pages + 31) / 32;
  if (tid < rows_old) { s_np[tid] = kv.npages[tid]; s_len[tid] = seq_len[tid]; }
  if (tid < rows_new) s_par[tid] = parent_row[tid];
  for (int i = tid; i < words; i += kReorderThreads) s_mark[i] = 0u;
  __syncthreads();
  for (int e = tid; e < rows_old * pps; e += kReorderThreads) if (e % pps < s_np[e / pps]) table_tmp[e] = kv.table[e];
  __syncthreads();
  // mark every page a new row keeps
  for (int e = tid; e < rows_new * pps; e += kReorderThreads) {
    const int j = e / pps, i = e % pps, p = s_par[j];
    if (i < s_np[p]) { const int pg = table_tmp[(size_t)p * pps + i]; atomicOr(&s_mark[pg >> 5], 1u << (pg & 31)); }
  }
  __syncthreads();
  if (tid == 0) {
    // release the unkept suffix of every old row (marking a released page stops a sibling that shares it from releasing it again)
    int top = kv.state[0];
    for (int k = 0; k < rows_old; ++k) {
      for (int i = s_np[k] - 1; i >= 0; --i) {
        const int pg = table_tmp[(size_t)k * pps + i];
        const uint32_t bit = 1u << (pg & 31);
        if (s_mark[pg >> 5] & bit) break;
        s_mark[pg >> 5] |= bit;
        kv.free_stack[top++] = pg;
      }
    }
    kv.state[0] = top;
  }
  __syncthreads();
  for (int e = tid; e < rows_new * pps; e += kReorderThreads) {
    const int j = e / pps, i = e % pps, p = s_par[j];
    if (i < s_np[p]) kv.table[e] = table_tmp[(size_t)p * pps + i];
  }
  if (tid < rows_new) { kv.npages[tid] = s_np[s_par[tid]]; seq_len[tid] = s_len[s_par[tid]]; }
  __syncthreads();
  if (tid == 0) {
    // copy-on-write of the page the next token is written to: the first row continuing a parent keeps it, the others get a copy
    int top = kv.state[0], n = 0;
    long long rows_copied = 0;
    uint64_t seen = 0;
    for (int j = 0; j < rows_new; ++j) {
      const int p = s_par[j], L = s_len[p], pw = L / pt;
      if (!((seen >> p) & 1ull)) { seen |= 1ull << p; continue; }
      if (pw >= s_np[p]) continue;                       // no page for a next token (the sequence is at its capacity)
      if (top <= 0) { kv.state[1] = 1; continue; }       // pool exhausted (unreachable: distinct pages <= rows * pages_per_seq)
      const int fresh = kv.free_stack[--top];
      kv.table[(size_t)j * pps + pw] = fresh;
      copy_list[1 + 3 * n] = table_tmp[(size_t)p * pps + pw];
      copy_list[2 + 3 * n] = fresh;
      copy_list[3 + 3 * n] = L % pt;
      rows_copied += L % pt;
      ++n;
    }
    copy_list[0] = n;
    kv.state[0] = top;
    if (cow_bytes) *cow_bytes += (unsigned long long)(rows_copied * kv.layers * kv.planes() * (FMT == KV_INT8 ? (long long)kKvQ8RowBytes : 128 * (long long)sizeof(bf16)));
  }
  // token history: columns gathered by parent, then this step's tokens as row t (one thread per history row: in place)
  const int t = *step_idx - 1;
  for (int pos = tid; pos < t; pos += kReorderThreads) {
    int32_t tmp[64];
    for (int j = 0; j < rows_new; ++j) tmp[j] = history[(size_t)pos * rows_old + s_par[j]];
    for (int j = 0; j < rows_new; ++j) history[(size_t)pos * rows_new + j] = tmp[j];
  }
  if (tid < rows_new) history[(size_t)t * rows_new + tid] = new_tok[tid];
  trace.done();
}
int kv_beam_reorder(int rows_old, int rows_new, const int32_t* parent_row, const int32_t* new_tok, int32_t* seq_len, const KvCache& kv,
                    int32_t* table_tmp, int32_t* history, const int32_t* step_idx, int32_t* copy_list, unsigned long long* cow_bytes,
                    cudaStream_t st, KvFormat fmt) {
  if (rows_old < 1 || rows_new < rows_old || rows_new > 64) { set_error("kv_beam_reorder: rows %d -> %d", rows_old, rows_new); return -1; }
  const size_t smem = (size_t)((kv.total_pages + 31) / 32) * 4;
  if (smem > 200u * 1024u) { set_error("kv_beam_reorder: %d pages exceed the page bitmap", kv.total_pages); return -1; }
  static bool opted_in = false;        // the first call is vcla_prefill's fork, outside any graph capture
  if (smem > 48u * 1024u && !opted_in) {
    VCLA_CUDA_OK(cudaFuncSetAttribute(kv_beam_reorder_kernel<KV_BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    VCLA_CUDA_OK(cudaFuncSetAttribute(kv_beam_reorder_kernel<KV_INT8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    opted_in = true;
  }
  if (fmt == KV_INT8)
    kv_beam_reorder_kernel<KV_INT8><<<1, kReorderThreads, smem, st>>>(rows_old, rows_new, parent_row, new_tok, seq_len, kv, table_tmp, history,
                                                                      step_idx, copy_list, cow_bytes);
  else
    kv_beam_reorder_kernel<<<1, kReorderThreads, smem, st>>>(rows_old, rows_new, parent_row, new_tok, seq_len, kv, table_tmp, history, step_idx,
                                                              copy_list, cow_bytes);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

__global__ void kv_page_copy_kernel(const KvCache kv, const int32_t* __restrict__ copy_list) {
  TraceScope trace(18);
  trace.dep();
  const int e = blockIdx.x;
  if (e >= copy_list[0]) return;
  const int src = copy_list[1 + 3 * e], dst = copy_list[2 + 3 * e], n = copy_list[3 + 3 * e];
  const KvPool layer = kv.layer(blockIdx.y);
  const uint4* s = reinterpret_cast<const uint4*>(layer.at(src, 0, 0, 0));
  uint4* d = reinterpret_cast<uint4*>(layer.at(dst, 0, 0, 0));
  const int per_plane = n * 16, plane_stride = kv.page_tokens * 16;   // 16 uint4 = one 128-wide bf16 row
  for (int i = threadIdx.x; i < kv.planes() * per_plane; i += blockDim.x) {
    const int plane = i / per_plane, off = i % per_plane;
    d[(size_t)plane * plane_stride + off] = s[(size_t)plane * plane_stride + off];
  }
  trace.done();
}
// KV_INT8: the int8 rows (8 uint4 each) and their fp32 scales, plane by plane
__global__ void kv_page_copy_q8_kernel(const KvCache kv, const int32_t* __restrict__ copy_list) {
  TraceScope trace(18);
  trace.dep();
  const int e = blockIdx.x;
  if (e >= copy_list[0]) return;
  const int src = copy_list[1 + 3 * e], dst = copy_list[2 + 3 * e], n = copy_list[3 + 3 * e];
  const KvPool layer = kv.layer(blockIdx.y);
  const uint4* s = reinterpret_cast<const uint4*>(layer.q8_at(src, 0, 0, 0));
  uint4* d = reinterpret_cast<uint4*>(layer.q8_at(dst, 0, 0, 0));
  const int per_plane = n * 8, plane_stride = kv.page_tokens * 8;
  for (int i = threadIdx.x; i < kv.planes() * per_plane; i += blockDim.x) {
    const int plane = i / per_plane, off = i % per_plane;
    d[(size_t)plane * plane_stride + off] = s[(size_t)plane * plane_stride + off];
  }
  const float* ss = layer.q8_scale(src, 0, 0, 0);
  float* ds = layer.q8_scale(dst, 0, 0, 0);
  for (int i = threadIdx.x; i < kv.planes() * n; i += blockDim.x) {
    const int plane = i / n, off = i % n;
    ds[(size_t)plane * kv.page_tokens + off] = ss[(size_t)plane * kv.page_tokens + off];
  }
  trace.done();
}
int kv_page_copy(const KvCache& kv, const int32_t* copy_list, int max_entries, cudaStream_t st, KvFormat fmt) {
  if (fmt == KV_INT8) kv_page_copy_q8_kernel<<<dim3(max_entries, kv.layers), 256, 0, st>>>(kv, copy_list);
  else kv_page_copy_kernel<<<dim3(max_entries, kv.layers), 256, 0, st>>>(kv, copy_list);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// weights: synthetic generator (bit-identical to oracle.hash_normal_bf16) and checkpoint repacking
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t fmix32(uint32_t h) {
  h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
  return h;
}
__global__ void fill_hash_normal_kernel(bf16* dst_bf16, float* dst_f32, int64_t n, uint32_t seed, float mul, float offset) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t a = fmix32((uint32_t)i * 0x9E3779B1u + seed);
    const uint32_t b = fmix32(a ^ 0x7F4A7C15u);
    const int tot = (int)(a & 0xFFFFu) + (int)(a >> 16) + (int)(b & 0xFFFFu) + (int)(b >> 16) - 131070;
    const float v = __fadd_rn(__fmul_rn((float)tot, mul), offset);   // no FMA contraction: must match numpy bit for bit
    const bf16 r = __float2bfloat16(v);
    if (dst_bf16) dst_bf16[i] = r;
    if (dst_f32) dst_f32[i] = __bfloat162float(r);
  }
}
int fill_hash_normal(bf16* dst_bf16, float* dst_f32, int64_t n, uint32_t seed, float mul, float offset, cudaStream_t st) {
  int64_t blocks = (n + 255) / 256;
  if (blocks > num_sms() * 16) blocks = num_sms() * 16;
  fill_hash_normal_kernel<<<(int)blocks, 256, 0, st>>>(dst_bf16, dst_f32, n, seed, mul, offset);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

template <typename T, typename O>
__global__ void convert_kernel(const T* src, int64_t n, O* dst) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = to_f32<T>(src[i]);
    if constexpr (sizeof(O) == 2) dst[i] = __float2bfloat16(v);
    else dst[i] = v;
  }
}
template <typename O>
static int convert_any(const void* src, int dtype, int64_t n, O* dst, cudaStream_t st) {
  int64_t blocks = (n + 255) / 256;
  if (blocks > num_sms() * 16) blocks = num_sms() * 16;
  if (blocks == 0) return 0;
  if (dtype == 0) convert_kernel<float, O><<<(int)blocks, 256, 0, st>>>((const float*)src, n, dst);
  else if (dtype == 1) convert_kernel<__half, O><<<(int)blocks, 256, 0, st>>>((const __half*)src, n, dst);
  else if (dtype == 2) convert_kernel<bf16, O><<<(int)blocks, 256, 0, st>>>((const bf16*)src, n, dst);
  else { set_error("convert: unknown dtype %d", dtype); return -1; }
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}
int convert_to_bf16(const void* src, int dtype, int64_t n, bf16* dst, cudaStream_t st) { return convert_any<bf16>(src, dtype, n, dst, st); }
int convert_to_f32(const void* src, int dtype, int64_t n, float* dst, cudaStream_t st) { return convert_any<float>(src, dtype, n, dst, st); }

__global__ void copy_rows_bf16_kernel(const bf16* src, int cols, bf16* dst, int ld) {
  const size_t r = blockIdx.x;
  for (int i = threadIdx.x; i < ld; i += blockDim.x) dst[r * ld + i] = (i < cols) ? src[r * cols + i] : __float2bfloat16(0.f);
}
int copy_rows_bf16(const bf16* src, int rows, int cols, bf16* dst, int ld, cudaStream_t st) {
  if (rows == 0) return 0;
  copy_rows_bf16_kernel<<<rows, 256, 0, st>>>(src, cols, dst, ld);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}
__global__ void interleave_rows32_kernel(const bf16* src, int cols, int which, bf16* dst) {
  const size_t j = blockIdx.x;
  const size_t r = (j >> 5) * 64 + (size_t)which * 32 + (j & 31);
  for (int i = threadIdx.x; i < cols; i += blockDim.x) dst[r * cols + i] = src[j * cols + i];
}
int interleave_rows32(const bf16* src, int rows, int cols, int which, bf16* dst, cudaStream_t st) {
  interleave_rows32_kernel<<<rows, 256, 0, st>>>(src, cols, which, dst);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

VCLA_DEFINE_TRACE_SETTER(trace_set_elementwise)

}  // namespace vcla
