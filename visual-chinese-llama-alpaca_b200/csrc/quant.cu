// Weight-only int8 (load_in_8bit): row-wise absmax quantisation of the LLaMA projections, and the moves between the stored layout
// and the caller's logical layout.
//
//   a = max_k |w[r, k]| (fp32), s[r] = a / 127, q[r, k] = clamp(rint(w[r, k] * (127 / a)), -127, 127)   (rint: half to even; a = 0: s = q = 0)
//
// Stored rows: within every 64-column block, byte 16 j4 + 4 s + j holds column 16 s + 2 j4 + {0, 1, 8, 9}[j] -- the order in which the
// decode GEMM's register fragments consume them (gemm_decode.cu).  The gate/up rows keep the engine's 32-row interleave.
#include "common.cuh"
#include "kernels.h"

namespace vcla {

// column of the 64-column block held by stored byte p, and the inverse
__host__ __device__ __forceinline__ int q8_logical_of_stored(int p) { return 16 * ((p >> 2) & 3) + 2 * (p >> 4) + (p & 1) + 8 * ((p >> 1) & 1); }
__host__ __device__ __forceinline__ int q8_stored_of_logical(int l) {
  const int r = l & 15;
  return 16 * ((r & 7) >> 1) + 4 * (l >> 4) + (r & 1) + 2 * (r >> 3);
}
__device__ __forceinline__ int q8_row(int r, int which) { return which < 0 ? r : (r / 32) * 64 + which * 32 + r % 32; }
__device__ __forceinline__ size_t q8_index(int row, int k, int cols) { return (size_t)row * cols + (k & ~63) + q8_stored_of_logical(k & 63); }

__device__ __forceinline__ float load_as_f32(const void* src, int dtype, size_t i) {
  if (dtype == 0) return reinterpret_cast<const float*>(src)[i];
  if (dtype == 1) return __half2float(reinterpret_cast<const __half*>(src)[i]);
  return __bfloat162float(reinterpret_cast<const bf16*>(src)[i]);
}

constexpr int kQ8Threads = 256;

// one CTA per row: the absmax is a max (exact, order free), the rest is elementwise
__global__ void __launch_bounds__(kQ8Threads) quantize_rows_q8_kernel(const void* src, int dtype, int cols, int which, int8_t* q, float* scale) {
  __shared__ float red[kQ8Threads / 32];
  const int r = blockIdx.x;
  const size_t off = (size_t)r * cols;
  float a = 0.f;
  for (int k = threadIdx.x; k < cols; k += kQ8Threads) a = fmaxf(a, fabsf(load_as_f32(src, dtype, off + k)));
  a = warp_max(a);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  a = red[0];
  for (int i = 1; i < kQ8Threads / 32; ++i) a = fmaxf(a, red[i]);
  const float inv = a > 0.f ? __fdiv_rn(127.f, a) : 0.f;
  const int row = q8_row(r, which);
  if (threadIdx.x == 0) scale[row] = __fdiv_rn(a, 127.f);
  for (int k = threadIdx.x; k < cols; k += kQ8Threads) {
    const float v = rintf(__fmul_rn(load_as_f32(src, dtype, off + k), inv));
    q[q8_index(row, k, cols)] = (int8_t)fminf(fmaxf(v, -127.f), 127.f);
  }
}

__global__ void place_rows_q8_kernel(const int8_t* q_src, const float* s_src, int cols, int which, int8_t* q, float* scale) {
  const int r = blockIdx.x, row = q8_row(r, which);
  if (threadIdx.x == 0) scale[row] = s_src[r];
  for (int k = threadIdx.x; k < cols; k += blockDim.x) q[q8_index(row, k, cols)] = q_src[(size_t)r * cols + k];
}

__global__ void read_rows_q8_kernel(const int8_t* q, const float* scale, int cols, int which, int8_t* q_out, float* s_out, float* f32_out) {
  const int r = blockIdx.x, row = q8_row(r, which);
  const float s = scale[row];
  if (s_out != nullptr && threadIdx.x == 0) s_out[r] = s;
  for (int k = threadIdx.x; k < cols; k += blockDim.x) {
    const int8_t v = q[q8_index(row, k, cols)];
    if (q_out != nullptr) q_out[(size_t)r * cols + k] = v;
    if (f32_out != nullptr) f32_out[(size_t)r * cols + k] = (float)v * s;
  }
}

// one thread per 8 output columns (16 B of bf16, so a warp's stores are contiguous).  Stored order: logical columns 8 v .. 8 v + 7 of a
// 64-column block are bytes 2 (v % 2) and 2 (v % 2) + 1 of the four words at 16 j4 + 4 (v / 2), j4 = 0..3 (in column order).
__device__ __forceinline__ uint32_t i8_pair_to_bf16x2(uint32_t word, int byte0) {
  return pack_bf16x2((float)(int8_t)(word >> (8 * byte0)), (float)(int8_t)(word >> (8 * byte0 + 8)));
}
__global__ void expand_rows_q8_kernel(const int8_t* q, size_t n_out16, int permuted, bf16* out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_out16) return;
  const int8_t* blk = q + (i >> 3) * 64;
  const int v = (int)(i & 7);
  uint32_t w[4];
  if (permuted) {
#pragma unroll
    for (int j4 = 0; j4 < 4; ++j4) w[j4] = i8_pair_to_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(blk + 16 * j4 + 4 * (v >> 1))), 2 * (v & 1));
  } else {
    const uint2 d = __ldg(reinterpret_cast<const uint2*>(blk + 8 * v));
    w[0] = i8_pair_to_bf16x2(d.x, 0); w[1] = i8_pair_to_bf16x2(d.x, 2); w[2] = i8_pair_to_bf16x2(d.y, 0); w[3] = i8_pair_to_bf16x2(d.y, 2);
  }
  reinterpret_cast<uint4*>(out)[i] = make_uint4(w[0], w[1], w[2], w[3]);
}

int quantize_rows_q8(const void* src, int dtype, int rows, int cols, int which, int8_t* q, float* scale, cudaStream_t st) {
  if (rows <= 0) return 0;
  if (cols % 64 != 0) { set_error("int8 weights need a multiple of 64 columns (got %d)", cols); return -1; }
  quantize_rows_q8_kernel<<<rows, kQ8Threads, 0, st>>>(src, dtype, cols, which, q, scale);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}
int place_rows_q8(const int8_t* q_src, const float* s_src, int rows, int cols, int which, int8_t* q, float* scale, cudaStream_t st) {
  if (rows <= 0) return 0;
  if (cols % 64 != 0) { set_error("int8 weights need a multiple of 64 columns (got %d)", cols); return -1; }
  place_rows_q8_kernel<<<rows, kQ8Threads, 0, st>>>(q_src, s_src, cols, which, q, scale);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}
int read_rows_q8(const int8_t* q, const float* scale, int rows, int cols, int which, int8_t* q_out, float* s_out, float* f32_out, cudaStream_t st) {
  if (rows <= 0) return 0;
  read_rows_q8_kernel<<<rows, kQ8Threads, 0, st>>>(q, scale, cols, which, q_out, s_out, f32_out);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}
int expand_rows_q8(const int8_t* q, int rows, int cols, int permuted, bf16* out, cudaStream_t st) {
  if (rows <= 0) return 0;
  if (cols % 64 != 0 || (reinterpret_cast<uintptr_t>(q) & 15) != 0 || (reinterpret_cast<uintptr_t>(out) & 15) != 0) {
    set_error("expand_rows_q8: needs 16 B aligned buffers and a multiple of 64 columns (got %d)", cols); return -1;
  }
  const size_t n = (size_t)rows * (cols / 8);
  expand_rows_q8_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(q, n, permuted, out);
  VCLA_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace vcla
