// fx_obs_stats.cu -- column moments of rollout observations for the policy's observation normalizer
// (fxenv_obs_moments): out[p][0][j] = sum (x - shift[p][j]), out[p][1][j] = sum (x - shift[p][j])^2 over the rows
// obs[slot][env][j] of every slot and every env of [env_begin, env_end) with env % num_pairs == p, in float64.
//
// Two passes, no atomics: the rows of a pair are cut into `chunks` contiguous ranges; a CTA of fx_moments_partial takes
// 128 columns of one range (4 row lanes x 128 columns: a warp reads 32 consecutive floats of one row, 128 bytes) and
// writes its float64 partial sums, which fx_moments_final adds chunk by chunk.  The cut depends on the shapes only (not
// on the device), so the same inputs give the same bits.  Memory-bound: every float is read once.
#include <cuda_runtime.h>
#include <stdint.h>

#include "fx_kernels.cuh"

namespace {

constexpr int kCols = 128;           // columns per CTA
constexpr int kLanes = 4;            // row lanes per CTA: lane y takes the rows y, y + 4, ... of the CTA's range
constexpr int kTargetCtas = 1024;    // CTAs of the first pass, about (fewer when a range would drop below kMinRows)
constexpr int kMinRows = 64;         // rows per range at least

// the first env >= env_begin of pair p, and the number of the slice's envs of pair p
__device__ __forceinline__ void pair_envs(int env_begin, int env_end, int P, int p, int& first, int& n) {
  first = env_begin + ((p - env_begin % P) % P + P) % P;
  n = first < env_end ? (env_end - first + P - 1) / P : 0;
}

__global__ void __launch_bounds__(kCols * kLanes)
fx_moments_partial(const float* __restrict__ obs, const int N, const int D, const int P, const int env_begin,
                   const int env_end, const int slots, const float* __restrict__ shift, const int chunks,
                   const int64_t rows_per_chunk, double* __restrict__ part) {
  __shared__ double red[kLanes - 1][2][kCols];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int j = blockIdx.x * kCols + tx;
  const int p = blockIdx.y / chunks, ch = blockIdx.y - p * chunks;
  int first, n;
  pair_envs(env_begin, env_end, P, p, first, n);
  const int64_t rows = (int64_t)slots * n;  // row r = (slot r / n, env first + (r % n) * P)
  const int64_t r0 = (int64_t)ch * rows_per_chunk;
  const int64_t r1 = r0 + rows_per_chunk < rows ? r0 + rows_per_chunk : rows;
  double s1 = 0.0, s2 = 0.0;
  if (j < D && r0 + ty < r1) {
    const double sh = (double)shift[(size_t)p * D + j];
    int64_t r = r0 + ty;
    int slot = (int)(r / n), k = (int)(r - (int64_t)slot * n);
    const int64_t row_step = (int64_t)P * D, slot_step = (int64_t)N * D;
    const float* x = obs + slot * slot_step + ((int64_t)first + (int64_t)k * P) * D + j;
    // the next row of this lane (4 rows on): k advances by 4 envs of the pair, wrapping into the next slots
    auto next = [&]() {
      k += kLanes;
      x += kLanes * row_step;
      while (k >= n) { k -= n; x += slot_step - n * row_step; }
    };
    for (; r + 3 * kLanes < r1; r += 4 * kLanes) {  // four loads in flight, then the adds in row order
      const float* a = x; next();
      const float* b = x; next();
      const float* c = x; next();
      const float* d = x; next();
      const float v0 = __ldcs(a), v1 = __ldcs(b), v2 = __ldcs(c), v3 = __ldcs(d);
      double t;
      t = (double)v0 - sh; s1 += t; s2 += t * t;
      t = (double)v1 - sh; s1 += t; s2 += t * t;
      t = (double)v2 - sh; s1 += t; s2 += t * t;
      t = (double)v3 - sh; s1 += t; s2 += t * t;
    }
    for (; r < r1; r += kLanes) {
      const double t = (double)__ldcs(x) - sh;
      s1 += t; s2 += t * t;
      next();
    }
  }
  if (ty > 0) { red[ty - 1][0][tx] = s1; red[ty - 1][1][tx] = s2; }
  __syncthreads();
  if (ty == 0 && j < D) {
#pragma unroll
    for (int y = 0; y < kLanes - 1; y++) { s1 += red[y][0][tx]; s2 += red[y][1][tx]; }
    double* o = part + ((size_t)p * chunks + ch) * 2 * D;
    o[j] = s1;
    o[D + j] = s2;
  }
}

// out[p][s][j] = sum over the chunks c, in order, of part[p][c][s][j]
__global__ void fx_moments_final(const double* __restrict__ part, const int chunks, const int P, const int D,
                                 double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)P * 2 * D) return;
  const int64_t p = i / (2 * D), sj = i - p * 2 * D;
  const double* src = part + (size_t)p * chunks * 2 * D + sj;
  double acc = 0.0;
  for (int c = 0; c < chunks; c++) acc += src[(size_t)c * 2 * D];
  out[i] = acc;
}

}  // namespace

cudaError_t fx_launch_obs_moments(const float* obs, int slots, int num_envs, int D, int num_pairs, int env_begin, int env_end,
                                  const float* shift, double* out, cudaStream_t stream) {
  const int P = num_pairs;
  const int col_blocks = (D + kCols - 1) / kCols;
  const int64_t max_rows = (int64_t)slots * ((env_end - env_begin + P - 1) / P);  // the largest pair's rows
  int64_t chunks = (kTargetCtas + (int64_t)col_blocks * P - 1) / ((int64_t)col_blocks * P);
  const int64_t by_rows = (max_rows + kMinRows - 1) / kMinRows;
  if (chunks > by_rows) chunks = by_rows;
  if (chunks < 1) chunks = 1;
  const int64_t rows_per_chunk = (max_rows + chunks - 1) / chunks;
  double* part = nullptr;
  cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&part), (size_t)P * chunks * 2 * D * sizeof(double), stream);
  if (e != cudaSuccess) return e;
  fx_moments_partial<<<dim3(col_blocks, (unsigned)(P * chunks)), dim3(kCols, kLanes), 0, stream>>>(
      obs, num_envs, D, P, env_begin, env_end, slots, shift, (int)chunks, rows_per_chunk, part);
  e = cudaGetLastError();
  if (e == cudaSuccess) {
    const int64_t total = (int64_t)P * 2 * D;
    fx_moments_final<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(part, (int)chunks, P, D, out);
    e = cudaGetLastError();
  }
  const cudaError_t e2 = cudaFreeAsync(part, stream);
  return e != cudaSuccess ? e : e2;
}
