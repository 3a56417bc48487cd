// fx_return_stats.cu -- moments of the discounted returns of a rollout for the reward normalizer (fxenv_return_moments).
// Per env i of [env_begin, env_end) (j = i - env_begin): the return R carried in ret[j] is kept only when the env has
// begun no episode since the last scan other than at this rollout's reset steps (begun[i] - n_reset == seen[j]), then
//   for t in 0 .. horizon-1:  if step t is not a reset step: R = R * gamma + reward[t][i], d = R - shift, S1 += d,
//                             S2 += d * d, n += 1;  if done[t][i]: R = 0
// and ret[j] = R, seen[j] = begun[i]; out = {S1, S2, n} over the slice, in float64.
//
// Two passes, no atomics: fx_return_scan runs one thread per env (a warp reads 32 consecutive rewards and done codes of
// one step) and a fixed tree adds its CTA's sums into one partial per CTA; fx_return_final adds the partials in CTA order.
// The cut depends on the slice width only, so the same inputs give the same bits.  The fp64 recursion is one dependent
// chain per env; the loads of the next kStage steps are issued before the current kStage steps are added, so a thread
// waits for memory about once per kStage steps, not once per step.
#include <cuda_runtime.h>
#include <stdint.h>

#include "fx_kernels.cuh"

namespace {

constexpr int kThreads = 64;   // envs per CTA: 64 CTAs at 4096 envs, so that the chains spread over the SMs
constexpr int kStage = 8;      // steps per prefetch stage

struct Stage {
  float r[kStage];
  uint8_t d[kStage];
};

__device__ __forceinline__ void load_stage(Stage& s, const float* __restrict__ reward, const uint8_t* __restrict__ done,
                                           const int64_t N, const int i, const int t0, const int H) {
#pragma unroll
  for (int k = 0; k < kStage; k++) {
    const int t = t0 + k;
    s.r[k] = t < H ? __ldcs(reward + (int64_t)t * N + i) : 0.0f;
    s.d[k] = t < H ? __ldg(done + (int64_t)t * N + i) : (uint8_t)0;
  }
}

__global__ void __launch_bounds__(kThreads)
fx_return_scan(const float* __restrict__ reward, const uint8_t* __restrict__ done, const uint8_t* __restrict__ prev_done,
               const int32_t* __restrict__ begun, const int N, const int H, const int env_begin, const int env_end,
               const double gamma, const double shift, double* __restrict__ ret, int32_t* __restrict__ seen,
               double* __restrict__ part) {
  __shared__ double red[3][kThreads];
  const int j = blockIdx.x * kThreads + threadIdx.x;
  const int i = env_begin + j;
  double s1 = 0.0, s2 = 0.0, n = 0.0;
  if (i < env_end) {
    // the reset steps: step 0 after prev_done, step t after done[t - 1]
    const uint8_t pd = prev_done[i];
    int n_reset = pd != 0;
    {
      int t = 0;
      for (; t + kStage <= H - 1; t += kStage) {
        uint8_t d[kStage];
#pragma unroll
        for (int k = 0; k < kStage; k++) d[k] = __ldg(done + (int64_t)(t + k) * N + i);
#pragma unroll
        for (int k = 0; k < kStage; k++) n_reset += d[k] != 0;
      }
      for (; t < H - 1; t++) n_reset += __ldg(done + (int64_t)t * N + i) != 0;
    }
    const int32_t b = begun[i];
    double R = (b - n_reset == seen[j]) ? ret[j] : 0.0;
    bool reset = pd != 0;
    Stage cur, nxt;
    load_stage(cur, reward, done, N, i, 0, H);
    for (int t0 = 0; t0 < H; t0 += kStage) {
      load_stage(nxt, reward, done, N, i, t0 + kStage, H);  // past the horizon: zeros, no loads
#pragma unroll
      for (int k = 0; k < kStage; k++) {
        if (t0 + k < H) {
          if (!reset) {
            R = R * gamma + (double)cur.r[k];
            const double d = R - shift;
            s1 += d;
            s2 += d * d;
            n += 1.0;
          }
          reset = cur.d[k] != 0;
          if (reset) R = 0.0;
        }
      }
      cur = nxt;
    }
    ret[j] = R;
    seen[j] = b;
  }
  red[0][threadIdx.x] = s1;
  red[1][threadIdx.x] = s2;
  red[2][threadIdx.x] = n;
  __syncthreads();
#pragma unroll
  for (int w = kThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
#pragma unroll
      for (int q = 0; q < 3; q++) red[q][threadIdx.x] += red[q][threadIdx.x + w];
    }
    __syncthreads();
  }
  if (threadIdx.x < 3) part[(size_t)blockIdx.x * 3 + threadIdx.x] = red[threadIdx.x][0];
}

// out[q] = sum over the CTAs, in order, of part[c][q]
__global__ void fx_return_final(const double* __restrict__ part, const int blocks, double* __restrict__ out) {
  const int q = threadIdx.x;
  if (q >= 3) return;
  double acc = 0.0;
  for (int c = 0; c < blocks; c++) acc += part[(size_t)c * 3 + q];
  out[q] = acc;
}

}  // namespace

cudaError_t fx_launch_return_moments(const float* reward, const uint8_t* done, const uint8_t* prev_done,
                                     const int32_t* begun, int num_envs, int horizon, int env_begin, int env_end,
                                     double gamma, double shift, double* ret, int32_t* seen, double* out,
                                     cudaStream_t stream) {
  const int blocks = (env_end - env_begin + kThreads - 1) / kThreads;
  double* part = nullptr;
  cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&part), (size_t)blocks * 3 * sizeof(double), stream);
  if (e != cudaSuccess) return e;
  fx_return_scan<<<blocks, kThreads, 0, stream>>>(reward, done, prev_done, begun, num_envs, horizon, env_begin, env_end,
                                                  gamma, shift, ret, seen, part);
  e = cudaGetLastError();
  if (e == cudaSuccess) {
    fx_return_final<<<1, 32, 0, stream>>>(part, blocks, out);
    e = cudaGetLastError();
  }
  const cudaError_t e2 = cudaFreeAsync(part, stream);
  return e != cudaSuccess ? e : e2;
}
