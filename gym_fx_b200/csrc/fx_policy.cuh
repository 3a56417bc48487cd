// fx_policy.cuh -- device-side parameters of the fused actor-critic policy kernel (fx_policy.cu) and its launcher.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define FX_POLICY_TILE_M 128   // env rows per CTA pair (two wgmma M = 64 warpgroups)
#define FX_POLICY_HIDDEN 256   // default hidden units of both layers (each CTA of a pair computes half = wgmma N)
#define FX_POLICY_ACTIONS 3

// fp32 parameters the epilogue reads directly (the two weight matrices travel as bf16 through TMA tensor maps);
// hidden = the policy's width (64, 128, 256 or 512)
struct FxPolicyDev {
  const float* b1;      // [hidden]
  const float* b2;      // [hidden]
  const float* head_w;  // [4][hidden]: rows 0..2 = actor head (one per action; continuous: row 0 = mean), row 3 = critic
  const float* head_b;  // [4] (continuous: {b_mu, log sigma, 0, b_v})
  uint16_t* h1;         // scratch, bf16 [num_envs rounded up to whole tiles][hidden]: where the two halves of h1 meet
  float4* head_part;    // scratch, [num_envs rounded up to whole tiles]: rank 1's partial head sums
  long long* dbg;       // timing build only (FXENV_TIMELINE): kernel-chain log, else nullptr
  // per-tile hand-over with the env-step kernel (FxTileSync in fx_kernels.cuh; nullptr: plain kernel order)
  int32_t* act_flag;    // [tiles]: set to step + 1 when the tile's actions are stored
  const int32_t* done_cnt;  // [tiles]: env-steps completed, counted by the step kernel
  int32_t* timeouts;    // [1]
};

// the hidden widths the kernel is instantiated for: 64, 128, 256, 512
bool fx_policy_width_ok(int hidden);
// dynamic shared memory of one policy CTA at that width (0 for an unsupported width)
size_t fx_policy_smem_bytes(int hidden);
// sets the dynamic shared-memory limit of every width and action mode
cudaError_t fx_policy_configure();
// One policy evaluation for all envs: obs (bf16 [num_envs][k_pad], through map_obs) -> action / log-prob / value.
// hidden: the width of both layers (fx_policy_width_ok; otherwise cudaErrorInvalidValue, nothing launched).
// continuous = false: action int32 [num_envs]; noise float32 [num_envs][3] Gumbel(0,1).
// continuous = true:  action float32 [num_envs]; noise float32 [num_envs] N(0,1).
// noise == nullptr: the in-kernel counter-based generator (seed, step).  greedy: argmax / mean, noise unused.
// map_w1 / map_w2: boxes of hidden / 2 rows (one CTA's half of the hidden units); map_h1: over FxPolicyDev::h1
// ([rows][hidden]), box 128 rows.
cudaError_t fx_launch_policy(const CUtensorMap& map_obs, const CUtensorMap& map_w1, const CUtensorMap& map_w2,
                             const CUtensorMap& map_h1, const FxPolicyDev& pol, int hidden, int num_envs, int k_pad,
                             const float* noise, unsigned long long seed, unsigned step, void* action, float* logp,
                             float* value, cudaStream_t stream, int env_begin = 0, int env_end = -1,  // env_begin: a multiple of FX_POLICY_TILE_M
                             bool tile_sync = false,  // true: wait for / publish per-tile flags (FxPolicyDev::act_flag ...)
                             bool continuous = false, bool greedy = false);

// fp32 [rows][cols] (nn.Linear layout) -> bf16 [rows][cols_pad], zero padded
cudaError_t fx_policy_pack(const float* src, uint16_t* dst, int rows, int cols, int cols_pad, cudaStream_t stream);
