// fx_policy.cuh -- device-side parameters of the fused actor-critic policy kernel (fx_policy.cu) and its launcher.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define FX_POLICY_TILE_M 128   // env rows per CTA pair (two wgmma M = 64 warpgroups)
#define FX_POLICY_HIDDEN 256   // default hidden units of both layers (each CTA of a pair computes half = wgmma N)
#define FX_POLICY_ACTIONS 3

// fp32 parameters the epilogue reads directly (the two weight matrices travel as bf16 through TMA tensor maps);
// hidden = the policy's width (64, 128, 256 or 512).  A separate actor and critic (fx_launch_policy(separate)) stacks
// the two networks, actor first: b1 / b2 [2][hidden], h1 [rows][2 hidden] (the actor's columns first), head_part
// [rows][2] (one partial sum per network); head_w / head_b keep their layout (rows 0..2 the actor's, row 3 the critic's).
// A population of M members (fx_launch_policy(tiles_per_member)) stacks whole members, member-major: b1 / b2
// [M][nets][hidden], head_w [M][4][hidden], head_b [M][4]; h1 and head_part are per env row and keep their layout.
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
// sets the dynamic shared-memory limit of every width, action mode and network layout
cudaError_t fx_policy_configure();
// One policy evaluation for all envs: obs (bf16 [num_envs][k_pad], through map_obs) -> action / log-prob / value.
// hidden: the width of both layers (fx_policy_width_ok; otherwise cudaErrorInvalidValue, nothing launched).
// continuous = false: action int32 [num_envs]; noise float32 [num_envs][3] Gumbel(0,1).
// continuous = true:  action float32 [num_envs]; noise float32 [num_envs] N(0,1).
// noise == nullptr: the in-kernel counter-based generator (seed, step).  greedy: argmax / mean, noise unused.
// map_w1 / map_w2: boxes of hidden / 2 rows (one CTA's half of the hidden units); map_h1: over FxPolicyDev::h1
// ([rows][hidden]), box 128 rows.
// separate: separate actor and critic networks (the stacked layout of FxPolicyDev; map_w1 / map_w2 over 2 hidden rows,
// map_h1 over 2 hidden columns), two CTA pairs per tile.  It always runs in plain kernel order: tile_sync is ignored,
// because the actor pair's act_flag would not tell the step kernel that the critic pair has read the observation slot.
// tiles_per_member (>= 1, else cudaErrorInvalidValue): the 128-env tiles of each population member; the tile of envs
// [128 t, 128 t + 128) runs member t / tiles_per_member (the stacked layout of FxPolicyDev; map_w1 / map_w2 over all
// members' rows).  A value of at least the tile count is a single policy, member 0.
cudaError_t fx_launch_policy(const CUtensorMap& map_obs, const CUtensorMap& map_w1, const CUtensorMap& map_w2,
                             const CUtensorMap& map_h1, const FxPolicyDev& pol, int hidden, int num_envs, int k_pad,
                             const float* noise, unsigned long long seed, unsigned step, void* action, float* logp,
                             float* value, cudaStream_t stream, int env_begin, int env_end,  // env_begin: a multiple of FX_POLICY_TILE_M; env_end < 0: num_envs
                             bool tile_sync,  // true: wait for / publish per-tile flags (FxPolicyDev::act_flag ...)
                             bool continuous, bool greedy, bool separate, int tiles_per_member);

// fp32 [rows][cols] (nn.Linear layout) -> bf16 [rows][cols_pad], zero padded
cudaError_t fx_policy_pack(const float* src, uint16_t* dst, int rows, int cols, int cols_pad, cudaStream_t stream);
