// fx_kernels.cuh -- device-side data layout shared by the kernels (fx_env_step.cuh, fx_kernels.cu) and fx_capi.cu
// (C-ABI host code).
#pragma once

#include "fx_core.cuh"

// One candle table per currency pair, resident in HBM (and, at benchmark sizes, in the 50 MB L2):
//   candles  float64 [T][n_cols] row-major (AoS rows: a W-row window of all columns is ONE contiguous span,
//            so the flat [W][F] observation block maps 1:1 onto a contiguous read when F == n_cols)
//   stats    float64 [T][F][2] = {mean, 1/std} of the rolling z-score window ENDING at that bar (precomputed at
//            load for every bar that has a full window behind it; pure function of the bar, SURVEY A.6)
//   minutes  int64 [T] minutes since the Unix epoch (session filter only) or nullptr
struct FxPairTable {
  const double* candles;
  const double* stats;
  const int64_t* minutes;
  int64_t T;
};

// Per-env state: struct-of-arrays over N envs.  The info columns of the C-ABI (FxInfoPtrs) point straight in here.
// Invariants at kernel boundaries: bar_index == t + 1, position == sign(psize), price == CLOSE[start + t], and the
// broker's cached value == equity -- so the step kernel only LOADS cash/psize/pprice/equity (+ counters) and
// re-derives the rest; prev_equity / price / position / bar_index are stored for the info columns.
struct FxDeviceState {
  double *cash, *psize, *pprice;                          // broker: cash, position size / average price
  double *equity, *prev_equity, *price, *commission_paid; // bridge (app/bt_bridge.py:30-66)
  double* dd_peak;                                        // dd_penalized_reward._peak
  double* sub_need;                                       // check_submitted cash bound of the entries [n_acc, n_orders)
  double* nbar;                                           // [N][6] {open, high, low, close, price_col value, -} of the candle the NEXT step call
                                                          // works on (row min(t+1, total_bars-1), or row t right after a reset): saves the
                                                          // dependent cursor -> candle round trip at the head of every step
  int64_t* start;                                         // first bar (table row) of the episode window
  int32_t *t, *total_bars, *position, *bar_index, *trades, *n_orders, *n_acc;
  int32_t *sh_len, *sh_head, *sh_last_step, *dd_last_step;
  uint32_t* flags;
  double* rstats;    // [N][FX_RS_N] end-of-run statistics: DrawDown / TradeAnalyzer / SQN state (fx_core.cuh FX_RS_*)
  double* sh_ring;   // [N][sharpe_window]
  double* welford;   // [N][FXENV_MAX_FEATURES][2] running {mean, M2} of each feature column over rows [0, s)
  uint32_t* o_meta;  // [N][cap + FXO_SLACK]  order table, entry-major per env (a warp scans one env coalesced)
  double *o_p0, *o_p1, *o_sz;
  // episode starts / records (fxenv_set_reset_starts, fxenv_get_episode_info; fx_episode_begin): in the slab rather
  // than in FxKernelParams, so that snapshots carry them and the cached graphs (P captured by value) stay valid
  int64_t* ep_lo;      // [N] first start bar of the range
  uint64_t* ep_span;   // [N] hi - lo + 1; 0 = no range: an episode restarts at its current start
  uint64_t* ep_seed;   // [1]
  int32_t* ep_begun;   // [N] episodes begun since create (the k of the next draw)
  int32_t* ep_done;    // [N] episodes recorded
  double* ep_last;     // [N][FXENV_EPISODE_STATS] record of the last finished episode
};

#define FX_NSTAMP 12

// How fx_rollout_kernel cuts the steps [0, n_steps) of a batch into rounds (one ticket = one env for the steps of one
// round): n_uniform rounds of `chunk` steps, then rounds [tail_start[i], tail_start[i + 1]); n_rounds in total.
#define FX_PLAN_TAIL 7
struct FxChunkPlan {
  int32_t chunk, n_uniform, n_rounds;
  int32_t tail_start[FX_PLAN_TAIL + 1];
};

struct FxKernelParams {
  FxConfig cfg;
  FxPairTable pair[FXENV_MAX_PAIRS];
  FxDeviceState st;
  double inv_initial_cash;  // 1 / (initial_cash or 1.0)
  int32_t* seq;             // [N + 1] per-env sequence words of a fxenv_step_many batch + the ticket counter (fx_rollout_kernel)
  long long* timing;        // debug (FXENV_TIMING=1): [N][FX_NSTAMP] clock64() phase stamps of the last step, else nullptr
  long long* timeline;      // debug (FXENV_TIMELINE=K, timing build): [K][N][2] globaltimer at start / end of every ticket
  int32_t obs_dim;
  int32_t cap;              // logical order-table capacity (multiple of 32); arrays hold cap + FXO_SLACK
  int32_t debug;            // timing experiments only (env FXENV_DEBUG, bit mask): 1 skip obs windows, 2 skip broker /
                            // strategy / reward, 4 plain launches (no programmatic dependent launch), 8 step_many always as
                            // the graph of single steps, 16 step_many always as the persistent launch
  int32_t resident_blocks;  // CTAs of the persistent rollout kernel resident at once on this device (SMs x occupancy)
  int32_t tame_data;        // 1: every loaded table value is finite and |x| < 1e100 (no NaN can arise in a z-score)
  int32_t fast_features;    // 5: F == n_cols == 5 with identity columns (the [W][5] block is one contiguous span)
  int32_t any_binary;       // 1: some feature column is a binary pass-through (feature_binary[])
  int32_t lean;             // 1: the configuration qualifies for the specialised kernels (fx_config_is_lean)
  int32_t num_sms;          // SMs of the device (fx_rollout_kernel: CTA b is the (b / num_sms)-th CTA of its SM)
  int32_t order_smem;       // 1: fx_rollout_kernel keeps each ticket's order table in shared memory (fx_order_smem_choice)
  // bracket audit (fxenv_set_bracket_audit): [N][audit_cap][FXENV_AU_FIELDS] ring and [N] record counters, or nullptr
  // (log off).  Outside the state slab: snapshots and the slab layout do not depend on the log.
  double* audit;
  int64_t* audit_written;
  int32_t audit_cap;
  // action repeat (fxenv_set_action_repeat): substeps per step (1 = off: the kernels without repeat run) and the
  // FXENV_REPEAT_* flags.  A setting of the handle, not env state: outside the slab, like the audit.
  int32_t repeat;
  uint32_t repeat_flags;
  // time limit (fxenv_set_time_limit): decisions per episode (0 = no limit) and the FXENV_TIME_LIMIT_* flags.  A setting
  // of the handle like the repeat; while either is set the host launches the truncation instantiations (fx_trunc_on).
  int32_t max_steps;
  uint32_t trunc_flags;
  // per-env broker and strategy values (fxenv_set_env_params): byte offset of the [N][FXENV_ENV_PARAMS] FxEnvParams rows
  // in the allocation of `seq` (fx_env_params), or 0 (off: the FxConfig values; the kernels without FX_V_PARAMS run).  A
  // setting of the handle outside the slab, like the audit.  An offset in the 4 bytes of padding before ep_steps rather
  // than a pointer of its own: a new 8-byte field would grow the kernel parameters and move every kernel argument after
  // them, changing the code of every existing kernel.  The table stays put while it is on, so that cached graphs read
  // values updated in place.
  uint32_t env_params_off;
  // [N] decisions of the current episode (a column of the state slab, so snapshots carry it; zeroed by fx_reset_env).
  // Addressed from here rather than from FxDeviceState so that no existing kernel parameter moves.
  int32_t* ep_steps;
};

__host__ __device__ inline bool fx_trunc_on(const FxKernelParams& P) { return P.max_steps > 0 || P.trunc_flags != 0u; }

// the per-env parameter table while it is on (env_params_off != 0)
__host__ __device__ inline const double* fx_env_params(const FxKernelParams& P) {
  return reinterpret_cast<const double*>(reinterpret_cast<const char*>(P.seq) + P.env_params_off);
}

// warps (= envs) per CTA of the step kernel.  One warp per CTA lets the second wave back-fill SM slots as soon as a
// single env finishes.
#ifndef FX_WARPS
#define FX_WARPS 1
#endif
// CTAs per SM the step kernel is compiled for: 16 warps per SM caps the registers at 128 (the sm_90a build spills
// 36-160 bytes per kernel).  Measured on one H100 SXM (700 W), bench.py --steps 1000, us/step with 16 / 12 CTAs per SM
// (12: 154 registers, no spills): cfg2 9.10 / 10.06, closed loop (cfg4) 45.7 / 47.9, cfg3 64.7 / 59.9, cfg5 91.1 / 85.3.
// The long-window shapes prefer fewer, spill-free warps; the 128-window shapes prefer occupancy.
#ifndef FX_MIN_BLOCKS
#define FX_MIN_BLOCKS (16 / FX_WARPS)   // 16 warps per SM => 128 registers
#endif
// warps per CTA of fx_rollout_kernel: with the order table resident in shared memory (13.7 KB per warp for W=128 and
// 256 orders), 4 warps share one 1 KB per-CTA reservation, so that 16 warps still fit an SM's 228 KB
#ifndef FX_RES_WARPS
#define FX_RES_WARPS 4
#endif
#define FX_ROLLOUT_WARPS(resident) ((resident) ? FX_RES_WARPS : FX_WARPS)

// host-callable launchers (fx_kernels.cu)
// one step of the envs [env_begin, env_end) (env_end < 0: all); the array arguments are the bases for env 0
// Fine-grained hand-over between the policy kernel and the env-step kernel of a closed-loop rollout (fxenv_rollout), per
// 128-env tile, instead of whole-kernel dependencies: the step kernel of step t starts an env as soon as the policy has
// published the tile's actions (act_flag[tile] >= t + 1), and the policy kernel of step t + 1 starts a tile as soon as
// its envs have finished step t (done_cnt[tile] == envs of the tile x (t + 1)).  Both kernels are launched with the
// programmatic-dependent-launch attribute and are resident together; a dependent grid is only launched once every CTA
// of its predecessor has started, so whoever is waited for is always running.  nullptr members: plain kernel order.
struct FxTileSync {
  int32_t* act_flag;   // [tiles] written by the policy kernel (release), polled by the step kernel (acquire)
  int32_t* done_cnt;   // [tiles] incremented by the step kernel (release), polled by the policy kernel (acquire)
  int32_t* timeouts;   // [1] number of polls that gave up (a bug or a lost launch: results are then invalid; tests assert 0)
  int32_t epoch;       // t + 1
};
#define FX_SYNC_TILE 128
#define FX_SYNC_MAX_POLLS (1 << 22)   // x ~64 ns: a poll gives up after ~0.3 s instead of hanging the device  // obs16: optional bf16 copy of the rows

// Observation normalizer of a closed-loop policy (fxenv_policy_set_obs_norm): every element the env kernels write to the
// bf16 copy becomes bf16_rn(clamp((x - mean) * rstd, -clip, clip)) with the statistics of the env's population member
// m = env / member_envs and pair p = env % num_pairs.  mean / rstd: float32 [members][num_pairs][stride16] (the bf16 row
// stride, so that a row of statistics is 16-byte aligned wherever a row of the copy is 8-byte aligned); clip: [members].
struct FxObsNorm {
  const float* mean;
  const float* rstd;
  const float* clip;
  int32_t member_envs;
  int32_t num_pairs;
};

// norm (with obs16 only): the normalized variant of the bf16 copy -- separate kernels, so that the plain ones are unchanged
cudaError_t fx_launch_step(const FxKernelParams& P, const void* actions, float* obs, float* reward, double* reward64,
                           uint8_t* terminated, cudaStream_t stream, int env_begin = 0, int env_end = -1,
                           uint16_t* obs16 = nullptr, int stride16 = 0, const FxTileSync* sync = nullptr,
                           const FxObsNorm* norm = nullptr);

cudaError_t fx_launch_reset(const FxKernelParams& P, const int64_t* start_bar, const uint8_t* mask, int first,
                            cudaStream_t stream);
cudaError_t fx_launch_observe(const FxKernelParams& P, float* obs, cudaStream_t stream, uint16_t* obs16 = nullptr,
                              int stride16 = 0, const FxObsNorm* norm = nullptr);
// Shifted column moments of rows [slots][num_envs][D] restricted to the envs [env_begin, env_end), by pair (env %
// num_pairs): out[p][0][j] = sum (x - shift[p][j]), out[p][1][j] = sum (x - shift[p][j])^2, in float64, in an order fixed
// by the shapes alone (fx_obs_stats.cu)
cudaError_t fx_launch_obs_moments(const float* obs, int slots, int num_envs, int D, int num_pairs, int env_begin, int env_end,
                                  const float* shift, double* out, cudaStream_t stream);
cudaError_t fx_launch_stats(const FxConfig& cfg, const double* candles, double* stats, int64_t T, cudaStream_t stream);
cudaError_t fx_configure_kernels(FxKernelParams& P);
// the same for the kernel half `half` (its FX_V_TRUNC | FX_V_PARAMS bits, see below); the halves with either bit are
// deferred to the first setter that turns the bit on, so that a handle that never does never loads their modules
cudaError_t fx_configure_half(FxKernelParams& P, unsigned half);
// rows_host: the per-env table ([N][FXENV_ENV_PARAMS]) whose costs decide instead of the config's, or nullptr
bool fx_config_is_lean(const FxKernelParams& P, const double* rows_host = nullptr);
cudaError_t fx_launch_rollout(const FxKernelParams& P, const void* actions, float* obs, int obs_slots, float* reward,
                              uint8_t* terminated, const FxChunkPlan& plan, unsigned seq_base, unsigned ticket_base,
                              bool reset_words, cudaStream_t stream);
int fx_rollout_blocks(const FxKernelParams& P);
int fx_rollout_warps(const FxKernelParams& P);  // warps of a fx_rollout_kernel launch (each draws one ticket past the last)
int fx_order_smem_choice(const FxKernelParams& P, int force);

// The variant key of the step / rollout kernels (DESIGN §4, "The variant key"): one bit per compile-time switch of
// fx_step_env, chosen from the handle by fx_variant_key (fx_kernels.cu).
enum : unsigned {
  FX_V_FAST5 = 1u,     // the 5-feature fast path (fast_features == 5)
  FX_V_LEAN = 2u,      // the LEAN specialisation (lean, fx_config_is_lean)
  FX_V_RESIDENT = 4u,  // the order table resident in shared memory (order_smem)
  FX_V_AUDIT = 8u,     // the bracket audit store (fxenv_set_bracket_audit)
  FX_V_REPEAT = 16u,   // the action repeat (fxenv_set_action_repeat, repeat > 1)
  FX_V_TRUNC = 32u,    // decision counts and truncation (fxenv_set_time_limit, fx_trunc_on)
  FX_V_PARAMS = 64u,   // per-env broker and strategy values (fxenv_set_env_params, env_params_off)
  FX_V_KEYS = 128u
};
enum { FX_N_STRATEGIES = FX_STRATEGY_ATR_SLTP + 1, FX_N_REWARDS = FX_REWARD_DD + 1 };
// The keys that have kernels: LEAN needs the fast path and the audit the ATR strategy.  (FX_V_RESIDENT selects a rollout
// kernel only: the step kernel ignores it.)
constexpr bool fx_variant_valid(int strategy, unsigned key) {
  return ((key & FX_V_LEAN) == 0u || (key & FX_V_FAST5) != 0u) &&
         ((key & FX_V_AUDIT) == 0u || strategy == FX_STRATEGY_ATR_SLTP);
}

typedef void (*FxStepKernelFn)(const FxKernelParams, const void*, float*, float*, double*, uint8_t*, int, int, uint16_t*, int,
                               const FxTileSync);
typedef void (*FxRolloutKernelFn)(const FxKernelParams, const char*, float*, int, float*, uint8_t*, const FxChunkPlan, unsigned,
                                  unsigned);
typedef void (*FxStepNormKernelFn)(const FxKernelParams, const void*, float*, float*, double*, uint8_t*, int, int, uint16_t*,
                                   int, const FxTileSync, const FxObsNorm);
struct FxEnvKernels {
  FxStepKernelFn step;
  FxRolloutKernelFn rollout;
  FxStepNormKernelFn step_norm;  // the step kernel with the normalized bf16 copy (fx_step_norm_kernel)
};
// The kernels are split over four translation units by the two bits FX_V_TRUNC and FX_V_PARAMS (the "half" of a key):
// fx_kernels.cu holds the keys with neither, fx_kernels_trunc.cu those with FX_V_TRUNC only, fx_kernels_params.cu those
// with FX_V_PARAMS only and fx_kernels_params_trunc.cu those with both.
FxEnvKernels fx_trunc_kernels(int strategy, int reward, unsigned key);
FxEnvKernels fx_params_kernels(int strategy, int reward, unsigned key);
FxEnvKernels fx_params_trunc_kernels(int strategy, int reward, unsigned key);
FxChunkPlan fx_rollout_plan(const FxKernelParams& P, int n_steps);  // the host's ticket accounting needs n_rounds
// tests: fx_variant_key(P), and whether the lookup has a step, a step-norm and a rollout kernel for the triple
// (strategy < FX_N_STRATEGIES, reward < FX_N_REWARDS, key < FX_V_KEYS)
unsigned fx_debug_variant_key(const FxKernelParams& P);
bool fx_debug_variant_exists(int strategy, int reward, unsigned key);
