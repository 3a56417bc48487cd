// fx_kernels.cu -- sm_90a kernels of the fused gym-fx env.step(): the host side (configuration, kernel choice,
// launches), the reset / observe / statistics kernels, and the step / rollout kernels of fx_env_step.cuh without
// truncation and per-env parameters (the other halves: fx_kernels_trunc.cu, fx_kernels_params.cu,
// fx_kernels_params_trunc.cu).
#include <cstdlib>

#include "fx_env_step.cuh"

namespace {

__global__ void fx_reset_kernel(const __grid_constant__ FxKernelParams P, const int64_t* __restrict__ start_bar,
                                const uint8_t* __restrict__ mask, int first) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  const FxConfig& c = P.cfg;
  if (env >= c.num_envs) return;
  const FxDeviceState& st = P.st;
  if (first) {  // plugin instances are brand new
    st.sh_len[env] = 0; st.sh_head[env] = 0; st.sh_last_step[env] = -1; st.dd_last_step[env] = -1;
    st.dd_peak[env] = 0.0;
  }
  if (mask && !mask[env]) return;
  fx_reset_env(P, env, start_bar ? start_bar[env] : st.start[env], start_bar == nullptr);
}

// writes the observation of the current state (what reset() returns): one warp per env.  NORM: the bf16 copy is the
// normalized one of `norm` (fx_observe_norm_kernel; obs16 is then never nullptr).
template <bool NORM>
__device__ __forceinline__ void fx_observe_body(const FxKernelParams& P, float* __restrict__ obs, uint16_t* __restrict__ obs16,
                                                const int stride16, const FxObsNorm* norm) {
  extern __shared__ __align__(16) unsigned char fx_smem[];
  const FxConfig& c = P.cfg;
  const FxDeviceState& st = P.st;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int env = blockIdx.x * FX_WARPS + warp;
  if (env >= c.num_envs) return;
  const int win_doubles = fx_window_doubles(c.window_size, c.n_cols);
  const WarpSmem ws = fx_carve(fx_smem + (size_t)warp * fx_warp_smem_bytes(win_doubles, 0), win_doubles, 0);
  const FxPairTable& tb = P.pair[env % c.num_pairs];
  FxEnvRegs e;
  e.equity = st.equity[env]; e.psize = st.psize[env]; e.price = st.price[env];
  e.position = st.position[env]; e.bar_index = st.bar_index[env];
  const int32_t total_bars = st.total_bars[env];
  const int64_t start = st.start[env];
  int s = e.bar_index;
  if (s < 1) s = 1;
  if (s > total_bars) s = total_bars;  // app/env.py:228
  float* row = obs + (int64_t)env * P.obs_dim;
  if constexpr (NORM) {
    const FxRow16N row16 = fx_norm_row(*norm, obs16, stride16, env);
    if (lane == 0) fx_write_scalars<false, FxRow16N>(P, e, total_bars, tb.candles[(start + s - 1) * (int64_t)c.n_cols + c.price_col], row, row16);
    fx_stream_windows<false, FxRow16N>(P, tb, env, lane, s, start, ws, row, row16);
  } else {
    uint16_t* row16 = obs16 ? obs16 + (int64_t)env * stride16 : nullptr;
    if (lane == 0) fx_write_scalars(P, e, total_bars, tb.candles[(start + s - 1) * (int64_t)c.n_cols + c.price_col], row, row16);
    fx_stream_windows<false>(P, tb, env, lane, s, start, ws, row, row16);
  }
}

__global__ void __launch_bounds__(FX_WARPS * 32) fx_observe_kernel(const __grid_constant__ FxKernelParams P, float* __restrict__ obs, uint16_t* __restrict__ obs16, const int stride16) {
  fx_observe_body<false>(P, obs, obs16, stride16, nullptr);
}

__global__ void __launch_bounds__(FX_WARPS * 32)
fx_observe_norm_kernel(const __grid_constant__ FxKernelParams P, float* __restrict__ obs, uint16_t* __restrict__ obs16,
                       const int stride16, const __grid_constant__ FxObsNorm norm) {
  fx_observe_body<true>(P, obs, obs16, stride16, &norm);
}

// Per-bar rolling z-score statistics (feature_window_preprocessor._scale_window :96-124 for a FULL window):
// stats[g][f] = {mean, 1/std} over rows (g-S, g], population std, std < 1e-8 -> 1.  One thread per (bar, feature).
__global__ void fx_stats_kernel(FxConfig c, const double* __restrict__ candles, double* __restrict__ stats, int64_t T) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int F = c.n_features, S = c.scaling_window, C = c.n_cols;
  if (idx >= T * F) return;
  const int64_t g = idx / F;
  const int f = (int)(idx - g * F);
  double m = 0.0, rc = 1.0;
  if (g + 1 >= S) {
    const double* p = candles + (g + 1 - S) * C + c.feature_cols[f];
    double acc = 0.0;
    for (int k = 0; k < S; k++) acc += p[(int64_t)k * C];
    m = acc / (double)S;
    double a2 = 0.0;
    for (int k = 0; k < S; k++) { const double d = p[(int64_t)k * C] - m; a2 += d * d; }
    double sd = sqrt(a2 / (double)S);
    if (sd < 1e-8) sd = 1.0;
    rc = 1.0 / sd;
  }
  stats[idx * 2 + 0] = m;
  stats[idx * 2 + 1] = rc;
}

size_t step_smem_bytes(const FxKernelParams& P) {
  const int ring_len = (P.cfg.reward == FX_REWARD_SHARPE) ? P.cfg.sharpe_window : 0;
  return fx_warp_smem_bytes(fx_window_doubles(P.cfg.window_size, P.cfg.n_cols), ring_len) * FX_WARPS;
}

int rollout_cta_warps(const FxKernelParams& P) { return FX_ROLLOUT_WARPS(P.order_smem != 0); }

// per CTA of fx_rollout_kernel, for the variant `resident`
size_t rollout_smem_bytes(const FxKernelParams& P, bool resident) {
  const int ring_len = (P.cfg.reward == FX_REWARD_SHARPE) ? P.cfg.sharpe_window : 0;
  const int tab = resident ? P.cap + FXO_SLACK : 0;
  return fx_warp_smem_bytes(fx_window_doubles(P.cfg.window_size, P.cfg.n_cols), ring_len, tab) * FX_ROLLOUT_WARPS(resident);
}

size_t observe_smem_bytes(const FxKernelParams& P) {
  return fx_warp_smem_bytes(fx_window_doubles(P.cfg.window_size, P.cfg.n_cols), 0) * FX_WARPS;
}

// shared-memory carve-out (percent of the SM's 228 KB) that holds `ctas` CTAs of `smem` bytes (+1 KB system use each)
int carveout_pct(size_t ctas, size_t smem) {
  const size_t want = ctas * (smem + 1024);
  int pct = (int)((want * 100 + 228 * 1024 - 1) / (228 * 1024));
  if (pct > 100) pct = 100;
  if (const char* cv = getenv("FXENV_CARVEOUT")) { const int v = atoi(cv); if (v >= pct && v <= 100) pct = v; }  // measurements
  return pct;
}

// The variant key (FX_V_*) of the handle's current settings: which step / rollout kernels a launch runs
unsigned fx_variant_key(const FxKernelParams& P) {
  unsigned key = 0u;
  if (P.fast_features == 5) key |= FX_V_FAST5;
  if (P.fast_features == 5 && P.lean) key |= FX_V_LEAN;
  if (P.order_smem) key |= FX_V_RESIDENT;
  if (P.audit != nullptr && P.cfg.strategy == FX_STRATEGY_ATR_SLTP) key |= FX_V_AUDIT;
  if (P.repeat > 1) key |= FX_V_REPEAT;
  if (fx_trunc_on(P)) key |= FX_V_TRUNC;
  if (P.env_params_off != 0u) key |= FX_V_PARAMS;
  return key;
}

// the lookup of each half, indexed by the half's FX_V_TRUNC | FX_V_PARAMS bits: this translation unit's part of the
// table, then the units that hold the others
static_assert(FX_V_PARAMS == 2 * FX_V_TRUNC, "a half's index is (key & FX_V_HALF) / FX_V_TRUNC");
FxEnvKernels (*const half_lookup[4])(int, int, unsigned) = {fx_variant_lookup<0u>, fx_trunc_kernels, fx_params_kernels,
                                                            fx_params_trunc_kernels};

FxEnvKernels env_kernels(const FxKernelParams& P, unsigned key) {
  return half_lookup[(key & FX_V_HALF) / FX_V_TRUNC](P.cfg.strategy, P.cfg.reward, key);
}

}  // namespace

// tests (fxenv_debug_variant_key, fxenv_debug_variant_exists): the key a launch on P runs, and whether the lookup has
// every kernel of a (strategy, reward, key)
unsigned fx_debug_variant_key(const FxKernelParams& P) { return fx_variant_key(P); }

bool fx_debug_variant_exists(int strategy, int reward, unsigned key) {
  FxKernelParams P = {};
  P.cfg.strategy = strategy;
  P.cfg.reward = reward;
  const FxEnvKernels k = env_kernels(P, key);
  return k.step != nullptr && k.step_norm != nullptr && k.rollout != nullptr;
}

// The resident-table rollout kernel when its CTAs fit an SM as many warps as the global-table one runs (16): each
// CTA at most 227 KB, and (16 / FX_ROLLOUT_WARPS(true)) CTAs plus their 1 KB reservations at most the SM's 228 KB.
// force: 0 / 1 = FXENV_ORDER_SMEM (measurements, tests), < 0 = decide by the budget.
int fx_order_smem_choice(const FxKernelParams& P, int force) {
  if (force >= 0) return force ? 1 : 0;
  const size_t cta = rollout_smem_bytes(P, true);
  const size_t ctas = (size_t)FX_ROLLOUT_MIN_BLOCKS * FX_WARPS / FX_ROLLOUT_WARPS(true);
  return (cta <= 227 * 1024 && ctas * (cta + 1024) <= 228 * 1024) ? 1 : 0;
}

// Attributes of one half of the step / rollout instantiations (half: its FX_V_TRUNC | FX_V_PARAMS bits) and the
// persistent grid: dynamic shared memory above the 48 KB default needs an explicit opt-in per kernel.  P.order_smem is
// decided.
cudaError_t fx_configure_half(FxKernelParams& P, unsigned half) {
  const size_t smem = step_smem_bytes(P), rsmem = rollout_smem_bytes(P, P.order_smem != 0);
  // ask for enough shared-memory carve-out that FX_MIN_BLOCKS CTAs (+1 KB system use each) fit on an SM
  const int pct = carveout_pct(FX_MIN_BLOCKS, smem);
  const int rcta = rollout_cta_warps(P);
  const int rpct = carveout_pct((size_t)FX_ROLLOUT_MIN_BLOCKS * FX_WARPS / rcta, rsmem);
  const int sms = P.num_sms;
  // every key of the handle's fast path and order-table choice: LEAN or not (which one runs is only known once the
  // candle tables are loaded), both states of the bracket audit (ATR strategy) and both states of the action repeat
  const unsigned fixed = FX_V_FAST5 | FX_V_RESIDENT | FX_V_TRUNC | FX_V_PARAMS;
  const unsigned want = (fx_variant_key(P) & (FX_V_FAST5 | FX_V_RESIDENT)) | half;
  for (unsigned key = 0u; key < FX_V_KEYS; key++) {
    if ((key & fixed) != want || !fx_variant_valid(P.cfg.strategy, key)) continue;
    const FxEnvKernels k = env_kernels(P, key);
    const FxStepKernelFn sk = k.step;
    const FxStepNormKernelFn nk = k.step_norm;
    const FxRolloutKernelFn rk = k.rollout;
    cudaError_t e = cudaFuncSetAttribute(sk, cudaFuncAttributePreferredSharedMemoryCarveout, pct);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(nk, cudaFuncAttributePreferredSharedMemoryCarveout, pct);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(rk, cudaFuncAttributePreferredSharedMemoryCarveout, rpct);
    if (e != cudaSuccess) return e;
    if (smem > 48 * 1024) {
      e = cudaFuncSetAttribute(sk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return e;
      e = cudaFuncSetAttribute(nk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return e;
    }
    if (rsmem > 48 * 1024) {
      e = cudaFuncSetAttribute(rk, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rsmem);
      if (e != cudaSuccess) return e;
    }
    // how many CTAs of the persistent rollout kernel the device holds at once (= its grid size).  The minimum over every
    // variant of the halves configured so far, the bracket audit's and the action repeat's included, whatever order the
    // halves were configured in: one grid size serves whichever variant a launch picks, so a change that raises those
    // kernels' registers or shared memory shrinks the grid with them off as well
    int per_sm = 0;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rk, rcta * 32, rsmem);
    if (e != cudaSuccess) return e;
    if (P.resident_blocks == 0 || sms * per_sm < P.resident_blocks) P.resident_blocks = sms * per_sm;
  }
  return P.resident_blocks < 1 ? cudaErrorInvalidConfiguration : cudaSuccess;
}

cudaError_t fx_configure_kernels(FxKernelParams& P) {
  const size_t smem = step_smem_bytes(P);
  if (smem > 227 * 1024) return cudaErrorInvalidValue;
  const char* os = getenv("FXENV_ORDER_SMEM");
  P.order_smem = fx_order_smem_choice(P, os ? atoi(os) : -1);
  if (rollout_smem_bytes(P, P.order_smem != 0) > 227 * 1024) return cudaErrorInvalidValue;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  P.num_sms = sms > 0 ? sms : 1;
  P.resident_blocks = 0;
  const cudaError_t e = fx_configure_half(P, 0u);
  if (e != cudaSuccess) return e;
  if (smem <= 48 * 1024) return cudaSuccess;
  const cudaError_t e2 = cudaFuncSetAttribute(fx_observe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)observe_smem_bytes(P));
  if (e2 != cudaSuccess) return e2;
  return cudaFuncSetAttribute(fx_observe_norm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)observe_smem_bytes(P));
}

// The LEAN contract of the specialised kernels (see fx_uses_running_stats): everything here is a property of the
// resolved configuration except `tame_data`, which is known once every pair's candle table has been loaded.  With a
// per-env table (rows_host) its rows' costs decide instead of the configuration's: the LEAN kernels leave commission,
// leverage and slippage out, and take only sl / tp / k_sl / k_tp from the row.
bool fx_config_is_lean(const FxKernelParams& P, const double* rows_host) {
  const FxConfig& c = P.cfg;
  if (P.fast_features != 5 || P.debug != 0 || !P.tame_data || P.any_binary) return false;
  if (c.action_mode != FX_ACTION_DISCRETE) return false;
  if (rows_host) {
    for (int i = 0; i < c.num_envs; i++) {
      const double* r = rows_host + (size_t)i * FXENV_ENV_PARAMS;
      if (r[FXENV_PARAM_COMMISSION] != 0.0 || r[FXENV_PARAM_LEVERAGE] != 1.0 || r[FXENV_PARAM_SLIPPAGE] != 0.0) return false;
    }
  } else if (c.commission != 0.0 || c.leverage != 1.0 || c.slippage_perc != 0.0) {
    return false;
  }
  if (c.children_same_bar || c.preproc != FX_PREPROC_FEATURE_WINDOW || c.scaling != FX_SCALING_ROLLING) return false;
  if (!(c.feature_clip > 0.0) || !c.include_price_window || !c.include_agent_state || (c.window_size & 3) || c.price_col > 4) return false;
  return true;
}

cudaError_t fx_launch_step(const FxKernelParams& P, const void* actions, float* obs, float* reward, double* reward64,
                           uint8_t* terminated, cudaStream_t stream, int env_begin, int env_end, uint16_t* obs16, int stride16,
                           const FxTileSync* sync, const FxObsNorm* norm) {
  if (env_end < 0) env_end = P.cfg.num_envs;
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3((env_end - env_begin + FX_WARPS - 1) / FX_WARPS);
  lc.blockDim = dim3(FX_WARPS * 32);
  lc.dynamicSmemBytes = step_smem_bytes(P);
  lc.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  lc.attrs = at;
  lc.numAttrs = (P.debug & 4) ? 0 : 1;  // FXENV_DEBUG & 4: plain stream-serialised launches (A/B timing only)
  const FxTileSync no_sync = {nullptr, nullptr, nullptr, 0};
  if (norm && obs16)
    return cudaLaunchKernelEx(&lc, env_kernels(P, fx_variant_key(P)).step_norm, P, actions, obs, reward, reward64, terminated,
                              env_begin, env_end, obs16, stride16, sync ? *sync : no_sync, *norm);
  return cudaLaunchKernelEx(&lc, env_kernels(P, fx_variant_key(P)).step, P, actions, obs, reward, reward64, terminated, env_begin,
                            env_end, obs16, stride16, sync ? *sync : no_sync);
}

int fx_rollout_blocks(const FxKernelParams& P) {
  const int w = rollout_cta_warps(P);
  int blocks = (P.cfg.num_envs + w - 1) / w;
  return blocks > P.resident_blocks ? P.resident_blocks : blocks;
}

int fx_rollout_warps(const FxKernelParams& P) { return fx_rollout_blocks(P) * rollout_cta_warps(P); }

// The rounds of a batch (FxChunkPlan): every ticket of round r is one env for the steps [start_r, start_{r+1}).  A longer
// chunk removes hand-overs (fence + sequence word + acquire round trip per ticket) but coarsens the work units: uniform chunks that leave >= 6 tickets per resident warp, at most 64 steps, the remainder as a
// shorter last round.  Uniform rounds dealt in env order are work-conserving: an env's previous ticket finished
// (N - warps) tickets ago, so nobody waits.  (Rounds that shrink towards the end of the batch -- "guided" scheduling, to
// shorten the tail in which warps run dry -- cost more in extra hand-overs than they save in the tail.)  When every env has a warp of its own the whole batch is
// one round: no hand-over at all.  FXENV_CHUNK=c forces chunks of c steps (measurements, tests).
// With the action repeat (P.repeat = k > 1) a step spans up to k bars: the 64-step bound becomes a bound of 64 bars,
// max(1, 64 / k) decisions, so that a ticket -- and the batch's tail -- is no longer than without the repeat.
FxChunkPlan fx_rollout_plan(const FxKernelParams& P, int n_steps) {
  const char* fe = getenv("FXENV_CHUNK");  // read per launch: tests switch it between batches
  const int forced = fe ? atoi(fe) : 0;
  const long long warps = fx_rollout_warps(P);
  const long long N = P.cfg.num_envs;
  const int max_chunk = P.repeat > 1 ? (64 / P.repeat > 1 ? 64 / P.repeat : 1) : 64;
  int chunk;
  if (forced > 0) chunk = forced;
  else if (N <= warps) chunk = n_steps;
  else { chunk = (int)((N * (long long)n_steps) / (warps * 6)); if (chunk > max_chunk) chunk = max_chunk; }
  if (chunk < 1) chunk = 1;
  if (chunk > n_steps) chunk = n_steps;
  FxChunkPlan pl = {};
  pl.chunk = chunk;
  pl.n_uniform = n_steps / chunk;
  pl.n_rounds = pl.n_uniform;
  pl.tail_start[0] = pl.n_uniform * chunk;
  if (pl.tail_start[0] < n_steps) { pl.tail_start[1] = n_steps; pl.n_rounds++; }  // the remainder: one shorter round
  return pl;
}

// seq_base / ticket_base: the values seq[] and the ticket counter hold when this launch starts (see fx_rollout_kernel);
// reset_words: zero them first with a stream-ordered memset (then both bases must be 0) -- used inside stream captures,
// where the host cannot track what the counters will hold at replay time.
cudaError_t fx_launch_rollout(const FxKernelParams& P, const void* actions, float* obs, int obs_slots, float* reward,
                              uint8_t* terminated, const FxChunkPlan& plan, unsigned seq_base, unsigned ticket_base,
                              bool reset_words, cudaStream_t stream) {
  const int N = P.cfg.num_envs;
  if (reset_words) {
    cudaError_t e = cudaMemsetAsync(P.seq, 0, ((size_t)N + 1) * sizeof(int32_t), stream);
    if (e != cudaSuccess) return e;
  }
  cudaLaunchConfig_t lc = {};
  lc.gridDim = dim3(fx_rollout_blocks(P));
  lc.blockDim = dim3(rollout_cta_warps(P) * 32);
  lc.dynamicSmemBytes = rollout_smem_bytes(P, P.order_smem != 0);
  lc.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  lc.attrs = at;
  lc.numAttrs = (reset_words || (P.debug & 4)) ? 0 : 1;  // behind a memset node: plain stream order
  return cudaLaunchKernelEx(&lc, env_kernels(P, fx_variant_key(P)).rollout, P, reinterpret_cast<const char*>(actions), obs,
                            obs_slots, reward, terminated, plan, seq_base, ticket_base);
}

cudaError_t fx_launch_reset(const FxKernelParams& P, const int64_t* start_bar, const uint8_t* mask, int first,
                            cudaStream_t stream) {
  const int N = P.cfg.num_envs;
  fx_reset_kernel<<<(N + 127) / 128, 128, 0, stream>>>(P, start_bar, mask, first);
  return cudaGetLastError();
}

cudaError_t fx_launch_observe(const FxKernelParams& P, float* obs, cudaStream_t stream, uint16_t* obs16, int stride16,
                              const FxObsNorm* norm) {
  const int N = P.cfg.num_envs;
  if (norm && obs16)
    fx_observe_norm_kernel<<<(N + FX_WARPS - 1) / FX_WARPS, FX_WARPS * 32, observe_smem_bytes(P), stream>>>(P, obs, obs16, stride16, *norm);
  else
    fx_observe_kernel<<<(N + FX_WARPS - 1) / FX_WARPS, FX_WARPS * 32, observe_smem_bytes(P), stream>>>(P, obs, obs16, stride16);
  return cudaGetLastError();
}

cudaError_t fx_launch_stats(const FxConfig& cfg, const double* candles, double* stats, int64_t T, cudaStream_t stream) {
  const int64_t total = T * cfg.n_features;
  const int threads = 128;
  fx_stats_kernel<<<(unsigned)((total + threads - 1) / threads), threads, 0, stream>>>(cfg, candles, stats, T);
  return cudaGetLastError();
}
