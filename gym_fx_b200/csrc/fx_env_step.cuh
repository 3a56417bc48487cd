// fx_env_step.cuh -- sm_90a kernels of the fused gym-fx env.step(): the step and rollout kernel templates, instantiated
// through fx_variant_lookup by fx_kernels.cu, fx_kernels_trunc.cu, fx_kernels_params.cu and fx_kernels_params_trunc.cu
// (the variants without / with truncation and per-env parameters, see fx_kernels.cuh).
//
// fx_step_env<STRATEGY, REWARD, V> is the whole env-step of ONE env by ONE warp (no block barrier anywhere):
//
//   load     one round trip: the env's state scalars (fx_step_load), its action, the candle of this step (saved by the
//            previous step) and the first 32 orders of its table;
//   prefetch lane 0 issues TMA bulk copies (cp.async.bulk + mbarrier) of the env's candle window (W rows x n_cols fp64,
//            one contiguous span of the table) and of the bar's z-score statistics into the warp's shared memory;
//            they land while the broker runs;
//   broker   backtrader's per-bar pass as ONE streaming sweep over the env's order table, 32 orders (one per lane) at
//            a time in registers with the next chunk in flight: bracket activation + trigger test and execution price
//            per lane (ballot), the few orders that trade are executed in FIFO order by uniform scalar fp64 code
//            (fx_core.cuh) with their fields broadcast by shuffle, then stable compaction + write-back of what
//            changed.  check_submitted is decided by a rigorous cash bound (the exact sequential simulation is a cold
//            path).  Then the drawdown analyzer (fx_step_drawdown), apply_action, publish, reward (fx_step_reward),
//            write-back;
//   observe  the observation row ([W,F] z-scored features | prices | returns | 4 agent scalars) is produced from the
//            staged window: fp64 math, coalesced fp32 streaming stores (>99% of the bytes).
//
// Two kernels wrap it: fx_step_kernel (one launch = one step of all N envs, one env per one-warp CTA, programmatic
// dependent launch) and fx_rollout_kernel (one launch = K steps: persistent warps pull (step, env) tickets and only
// honour per-env dependencies).  Both are compiled once per (strategy, reward, variant key FX_V_*) so each instance
// only carries the code its configuration can reach.  No tensor cores: there is no contraction on this path.
//
// Reference call stack being replaced: app/env.py:131-172 -> app/bt_bridge.py:119-150 -> strategy / reward /
// preprocessor plugins + backtrader (per-function citations in fx_core.cuh).
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <utility>

#include "fx_kernels.cuh"

#define FX_FULL 0xffffffffu
#ifndef FX_LONG_UNROLL
#define FX_LONG_UNROLL 2   // unroll factor of the 16-byte emit loop for long windows
#endif
#ifndef FX_LONG_MIN_W
#define FX_LONG_MIN_W 384  // windows of at least this many rows use the unrolled loop
#endif
constexpr int kLongUnroll = FX_LONG_UNROLL;  // (a macro is not expanded inside #pragma unroll)

namespace {

// per-warp shared memory: the TMA-staged candle window + z-score statistics (+ the Sharpe ring) + one mbarrier
// (+ the env's order table in the resident-table rollout kernel)
struct WarpSmem {
  double *win, *stat, *ring;  // stat: [F][2] = {mean, 1/std} per feature (the layout of the per-bar statistics table)
  double* carry;              // FX_CARRY_*: the env's scalar state between two steps run by the same warp (fx_rollout_kernel)
  double *op0, *op1, *osz;    // [cap + FXO_SLACK] each: the order table of the env a ticket owns (RESIDENT), else unused
  uint32_t* ometa;
  unsigned long long* bar;
};

// Carry record (8-byte slots): what the next env-step loads in its first round trip.  A warp that keeps an env for several
// consecutive steps (a ticket of fx_rollout_kernel) reads it here instead of from the state arrays in global memory --
// which are still written every step -- and so starts its broker pass one L2 round trip earlier.
enum {
  FX_CARRY_CASH = 0, FX_CARRY_PSIZE, FX_CARRY_PPRICE, FX_CARRY_EQUITY, FX_CARRY_COMM, FX_CARRY_SUBNEED,
  FX_CARRY_NBAR,                       // 5 slots: o, h, l, c, price column of the candle the next step works on
  FX_CARRY_FLAGS_T = FX_CARRY_NBAR + 5, // int2 {flags, t}
  FX_CARRY_BARS_N,                     // int2 {total_bars, n_orders}
  FX_CARRY_NACC_TRADES,                // int2 {n_acc, trades}
  FX_CARRY_START,                      // int64
  FX_CARRY_SHARPE,                     // int2 {deque length, head}; the deque itself stays in WarpSmem::ring
  FX_CARRY_SHARPE_LAST,                // int2 {last step seen by the Sharpe plugin, table bound (fx_carry_tab_hi)}
  FX_CARRY_RSTATS,                     // FX_RS_N slots
  FX_CARRY_N = FX_CARRY_RSTATS + FX_RS_N
};

// RESIDENT: entries [0, hi) of the warp's copy of the order table may differ from global memory (the second int32 of an
// existing slot: the layout of the other kernels stays as it is)
__device__ __forceinline__ int32_t* fx_carry_tab_hi(double* carry) {
  return reinterpret_cast<int32_t*>(carry + FX_CARRY_SHARPE_LAST) + 1;
}

// FX_V_TRUNC: the carried decision count of the episode (the carry record's extra field) lives in the second half of the
// 16 bytes fx_warp_smem_bytes reserves for the 8-byte mbarrier, so that the slice -- and the kernels without truncation
// -- keep their size
__device__ __forceinline__ int32_t* fx_carry_dec(const WarpSmem& ws) { return reinterpret_cast<int32_t*>(ws.bar + 1); }

__host__ __device__ inline int fx_window_doubles(int W, int C) { return (W * C + 2 + 1) & ~1; }  // +1 alignment, even

// tab_entries: cap + FXO_SLACK for the resident-table rollout kernel, else 0 (a multiple of 32: 28 B per entry keep the
// mbarrier 8-byte aligned)
__host__ __device__ inline size_t fx_warp_smem_bytes(int win_doubles, int ring_len, int tab_entries = 0) {
  size_t b = (size_t)win_doubles * 8 + 2 * FXENV_MAX_FEATURES * 8 + (size_t)ring_len * 8 + FX_CARRY_N * 8 +
             (size_t)tab_entries * (3 * 8 + 4) + 16;
  return (b + 15) & ~(size_t)15;
}

__device__ __forceinline__ WarpSmem fx_carve(unsigned char* base, int win_doubles, int ring_len, int tab_entries = 0) {
  WarpSmem w;
  double* d = reinterpret_cast<double*>(base);
  w.win = d; d += win_doubles;
  w.stat = d; d += 2 * FXENV_MAX_FEATURES;
  w.ring = d; d += ring_len;
  w.carry = d; d += FX_CARRY_N;
  w.op0 = d; d += tab_entries;
  w.op1 = d; d += tab_entries;
  w.osz = d; d += tab_entries;
  w.ometa = reinterpret_cast<uint32_t*>(d);
  w.bar = reinterpret_cast<unsigned long long*>(w.ometa + tab_entries);
  return w;
}

// entries [0, n) of an order table from one copy to the other (global <-> the warp's shared memory), coalesced
__device__ __forceinline__ void fx_table_copy(uint32_t* __restrict__ dm, double* __restrict__ d0, double* __restrict__ d1,
                                              double* __restrict__ ds, const uint32_t* __restrict__ sm,
                                              const double* __restrict__ s0, const double* __restrict__ s1,
                                              const double* __restrict__ ss, const int n, const int lane) {
#pragma unroll 4
  for (int k = lane; k < n; k += 32) { dm[k] = sm[k]; d0[k] = s0[k]; d1[k] = s1[k]; ds[k] = ss[k]; }
}

// ---- TMA (cp.async.bulk) staging of the env's candle window: rows [left, s) of its episode, one contiguous span ----
// fx_window_init (lane 0, at kernel top so that the init fence overlaps the state loads) arms the warp's mbarrier;
// fx_window_issue starts the bulk copy and returns the element shift (0/1) that makes the global source 16-byte
// aligned; fx_window_wait blocks until the bytes have landed.  The table is allocated with 32 B of tail padding.
__device__ __forceinline__ void fx_window_init(int lane, const WarpSmem& ws) {
  if (lane == 0) {
    const unsigned bar_a = (unsigned)__cvta_generic_to_shared(ws.bar);
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // CTA-scope: the cluster-scope init fence costs an L1 invalidate (CCTL.IVALL)
  }
}

__device__ __forceinline__ int fx_window_issue(const FxPairTable& tb, int C, int64_t start, int left, int have, int lane,
                                               const WarpSmem& ws, const double* stats_row = nullptr, int n_features = 0) {
  const int64_t e0 = (start + left) * (int64_t)C;
  const int shift = (int)(e0 & 1);
  const unsigned bytes = (unsigned)(((have * C + shift + 1) & ~1) * 8);
  if (lane == 0) {
    // a persistent warp reuses this buffer: its previous env-step may have written ws.stat with ordinary stores (warm-up
    // statistics) -- order them before the bulk copies (async proxy) that overwrite the same bytes
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    const unsigned bar_a = (unsigned)__cvta_generic_to_shared(ws.bar);
    const unsigned dst_a = (unsigned)__cvta_generic_to_shared(ws.win);
    const unsigned sbytes = stats_row ? (unsigned)n_features * 16u : 0u;  // {mean, 1/std} rows are 16-byte multiples
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes + sbytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst_a), "l"(tb.candles + (e0 - shift)), "r"(bytes), "r"(bar_a) : "memory");
    if (stats_row)  // the bar's z-score statistics ride on the same mbarrier: no register ever holds them
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   ::"r"((unsigned)__cvta_generic_to_shared(ws.stat)), "l"(stats_row), "r"(sbytes), "r"(bar_a) : "memory");
  }
  return shift;
}

// `phase` = how many copies this warp's mbarrier has completed before (a persistent warp reuses it for every env-step)
__device__ __forceinline__ void fx_window_wait(const WarpSmem& ws, unsigned phase = 0u) {
  __syncwarp();
  const unsigned bar_a = (unsigned)__cvta_generic_to_shared(ws.bar);
  unsigned ok = 0;
  while (!ok)
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"(bar_a), "r"(phase & 1u) : "memory");
}

// GymFxEnv.reset (app/env.py:102-129): fresh bridge/broker/strategy; broker.next() on bar 0 with nothing pending
// (value = cash) and the first _publish_obs.  Reward-plugin state persists across episodes, like the plugin
// instance does in the reference (its `step <= last_step` rule then clears it on the next compute_reward).
__device__ __forceinline__ void fx_reset_regs(const FxConfig& c, FxEnvRegs& e, double close0) {
  e.cash = c.initial_cash; e.value = c.initial_cash; e.psize = 0.0; e.pprice = 0.0;
  e.equity = c.initial_cash; e.prev_equity = c.initial_cash; e.commission_paid = 0.0;
  e.trades = 0; e.position = 0; e.flags = 0u;
  e.price = close0; e.bar_index = 1;
}

__device__ __forceinline__ void fx_store_all(const FxDeviceState& st, int env, const FxEnvRegs& e) {
  st.cash[env] = e.cash; st.psize[env] = e.psize; st.pprice[env] = e.pprice;
  st.equity[env] = e.equity; st.prev_equity[env] = e.prev_equity; st.price[env] = e.price;
  st.commission_paid[env] = e.commission_paid;
  st.position[env] = e.position; st.bar_index[env] = e.bar_index; st.trades[env] = e.trades;
  st.flags[env] = e.flags;
}

__device__ __forceinline__ int32_t fx_total_bars(const FxConfig& c, int64_t T, int64_t start) {
  int64_t tb = T - start;
  if (c.episode_bars > 0 && c.episode_bars < tb) tb = c.episode_bars;
  return (int32_t)tb;
}

__device__ __forceinline__ uint64_t fx_splitmix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// LEAN (compile time, see fx_config_is_lean): the BASELINE family of configurations -- discrete actions, no commission /
// leverage / slippage, backtrader's next-bar child activation, feature_window preprocessor over the 5 OHLCV columns with
// a rolling z-score, clipping, price window and agent state, finite data.  The specialised kernels leave out every branch
// and constant-bank read those settings make dead; results are bit-identical to the general kernels.
template <bool LEAN = false>
__device__ __forceinline__ bool fx_uses_running_stats(const FxConfig& c) {
  return LEAN || (c.preproc == FX_PREPROC_FEATURE_WINDOW && c.scaling != FX_SCALING_NONE);
}

// GymFxEnv.reset of one env, by one thread (fx_reset_kernel; lane 0 of fx_step_env's auto-reset branch).  The episode it
// ends, if that ever took a step, is latched from the state arrays into ep_last.  The new one starts at `start` (clamped
// to the table), or, with `draw` and a start range set, at a bar drawn from the range (include/fxenv.h,
// fxenv_set_reset_starts).  Scalar and out of line: the step kernels' registers belong to the stepping path.
__device__ __noinline__ void fx_reset_env(const FxKernelParams& P, const int env, int64_t start, const bool draw) {
  const FxConfig& c = P.cfg;
  const FxDeviceState& st = P.st;
  const FxPairTable& tb = P.pair[env % c.num_pairs];
  const int32_t k = st.ep_begun[env];
  const uint32_t flags = st.flags[env];
  if (flags & FX_FLAG_STARTED) {
    double* r = st.ep_last + (int64_t)env * FXENV_EPISODE_STATS;
    const double* rs = st.rstats + (int64_t)env * FX_RS_N;
    r[FXENV_EP_START] = (double)st.start[env];
    r[FXENV_EP_BARS] = (double)st.bar_index[env];
    r[FXENV_EP_EQUITY] = st.equity[env];
    r[FXENV_EP_COMMISSION] = st.commission_paid[env];
    r[FXENV_EP_END_FLAGS] = (double)(flags & (FX_FLAG_TERMINATED | FX_FLAG_EXHAUSTED | FX_FLAG_BROKE | FX_FLAG_TRUNCATED));
    r[FXENV_EP_DD_MAX_PCT] = rs[FX_RS_DD_MAX_PCT];
    r[FXENV_EP_DD_MAX_MONEY] = rs[FX_RS_DD_MAX_MONEY];
    r[FXENV_EP_PNL_NET] = rs[FX_RS_PNL_NET];
    r[FXENV_EP_PNL_SQ] = rs[FX_RS_PNL_SQ];
    r[FXENV_EP_OPENED] = rs[FX_RS_OPENED];
    r[FXENV_EP_CLOSED] = (double)st.trades[env];
    r[FXENV_EP_WON] = rs[FX_RS_WON];
    r[FXENV_EP_LOST] = rs[FX_RS_LOST];
    r[FXENV_EP_INDEX] = (double)(k - 1);
    st.ep_done[env] += 1;
  }
  st.ep_begun[env] = k + 1;
  const uint64_t span = st.ep_span[env];
  if (draw && span != 0) {
    const uint64_t h = fx_splitmix64(st.ep_seed[0] ^ (((uint64_t)(uint32_t)env << 32) | (uint64_t)(uint32_t)k));
    start = st.ep_lo[env] + (int64_t)__umul64hi(h, span);
  }
  if (start < 0) start = 0;
  if (start > tb.T - 1) start = tb.T - 1;
  FxEnvRegs e;
  fx_reset_regs(c, e, tb.candles[start * (int64_t)c.n_cols + 3]);
  fx_store_all(st, env, e);
  st.start[env] = start;
  st.t[env] = 0;
  st.total_bars[env] = fx_total_bars(c, tb.T, start);
  st.n_orders[env] = 0;
  st.n_acc[env] = 0;
  st.sub_need[env] = 0.0;
  P.ep_steps[env] = 0;
  for (int j = 0; j < FX_RS_N; j++) st.rstats[(int64_t)env * FX_RS_N + j] = (j == FX_RS_DD_MAXVALUE) ? c.initial_cash : 0.0;
  for (int j = 0; j < 5; j++) st.nbar[(int64_t)env * 6 + j] = tb.candles[start * (int64_t)c.n_cols + (j < 4 ? j : c.price_col)];
  if (fx_uses_running_stats(c)) {
    for (int f = 0; f < c.n_features; f++) {
      const int64_t wi = ((int64_t)env * FXENV_MAX_FEATURES + f) * 2;
      st.welford[wi] = tb.candles[start * (int64_t)c.n_cols + c.feature_cols[f]];
      st.welford[wi + 1] = 0.0;
    }
  }
}

// z-score statistics of the history window ending at local row s-1, for lane f < F: {mean, 1/std}.
// Full rolling window: the per-bar table computed at load time.  Otherwise (warm-up, expanding): the env's running
// Welford state (wm, wm2 = the lane's feature, already including row s-1).  Returns false -> raw (unscaled) values.
template <bool LEAN = false>
__device__ __forceinline__ bool fx_scaling_active(const FxConfig& c, int s, int& hn) {
  if (!fx_uses_running_stats<LEAN>(c)) return false;
  hn = s;
  if ((LEAN || c.scaling == FX_SCALING_ROLLING) && hn > c.scaling_window) hn = c.scaling_window;
  return hn >= 2;
}

template <bool LEAN = false>
__device__ __forceinline__ bool fx_stats_from_table(const FxConfig& c, const FxPairTable& tb, int hn) {
  return (LEAN || (c.scaling == FX_SCALING_ROLLING && tb.stats != nullptr)) && hn == c.scaling_window;
}

// 1 / n for a small positive integer: float reciprocal + two Newton steps in fp64 (relative error < 1e-15), ~8 instructions
// instead of the ~35 of an IEEE fp64 division.  Only the observation statistics use it (tolerance 1e-5 on float32 values).
__device__ __forceinline__ double fx_rcp_int(int n) {
  const double x = (double)n;
  double y = (double)__frcp_rn((float)n);
  y = y * (2.0 - x * y);
  y = y * (2.0 - x * y);
  return y;
}

// {mean, 1 / std} of the running Welford state over hn rows; population std, std < 1e-8 -> 1 (feature_window_preprocessor.py
// :110-116).  1/std by rsqrt + Newton (relative error < 1e-14) instead of division, square root and division.
__device__ __forceinline__ void fx_welford_to_stats(double wm, double wm2, int hn, double& m, double& r) {
  const double var = wm2 * fx_rcp_int(hn);
  m = wm;
  if (var < 1e-16) { r = 1.0; return; }                      // std < 1e-8 -> unscaled
  if (!(var <= 1.0e300)) { r = 1.0 / sqrt(var); return; }    // inf / NaN in the data: IEEE semantics (NaN -> 0 downstream)
  double y = (double)rsqrtf((float)var);
  y = y * (1.5 - 0.5 * var * y * y);
  y = y * (1.5 - 0.5 * var * y * y);
  r = y;
}

// Welford update with the n-th row (n >= 1 after the update), 1/n by fx_rcp_int
__device__ __forceinline__ void fx_welford_step(double& mean, double& m2, double x, int n) {
  const double d = x - mean;
  mean += d * fx_rcp_int(n);
  m2 += d * (x - mean);
}

// self-contained version for the paths that are not latency critical (terminated envs, observe kernel)
__device__ __forceinline__ bool fx_prepare_stats(const FxKernelParams& P, const FxPairTable& tb, int env, int lane, int s,
                                                 int64_t start, double* sstat) {
  const FxConfig& c = P.cfg;
  int hn;
  if (!fx_scaling_active(c, s, hn)) return false;
  if (lane < c.n_features) {
    double m, r;
    if (fx_stats_from_table(c, tb, hn)) {
      const double* sp = tb.stats + ((start + s - 1) * (int64_t)c.n_features + lane) * 2;
      m = sp[0]; r = sp[1];
    } else {
      const int64_t wi = ((int64_t)env * FXENV_MAX_FEATURES + lane) * 2;
      fx_welford_to_stats(P.st.welford[wi], P.st.welford[wi + 1], hn, m, r);
    }
    sstat[2 * lane] = m; sstat[2 * lane + 1] = r;
  }
  __syncwarp();
  return true;
}

// Optional second copy of the observation row in bfloat16 (round-to-nearest-even of the float32 value), K-padded row
// stride: the A operand of the fused policy kernel (fx_policy.cu).  o16 == nullptr: not requested.
__device__ __forceinline__ void fx_st16(uint16_t* o16, int j, float v) {
  if (o16) o16[j] = __bfloat16_as_ushort(__float2bfloat16_rn(v));
}
__device__ __forceinline__ void fx_st16x4(uint16_t* o16, int j, float4 v) {  // j % 4 == 0, row 8-byte aligned
  if (o16) {
    const __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
    uint2 u;
    u.x = *reinterpret_cast<const uint32_t*>(&lo); u.y = *reinterpret_cast<const uint32_t*>(&hi);
    *reinterpret_cast<uint2*>(o16 + j) = u;
  }
}

// ---- observation windows: preprocessor.make_observation (features | prices | returns) in the flat VecEnv layout ----
// `win` = the staged rows [left, s) (shift already applied): element (k, col) at win[k * C + col].
// float32 finishing of one feature value: np.clip then np.nan_to_num (feature_window_preprocessor.py:119-123)
// TAME: every table value is finite and below 1e100 in magnitude (checked at fxenv_load_candles), so a z-score can
// overflow to +-inf but never be NaN and the nan -> 0 fix-up is dead code.
template <bool CLIP, bool TAME>
__device__ __forceinline__ float fx_finish_t(float v, float clipf) {
  if (!TAME) v = (v != v) ? 0.0f : v;
  if (CLIP) return fminf(fmaxf(v, -clipf), clipf);  // also maps +-inf to +-clip
  return isinf(v) ? (v > 0.0f ? clipf : -clipf) : v;
}

// LONG: windows of several hundred rows, where loop overhead outweighs instruction-cache footprint (the loops are unrolled)
template <bool FAST5, bool CLIP, bool TAME, bool LONG, bool O16>
__device__ __noinline__ void fx_emit_windows_t(const FxKernelParams& P, int lane, int s, bool scale,
                                               const double* __restrict__ win, const double* sstat,
                                               float* __restrict__ out, uint16_t* __restrict__ o16_) {
  uint16_t* __restrict__ const o16 = O16 ? o16_ : nullptr;  // O16 == false: the bf16 copy is compiled out
  const FxConfig& c = P.cfg;
  const int W = c.window_size, C = c.n_cols;
  int left = s - W;
  if (left < 0) left = 0;
  const int pad = W - (s - left);  // left padding with the first available row
  int off = 0;
  if (c.preproc == FX_PREPROC_FEATURE_WINDOW) {
    const int F = c.n_features;
    const float clipf = (float)c.feature_clip;
    const int total = W * F;
    if (FAST5 && pad == 0 && (reinterpret_cast<uintptr_t>(out) & 7) == 0) {  // row must be 8-byte aligned for float2
      // F == n_cols == 5, identity columns, full window: the [W][5] block is the staged span itself.  A lane owns the
      // element PAIR (2*lane, 2*lane+1) of every 60-element (12-row) pass: its two features -- hence their mean and
      // 1/std -- are loop-invariant, and each pass ends in one 8-byte streaming store per lane (30 lanes active).
      if (lane < 30) {
        const int f0 = (2 * lane) % 5, f1 = (2 * lane + 1) % 5;
        const bool z0 = scale && !c.feature_binary[f0], z1 = scale && !c.feature_binary[f1];
        const double m0 = z0 ? sstat[2 * f0] : 0.0, r0 = z0 ? sstat[2 * f0 + 1] : 1.0;
        const double m1 = z1 ? sstat[2 * f1] : 0.0, r1 = z1 ? sstat[2 * f1 + 1] : 1.0;
        const int npair = total >> 1;  // total = 5 W; an odd W leaves one tail element
        // Short windows: not unrolled on purpose -- 16 warps per SM sit at different places of a ~65 KB kernel, and the
        // smaller loop body is worth more in instruction-cache hits than the saved loop overhead; long windows (cfg5,
        // W=512) gain from unrolling, hence the LONG variant.
#define FX_PAIR_BODY                                                        \
          const double x0 = win[2 * q], x1 = win[2 * q + 1];                \
          float2 v;                                                         \
          v.x = fx_finish_t<CLIP, TAME>((float)((x0 - m0) * r0), clipf);    \
          v.y = fx_finish_t<CLIP, TAME>((float)((x1 - m1) * r1), clipf);    \
          __stcs(reinterpret_cast<float2*>(out) + q, v);                    \
          fx_st16(o16, 2 * q, v.x); fx_st16(o16, 2 * q + 1, v.y);
        if (LONG) {
#pragma unroll 4
          for (int q = lane; q < npair; q += 30) { FX_PAIR_BODY }
        } else {
#pragma unroll 1
          for (int q = lane; q < npair; q += 30) { FX_PAIR_BODY }
        }
#undef FX_PAIR_BODY
        if ((total & 1) && lane == 0) {
          const int j = total - 1, f = j % 5;
          const bool z = scale && !c.feature_binary[f];
          const double x = win[j];
          const float vt = fx_finish_t<CLIP, TAME>(z ? (float)((x - sstat[2 * f]) * sstat[2 * f + 1]) : (float)x, clipf);
          __stcs(out + j, vt);
          fx_st16(o16, j, vt);
        }
      }
    } else {
      // general path: (row, feature) advanced incrementally, no integer division in the loop
      int w = lane / F, f = lane - w * F;
      const int dw = 32 / F, df = 32 - dw * F;
      for (int j = lane; j < total; j += 32) {
        int k = w - pad;
        if (k < 0) k = 0;
        const double x = win[k * C + c.feature_cols[f]];
        const float v = (scale && !c.feature_binary[f]) ? (float)((x - sstat[2 * f]) * sstat[2 * f + 1]) : (float)x;
        const float vf = fx_finish_t<CLIP, TAME>(v, clipf);
        __stcs(out + j, vf);
        fx_st16(o16, j, vf);
        w += dw; f += df;
        if (f >= F) { f -= F; w += 1; }
      }
    }
    off = total;
  }
  const bool inc_price = (c.preproc == FX_PREPROC_DEFAULT) || c.include_price_window;
  if (inc_price) {
    const int pc = c.price_col;
    float* __restrict__ op = out + off;
#define FX_PRICE_BODY                                                       \
      int k = w - pad;                                                      \
      if (k < 0) k = 0;                                                     \
      int k1 = w - 1 - pad;                                                 \
      if (k1 < 0) k1 = 0;                                                   \
      const double p = win[k * C + pc];                                     \
      const double prev = win[k1 * C + pc];                                 \
      const float rt = (w == 0) ? 0.0f : (float)(p - prev);                 \
      __stcs(op + w, (float)p);                                             \
      __stcs(op + W + w, rt);                                               \
      fx_st16(o16, off + w, (float)p); fx_st16(o16, off + W + w, rt);
    if (LONG) {
#pragma unroll 4
      for (int w = lane; w < W; w += 32) { FX_PRICE_BODY }
    } else {
#pragma unroll 1
      for (int w = lane; w < W; w += 32) { FX_PRICE_BODY }
    }
#undef FX_PRICE_BODY
  }
}

// The BASELINE shape (F == n_cols == 5 identity columns, full window, W % 4 == 0, 16-byte aligned row, price window on):
// 16-byte streaming stores.  A lane owns the float4 q = lane + 30 * it of the [W][5] block (30 lanes active): its four
// features are (4 * (lane % 5) + i) % 5 in every iteration, so their scale factors stay in registers, and a z-score is
// ONE fp64 fma, x * (1/std) + (-mean / std) (the reference computes (x - mean) / std in fp64 and casts to float32; the
// difference is far below half a float32 ulp, see DESIGN.md section 2).  prices | returns: a lane owns 4 consecutive rows.
// PAD: the episode is younger than the window (s < W rows staged): output row w shows staged row max(0, w - pad), i.e. the
// first row repeated `pad` times (feature_window_preprocessor.py:153-160,197-204) -- the first W steps of every episode.
// What it needs of the configuration arrives BY VALUE: as a non-inlined function taking a reference to the kernel parameters
// it read them with generic loads (a constant-bank address formed at run time), ~10 dependent round trips at the top of
// every row.  (It is now inlined as well.)  NOBIN: no binary pass-through feature (LEAN contract).
template <bool CLIP, bool TAME, bool O16, bool PAD, bool LONG, bool NOBIN>
__device__ __forceinline__ void fx_emit_fast5_q(const int lane, const bool scale, const double* __restrict__ win,
                                             const double* sstat, float* __restrict__ out, uint16_t* __restrict__ o16_,
                                             const int pad, const int W, const float clipf, const int pc,
                                             const unsigned binary_mask) {
  uint16_t* __restrict__ const o16 = O16 ? o16_ : nullptr;
  const int pad5 = 5 * pad;
  if (lane < 30) {
    const int l5 = lane % 5;
    double r[4], a[4];
    int fi[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      int f = i - l5;                      // (4 * l5 + i) % 5, with 4 = -1 (mod 5)
      if (f < 0) f += 5;
      fi[i] = f;
      const bool z = scale && (NOBIN || !((binary_mask >> f) & 1u));
      const double2 mr = *reinterpret_cast<const double2*>(sstat + 2 * f);  // {mean, 1/std}
      r[i] = z ? mr.y : 1.0;
      a[i] = z ? -(mr.x * mr.y) : 0.0;
    }
    const int nq = (5 * W) >> 2;
    float4* __restrict__ o4 = reinterpret_cast<float4*>(out);
    // short windows: not unrolled -- the warps of an SM sit at different places of a large kernel, and the smaller loop
    // body is worth more in instruction-cache hits than the saved loop overhead; LONG (W >= 384): unrolled by 2
#pragma unroll(LONG ? kLongUnroll : 1)
    for (int q = lane; q < nq; q += 30) {
      double x[4];
      if (PAD) {  // element j of the block comes from staged element j - 5 * pad, or from row 0 (same feature) in the pad
#pragma unroll
        for (int i = 0; i < 4; i++) { const int j = 4 * q + i - pad5; x[i] = win[j >= 0 ? j : fi[i]]; }
      } else {
        const double* __restrict__ xs = win + 4 * q;  // the staged span may start on an odd double: 8-byte loads
        x[0] = xs[0]; x[1] = xs[1]; x[2] = xs[2]; x[3] = xs[3];
      }
      float4 v;
      v.x = fx_finish_t<CLIP, TAME>((float)fma(x[0], r[0], a[0]), clipf);
      v.y = fx_finish_t<CLIP, TAME>((float)fma(x[1], r[1], a[1]), clipf);
      v.z = fx_finish_t<CLIP, TAME>((float)fma(x[2], r[2], a[2]), clipf);
      v.w = fx_finish_t<CLIP, TAME>((float)fma(x[3], r[3], a[3]), clipf);
      __stcs(o4 + q, v);
      fx_st16x4(o16, 4 * q, v);
    }
  }
  float* __restrict__ op = out + 5 * W;
#pragma unroll 1
  for (int w0 = 4 * lane; w0 < W; w0 += 128) {
    double pm, p0, p1, p2, p3;
    if (PAD) {
      const int k = w0 - pad;  // staged row of output row w0 (negative inside the pad: row 0)
      pm = win[(k - 1 > 0 ? k - 1 : 0) * 5 + pc];
      p0 = win[(k > 0 ? k : 0) * 5 + pc]; p1 = win[(k + 1 > 0 ? k + 1 : 0) * 5 + pc];
      p2 = win[(k + 2 > 0 ? k + 2 : 0) * 5 + pc]; p3 = win[(k + 3 > 0 ? k + 3 : 0) * 5 + pc];
    } else {
      const double* __restrict__ pr = win + w0 * 5 + pc;
      pm = (w0 > 0) ? pr[-5] : pr[0];
      p0 = pr[0]; p1 = pr[5]; p2 = pr[10]; p3 = pr[15];
    }
    float4 pv, rv;
    pv.x = (float)p0; pv.y = (float)p1; pv.z = (float)p2; pv.w = (float)p3;
    rv.x = (w0 > 0) ? (float)(p0 - pm) : 0.0f; rv.y = (float)(p1 - p0); rv.z = (float)(p2 - p1); rv.w = (float)(p3 - p2);
    __stcs(reinterpret_cast<float4*>(op + w0), pv);
    __stcs(reinterpret_cast<float4*>(op + W + w0), rv);
    fx_st16x4(o16, 5 * W + w0, pv);
    fx_st16x4(o16, 6 * W + w0, rv);
  }
}

template <bool FAST5, bool O16 = true, bool LEAN = false>
__device__ __forceinline__ void fx_emit_windows(const FxKernelParams& P, int lane, int s, bool scale,
                                                const double* __restrict__ win, const double* sstat,
                                                float* __restrict__ out, uint16_t* __restrict__ o16 = nullptr) {
  const int pad = P.cfg.window_size - s;  // > 0: the first rows of the window repeat the episode's first bar
  if (LEAN) {  // window % 4 == 0, price window, clip > 0 and finite data are part of the LEAN contract
    if ((reinterpret_cast<uintptr_t>(out) & 15) == 0) {
      const int W = P.cfg.window_size, pc = P.cfg.price_col;
      const float clipf = (float)P.cfg.feature_clip;
      if (pad > 0) fx_emit_fast5_q<true, true, O16, true, false, true>(lane, scale, win, sstat, out, o16, pad, W, clipf, pc, 0u);
      else if (W >= FX_LONG_MIN_W) fx_emit_fast5_q<true, true, O16, false, true, true>(lane, scale, win, sstat, out, o16, 0, W, clipf, pc, 0u);
      else fx_emit_fast5_q<true, true, O16, false, false, true>(lane, scale, win, sstat, out, o16, 0, W, clipf, pc, 0u);
    } else {
      fx_emit_windows_t<true, true, true, false, O16>(P, lane, s, scale, win, sstat, out, o16);
    }
    return;
  }
  if (FAST5 && (P.cfg.window_size & 3) == 0 && P.cfg.include_price_window && P.cfg.feature_clip > 0.0 && P.tame_data &&
      (reinterpret_cast<uintptr_t>(out) & 15) == 0) {
    const int W = P.cfg.window_size, pc = P.cfg.price_col;
    const float clipf = (float)P.cfg.feature_clip;
    unsigned bm = 0u;  // binary pass-through features keep their raw value
    if (P.any_binary) {
#pragma unroll
      for (int f = 0; f < 5; f++) bm |= P.cfg.feature_binary[f] ? (1u << f) : 0u;
    }
    if (pad > 0) fx_emit_fast5_q<true, true, O16, true, false, false>(lane, scale, win, sstat, out, o16, pad, W, clipf, pc, bm);
    else if (W >= FX_LONG_MIN_W) fx_emit_fast5_q<true, true, O16, false, true, false>(lane, scale, win, sstat, out, o16, 0, W, clipf, pc, bm);
    else fx_emit_fast5_q<true, true, O16, false, false, false>(lane, scale, win, sstat, out, o16, 0, W, clipf, pc, bm);
    return;
  }
  const bool lng = P.cfg.window_size >= 384;
  if (P.cfg.feature_clip > 0.0) {
    if (P.tame_data) {
      if (lng) fx_emit_windows_t<FAST5, true, true, true, O16>(P, lane, s, scale, win, sstat, out, o16);
      else fx_emit_windows_t<FAST5, true, true, false, O16>(P, lane, s, scale, win, sstat, out, o16);
    } else {
      fx_emit_windows_t<FAST5, true, false, false, O16>(P, lane, s, scale, win, sstat, out, o16);
    }
  } else {
    fx_emit_windows_t<FAST5, false, false, false, O16>(P, lane, s, scale, win, sstat, out, o16);
  }
}

// issue + wait + emit in one go (terminated path, observe kernel)
template <bool FAST5>
__device__ __forceinline__ void fx_stream_windows(const FxKernelParams& P, const FxPairTable& tb, int env, int lane, int s,
                                                  int64_t start, const WarpSmem& ws, float* __restrict__ out,
                                                  uint16_t* __restrict__ o16 = nullptr) {
  const int W = P.cfg.window_size;
  int left = s - W;
  if (left < 0) left = 0;
  fx_window_init(lane, ws);
  __syncwarp();
  const int shift = fx_window_issue(tb, P.cfg.n_cols, start, left, s - left, lane, ws);
  const bool scale = fx_prepare_stats(P, tb, env, lane, s, start, ws.stat);
  fx_window_wait(ws);
  fx_emit_windows<FAST5>(P, lane, s, scale, ws.win + shift, ws.stat, out, o16);
}

__device__ __forceinline__ int fx_scalar_offset(const FxConfig& c) {
  const int W = c.window_size;
  if (c.preproc == FX_PREPROC_DEFAULT) return 2 * W;
  return W * c.n_features + (c.include_price_window ? 2 * W : 0);
}

// the 4 agent scalars at the end of the row (one lane)
// `last` = price_column of the last window row (local row bar_index - 1)
template <bool LEAN = false>
__device__ __forceinline__ void fx_write_scalars(const FxKernelParams& P, const FxEnvRegs& e, int32_t total_bars,
                                                 double last, float* __restrict__ out, uint16_t* __restrict__ o16 = nullptr) {
  const FxConfig& c = P.cfg;
  const bool inc_agent = LEAN || (c.preproc == FX_PREPROC_DEFAULT) || c.include_agent_state;
  if (!inc_agent) return;
  const bool inc_price = LEAN || (c.preproc == FX_PREPROC_DEFAULT) || c.include_price_window;
  double ref;
  if (!LEAN && c.preproc == FX_PREPROC_DEFAULT) ref = last;  // default_preprocessor.py:63
  else ref = inc_price ? (double)(float)last : e.price;     // feature_window_preprocessor.py:218-222
  float sc[4];
  fx_agent_scalars(c, e, total_bars, ref, P.inv_initial_cash, sc);
  const int so = LEAN ? 7 * c.window_size : fx_scalar_offset(c);
  float* o = out + so;
  o[0] = sc[0]; o[1] = sc[1]; o[2] = sc[2]; o[3] = sc[3];
  fx_st16(o16, so, sc[0]); fx_st16(o16, so + 1, sc[1]); fx_st16(o16, so + 2, sc[2]); fx_st16(o16, so + 3, sc[3]);
}

// ---- Sharpe: lane-parallel evaluation of the deque statistics -----------------------------------------------------
// The reference sums the <= window returns with Python's compensated sum() (sequential Neumaier).  Here every lane
// accumulates its share as an error-free (hi, lo) pair (Knuth two-sum; the build uses -fmad=false so each operation
// rounds once) and the pairs are merged across the warp: the total is accurate to ~1e-32 relative before the final
// rounding, i.e. it can differ from the reference's result only where Neumaier itself is not correctly rounded
// (<= 1 ulp; the reward tolerance is 1e-9 in fp64, 1e-5 in fp32).  All-equal and all-zero windows stay exact, so the
// `std <= 0 -> 0.0` rule fires exactly when the reference's does (flat episodes).
__device__ __forceinline__ void fx_two_sum(double a, double b, double& s, double& e) {
  s = a + b;
  const double bb = s - a;
  e = (a - (s - bb)) + (b - bb);
}

__device__ __forceinline__ void fx_dd_add(double& hi, double& lo, double x) {
  double s, e;
  fx_two_sum(hi, x, s, e);
  lo += e;
  hi = s;
}

__device__ __forceinline__ double fx_dd_warp_total(double hi, double lo) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double h2 = __shfl_xor_sync(FX_FULL, hi, o), l2 = __shfl_xor_sync(FX_FULL, lo, o);
    double s, e;
    fx_two_sum(hi, h2, s, e);
    e += lo + l2;
    hi = s + e;           // fast two-sum renormalisation
    lo = e - (hi - s);
  }
  return hi + lo;
}

__device__ __forceinline__ double fx_sharpe_eval_warp(const double* ring, int W, int n, int head, double ann, int lane) {
  if (n < 2) return 0.0;
  double hi = 0.0, lo = 0.0;
  for (int i = lane; i < n; i += 32) { int idx = head + i; if (idx >= W) idx -= W; fx_dd_add(hi, lo, ring[idx]); }
  const double mean = fx_dd_warp_total(hi, lo) / (double)n;
  hi = 0.0; lo = 0.0;
  for (int i = lane; i < n; i += 32) {
    int idx = head + i; if (idx >= W) idx -= W;
    const double d = ring[idx] - mean;
    fx_dd_add(hi, lo, d * d);
  }
  const double var = fx_dd_warp_total(hi, lo) / (double)(n - 1);
  const double sd = sqrt(var);
  if (sd <= 0.0) return 0.0;
  return (mean / sd) * sqrt(ann);
}

// End-of-run statistics record of the env (fx_core.cuh FX_RS_*): field i lives in lane i of ONE register -- a single
// coalesced load with the state, a single coalesced store if anything changed.  get() broadcasts by shuffle, so the
// callers (uniform scalar code) must be convergent; set() keeps the value in the owning lane.
struct FxRunStatsWarp {
  double& v;
  int lane;
  __device__ __forceinline__ double get(int i) const { return __shfl_sync(FX_FULL, v, i); }
  __device__ __forceinline__ void set(int i, double x) const { if (lane == i) v = x; }
  __device__ __forceinline__ void add(int i, double x) const { if (lane == i) v += x; }  // no broadcast needed
};

// ---- the fused step --------------------------------------------------------------------------------------------
#define FX_OP_KILL 1u
#define FX_OP_ACTIVATE 2u
#define FX_OP_ACTIVATE_NEXT 4u

__device__ __forceinline__ uint32_t fx_apply_op(uint32_t m, uint32_t op) {
  if (op & FX_OP_KILL) return m | FXO_DEAD;
  if (op & FX_OP_ACTIVATE) return m | FXO_ACTIVE;
  if (op & FX_OP_ACTIVATE_NEXT) return m | FXO_ACTIVATE_NEXT;
  return m;
}

// Bracket audit (include/fxenv.h, fxenv_set_bracket_audit): the env's next record into its ring, lane i storing field i
// (the decision is warp-uniform), then the counter.  One warp owns the env for the step, so no atomics.  Only the
// FX_V_AUDIT instantiations contain it.
__device__ __noinline__ void fx_audit_store(const FxKernelParams& P, const int env, const int lane, const FxAudit& au,
                                            const int64_t bar, const double entry) {
  long long w = (lane == 0) ? (long long)P.audit_written[env] : 0ll;
  w = __shfl_sync(FX_FULL, w, 0);
  const double nan = __longlong_as_double(0x7FF8000000000000ll);
  const bool fc = au.kind == FXENV_AU_KIND_FORCE_CLOSE;
  double v = (double)au.kind;
  if (lane == FXENV_AU_BAR) v = (double)bar;
  else if (lane == FXENV_AU_EPISODE) v = (double)(P.st.ep_begun[env] - 1);
  else if (lane == FXENV_AU_ENTRY) v = entry;
  else if (lane == FXENV_AU_STOP) v = fc ? nan : au.stop;
  else if (lane == FXENV_AU_LIMIT) v = fc ? nan : au.limit;
  else if (lane == FXENV_AU_SIZE) v = au.size;
  else if (lane == FXENV_AU_ATR) v = fc ? nan : au.atr;
  if (lane < FXENV_AU_FIELDS) P.audit[((int64_t)env * P.audit_cap + w % P.audit_cap) * FXENV_AU_FIELDS + lane] = v;
  if (lane == 0) P.audit_written[env] = (int64_t)(w + 1);
}

// Action repeat (include/fxenv.h, fxenv_set_action_repeat): the FX_V_REPEAT instantiations run a step of up to P.repeat
// substeps.  One fx_step_env call runs one substep; this record is what the substeps of one step share.
struct FxSubstep {
  double racc;  // float64 sum of the rewards of the step's substeps so far
  int j;        // index of this substep
  bool ended;   // out: this substep ended the step (the last one, a terminating one, or the step of a terminated env)
};

// Where one env-step writes: the BASES of the caller's arrays (kernel parameters: they cost no registers).  The step's
// element of actions / reward / terminated is at index step_row + env (step_row = step * num_envs), its observation row
// at obs_slot_row + env (obs_slot_row = slot * num_envs), its bf16 copy (single-step kernel only) at row env of obs16.
// Addresses are formed where they are used.
struct FxStepOut {
  float* obs;
  uint16_t* obs16;
  float* reward;
  double* reward64;
  uint8_t* terminated;
  unsigned step_row, obs_slot_row;
  int stride16;
};
__device__ __forceinline__ size_t fx_out_idx(const FxStepOut& o, int env) { return (size_t)o.step_row + (size_t)env; }
__device__ __forceinline__ float* fx_obs_row(const FxKernelParams& P, const FxStepOut& o, int env) {
  return o.obs + ((size_t)o.obs_slot_row + (size_t)env) * (size_t)P.obs_dim;
}
template <bool O16>
__device__ __forceinline__ uint16_t* fx_obs_row16(const FxStepOut& o, int env) {
  return (O16 && o.obs16) ? o.obs16 + (size_t)env * (size_t)o.stride16 : nullptr;
}

// Phase stamps of the timing build (make TIMING=1, tools/phase_timing.py): lane 0 writes stamp i of the env's FX_NSTAMP
// (clock64, %globaltimer or a count).  In the release build the struct is empty and every call compiles to nothing.
struct FxStamps {
#ifdef FXENV_ENABLE_TIMING
  long long* p;  // nullptr: FXENV_TIMING is off
  __device__ __forceinline__ void put(int lane, int i, long long v) const { if (p && lane == 0) p[i] = v; }
  __device__ __forceinline__ void at(int lane, int i) const { if (p && lane == 0) p[i] = clock64(); }
  // taken only after `dep` (a loaded value) has actually arrived in a register
  __device__ __forceinline__ void after(int lane, int i, unsigned long long dep) const {
    if (p) { long long t; asm volatile("mov.u64 %0, %%clock64;" : "=l"(t) : "l"(dep)); if (lane == 0) p[i] = t; }
  }
  __device__ __forceinline__ void global(int lane, int i) const {
    if (p && lane == 0) { long long g; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g)); p[i] = g; }
  }
  __device__ __forceinline__ void begin(const FxKernelParams& P, int env, int lane) {
    p = P.timing ? P.timing + (int64_t)env * FX_NSTAMP : nullptr;
    at(lane, 0);
    global(lane, 10);
  }
  // keep two consecutive steps: the stamps move to slot = parity of the (pre-step) cursor t
  __device__ __forceinline__ void to_slot(const FxKernelParams& P, int env, int32_t t, int lane) {
    if (!p) return;
    long long* nb = P.timing + ((int64_t)(t & 1) * P.cfg.num_envs + env) * FX_NSTAMP;
    if (lane == 0) { nb[0] = p[0]; nb[10] = p[10]; }
    p = nb;
  }
#else
  __device__ __forceinline__ void put(int, int, long long) const {}
  __device__ __forceinline__ void at(int, int) const {}
  __device__ __forceinline__ void after(int, int, unsigned long long) const {}
  __device__ __forceinline__ void global(int, int) const {}
  __device__ __forceinline__ void begin(const FxKernelParams&, int, int) {}
  __device__ __forceinline__ void to_slot(const FxKernelParams&, int, int32_t, int) {}
#endif
};

// The broker and strategy values of an env-step (FxEnvParams, fx_core.cuh): in the kernels without FX_V_PARAMS the
// configuration itself (a reference to the kernel parameters, as before), in those with it the env's row of the table,
// loaded one field per lane (`v`, lanes 0..6) with the state and broadcast here.
template <bool PARAMS>
struct FxStepParams {
  static __device__ __forceinline__ const FxConfig& get(const FxConfig& c, double) { return c; }
};
template <>
struct FxStepParams<true> {
  static __device__ __forceinline__ FxEnvParams get(const FxConfig&, double v) {
    FxEnvParams p;
    p.commission = __shfl_sync(FX_FULL, v, FXENV_PARAM_COMMISSION);
    p.leverage = __shfl_sync(FX_FULL, v, FXENV_PARAM_LEVERAGE);
    p.slippage_perc = __shfl_sync(FX_FULL, v, FXENV_PARAM_SLIPPAGE);
    p.sl_pips = __shfl_sync(FX_FULL, v, FXENV_PARAM_SL_PIPS);
    p.tp_pips = __shfl_sync(FX_FULL, v, FXENV_PARAM_TP_PIPS);
    p.k_sl = __shfl_sync(FX_FULL, v, FXENV_PARAM_K_SL);
    p.k_tp = __shfl_sync(FX_FULL, v, FXENV_PARAM_K_TP);
    return p;
  }
};

// ---- phases of fx_step_env as functions of their own: the state load, the drawdown analyzer and the reward ---------
// Each takes what it reads by value or const reference, returns what it produces, and takes by reference only what it
// updates (the env's FxEnvRegs, the lane's run-statistics field).  They are inlined and compile to the same code as
// when written out.  The other phases stay written out in fx_step_env: cut into functions they compile differently.

// The env's scalar state besides FxEnvRegs, as fx_step_load reads it (the state arrays or the carry record)
struct FxStepState {
  uint32_t flags;
  int32_t t, total_bars;
  int64_t start;
  int n, n_acc;     // entries of the order table; the first one created by the previous strategy call
  double sub_need;  // check_submitted cash bound of the entries [n_acc, n)
  int32_t dec;      // TRUNC: decisions of the episode before this step
  FxBar nb;         // the candle this step works on, saved by the previous step (FxDeviceState::nbar)
  double nb_price;  // its price column
};

// ---- round trip 1: one batch of independent state loads (invariants: see FxDeviceState); rsv: field `lane` of the
//      DrawDown / TradeAnalyzer / SQN record
template <bool TRUNC, bool CARRY>
__device__ __forceinline__ FxStepState fx_step_load(const FxKernelParams& P, const int env, const int lane, const WarpSmem& ws,
                                                    const bool carry_in, FxEnvRegs& e, double& rsv) {
  const FxDeviceState& st = P.st;
  FxStepState s;
  s.dec = 0;
  if (CARRY && carry_in) {  // the record this warp left behind one step ago (shared memory: broadcast reads)
    const double* __restrict__ cr = ws.carry;
    const int2 ft = *reinterpret_cast<const int2*>(cr + FX_CARRY_FLAGS_T);
    const int2 bn = *reinterpret_cast<const int2*>(cr + FX_CARRY_BARS_N);
    const int2 at = *reinterpret_cast<const int2*>(cr + FX_CARRY_NACC_TRADES);
    s.flags = (uint32_t)ft.x; s.t = ft.y; s.total_bars = bn.x; s.n = bn.y; s.n_acc = at.x; e.trades = at.y;
    s.start = *reinterpret_cast<const long long*>(cr + FX_CARRY_START);
    s.sub_need = cr[FX_CARRY_SUBNEED];
    e.cash = cr[FX_CARRY_CASH]; e.psize = cr[FX_CARRY_PSIZE]; e.pprice = cr[FX_CARRY_PPRICE]; e.equity = cr[FX_CARRY_EQUITY];
    e.commission_paid = cr[FX_CARRY_COMM];
    s.nb.o = cr[FX_CARRY_NBAR]; s.nb.h = cr[FX_CARRY_NBAR + 1]; s.nb.l = cr[FX_CARRY_NBAR + 2]; s.nb.c = cr[FX_CARRY_NBAR + 3];
    s.nb_price = cr[FX_CARRY_NBAR + 4];
    if (TRUNC) s.dec = *fx_carry_dec(ws);
    if (lane < FX_RS_N) rsv = cr[FX_CARRY_RSTATS + lane];
  } else {
    s.flags = st.flags[env];
    s.t = st.t[env];
    s.total_bars = st.total_bars[env];
    s.start = st.start[env];
    s.n = st.n_orders[env];
    s.n_acc = st.n_acc[env];
    s.sub_need = st.sub_need[env];
    e.cash = st.cash[env]; e.psize = st.psize[env]; e.pprice = st.pprice[env]; e.equity = st.equity[env];
    e.commission_paid = st.commission_paid[env]; e.trades = st.trades[env];
    // the candle this call works on was saved by the previous call (FxDeviceState::nbar): it travels in this same round trip
    const double2* __restrict__ nb2 = reinterpret_cast<const double2*>(st.nbar + (int64_t)env * 6);
    const double2 nb_oh = nb2[0], nb_lc = nb2[1];
    s.nb.o = nb_oh.x; s.nb.h = nb_oh.y; s.nb.l = nb_lc.x; s.nb.c = nb_lc.y;
    s.nb_price = st.nbar[(int64_t)env * 6 + 4];
    if (TRUNC) s.dec = P.ep_steps[env];
    if (lane < FX_RS_N) rsv = st.rstats[(int64_t)env * FX_RS_N + lane];  // DrawDown / TradeAnalyzer / SQN state
  }
  e.value = e.equity;
  return s;
}

// DrawDown analyzer: one notify_fund + next per bar.  With no position and no execution the value is the one of
// the previous bar and nothing can change.
__device__ __forceinline__ void fx_step_drawdown(const FxDeviceState& st, const int env, const int lane, const FxEnvRegs& e,
                                                 const bool any_fill, double& rsv) {
  if (any_fill || e.psize != 0.0) {
    // fx_rs_drawdown in the lane layout: ONE broadcast (the peak), then lanes 0 / 1 / 2 each test their own field;
    // the percent needs its division only when it can set a new maximum.  The record goes back to memory only when
    // something in it changed (an execution, a new peak, a new maximum drawdown).
    const double peak0 = __shfl_sync(FX_FULL, rsv, FX_RS_DD_MAXVALUE);
    const double peak = e.value > peak0 ? e.value : peak0;
    const double md = peak - e.value;
    double cand = (lane == FX_RS_DD_MAXVALUE) ? peak : md;
    const bool pct_may = (lane == FX_RS_DD_MAX_PCT) && (100.0 * md > rsv * peak * 0.999999);
    if (__any_sync(FX_FULL, pct_may)) { if (lane == FX_RS_DD_MAX_PCT) cand = pct_may ? 100.0 * md / peak : 0.0; }
    else if (lane == FX_RS_DD_MAX_PCT) cand = 0.0;
    const bool up = (lane <= FX_RS_DD_MAX_PCT) && (cand > rsv);
    if (up) rsv = cand;
    if (any_fill || __any_sync(FX_FULL, up)) { if (lane < FX_RS_N) st.rstats[(int64_t)env * FX_RS_N + lane] = rsv; }
  }
}

// ---- reward plugin (app/env.py:148-155)
template <int REWARD, bool CARRY>
__device__ __forceinline__ double fx_step_reward(const FxKernelParams& P, const FxEnvRegs& e, const int env, const int lane,
                                                 const WarpSmem& ws, const bool carry_in) {
  const FxConfig& c = P.cfg;
  const FxDeviceState& st = P.st;
  double r;
  if (REWARD == FX_REWARD_PNL) {
    r = fx_reward_pnl(c, e);
  } else if (REWARD == FX_REWARD_DD) {
    double peak = st.dd_peak[env];
    int32_t last = st.dd_last_step[env];
    r = fx_reward_dd(c, e, peak, last);
    if (lane == 0) { st.dd_peak[env] = peak; st.dd_last_step[env] = last; }
  } else {
    // deque of per-step returns: stage the ring in shared memory (coalesced), push, evaluate in Python order
    const int Wn = c.sharpe_window;
    double* gring = st.sh_ring + (int64_t)env * Wn;
    int32_t len, head, last;
    if (CARRY && carry_in) {  // this warp ran the env's previous step: its copy of the deque is current
      const int2 lh = *reinterpret_cast<const int2*>(ws.carry + FX_CARRY_SHARPE);
      len = lh.x; head = lh.y;
      last = *reinterpret_cast<const int32_t*>(ws.carry + FX_CARRY_SHARPE_LAST);
    } else {
      len = st.sh_len[env]; head = st.sh_head[env]; last = st.sh_last_step[env];
      for (int k = lane; k < Wn; k += 32) ws.ring[k] = gring[k];
      __syncwarp();
    }
    const double ret = (e.equity - e.prev_equity) / c.reward_initial_cash;
    int slot;  // where the new return lands (same rule as fx_sharpe_push)
    if (e.bar_index <= last) slot = 0; else slot = (len == Wn) ? head : (head + len) % Wn;
    const int nn = fx_sharpe_push(ws.ring, 1, Wn, len, head, last, e.bar_index, ret);
    __syncwarp();
    r = fx_sharpe_eval_warp(ws.ring, Wn, nn, head, c.annualization_factor, lane);
    if (lane == 0) {
      gring[slot] = ret;
      st.sh_len[env] = len; st.sh_head[env] = head; st.sh_last_step[env] = last;
      if (CARRY) {
        *reinterpret_cast<int2*>(ws.carry + FX_CARRY_SHARPE) = make_int2(len, head);
        *reinterpret_cast<int32_t*>(ws.carry + FX_CARRY_SHARPE_LAST) = last;
      }
    }
  }
  return r;
}

// One env-step of one env by one warp (everything between the cross-kernel dependency wait and the release).
// V: the variant key (FX_V_*).
// CARRY (fx_rollout_kernel): the step leaves the env's scalar state in ws.carry and returns true if that record is valid;
// carry_in = the previous call of this warp was the same env's previous step and returned true.
// RESIDENT (with CARRY): the env's order table lives in ws.op0/op1/osz/ometa while the carry record is valid -- loaded
// from global memory by a step without carry_in, written back by a step that returns false (terminated branch) and by
// the caller at the end of its ticket (fx_rollout_kernel).
// REPEAT (with CARRY): the call is substep sub->j of a step.  A substep that does not end the step issues no window
// copy, stages no statistics and stores no row, reward or flag (the running Welford statistics still advance); it adds
// its reward to sub->racc and leaves the carry record for the next substep.
template <int STRATEGY, int REWARD, unsigned V, bool O16, bool CARRY = false>
__device__ __forceinline__ bool fx_step_env(const FxKernelParams& P, const void* __restrict__ actions, float* __restrict__ obs,
                                            float* __restrict__ reward, double* __restrict__ reward64,
                                            uint8_t* __restrict__ terminated, const int env, const int lane, const WarpSmem& ws,
                                            const unsigned phase = 0u, const unsigned step_row = 0u, const unsigned obs_slot_row = 0u,
                                            uint16_t* __restrict__ obs16 = nullptr, const int stride16 = 0,
                                            const bool carry_in = false, FxSubstep* sub = nullptr) {
  const FxStepOut o{obs, obs16, reward, reward64, terminated, step_row, obs_slot_row, stride16};
  constexpr bool FAST5 = (V & FX_V_FAST5) != 0, LEAN = (V & FX_V_LEAN) != 0, RESIDENT = (V & FX_V_RESIDENT) != 0;
  constexpr bool AUDIT = (V & FX_V_AUDIT) != 0, REPEAT = (V & FX_V_REPEAT) != 0, TRUNC = (V & FX_V_TRUNC) != 0;
  constexpr bool PARAMS = (V & FX_V_PARAMS) != 0;
  constexpr bool ATR = STRATEGY == FX_STRATEGY_ATR_SLTP;
  static_assert(!REPEAT || CARRY, "substeps hand the env over through the carry record");
  static_assert(!RESIDENT || CARRY, "the shared copy of the order table lives as long as the carry record");
  const FxConfig& c = P.cfg;
  const FxDeviceState& st = P.st;
  const int C = c.n_cols;
  const int capP = P.cap + FXO_SLACK;
  const int pair = (c.num_pairs == 1) ? 0 : env % c.num_pairs;
  const FxPairTable& tb = P.pair[pair];
  FxStamps ts;
  ts.begin(P, env, lane);

  // ---- round trip 1: one batch of independent state loads (invariants: see FxDeviceState)
  FxEnvRegs e;
  double rsv = 0.0;
  double prow = 0.0;  // PARAMS: field `lane` of the env's row (lanes 0..6)
  if (PARAMS && lane < FXENV_ENV_PARAMS) prow = fx_env_params(P)[(int64_t)env * FXENV_ENV_PARAMS + lane];
  FxStepState s0 = fx_step_load<TRUNC, CARRY>(P, env, lane, ws, carry_in, e, rsv);
  // the step's own copies (the timeline advances flags and t, an auto-reset moves start and total_bars): using the
  // fields of s0 in their place compiles to different code
  uint32_t flags = s0.flags;
  int32_t t = s0.t, total_bars = s0.total_bars;
  int64_t start = s0.start;
  int n = s0.n, n_acc = s0.n_acc;
  double sub_need = s0.sub_need;
  int32_t dec = s0.dec;
  double2 nb_oh, nb_lc;
  nb_oh.x = s0.nb.o; nb_oh.y = s0.nb.h; nb_lc.x = s0.nb.l; nb_lc.y = s0.nb.c;
  double nb_price = s0.nb_price;
  int action_raw_i = 0;
  float action_raw_f = 0.0f;
  if (!LEAN && c.action_mode == FX_ACTION_CONTINUOUS) action_raw_f = reinterpret_cast<const float*>(actions)[fx_out_idx(o, env)];
  else action_raw_i = reinterpret_cast<const int32_t*>(actions)[fx_out_idx(o, env)];
  // the first 32 orders of the table sit at an address that only depends on the env: they travel with the state
  // (RESIDENT: the table is read from the warp's shared memory instead, no prefetch)
  const int64_t obase = (int64_t)env * capP;
  uint32_t* __restrict__ gmeta = RESIDENT ? ws.ometa : st.o_meta + obase;
  double* __restrict__ gp0 = RESIDENT ? ws.op0 : st.o_p0 + obase;
  double* __restrict__ gp1 = RESIDENT ? ws.op1 : st.o_p1 + obase;
  double* __restrict__ gsz = RESIDENT ? ws.osz : st.o_sz + obase;
  uint32_t pm0 = 0u;
  double pp0 = 0.0, pp1 = 0.0, psz = 0.0;
  if (!RESIDENT) { pm0 = gmeta[lane]; pp0 = gp0[lane]; pp1 = gp1[lane]; psz = gsz[lane]; }
  const FxRunStatsWarp rs{rsv, lane};

  ts.to_slot(P, env, t, lane);
  ts.after(lane, 2, (unsigned long long)flags + (unsigned long long)t + (unsigned long long)start + (unsigned long long)total_bars);

  // ---- terminated envs: the reference answers (obs, 0.0, True) without touching plugins (app/env.py:137-138);
  //      with auto_reset (build-side extension) the env restarts its episode window instead.  A truncated env is
  //      treated alike, answering FXENV_DONE_TRUNCATED -- also in the kernels without truncation: the flag is env state
  //      and outlives the setting (a limit turned off, or a snapshot restored, before the cut env's reset step), and
  //      its episode is over all the same (their 0 / 1 output then answers 1)
  if (flags & (FX_FLAG_TERMINATED | FX_FLAG_TRUNCATED)) {
    if (RESIDENT && carry_in)  // this step returns false: the next one reloads the table from global memory
      fx_table_copy(st.o_meta + obase, st.o_p0 + obase, st.o_p1 + obase, st.o_sz + obase, gmeta, gp0, gp1, gsz,
                    *fx_carry_tab_hi(ws.carry), lane);
    if (c.auto_reset) {
      // a new episode (fx_reset_env, lane 0: the finished one is latched, the start drawn, the state arrays re-initialised);
      // the warp then continues from the new start
      if (lane == 0) fx_reset_env(P, env, start, true);
      __syncwarp();
      start = st.start[env];
      total_bars = fx_total_bars(c, tb.T, start);
      fx_reset_regs(c, e, tb.candles[start * (int64_t)C + 3]);
    } else {
      e.flags = flags;
      e.bar_index = t + 1;
      e.position = e.psize > 0.0 ? 1 : (e.psize < 0.0 ? -1 : 0);
      e.price = tb.candles[(start + t) * (int64_t)C + 3];
    }
    if (lane == 0) {
      o.reward[fx_out_idx(o, env)] = 0.0f;
      if (o.reward64) o.reward64[fx_out_idx(o, env)] = 0.0;
      o.terminated[fx_out_idx(o, env)] = c.auto_reset ? 0 : ((TRUNC && !(flags & FX_FLAG_TERMINATED)) ? FXENV_DONE_TRUNCATED : 1);
      fx_write_scalars<LEAN>(P, e, total_bars, tb.candles[(start + e.bar_index - 1) * (int64_t)C + c.price_col], fx_obs_row(P, o, env), fx_obs_row16<O16>(o, env));
    }
    {
      const int s = e.bar_index;
      int left = s - c.window_size;
      if (left < 0) left = 0;
      __syncwarp();
      const int shift = fx_window_issue(tb, C, start, left, s - left, lane, ws);
      const bool scale = fx_prepare_stats(P, tb, env, lane, s, start, ws.stat);
      fx_window_wait(ws, phase);
      fx_emit_windows<FAST5, O16, LEAN>(P, lane, s, scale, ws.win + shift, ws.stat, fx_obs_row(P, o, env), fx_obs_row16<O16>(o, env));
    }
    if (REPEAT) sub->ended = true;  // rule 1 of the repeat: a terminated env runs this one substep
    return false;  // (the carry record does not follow resets / ended episodes: the next step reloads the arrays)
  }

  // the values the broker and the strategy read (the configuration's, or the env's row: PARAMS)
  const auto& pc = FxStepParams<PARAMS>::get(c, prow);

  // ---- step <-> bar timeline (SURVEY A.1): the first step does not advance; later steps advance or exhaust
  bool exhausted = false, advance = false;
  if (!(flags & FX_FLAG_STARTED)) flags |= FX_FLAG_STARTED;
  else if (t + 1 >= total_bars) exhausted = true;  // strategy.stop(): bridge state unchanged (app/bt_bridge.py:152-155)
  else { t += 1; advance = true; }
  e.flags = flags;
  const int dbg = LEAN ? 0 : P.debug;
  if (RESIDENT && !carry_in && !(dbg & 2)) {  // first step of a ticket: the table into shared memory
    fx_table_copy(gmeta, gp0, gp1, gsz, st.o_meta + obase, st.o_p0 + obase, st.o_p1 + obase, st.o_sz + obase, n, lane);
    if (lane == 0) *fx_carry_tab_hi(ws.carry) = n;
    __syncwarp();
  }

  // ---- the broker can start right away (candle + first 32 orders arrived with the state); what only the observation
  //      needs -- the candle window and the bar's z-score statistics -- is fetched by TMA bulk copies into shared
  //      memory while the broker runs, without occupying registers
  const int s_obs = t + 1;  // bar_index after this step
  const double* __restrict__ row = tb.candles + (start + t) * (int64_t)C;
  FxBar b;
  b.o = nb_oh.x; b.h = nb_oh.y; b.l = nb_lc.x; b.c = nb_lc.y;
  const double last_price = nb_price;
  int hn = 0;
  const bool scale = fx_scaling_active<LEAN>(c, s_obs, hn);
  const bool table_stats = scale && fx_stats_from_table<LEAN>(c, tb, hn);
  const bool welford_live = advance && fx_uses_running_stats<LEAN>(c) && ((!LEAN && c.scaling == FX_SCALING_EXPANDING) || t + 1 <= c.scaling_window);

  int win_left = s_obs - c.window_size;
  if (win_left < 0) win_left = 0;
  int win_shift = 0;
  // REPEAT: only the step's last substep is known to emit here; one that ends the step by terminating emits as well, and
  // issues its copy then (cold path).  Without the repeat every call emits.
  const bool last_sub = !REPEAT || sub->j + 1 >= P.repeat;
  bool emit = last_sub;
  __syncwarp();
  if (!(dbg & 1) && last_sub)  // the observation window and (steady state) the bar's z-score statistics: TMA -> shared memory
    win_shift = fx_window_issue(tb, C, start, win_left, s_obs - win_left, lane, ws,
                                table_stats ? tb.stats + (start + t) * (int64_t)c.n_features * 2 : nullptr, c.n_features);

  ts.after(lane, 1, __double_as_longlong(b.o) + __double_as_longlong(b.c));  // the new bar has arrived


  double nbar_next = 0.0;
  if (!(dbg & 2)) {
    int n_live = n;
    bool any_fill = false;  // cash / position / commission / trade counters only change when an order executes

    if (advance) {
      if (n > 0) {
        // ---- check_submitted: the entries created by the previous strategy call are [n_acc, n); their cash bound
        //      was stored when they were created.  If cash covers it nobody can be rejected; otherwise the exact
        //      sequential simulation (cold path) runs on the table in place.
        int first_sub = n_acc;
        bool reload0 = false;
        if (n_acc < n && !(e.cash >= sub_need * 1.001)) {
          FxOrderTab tg;
          tg.meta = gmeta; tg.p0 = gp0; tg.p1 = gp1; tg.sz = gsz;
          tg.n = n; tg.cap = P.cap; tg.dirty_from = n; tg.ndead = 0; tg.sub_need = 0.0; tg.bound_per = 0.0;
          fx_check_submitted(pc, e, tg, first_sub);  // clears SUBMITTED / marks DEAD in place
          __syncwarp();
          first_sub = n;    // nothing left to accept in the pass below
          reload0 = true;   // the prefetched chunk may be stale
        }
        ts.at(lane, 3);
        // ---- BackBroker.next(): ONE streaming pass over the table, 32 entries (one per lane) at a time, in registers:
        //      activate queued children -> trigger test (ballot) -> execute the hits in FIFO order (fields broadcast by
        //      shuffle from the owning lane) -> stable compaction + write-back of what changed.
        int w = 0;
        int n_fills = 0;  // (timing build only)
        uint32_t carry = 0u;  // operation for the first entry of the next chunk (bracket pair of a parent in lane 31)
        if (!RESIDENT && reload0 && lane < n) { pm0 = gmeta[lane]; pp0 = gp0[lane]; pp1 = gp1[lane]; psz = gsz[lane]; }
        for (int k0 = 0; k0 < n; k0 += 32) {
          const int k = k0 + lane;
          const bool valid = k < n;
          // the chunk in flight: entries [k0+32, k0+64) are requested now and consumed by the next iteration (this
          // iteration only writes at indices <= k, so what it fetches stays valid); RESIDENT: read from shared memory
          if (RESIDENT && valid) { pm0 = gmeta[k]; pp0 = gp0[k]; pp1 = gp1[k]; psz = gsz[k]; }
          const uint32_t m0 = pm0;
          const double p0 = pp0, p1 = pp1, sz = psz;
          if (!RESIDENT && k + 32 < n) { pm0 = gmeta[k + 32]; pp0 = gp0[k + 32]; pp1 = gp1[k + 32]; psz = gsz[k + 32]; }
          uint32_t m = 0u;
          if (valid) {
            m = fx_entry_begin_bar(m0);
            if (k >= first_sub) m &= ~FXO_SUBMITTED;  // accepted by the cash bound
            if (lane == 0) m = fx_apply_op(m, carry);
          }
          carry = 0u;
          double px_lane = 0.0;  // execution price of this lane's entry, should it trade on this bar
          const bool hit = fx_entry_fill(LEAN ? 0.0 : pc.slippage_perc, m, p0, p1, b, px_lane);
          uint32_t hm = __ballot_sync(FX_FULL, valid && !(m & FXO_DEAD) && hit);
          while (hm) {
            const int l = __ffs(hm) - 1;
            hm &= hm - 1;
            const uint32_t bm = __shfl_sync(FX_FULL, m, l);  // current state: an earlier fill may have changed it
            if (bm & (FXO_DEAD | FXO_SUBMITTED)) continue;
            const uint32_t kind = bm & FXO_KIND_MASK;
            if (kind == FXO_PAIR && !(bm & FXO_ACTIVE)) continue;
            // Completed or Margin: either way the entry leaves the table (a PAIR: sibling / group cancelled)
            const bool margin = fx_execute<LEAN>(pc, e, __shfl_sync(FX_FULL, sz, l), __shfl_sync(FX_FULL, px_lane, l), rs);
            any_fill = true;
            n_fills++;
            if (lane == l) m |= FXO_DEAD;
            if (kind == FXO_PARENT) {
              const uint32_t op = margin ? FX_OP_KILL : ((!LEAN && c.children_same_bar) ? FX_OP_ACTIVATE : FX_OP_ACTIVATE_NEXT);
              if (l < 31) { if (lane == l + 1) m = fx_apply_op(m, op); }
              else carry = op;
            }
          }
          const bool keep = valid && !(m & FXO_DEAD);
          const uint32_t km = __ballot_sync(FX_FULL, keep);
          if (keep) {
            const int dst = w + __popc(km & ((1u << lane) - 1u));
            if (dst != k) { gmeta[dst] = m; gp0[dst] = p0; gp1[dst] = p1; gsz[dst] = sz; }
            else if (m != m0) gmeta[dst] = m;
          }
          w += __popc(km);
        }
        n_live = w;
        ts.put(lane, 4, ((long long)n << 32) | (long long)n_fills);  // debug: table size, fills
      }
      fx_mark_to_market<LEAN>(pc, e, b.c);
      // DrawDown analyzer: one notify_fund + next per bar.  With no position and no execution the value is the one of
      // the previous bar and nothing can change.
      fx_step_drawdown(st, env, lane, e, any_fill, rsv);
    }
    ts.at(lane, 5);  // broker pass done, marked to market
    // candle of the next call (lanes 0..4): requested now, stored at the end of the env-step
    if (lane < 5) {
      const int tn = (t + 1 < total_bars) ? t + 1 : total_bars - 1;
      nbar_next = tb.candles[(start + tn) * (int64_t)C + (lane < 4 ? lane : c.price_col)];
    }

    double r;
    int n_final = n_live, n_acc_new = n_live;
    double sub_need_new = 0.0;
    if (!exhausted) {
      // hold mode: the substeps after the first run the coerced hold action 0 itself
      const bool hold = REPEAT && sub->j > 0 && (P.repeat_flags & FXENV_REPEAT_HOLD);
      const int action = hold ? 0
                              : (!LEAN && c.action_mode == FX_ACTION_CONTINUOUS) ? fx_coerce_continuous(c, action_raw_f)
                                                                                  : fx_coerce_discrete(action_raw_i);
      double atr = 0.0;
      bool atr_ready = false;
      if (ATR && action != 0) {
        // simple-mean ATR over the env's TR deque; TR(k) is a pure function of the table (SURVEY A.6): lanes fetch the
        // last min(t+1, period) bars in parallel, then the deque-order compensated sum (Python's sum()) runs uniformly
        const int period = c.atr_period;
        const int nb = (t + 1 < period) ? t + 1 : period;
        double s_ = 0.0, comp = 0.0;
        for (int j0 = 0; j0 < nb; j0 += 32) {
          double tr = 0.0;
          const int j = j0 + lane;
          if (j < nb) {
            const int k = t - nb + 1 + j;
            const double* rr = tb.candles + (start + k) * (int64_t)C;
            tr = fx_true_range(rr[1], rr[2], (k > 0) ? rr[3 - C] : 0.0, k > 0);
          }
          const int lim = (nb - j0 < 32) ? nb - j0 : 32;
          for (int q = 0; q < lim; q++) {
            const double x = __shfl_sync(FX_FULL, tr, q);
            if (j0 + q == 0) s_ = x; else fx_neumaier_add(s_, comp, x);
          }
        }
        atr = fx_neumaier_done(s_, comp) / (double)nb;
        atr_ready = nb >= period;
      }
      const bool has_min = (tb.minutes != nullptr);
      const int64_t minutes = (ATR && c.session_filter && has_min) ? tb.minutes[start + t] : 0;
      // new orders are appended straight to the (compacted) table (RESIDENT: the shared copy); their check_submitted cash
      // bound is accumulated by fx_push and kept in the env state for the next step
      FxOrderTab tg;
      tg.meta = gmeta; tg.p0 = gp0; tg.p1 = gp1; tg.sz = gsz;
      tg.n = n_live; tg.cap = P.cap; tg.dirty_from = n_live; tg.ndead = 0; tg.sub_need = 0.0; tg.bound_per = LEAN ? 1.0 : fx_bound_per(pc);
      FxAudit au;
      au.kind = FXENV_AU_KIND_NONE;
      fx_apply_action(c, pc, STRATEGY, e, tg, action, b, pair, atr, atr_ready, has_min, minutes, au);
      if (AUDIT && au.kind != FXENV_AU_KIND_NONE) fx_audit_store(P, env, lane, au, start + t, b.c);
      n_final = tg.n;
      sub_need_new = tg.sub_need;
      fx_publish(e, b.c, t);
      if (e.equity <= c.min_equity) e.flags |= FX_FLAG_TERMINATED | FX_FLAG_BROKE;  // app/bt_bridge.py:140-143
    } else {
      // the episode window ran out: a truncation with FXENV_TIME_LIMIT_WINDOW (equity > min_equity here: an env at or
      // below it terminated as broke on an earlier step)
      e.flags |= (TRUNC && (P.trunc_flags & FXENV_TIME_LIMIT_WINDOW)) ? (FX_FLAG_EXHAUSTED | FX_FLAG_TRUNCATED)
                                                                         : (FX_FLAG_TERMINATED | FX_FLAG_EXHAUSTED);
      e.prev_equity = st.prev_equity[env];
      e.bar_index = t + 1;
      e.position = e.psize > 0.0 ? 1 : (e.psize < 0.0 ? -1 : 0);
      e.price = b.c;
      n_acc_new = n_acc; sub_need_new = sub_need;  // nothing was processed
    }
    ts.at(lane, 6);  // strategy + publish

    // ---- reward plugin (app/env.py:148-155)
    r = fx_step_reward<REWARD, CARRY>(P, e, env, lane, ws, carry_in);
    const bool term = ((e.flags & FX_FLAG_TERMINATED) != 0u) || (e.equity <= c.min_equity);  // app/env.py:157
    bool trunc = TRUNC && (e.flags & FX_FLAG_TRUNCATED) != 0u;  // the window ran out (FXENV_TIME_LIMIT_WINDOW)
    if (REPEAT) {  // the step's reward: the substeps' sum in substep order, from r0; a terminating substep ends the step
      if (sub->j > 0) r = sub->racc + r;
      sub->racc = r;
      emit = emit || term || trunc;
    }
    if (TRUNC && (!REPEAT || emit)) {  // one decision more; the limit cuts an episode that did not terminate
      dec += 1;
      if (!term && !trunc && P.max_steps > 0 && dec >= P.max_steps) { e.flags |= FX_FLAG_TRUNCATED; trunc = true; }
    }
    ts.at(lane, 7);  // reward

    // ---- write back (lane 0): always-changing columns, then the ones a fill touched
    if (lane == 0) {
      st.t[env] = t; st.flags[env] = e.flags;
      st.equity[env] = e.equity; st.prev_equity[env] = e.prev_equity; st.price[env] = e.price;
      st.position[env] = e.position; st.bar_index[env] = e.bar_index;
      if (any_fill) {
        st.cash[env] = e.cash; st.psize[env] = e.psize; st.pprice[env] = e.pprice;
        st.commission_paid[env] = e.commission_paid; st.trades[env] = e.trades;
      }
      if (n_final != n) st.n_orders[env] = n_final;
      if (n_acc_new != n_acc) st.n_acc[env] = n_acc_new;
      if (sub_need_new != sub_need) st.sub_need[env] = sub_need_new;
      if (TRUNC) P.ep_steps[env] = dec;
      if (!REPEAT || emit) {
        o.reward[fx_out_idx(o, env)] = (float)r;
        if (o.reward64) o.reward64[fx_out_idx(o, env)] = r;
        o.terminated[fx_out_idx(o, env)] = term ? 1 : ((TRUNC && trunc) ? FXENV_DONE_TRUNCATED : 0);
        fx_write_scalars<LEAN>(P, e, total_bars, last_price, fx_obs_row(P, o, env), fx_obs_row16<O16>(o, env));
      }
      if (CARRY) {  // what the env's next step starts from, should this warp run it (the arrays above stay authoritative)
        double* __restrict__ cr = ws.carry;
        cr[FX_CARRY_CASH] = e.cash; cr[FX_CARRY_PSIZE] = e.psize; cr[FX_CARRY_PPRICE] = e.pprice; cr[FX_CARRY_EQUITY] = e.equity;
        cr[FX_CARRY_COMM] = e.commission_paid; cr[FX_CARRY_SUBNEED] = sub_need_new;
        *reinterpret_cast<int2*>(cr + FX_CARRY_FLAGS_T) = make_int2((int)e.flags, t);
        *reinterpret_cast<int2*>(cr + FX_CARRY_BARS_N) = make_int2(total_bars, n_final);
        *reinterpret_cast<int2*>(cr + FX_CARRY_NACC_TRADES) = make_int2(n_acc_new, e.trades);
        *reinterpret_cast<long long*>(cr + FX_CARRY_START) = start;
        if (TRUNC) *fx_carry_dec(ws) = dec;
        if (RESIDENT) {  // every index this ticket wrote is below the largest table size it saw: the write-back range,
                         // which leaves the global arrays exactly as the global-table kernel does (stale entries included)
          int32_t* hi = fx_carry_tab_hi(cr);
          if (n_final > *hi) *hi = n_final;
        }
      }
    }
  } else {  // timing experiment only (FXENV_DEBUG & 2): cursor only
    if (lane == 0) { st.t[env] = t; st.flags[env] = flags; st.bar_index[env] = t + 1; o.reward[fx_out_idx(o, env)] = 0.f; o.terminated[fx_out_idx(o, env)] = 0; }
  }
  ts.at(lane, 8);  // scalars written back

  // ---- observation windows (app/env.py:160 -> preprocessor.make_observation) from the staged copy.  They depend on
  // the bar cursor only (not on what the broker / strategy did); emitting them right after the order sweep (so that
  // the row's stores drain under the strategy / reward / write-back) was measured and is slower.
  // Running z-score statistics while the history window is still growing (or expanding_zscore): warm-up path, one
  // extra round trip here instead of registers held across the broker pass.
  if (REPEAT && emit && !last_sub && !(dbg & 1)) {
    __syncwarp();
    win_shift = fx_window_issue(tb, C, start, win_left, s_obs - win_left, lane, ws,
                                table_stats ? tb.stats + (start + t) * (int64_t)c.n_features * 2 : nullptr, c.n_features);
  }
  if (lane < c.n_features && (welford_live || ((!REPEAT || emit) && scale && !table_stats))) {
    const int64_t wi = ((int64_t)env * FXENV_MAX_FEATURES + lane) * 2;
    double wf_m = st.welford[wi], wf_m2 = st.welford[wi + 1];
    if (welford_live) {
      fx_welford_step(wf_m, wf_m2, row[c.feature_cols[lane]], t + 1);
      st.welford[wi] = wf_m; st.welford[wi + 1] = wf_m2;
    }
    if ((!REPEAT || emit) && scale && !table_stats) {
      double st_m, st_r;
      fx_welford_to_stats(wf_m, wf_m2, hn, st_m, st_r);
      ws.stat[2 * lane] = st_m; ws.stat[2 * lane + 1] = st_r;
    }
  }
  __syncwarp();
  if ((!REPEAT || emit) && !(dbg & 1)) {
    fx_window_wait(ws, phase);
    fx_emit_windows<FAST5, O16, LEAN>(P, lane, s_obs, scale, ws.win + win_shift, ws.stat, fx_obs_row(P, o, env), fx_obs_row16<O16>(o, env));
  }
  if (lane < 5 && !(dbg & 2)) st.nbar[(int64_t)env * 6 + lane] = nbar_next;
  if (CARRY) {
    if (lane < 5) ws.carry[FX_CARRY_NBAR + lane] = nbar_next;
    if (lane < FX_RS_N) ws.carry[FX_CARRY_RSTATS + lane] = rsv;
  }
  if (REPEAT) sub->ended = emit;
  ts.at(lane, 9);
  ts.global(lane, 11);
  return CARRY && !(dbg & 2);
}

// One step of up to P.repeat substeps (the REPEAT instantiations): substeps run until one ends the step.  They hand the
// env to each other through the carry record (RESIDENT: and the shared copy of the order table), so only the first one
// loads it from global memory.  Returns what the last substep returned.
template <int STRATEGY, int REWARD, unsigned V, bool O16>
__device__ __forceinline__ bool fx_step_repeat(const FxKernelParams& P, const void* __restrict__ actions, float* __restrict__ obs,
                                               float* __restrict__ reward, double* __restrict__ reward64,
                                               uint8_t* __restrict__ terminated, const int env, const int lane, const WarpSmem& ws,
                                               const unsigned phase, const unsigned step_row, const unsigned obs_slot_row,
                                               uint16_t* __restrict__ obs16, const int stride16, bool carry) {
  FxSubstep sub;
  sub.racc = 0.0;
  sub.ended = false;
#pragma unroll 1
  for (sub.j = 0;; ++sub.j) {
    carry = fx_step_env<STRATEGY, REWARD, V, O16, true>(P, actions, obs, reward, reward64, terminated, env, lane, ws, phase,
                                                        step_row, obs_slot_row, obs16, stride16, carry, &sub);
    if (sub.ended) break;
    __syncwarp();  // the substep's stores (state arrays, carry record) before the next substep's loads
  }
  return carry;
}

__device__ __forceinline__ int fx_ld_acquire(const int32_t* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void fx_st_release(int32_t* p, int v) {
  asm volatile("st.release.gpu.global.s32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}

// The single-step kernel: one warp per env, one env per CTA.  Launched with the programmatic-dependent-launch attribute:
// the NEXT kernel of the stream / graph may be scheduled while this grid drains (its CTAs take SM slots as ours exit and
// park at their own griddepcontrol.wait), which hides the launch gap between dependent steps.  Everything that touches
// memory written by the previous kernel comes after the wait.
template <int STRATEGY, int REWARD, unsigned V>
__global__ void __launch_bounds__(FX_WARPS * 32, FX_MIN_BLOCKS)
fx_step_kernel(const __grid_constant__ FxKernelParams P, const void* __restrict__ actions, float* __restrict__ obs,
               float* __restrict__ reward, double* __restrict__ reward64, uint8_t* __restrict__ terminated,
               const int env_begin, const int env_end, uint16_t* __restrict__ obs16, const int stride16, const FxTileSync sync) {
  static_assert((V & FX_V_RESIDENT) == 0, "the step kernel keeps no order table in shared memory");
  extern __shared__ __align__(16) unsigned char fx_smem[];
  const FxConfig& c = P.cfg;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int env = env_begin + blockIdx.x * FX_WARPS + warp;  // a launch covers the envs [env_begin, env_end)
  if (env >= env_end) return;
  const int ring_len = (REWARD == FX_REWARD_SHARPE) ? c.sharpe_window : 0;
  const int win_doubles = fx_window_doubles(c.window_size, c.n_cols);
  const WarpSmem ws = fx_carve(fx_smem + (size_t)warp * fx_warp_smem_bytes(win_doubles, ring_len), win_doubles, ring_len);
  asm volatile("griddepcontrol.launch_dependents;");
  fx_window_init(lane, ws);  // mbarrier init + fence
#ifdef FXENV_ENABLE_TIMING  // kernel-chain probe (tools/chain_probe.py): CTA 0 logs {kind, entry, after the wait, exit}
  long long* klog = nullptr;
  if (P.timeline && blockIdx.x == 0 && lane == 0 && obs16) {
    long long g0; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g0));
    const unsigned long long seqno = atomicAdd(reinterpret_cast<unsigned long long*>(P.timeline), 1ull);
    klog = P.timeline + 8 + (seqno % 1024ull) * 4;
    klog[0] = 1; klog[1] = g0;
  }
#endif
  if (sync.act_flag) {  // closed loop: this env's action is ready once the policy has published its 128-env tile
    if (lane == 0) {
      const int32_t* f = sync.act_flag + env / FX_SYNC_TILE;
      int polls = 0;
      while (fx_ld_acquire(f) < sync.epoch) {
        if (++polls > FX_SYNC_MAX_POLLS) { atomicAdd(sync.timeouts, 1); break; }
        __nanosleep(64);
      }
    }
    __syncwarp();
  } else {
    asm volatile("griddepcontrol.wait;" ::: "memory");
  }
#ifdef FXENV_ENABLE_TIMING
  if (klog) { long long g1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g1)); klog[2] = g1; }
#endif
  // the bf16 copy of the row (closed loop only) is a compile-time variant: no per-store pointer tests in the plain step
  if constexpr ((V & FX_V_REPEAT) != 0) {  // action repeat: the step's substeps (the emitting one writes both rows)
    if (obs16) fx_step_repeat<STRATEGY, REWARD, V, true>(P, actions, obs, reward, reward64, terminated, env, lane, ws, 0u, 0u, 0u, obs16, stride16, false);
    else fx_step_repeat<STRATEGY, REWARD, V, false>(P, actions, obs, reward, reward64, terminated, env, lane, ws, 0u, 0u, 0u, nullptr, 0, false);
  } else {
    if (obs16) fx_step_env<STRATEGY, REWARD, V, true>(P, actions, obs, reward, reward64, terminated, env, lane, ws, 0u, 0u, 0u, obs16, stride16);
    else fx_step_env<STRATEGY, REWARD, V, false>(P, actions, obs, reward, reward64, terminated, env, lane, ws);
  }
  if (sync.done_cnt) {  // this env's row (float32 and bf16) and state are complete: count it for its tile
    __syncwarp();
    if (lane == 0) {
      asm volatile("fence.proxy.async;" ::: "memory");  // the policy kernel reads the bf16 rows through TMA (async proxy)
      asm volatile("red.release.gpu.global.add.s32 [%0], 1;" :: "l"(sync.done_cnt + env / FX_SYNC_TILE) : "memory");
    }
  }
#ifdef FXENV_ENABLE_TIMING
  if (klog) { long long g2; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g2)); klog[3] = g2; }
#endif
}

// ---- K steps in ONE launch (fxenv_step_many): persistent warps pull (step chunk, env) tickets ----------------------
// The actions of the whole batch are supplied up front, so an env only depends on ITS OWN previous step.  A grid that
// fits the device at once keeps every warp slot busy for the whole batch: a warp takes the next ticket g from a
// global counter (round ch = g / N, env = g % N: all envs of a round are handed out before the next round), waits until
// seq[env] == first step of the round (acquire; the warp that ran the env's previous round released it), runs the round's
// consecutive steps of that env (FxChunkPlan), publishes seq[env] = first step of the next round (release).  No kernel boundary, CTA turnaround
// or grid-wide barrier between steps; heavy env-steps (many fills) only delay their own env.  The hand-over between
// warps costs a fence that drains the row's streaming stores, the sequence-word store and an acquire round trip
// (~20 % of a step at chunk = 1): the chunk length amortises it (fx_rollout_plan).  No deadlock: the ticket an env-step
// waits for is lower than its own, and every ticket handed out belongs to a running warp that needs nothing from higher
// tickets.  seq[] and the counter are epoch-based (see below), or zeroed by a stream-ordered memset inside captures.
// RESIDENT (FxKernelParams::order_smem): a ticket keeps its env's order table in the warp's shared memory, loaded by its
// first step and written back before the release -- no order-table round trip on the steps in between.  The table
// (28 B per entry) does not fit next to 16 one-warp CTAs per SM with their 1 KB reservation each: FX_RES_WARPS warps per
// CTA instead, still 16 warps per SM (the warps are independent; there is no block barrier).
#ifndef FX_ROLLOUT_MIN_BLOCKS
#define FX_ROLLOUT_MIN_BLOCKS FX_MIN_BLOCKS
#endif
template <int STRATEGY, int REWARD, unsigned V>
__global__ void __launch_bounds__(FX_ROLLOUT_WARPS((V & FX_V_RESIDENT) != 0) * 32,
                                  FX_ROLLOUT_MIN_BLOCKS * FX_WARPS / FX_ROLLOUT_WARPS((V & FX_V_RESIDENT) != 0))
fx_rollout_kernel(const __grid_constant__ FxKernelParams P, const char* __restrict__ actions, float* __restrict__ obs,
                  const int obs_slots, float* __restrict__ reward, uint8_t* __restrict__ terminated,
                  const __grid_constant__ FxChunkPlan plan, const unsigned seq_base, const unsigned ticket_base) {
  constexpr bool RESIDENT = (V & FX_V_RESIDENT) != 0;
  extern __shared__ __align__(16) unsigned char fx_smem[];
  const FxConfig& c = P.cfg;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ring_len = (REWARD == FX_REWARD_SHARPE) ? c.sharpe_window : 0;
  const int win_doubles = fx_window_doubles(c.window_size, c.n_cols);
  const int tab = RESIDENT ? P.cap + FXO_SLACK : 0;
  const WarpSmem ws = fx_carve(fx_smem + (size_t)warp * fx_warp_smem_bytes(win_doubles, ring_len, tab), win_doubles, ring_len, tab);
  asm volatile("griddepcontrol.launch_dependents;");  // the next batch's launch latency hides behind this one
  fx_window_init(lane, ws);
  const unsigned N = (unsigned)c.num_envs;
  const unsigned total = N * (unsigned)plan.n_rounds;  // tickets; N * n_steps < 2^31 (checked by the caller)
  unsigned* ticket = reinterpret_cast<unsigned*>(P.seq + N);
  asm volatile("griddepcontrol.wait;" ::: "memory");  // everything below touches memory the previous launch wrote
  // seq[] and the ticket counter are never reset: this launch's values start at seq_base / ticket_base (kept by the
  // host: every launch leaves seq[env] = seq_base + n_steps and the counter at ticket_base + total + #warps, because
  // each warp draws exactly one ticket >= total).  Unsigned differences make the 2^32 wrap harmless.
  unsigned g = 0u;
  if (lane == 0) g = atomicAdd(ticket, 1u) - ticket_base;
  g = __shfl_sync(FX_FULL, g, 0);
  unsigned phase = 0u;
  while (g < total) {
    // the ticket after this one is requested now: its atomic round trip hides behind the env-step
    unsigned g_next = 0u;
    if (lane == 0) g_next = atomicAdd(ticket, 1u) - ticket_base;
    const unsigned ch = g / N, env = g - ch * N;
    unsigned k, k_end;  // the steps of round ch (FxChunkPlan)
    if (ch < (unsigned)plan.n_uniform) { k = ch * (unsigned)plan.chunk; k_end = k + (unsigned)plan.chunk; }
    else { k = (unsigned)plan.tail_start[ch - plan.n_uniform]; k_end = (unsigned)plan.tail_start[ch - plan.n_uniform + 1]; }
    if (k > 0u) {
      if (lane == 0) { while ((unsigned)fx_ld_acquire(P.seq + env) != seq_base + k) __nanosleep(32); }
      __syncwarp();
    }
    // the warp keeps the env for `chunk` consecutive steps: between them the state goes through memory as always, but
    // within one warp (__syncwarp orders it) -- no fence, no sequence word, no acquire round trip
    bool carry = false;  // ws.carry holds this env's state as of step k (the warp ran step k - 1 itself)
    unsigned slot_row = (k % (unsigned)obs_slots) * N;  // row offset of step k's slot in the observation ring
#pragma unroll 1
    for (; k < k_end; ++k) {
#if defined(FXENV_ENABLE_TIMING) || defined(FXENV_ENABLE_TIMELINE)
      if (P.timeline && lane == 0) { long long g__; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g__)); P.timeline[((size_t)k * N + env) * 2] = g__; }
#endif
      if constexpr ((V & FX_V_REPEAT) != 0)  // action repeat: the decision's substeps, one window copy among them
        carry = fx_step_repeat<STRATEGY, REWARD, V, false>(P, actions, obs, reward, nullptr, terminated, (int)env, lane, ws, phase,
                                                           k * N, slot_row, nullptr, 0, carry);
      else
        carry = fx_step_env<STRATEGY, REWARD, V, false, true>(P, actions, obs, reward, nullptr, terminated, (int)env, lane, ws, phase,
                                                              k * N, slot_row, nullptr, 0, carry);
      slot_row += N;
      if (slot_row == (unsigned)obs_slots * N) slot_row = 0u;
      __syncwarp();
      phase++;  // every step (every decision, with the repeat) issued and waited on exactly one copy
#if defined(FXENV_ENABLE_TIMING) || defined(FXENV_ENABLE_TIMELINE)
      if (P.timeline && lane == 0) { long long g__; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g__)); P.timeline[((size_t)k * N + env) * 2 + 1] = g__; }
#endif
    }
    if (RESIDENT && carry) {  // the shared copy is the current table: back to global memory, published by the release
      const int64_t ob = (int64_t)env * (P.cap + FXO_SLACK);
      const int n = *fx_carry_tab_hi(ws.carry);
      fx_table_copy(P.st.o_meta + ob, P.st.o_p0 + ob, P.st.o_p1 + ob, P.st.o_sz + ob, ws.ometa, ws.op0, ws.op1, ws.osz, n, lane);
      __syncwarp();
    }
    if (lane == 0) fx_st_release(P.seq + env, (int)(seq_base + k_end));
    g = __shfl_sync(FX_FULL, g_next, 0);
  }
}

// The kernels of one (strategy, reward, key) of the half HALF (its FX_V_TRUNC | FX_V_PARAMS bits): none for a key of
// another half or one that fx_variant_valid rejects.  The step kernel has no resident order table, so keys with and
// without FX_V_RESIDENT share it.
constexpr unsigned FX_V_HALF = FX_V_TRUNC | FX_V_PARAMS;
template <unsigned HALF, int STRATEGY, int REWARD, unsigned V>
FxEnvKernels fx_variant_entry() {
  if constexpr ((V & FX_V_HALF) == HALF && fx_variant_valid(STRATEGY, V))
    return {fx_step_kernel<STRATEGY, REWARD, V & ~FX_V_RESIDENT>, fx_rollout_kernel<STRATEGY, REWARD, V>};
  else
    return {nullptr, nullptr};
}

template <unsigned HALF, size_t... I>
FxEnvKernels fx_variant_table(int strategy, int reward, unsigned key, std::index_sequence<I...>) {
  static const FxEnvKernels table[] = {
      fx_variant_entry<HALF, (int)(I / (FX_N_REWARDS * FX_V_KEYS)), (int)(I / FX_V_KEYS % FX_N_REWARDS), (unsigned)(I % FX_V_KEYS)>()...};
  return table[((size_t)strategy * FX_N_REWARDS + (size_t)reward) * FX_V_KEYS + key];
}

// The lookup over every (strategy, reward, key) whose FX_V_TRUNC | FX_V_PARAMS bits are HALF: the translation unit that
// calls it instantiates exactly those kernels.
template <unsigned HALF>
FxEnvKernels fx_variant_lookup(int strategy, int reward, unsigned key) {
  return fx_variant_table<HALF>(strategy, reward, key, std::make_index_sequence<FX_N_STRATEGIES * FX_N_REWARDS * FX_V_KEYS>());
}

}  // namespace
