/*
 * include/fxenv.h -- C-ABI of libfxenv.so: the H100-native (sm_90a) vectorised gym-fx env.step() hot path.
 *
 * The reference (harveybc/gym-fx) is pure Python and has no FFI of its own; the boundary below is what a
 * Python binding (ctypes, see INTEGRATION.md) of its per-tick path would bind.  Each entry point cites the
 * reference interface it replaces (paths relative to the reference tree):
 *
 *   fxenv_create / fxenv_destroy   GymFxEnv.__init__ / close            app/env.py:36-97, 177-178
 *   fxenv_load_candles             data_feed load_data -> dataframe     data_feed_plugins/default_data_feed.py:36-56
 *                                  + GymFxEnv.dataframe / total_bars    app/env.py:63-68
 *   fxenv_reset                    GymFxEnv.reset                       app/env.py:102-129 (+ bt_bridge.py:33-66)
 *   fxenv_step / fxenv_step_host   GymFxEnv.step                        app/env.py:131-172
 *                                  (BTBridgeStrategy.next               app/bt_bridge.py:119-150,
 *                                   strategy apply_action               strategy_plugins/direct_{fixed,atr}_sltp.py,
 *                                   backtrader BackBroker.next          [external],
 *                                   reward compute_reward               reward_plugins/{pnl,sharpe,dd_penalized}_reward.py,
 *                                   preprocessor make_observation       preprocessor_plugins/{default,feature_window}_preprocessor.py)
 *   fxenv_observe                  GymFxEnv._make_observation           app/env.py:226-242
 *   fxenv_get_info                 GymFxEnv._make_info                  app/env.py:244-254
 *   fxenv_get_state/set_state      (no counterpart: env snapshot, SURVEY 8f #4)
 *   fxenv_rollout / fxenv_rollout_ex  the caller loop of app/main.py:57-65 with a learned policy (see below);
 *                                  continuous actions are the Box(-1, 1, (1,)) of app/env.py:71-80, 187-204
 *   fxenv_set_action_repeat        (no counterpart: k bars per step, one decision per step; its contract below)
 *   fxenv_set_time_limit           (no counterpart: Gymnasium's max_episode_steps and truncation; its contract below)
 *   fxenv_set_env_params           (no counterpart: per-env commission / leverage / slippage / SL / TP; its contract below)
 *   fxenv_policy_set_obs_norm      (no counterpart: the policy's running observation normalizer, SB3 VecNormalize /
 *   fxenv_obs_moments               CleanRL NormalizeObservation; its contract below)
 *   fxenv_return_moments           (no counterpart: SB3 VecNormalize(norm_reward), gymnasium NormalizeReward; its contract
 *                                   below)
 *
 * Conventions: every function returns 0 on success, <0 on error (see FXENV_E_*); fxenv_last_error() gives the
 * message.  No exceptions or aborts cross the ABI.  The library owns env state (device struct-of-arrays) behind
 * an opaque handle; the CALLER owns every I/O buffer and passes raw pointers (+ a cudaStream_t as void*).
 * "_dev" pointers are device memory, "_host" pointers host memory (pinned for best speed).  A handle is bound
 * to the CUDA device that was current at fxenv_create and is not thread-safe.  No host synchronisation happens
 * inside fxenv_step/fxenv_reset/fxenv_observe: work is enqueued on the caller's stream.
 */
#ifndef FXENV_H_
#define FXENV_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FXENV_ABI_VERSION 2
#define FXENV_MAX_PAIRS 8
#define FXENV_MAX_FEATURES 16
#define FXENV_MAX_COLS 16

/* status codes */
#define FXENV_OK 0
#define FXENV_E_INVALID (-1)   /* bad argument / unsupported configuration */
#define FXENV_E_CUDA (-2)      /* a CUDA runtime call failed */
#define FXENV_E_STATE (-3)     /* call out of order (e.g. step before candles were loaded / before reset) */
#define FXENV_E_NOMEM (-4)

/* enumerations used in FxConfig */
enum { FX_ACTION_DISCRETE = 0, FX_ACTION_CONTINUOUS = 1 };
enum { FX_STRATEGY_DEFAULT = 0, FX_STRATEGY_FIXED_SLTP = 1, FX_STRATEGY_ATR_SLTP = 2 };
enum { FX_PREPROC_DEFAULT = 0, FX_PREPROC_FEATURE_WINDOW = 1 };
enum { FX_SCALING_NONE = 0, FX_SCALING_ROLLING = 1, FX_SCALING_EXPANDING = 2 };
enum { FX_REWARD_PNL = 0, FX_REWARD_SHARPE = 1, FX_REWARD_DD = 2 };
enum { FX_SIZE_FX_UNITS = 0, FX_SIZE_NOTIONAL = 1 };

/* per-env status bits (FxInfoPtrs.flags) */
#define FX_FLAG_STARTED 1u        /* the first step() (which does not advance the bar) has happened */
#define FX_FLAG_TERMINATED 2u     /* bridge.terminated                    app/bt_bridge.py:141,154 */
#define FX_FLAG_EXHAUSTED 4u      /* data ran out (strategy.stop())       app/bt_bridge.py:152-155 */
#define FX_FLAG_BROKE 8u          /* equity <= min_equity                 app/bt_bridge.py:203-204 */
#define FX_FLAG_ORDER_OVERFLOW 16u/* order table full: an order was dropped (the reference is unbounded) */
#define FX_FLAG_TRADE_PRICE_OWN 32u /* statistics bookkeeping: the open trade's average price differs from the position's */
/* FX_FLAG_TRUNCATED (64u): see fxenv_set_time_limit */

/*
 * The reference resolves one "dict of everything" at call time (app/config.py:1-45, plugin_params of every
 * plugin, app/main.py:42-45).  The host side resolves it ONCE, per each plugin's own precedence rules, into
 * this POD.  All doubles are used exactly as the reference uses the corresponding Python float.
 */
typedef struct FxConfig {
  int32_t struct_size;              /* = sizeof(FxConfig); checked by fxenv_create */
  int32_t num_envs;
  int32_t num_pairs;                /* candle tables; env i trades pair (i % num_pairs) */
  int32_t n_cols;                   /* float64 columns per candle row; cols 0..4 = OPEN,HIGH,LOW,CLOSE,VOLUME */
  int32_t order_capacity;           /* order-table entries per env (0 = default 128) */
  int32_t auto_reset;               /* 1: an env that terminated at step k is reset at step k+1 */
  int64_t episode_bars;             /* bars per episode window; 0 = from the start bar to the end of the table */

  /* GymFxEnv                                                         app/env.py:56-80 */
  double initial_cash;
  double position_size;             /* default order flow size         app/bt_bridge.py:172 */
  double min_equity;
  int32_t action_mode;              /* FX_ACTION_*                     app/env.py:71-80,187-204 */
  int32_t _pad0;
  double continuous_action_threshold;

  /* default_broker -> backtrader BackBroker                          broker_plugins/default_broker.py:35-53 */
  double commission;                /* fraction of notional */
  double leverage;
  double slippage_perc;             /* fraction of price per fill, set_slippage_perc(perc, slip_open/limit/match=True) */
  int32_t children_same_bar;        /* 0 (backtrader: bracket children activate next cycle) | 1 */

  /* strategy plugin                                                  strategy_plugins/direct_{fixed,atr}_sltp.py */
  int32_t strategy;                 /* FX_STRATEGY_* */
  double strat_position_size;
  double sl_pips, tp_pips, pip_size;              /* direct_fixed_sltp.py:24-29 */
  double pair_pip_size[FXENV_MAX_PAIRS];          /* per-pair override of pip_size (0 = use pip_size) */
  int32_t atr_period;                             /* direct_atr_sltp.py:49-86 */
  int32_t use_rel_volume;
  double k_sl, k_tp;
  double rel_volume, strat_leverage, min_order_volume, max_order_volume;
  int32_t size_mode;                /* FX_SIZE_* */
  int32_t use_min_frac, use_max_frac;
  int32_t session_filter;
  double min_sltp_frac, max_sltp_frac;
  int32_t entry_dow_start, entry_hour_start, force_close_dow, force_close_hour;

  /* preprocessor plugin                                              preprocessor_plugins/ *.py */
  int32_t preproc;                  /* FX_PREPROC_* */
  int32_t window_size;
  int32_t price_col;                /* column index of price_column */
  int32_t n_features;
  int32_t feature_cols[FXENV_MAX_FEATURES];
  int32_t feature_binary[FXENV_MAX_FEATURES];
  int32_t scaling;                  /* FX_SCALING_* */
  int32_t scaling_window;
  int32_t include_price_window, include_agent_state;
  double feature_clip;
  double obs_position_size;         /* config.get("position_size", 1.0) as read by the preprocessors */

  /* reward plugin                                                    reward_plugins/ *.py */
  int32_t reward;                   /* FX_REWARD_* */
  int32_t sharpe_window;
  double reward_initial_cash;       /* float(config["initial_cash"]) or 1.0 */
  double reward_scale;
  double annualization_factor;
  double penalty_lambda;
} FxConfig;

typedef struct FxEnv FxEnv;

/* Device pointers to the per-env info columns (arrays of num_envs), valid until fxenv_destroy.
 * Mirrors GymFxEnv._make_info (app/env.py:244-254) + step()'s additions (:162-166). */
typedef struct FxInfoPtrs {
  const double* equity;
  const double* prev_equity;        /* pnl = equity - prev_equity */
  const double* price;
  const double* cash;
  const double* position_size;      /* signed units held */
  const double* position_price;
  const double* commission_paid;
  const int32_t* position;          /* -1 / 0 / +1 */
  const int32_t* bar_index;         /* bridge.bar_index = len(data) = local bar + 1 */
  const int32_t* total_bars;
  const int32_t* trades;
  const int32_t* n_orders;          /* live order-table entries */
  const uint32_t* flags;            /* FX_FLAG_* */
  /* [num_envs][FXENV_RUN_STATS] float64: what backtrader's DrawDown / TradeAnalyzer / SQN analyzers (attached by
   * app/bt_bridge.py:230-234) hold for the current episode -- the inputs of GymFxEnv.summary()
   * (app/env.py:256-271 -> metrics_plugins/default_metrics.py:48-60).  Field order: FXENV_RS_*. */
  const double* run_stats;
} FxInfoPtrs;

#define FXENV_RUN_STATS 12
enum {
  FXENV_RS_DD_MAXVALUE = 0, /* running peak of the broker value */
  FXENV_RS_DD_MAX_MONEY,    /* drawdown.max.moneydown */
  FXENV_RS_DD_MAX_PCT,      /* drawdown.max.drawdown (percent) */
  FXENV_RS_TR_PNL, FXENV_RS_TR_COMM, FXENV_RS_TR_PRICE, /* the open trade (TR_PRICE valid only with FX_FLAG_TRADE_PRICE_OWN) */
  FXENV_RS_PNL_NET,         /* trades.pnl.net.total (average = / closed trades = FxInfoPtrs.trades) */
  FXENV_RS_PNL_SQ,          /* sum of squares of the closed trades' net pnl: with n = FxInfoPtrs.trades, mean = PNL_NET / n,
                             * sqn = sqrt(n) * mean / sqrt(PNL_SQ / n - mean^2)  (n > 1) */
  FXENV_RS_SPARE,
  FXENV_RS_OPENED,          /* trades.total.total */
  FXENV_RS_WON, FXENV_RS_LOST
};

int fxenv_abi_version(void);

/* Replaces GymFxEnv.__init__ (app/env.py:36-97: config resolution, spaces, min_equity) and, per reset, build_cerebro /
 * build_bt_broker (app/bt_bridge.py:207-238, broker_plugins/default_broker.py:35-53).  Validates the POD config and
 * allocates the per-env device state; fails (no CPU path) when no CUDA device is available. */
int fxenv_create(const FxConfig* cfg, FxEnv** out);
/* Replaces GymFxEnv.close (app/env.py:177-178). */
int fxenv_destroy(FxEnv* env);
const char* fxenv_last_error(const FxEnv* env); /* env may be NULL: error of the last failed fxenv_create */

/* Replaces data_feed.load_data + build_bt_feed (data_feed_plugins/default_data_feed.py:36-79: the dataframe the env
 * keeps, app/env.py:62-67, incl. its "too short for the window" ValueError).
 * Copies a host float64 [T, n_cols] row-major candle table (and optional int64 [T] minutes-since-epoch
 * timestamps, needed only by the ATR session filter) to the device, and precomputes the per-bar rolling
 * z-score statistics.  Synchronous.  A table may be loaded again at any time, in place of the pair's previous one: the
 * cached step-many graphs and each policy's rollout graph are captured again on their next use, with the new table and
 * the kernel choice its data make (fxenv_debug_lean). */
int fxenv_load_candles(FxEnv* env, int pair_id, const double* candles_host, int64_t T, const int64_t* minutes_host);

/* Replaces the observation_space bookkeeping of app/env.py:81-90.
 * Number of float32 per observation row and the offsets of its parts (flat layout, SURVEY A.2):
 * [features W*F | prices W | returns W | position | equity_norm | unrealized_pnl_norm | steps_remaining_norm] */
int64_t fxenv_obs_dim(const FxEnv* env);

/* Replaces GymFxEnv.reset (app/env.py:102-129: new bridge / broker / feed, first publish at bar 0).
 * start_bar_dev: int64 [num_envs] first bar (row of the pair's table) of each env's episode window, or NULL to
 * keep the current ones (all 0 after create).  mask_dev: uint8 [num_envs], reset only where != 0, or NULL = all. */
int fxenv_reset(FxEnv* env, const int64_t* start_bar_dev, const uint8_t* mask_dev, void* stream);

/* Replaces _make_observation for the current state (app/env.py:226-242 -> preprocessor.make_observation).
 * Writes the observation of the current state (what reset() returns). obs_dev: float32 [num_envs, obs_dim]. */
int fxenv_observe(FxEnv* env, float* obs_dev, void* stream);

/* Replaces GymFxEnv.step (app/env.py:131-172) and everything below it: BTBridgeStrategy.next (app/bt_bridge.py:119-150),
 * the strategy / reward / preprocessor plugins and backtrader's broker pass.
 * One env.step() for every env.  actions_dev: int32 [num_envs] (discrete) or float32 [num_envs] (continuous).
 * obs_dev float32 [num_envs, obs_dim]; reward_dev float32 [num_envs]; terminated_dev uint8 [num_envs].
 * reward64_dev: optional float64 [num_envs] copy of the reward before the float32 cast (may be NULL). */
int fxenv_step(FxEnv* env, const void* actions_dev, float* obs_dev, float* reward_dev, uint8_t* terminated_dev,
               double* reward64_dev, void* stream);

/* n_steps consecutive steps with the actions of the whole batch supplied up front (replayed / random / scripted
 * drivers: strategy_plugins/default_strategy.py:38-53, the loop of app/main.py:57-65); step k reads
 * actions_dev + k*num_envs and writes reward/terminated at k*num_envs; obs rows go to
 * obs_dev + (k % obs_slots)*num_envs*obs_dim (obs_slots >= 1).  Results are identical to n_steps calls of fxenv_step.
 * Two engines (fxenv_step_many_engine): 1 = one persistent launch whose warps pull (round of consecutive steps, env)
 * tickets and honour per-env dependencies only (every batch of more than one step); 0 = a CUDA graph of n_steps
 * single-step launches, cached by pointer set. */
int fxenv_step_many(FxEnv* env, int n_steps, const void* actions_dev, float* obs_dev, int obs_slots,
                    float* reward_dev, uint8_t* terminated_dev, void* stream);

/* Which engine fxenv_step_many would use for a batch of n_steps (1 persistent launch / 0 graph of steps), <0 on error. */
int fxenv_step_many_engine(const FxEnv* env, int n_steps);

/* Same as fxenv_step for callers that hold numpy / host buffers like the reference's own loop (app/main.py:57-65,
 * tools/smoke_test.py:79-83).  Reference-facing call with HOST buffers: H2D actions, one step, D2H obs/reward/terminated, then waits. */
int fxenv_step_host(FxEnv* env, const void* actions_host, float* obs_host, float* reward_host,
                    uint8_t* terminated_host);

/* Replaces GymFxEnv._make_info (app/env.py:244-254): zero-copy device views instead of a dict of Python floats. */
int fxenv_get_info(FxEnv* env, FxInfoPtrs* out);

/* No reference counterpart (its env cannot be cloned: one daemon thread per instance, app/bt_bridge.py:30-66).
 * Snapshot / restore of the whole env state (host buffer of fxenv_state_bytes() bytes). Synchronous. */
int64_t fxenv_state_bytes(const FxEnv* env);
int fxenv_get_state(FxEnv* env, void* buf_host, int64_t nbytes);
int fxenv_set_state(FxEnv* env, const void* buf_host, int64_t nbytes);

/* Kernels launched by this handle since creation (bench.py's gpu_launches). */
int64_t fxenv_launch_count(const FxEnv* env);

/* ---- episode starts and episode records (no reference counterpart: a Gymnasium vector env begins a NEW episode on
 * auto-reset, and RecordEpisodeStatistics keeps the results of the one that ended) ----------------------------------
 * Start ranges: env i may be given an inclusive range [lo_i, hi_i] of start bars (rows of its pair's table) and the
 * handle a 64-bit seed.  An episode begun from the ranges -- every auto-reset, and fxenv_reset with start_bar_dev == NULL
 * (an explicit start_bar_dev still wins) -- starts at
 *   start = lo + umulhi64(splitmix64(seed ^ ((uint64)i << 32 | (uint32)k)), hi - lo + 1)
 * where k counts the episodes env i has begun since fxenv_create (explicit resets included) and splitmix64 is the
 * standard finaliser (z += 0x9E3779B97F4A7C15; z = (z ^ z >> 30) * 0xBF58476D1CE4E5B9; z = (z ^ z >> 27) *
 * 0x94D049BB133111EB; z ^ z >> 31).  Without ranges (the default) an episode restarts at the env's current start.
 * lo_host / hi_host: int64 [num_envs], 0 <= lo <= hi <= T_pair - 1 for pair i % num_pairs; both NULL clears the ranges.
 * Needs the candles loaded (FXENV_E_STATE otherwise).  Synchronous.  The ranges, the seed and the counters live in the
 * env state: snapshots carry them. */
int fxenv_set_reset_starts(FxEnv* env, const int64_t* lo_host, const int64_t* hi_host, uint64_t seed);

/* Episode record: when a reset (auto or explicit) ends an episode that has FX_FLAG_STARTED, the env stores what its
 * analyzers held at the end of it in last_episode and increments episodes_done, once per episode.  The record keeps the
 * last finished episode per env; the first reset after create records nothing. */
#define FXENV_EPISODE_STATS 14
enum {
  FXENV_EP_START = 0,       /* first bar (table row) of the episode */
  FXENV_EP_BARS,            /* bars it ran (bridge.bar_index) */
  FXENV_EP_EQUITY,          /* final equity */
  FXENV_EP_COMMISSION,      /* commission paid */
  FXENV_EP_END_FLAGS,       /* flags & (FX_FLAG_TERMINATED | FX_FLAG_EXHAUSTED | FX_FLAG_BROKE | FX_FLAG_TRUNCATED);
                             * 0 = cut short by a reset */
  FXENV_EP_DD_MAX_PCT,      /* drawdown.max.drawdown (percent) */
  FXENV_EP_DD_MAX_MONEY,    /* drawdown.max.moneydown */
  FXENV_EP_PNL_NET,         /* trades.pnl.net.total */
  FXENV_EP_PNL_SQ,          /* sum of squares of the closed trades' net pnl */
  FXENV_EP_OPENED,          /* trades opened */
  FXENV_EP_CLOSED,          /* trades closed */
  FXENV_EP_WON, FXENV_EP_LOST,
  FXENV_EP_INDEX            /* the episode's k (see fxenv_set_reset_starts) */
};

/* Device pointers into the env state, valid until fxenv_destroy. */
typedef struct FxEpisodePtrs {
  const int64_t* start;           /* [num_envs] first bar of the current episode */
  const int32_t* episodes_done;   /* [num_envs] episodes recorded since create */
  const double* last_episode;     /* [num_envs][FXENV_EPISODE_STATS], FXENV_EP_* order (zeros until the first record) */
} FxEpisodePtrs;

int fxenv_get_episode_info(FxEnv* env, FxEpisodePtrs* out);

/* ---- bracket audit: the GYMFX_BRACKET_AUDIT log of direct_atr_sltp (strategy_plugins/direct_atr_sltp.py:35-45,
 * :138-142, :188-191, :199-202) -----------------------------------------------------------------------------------
 * With the log on, every env-step of the ATR strategy that the reference would log writes one record of
 * FXENV_AU_FIELDS doubles into a per-env ring of `capacity` records:
 *   long_bracket / short_bracket: action 1 / 2 once the session entry check and the ready / atr > 0 / size > 0 /
 *     close > 0 checks pass, and only when the position is <= 0 / >= 0 (a short / long is closed first, same call);
 *   session_force_close: the bar is in the close zone and the position is non-zero, whatever the action.
 * A record is written whether or not its orders later fill or are rejected, and also when the order table had no room
 * for them (FX_FLAG_ORDER_OVERFLOW drops the orders, the reference's unbounded list would have taken them).  At most one
 * record per env-step; records of one env stay in call order.  The other strategies write nothing.
 * written[i] counts env i's records since the log was enabled; record j of env i sits at
 * records[(i * capacity + j % capacity) * FXENV_AU_FIELDS].  The ring and the counters live outside the env state:
 * fxenv_state_bytes and snapshots do not include them, and fxenv_reset / fxenv_set_state leave them alone. */
#define FXENV_AU_FIELDS 8
enum {
  FXENV_AU_KIND = 0,   /* FXENV_AU_KIND_* */
  FXENV_AU_BAR,        /* table row of the signal bar (start + t) */
  FXENV_AU_EPISODE,    /* the episode's k (FXENV_EP_INDEX) */
  FXENV_AU_ENTRY,      /* close of the signal bar */
  FXENV_AU_STOP,       /* stop price passed to buy_bracket / sell_bracket (NaN for a force-close) */
  FXENV_AU_LIMIT,      /* limit price (NaN for a force-close) */
  FXENV_AU_SIZE,       /* _compute_size; for a force-close the signed position before the close fills */
  FXENV_AU_ATR         /* simple-mean ATR (NaN for a force-close) */
};
enum { FXENV_AU_KIND_NONE = 0, FXENV_AU_KIND_LONG = 1, FXENV_AU_KIND_SHORT = 2, FXENV_AU_KIND_FORCE_CLOSE = 3 };

/* capacity > 0: (re)allocates the ring for capacity records per env and zeroes the counters (log on); 0: frees it (log
 * off); < 0 or too large: FXENV_E_INVALID.  Accepted for every strategy.  Synchronous. */
int fxenv_set_bracket_audit(FxEnv* env, int32_t capacity);

/* Device pointers of the log, valid until the next fxenv_set_bracket_audit / fxenv_destroy; all NULL / 0 when off. */
typedef struct FxAuditPtrs {
  const double* records;    /* [num_envs][capacity][FXENV_AU_FIELDS] */
  const int64_t* written;   /* [num_envs] */
  int32_t capacity;
} FxAuditPtrs;

int fxenv_get_bracket_audit(FxEnv* env, FxAuditPtrs* out);

/* ---- action repeat: one step spans up to k bars, with one observation and one decision per step (no reference
 * counterpart: the frame_skip of vectorised RL envs; "act every k bars") --------------------------------------------
 * A handle has an action repeat k (1 <= k <= FXENV_MAX_REPEAT, default 1) and a mode:
 *   repeat (flags 0, the default): the step's action is applied on each of the k bars (Atari frame-skip);
 *   hold (FXENV_REPEAT_HOLD): the action is applied on the first bar only; the other bars run with the hold action --
 *     the coerced action 0 itself, not a raw action that is thresholded.
 * One step of fxenv_step / fxenv_step_host, and one decision of fxenv_step_many and fxenv_rollout, consists of up to k
 * SUBSTEPS, each exactly one step of the library without repeat (so parity with the reference covers each of them):
 *   1. An env that is terminated when the step begins runs one substep only: what a step does today (the auto-reset
 *      step: reward 0, not done, observation of the new episode; without auto-reset (obs, 0.0, True)).  Substeps never
 *      continue into a new episode.
 *   2. Otherwise substeps j = 0, 1, ... run in order; the step stops after substep k - 1 or after the first substep that
 *      terminates (broke, or data exhausted).  "The first step does not advance the bar" holds per substep: the first
 *      decision of an episode covers k - 1 new bars, as the expanded action stream does in the reference.
 *   3. The observation is that of the state after the last substep run, `terminated` is that substep's flag, and the
 *      reward is the float64 sum of the substep rewards in substep order, starting from r0 (so k = 1 keeps the sign of
 *      a zero): reward64 is that sum, reward (float) of it.  With the Sharpe reward this is a sum of k rolling Sharpe
 *      values.
 *   4. All state advances per substep: account, order table, run statistics, Sharpe deque, drawdown peak, running
 *      z-score statistics, episode records and the bracket audit (one record per bar that logs, with that bar's row).
 *      The info columns after a step are those after its last substep.
 * Equivalently: for every env, the outputs of a step equal those of the library without repeat driven by the env's
 * expanded action stream, taken at the step's last substep, with the rewards summed as above.
 * k and the mode belong to the handle, like the bracket audit, and are not env state: fxenv_state_bytes, snapshots,
 * fxenv_reset and fxenv_set_state neither include nor change them.  Changing them drops the cached step-many graphs and
 * makes each policy re-capture its rollout graph.  Out-of-range repeat or unknown flag bits: FXENV_E_INVALID. */
#define FXENV_MAX_REPEAT 256
#define FXENV_REPEAT_HOLD 1u
int fxenv_set_action_repeat(FxEnv* env, int32_t repeat, uint32_t flags);

/* ---- time limit and truncation: an episode cut short is reported as truncated, not terminated (no reference
 * counterpart: Gymnasium's max_episode_steps / TimeLimit; a learner bootstraps through a truncation) ----------------
 * max_steps > 0 ends an episode at the end of its max_steps-th DECISION: one step of fxenv_step / fxenv_step_host, one
 * decision of fxenv_step_many / fxenv_rollout (with an action repeat k it spans up to k bars).  The first step of an
 * episode (it does not advance the bar) is decision 1; an auto-reset step belongs to neither episode and does not
 * count.  max_steps = 0: no limit.  FXENV_TIME_LIMIT_WINDOW: the step that finds the episode window exhausted (at
 * FxConfig.episode_bars or at the end of the table) sets FX_FLAG_EXHAUSTED | FX_FLAG_TRUNCATED instead of
 * FX_FLAG_EXHAUSTED | FX_FLAG_TERMINATED.  Broke stays a termination.
 *   Precedence: a decision that terminates the episode (broke, or exhaustion without the WINDOW flag) reports a
 *     termination only, even if it also reaches the limit.  FX_FLAG_TRUNCATED and FX_FLAG_TERMINATED are never set
 *     together.
 *   After a truncation the env behaves exactly as after a termination: with auto_reset the next step is the reset
 *     step (the new episode, reward 0, code 0); without it every later step returns the same observation, reward 0 and
 *     FXENV_DONE_TRUNCATED.
 *   Outputs: while truncation is on (max_steps > 0 or the WINDOW flag), the uint8 terminated / done output of
 *     fxenv_step, fxenv_step_host, fxenv_step_many and FxRollout.done carries a code: 0, FXENV_DONE_TERMINATED or
 *     FXENV_DONE_TRUNCATED (non-zero still means "episode over").  While it is off they are 0 / 1 as without it.
 *   State: each env counts the decisions of its episode in the env state (snapshots carry the count; a reset zeroes
 *     it).  The limit and the flags belong to the handle, like the action repeat: fxenv_state_bytes, snapshots,
 *     fxenv_reset and fxenv_set_state neither include nor change them.
 * Synchronous.  Zeroes every env's decision count (an episode already running gets max_steps more decisions), drops the
 * cached step-many graphs and makes each policy re-capture its rollout graph.  max_steps < 0 or unknown flag bits:
 * FXENV_E_INVALID. */
#define FX_FLAG_TRUNCATED 64u          /* the episode was cut by the time limit / window (above); never with TERMINATED */
#define FXENV_TIME_LIMIT_WINDOW 1u     /* data exhaustion of the episode window is a truncation, not a termination */
#define FXENV_DONE_TERMINATED 1
#define FXENV_DONE_TRUNCATED 2
int fxenv_set_time_limit(FxEnv* env, int32_t max_steps, uint32_t flags);

/* ---- per-env broker and strategy parameters (no reference counterpart: one reference env has one configuration; a
 * handle of N envs can run N of them, e.g. a backtest grid over SL x TP x commission, or costs drawn per env for RL) ----
 * params_host: float64 [num_envs][FXENV_ENV_PARAMS] row-major, or NULL (off: every env uses the FxConfig values).
 * Row i replaces, for env i only, the FxConfig field of the same meaning everywhere the library uses it:
 *   FXENV_PARAM_COMMISSION / _LEVERAGE / _SLIPPAGE   commission, leverage, slippage_perc of the broker: executions,
 *       check_submitted's pseudo-executions and its cash bound, the mark to market, every slipped fill price, margin;
 *   FXENV_PARAM_SL_PIPS / _TP_PIPS                   sl_pips, tp_pips of direct_fixed_sltp;
 *   FXENV_PARAM_K_SL / _K_TP                         k_sl, k_tp of direct_atr_sltp.
 * Fields the strategy does not use are accepted and ignored.  Not replaced: strat_leverage (ATR rel-volume sizing),
 * position sizes, pip sizes, initial cash, every preprocessor and reward field.
 * Validation, per row, as fxenv_create checks the config: every field finite, leverage > 0, 0 <= slippage < 1.  A bad
 * row is FXENV_E_INVALID (fxenv_last_error names the env and the field) and leaves the table in force before the call.
 * The table belongs to the handle, like the time limit: fxenv_state_bytes, snapshots, fxenv_reset and fxenv_set_state
 * neither include nor change it.  Synchronous: the call waits for the device before it copies.
 *   A call that keeps the table on and the kernel choice (fxenv_debug_lean) the same updates the values in place: the
 *     cached step-many graphs and the policies' rollout graphs stay valid and read the new values.  Turning the table
 *     on or off, or a change of the LEAN choice, drops those graphs as the other setters do.
 *   LEAN (fxenv_debug_lean): decided on the table's values while it is on -- every row with commission 0, leverage 1 and
 *     slippage 0, and the rest of the configuration qualifying.
 *   New values apply from the next env-step on.  Orders already in the table keep their stop / limit prices; their
 *     later fills, the cash bound of orders submitted before the call included, use the new costs. */
#define FXENV_ENV_PARAMS 7
enum { FXENV_PARAM_COMMISSION = 0, FXENV_PARAM_LEVERAGE, FXENV_PARAM_SLIPPAGE,
       FXENV_PARAM_SL_PIPS, FXENV_PARAM_TP_PIPS, FXENV_PARAM_K_SL, FXENV_PARAM_K_TP };
int fxenv_set_env_params(FxEnv* env, const double* params_host);

/* ---- closed loop: a policy on the device between the steps ------------------------------------------------------
 * Replaces the caller loop of app/main.py:57-65 (`action = strategy.decide_action(obs, info, step); env.step(action)`)
 * for a learned actor-critic MLP(hidden, hidden) (default 256, BASELINE configs[3]: PPO MLP(256,256)): observation rows
 * never leave the GPU, and the policy is one fused tensor-core kernel per step (wgmma / TMA / clusters,
 * gym_fx_b200/csrc/fx_policy.cu), chained to the env step kernel by programmatic dependent launches.  The actor head
 * follows the env's FxConfig.action_mode:
 *
 *   h1 = tanh(obs W1^T + b1), h2 = tanh(h1 W2^T + b2), value = h2 wv + bv
 *   FX_ACTION_DISCRETE:   logits = h2 Wpi^T + bpi (3)
 *                         action = argmax(logits + Gumbel noise), logp = log_softmax(logits)[action]
 *   FX_ACTION_CONTINUOUS: mu = h2 wmu + bmu, learned state-independent log sigma
 *                         action = mu + sigma * eps, eps ~ N(0, 1), logp = -eps^2 / 2 - log sigma - log(2 pi) / 2
 *                         (not clipped: the env step thresholds the raw value, app/env.py:187-204)
 *   greedy (fxenv_rollout_ex, FXENV_ROLLOUT_GREEDY): action = argmax(logits) (first maximum) / mu, with the log-prob of
 *                         that action (continuous: -log sigma - log(2 pi) / 2); no noise is read or generated.
 * The two hidden layers run in bfloat16 with float32 accumulation (the env step writes a bfloat16 copy of each row for
 * this purpose); biases, heads, sampling and log-prob in float32. */
typedef struct FxPolicy FxPolicy;

/* DEVICE pointers to float32 parameters in torch.nn.Linear layout ([out][in] row-major); hidden = the policy's width
 * (fxenv_policy_create_ex).  A policy created with FXENV_POLICY_SEPARATE (separate actor and critic networks) takes
 * both trunks stacked, the actor's first: w1 [2][hidden][obs_dim], b1 [2][hidden], w2 [2][hidden][hidden],
 * b2 [2][hidden]; w_pi / b_pi are the actor's head and w_v / b_v the critic's, as below. */
typedef struct FxPolicyWeights {
  const float* w1;   /* [hidden][obs_dim] */
  const float* b1;   /* [hidden] */
  const float* w2;   /* [hidden][hidden] */
  const float* b2;   /* [hidden] */
  const float* w_pi; /* discrete: [3][hidden] (one row per action);  continuous: [1][hidden] (the mean) */
  const float* b_pi; /* discrete: [3];                               continuous: [2] = {b_mu, log sigma} */
  const float* w_v;  /* [hidden] */
  const float* b_v;  /* [1] */
} FxPolicyWeights;

/* Buffers of one rollout of `horizon` steps (all DEVICE, caller-owned).  Step t: the policy reads the observation of
 * slot t % obs_slots, writes actions/logp/value at [t], the env step writes reward/done at [t] and the next observation
 * into slot (t + 1) % obs_slots; value[horizon] is the value of the last observation (bootstrap).  obs_slots >= 2
 * (horizon + 1 keeps every observation for the learner). */
typedef struct FxRollout {
  int32_t horizon;
  int32_t obs_slots;
  float* obs;           /* [obs_slots][num_envs][obs_dim] */
  void* actions;        /* [horizon][num_envs]: int32 (discrete) or float32 (continuous) */
  float* logp;          /* [horizon][num_envs] */
  float* value;         /* [horizon + 1][num_envs] */
  float* reward;        /* [horizon][num_envs] */
  uint8_t* done;        /* [horizon][num_envs] */
  const float* gumbel;  /* sampling noise, or NULL: counter-based generator from `seed`.  Discrete: [horizon][num_envs][3]
                         * Gumbel(0,1); continuous: [horizon][num_envs] standard normal.  Unused by greedy rollouts. */
  uint64_t seed;
} FxRollout;

/* fxenv_rollout_ex flags */
#define FXENV_ROLLOUT_GREEDY 1u   /* evaluation: the most likely action (argmax of the logits / the mean), no sampling */

/* fxenv_policy_create_ex2 flags */
#define FXENV_POLICY_SEPARATE 1u  /* separate actor and critic networks of the same width instead of one shared body:
                                   * the actor MLP gives the logits / mean, the critic MLP the value (the default layout
                                   * of Stable-Baselines3's and CleanRL's PPO).  Each network runs as its own pair of
                                   * kernel CTAs per 128-env tile.  Its rollouts always hand tiles over in kernel order
                                   * (FXENV_TILE_SYNC does not apply). */

/* Discrete or continuous, as FxConfig.action_mode.  `hidden` is the width of both hidden layers: 64, 128, 256 or 512
 * (anything else: FXENV_E_INVALID).  A 512-wide policy runs one kernel CTA per SM instead of two.  flags:
 * FXENV_POLICY_* (unknown bits: FXENV_E_INVALID).  fxenv_policy_create(env, out) is fxenv_policy_create_ex(env, 256,
 * out), and fxenv_policy_create_ex(env, hidden, out) is fxenv_policy_create_ex2(env, hidden, 0, out). */
int fxenv_policy_create(FxEnv* env, FxPolicy** out);
int fxenv_policy_create_ex(FxEnv* env, int32_t hidden, FxPolicy** out);
int fxenv_policy_create_ex2(FxEnv* env, int32_t hidden, uint32_t flags, FxPolicy** out);
/* Policy population: `members` (>= 1) independent actor-critic networks of one width and layout (flags), each on its
 * own contiguous slice of the envs: member m acts for envs [m N / members, (m + 1) N / members), N = num_envs.  On its
 * slice a member gives bit for bit what a single policy with its weights gives there, from the same state and noise
 * (caller noise, the in-kernel generator and greedy mode alike).  members > 1 needs N to be a multiple of
 * 128 x members, so that no 128-env kernel tile mixes members; members < 1 or an N that does not divide:
 * FXENV_E_INVALID.  fxenv_policy_create_ex2(env, hidden, flags, out) is fxenv_policy_create_ex3(env, hidden, flags,
 * 1, out).  A rollout runs every member in the same kernels as one policy. */
int fxenv_policy_create_ex3(FxEnv* env, int32_t hidden, uint32_t flags, int32_t members, FxPolicy** out);
/* Converts / copies the parameters into the policy's own device buffers (stream-ordered; call after every optimiser
 * step).  fxenv_policy_set_weights(pol, w, s) is fxenv_policy_set_member_weights(pol, 0, w, s). */
int fxenv_policy_set_weights(FxPolicy* pol, const FxPolicyWeights* weights_dev, void* stream);
/* The same for one member of a population (FxPolicyWeights as for a single policy of the population's width and
 * layout); member outside [0, members): FXENV_E_INVALID.  A rollout needs weights for every member (FXENV_E_STATE
 * until then).  Updating one member leaves the others' parameters and the cached rollout graph as they are. */
int fxenv_policy_set_member_weights(FxPolicy* pol, int32_t member, const FxPolicyWeights* weights_dev, void* stream);
int fxenv_policy_destroy(FxPolicy* pol);
/* `horizon` closed-loop steps starting from the env's current state; everything is enqueued on `stream`
 * (2 * horizon + 2 kernels; the launch sequence is cached as a CUDA graph per buffer set and flags).
 * fxenv_rollout(...) is fxenv_rollout_ex(..., 0, ...); flags: FXENV_ROLLOUT_* (unknown bits are an error). */
int fxenv_rollout(FxEnv* env, FxPolicy* pol, const FxRollout* io, void* stream);
int fxenv_rollout_ex(FxEnv* env, FxPolicy* pol, const FxRollout* io, uint32_t flags, void* stream);
/* Inside a rollout the policy kernel and the env-step kernel hand 128-env tiles to each other through flags in device
 * memory instead of whole-kernel dependencies; a poll that is never answered gives up after ~0.3 s instead of hanging
 * the device.  Returns how many polls of the LAST rollout gave up (0 unless something is broken; then that rollout's
 * results are invalid), or <0.  Synchronises the device. */
int fxenv_policy_sync_timeouts(FxPolicy* pol);

/* Observation normalizer of the policy.  The policy reads the observation in bfloat16; with a normalizer on, every
 * element the env kernels write to that copy is
 *     bf16_rn(min(max((x - mean[m][p][j]) * rstd[m][p][j], -clip[m]), clip[m]))
 * each operation rounded in float32 (torch's clamp((x - mean) * rstd, -clip, clip) gives the same bits), x the float32
 * value of the row, m = env / (num_envs / members) the env's member and p = env % num_pairs its pair.  The float32
 * rows of FxRollout.obs, the env's outputs and state, and fxenv_step / fxenv_step_many do not change.
 * Member `member`'s normalizer: mean_dev / rstd_dev float32 [num_pairs][obs_dim] DEVICE, copied stream-ordered into the
 * policy; clip > 0 (+inf allowed); both NULL clears it.  A rollout needs every member on or every member off (mixed:
 * FXENV_E_STATE).  Turning it on or off drops the cached rollout graph; a value update keeps it (like
 * fxenv_policy_set_member_weights).  An invalid member, clip <= 0 or NaN, or only one of the two pointers NULL:
 * FXENV_E_INVALID, and the policy stays as it was. */
int fxenv_policy_set_obs_norm(FxPolicy* pol, int32_t member, const float* mean_dev, const float* rstd_dev, float clip,
                              void* stream);
/* The normalizer's statistics of rollout observations: obs_dev float32 [slots][num_envs][obs_dim] DEVICE (FxRollout.obs
 * layout), over every slot and the envs [env_begin, env_end) (a member's slice, or all), grouped by pair p = env %
 * num_pairs.  out_dev float64 [num_pairs][2][obs_dim] DEVICE receives S1 = sum (x - shift) and S2 = sum (x - shift)^2,
 * the difference formed in float64 from float32 shift_dev [num_pairs][obs_dim] (the running mean: shifted sums of
 * several ranks add up with one all-reduce SUM when every rank uses the same shift).  The summation order depends on
 * the shapes only: the same inputs give the same bits.  Stream-ordered.  slots < 1 or a range outside [0, num_envs)
 * or empty: FXENV_E_INVALID. */
int fxenv_obs_moments(FxEnv* env, const float* obs_dev, int32_t slots, int32_t env_begin, int32_t env_end,
                      const float* shift_dev, double* out_dev, void* stream);
/* The reward normalizer's statistics: moments of the discounted return of every env, carried across rollouts.
 * reward_dev float32 [horizon][num_envs], done_dev uint8 [horizon][num_envs] (FxRollout.reward / done: 0, or 1 / 2 =
 * terminated / truncated), prev_done_dev uint8 [num_envs] (the done of the step before the rollout), all DEVICE.  Over
 * the envs [env_begin, env_end) (a member's slice, or all); ret_dev float64 and seen_dev int32 DEVICE, env_end -
 * env_begin entries each, env i at [i - env_begin], read and written.  For each env, with begun = the episodes the env
 * has begun since fxenv_create (every reset, auto or explicit, counts; snapshots carry it):
 *   reset(t) = t == 0 ? prev_done[i] != 0 : done[t-1][i] != 0      (the learner's reset steps)
 *   R = begun - (number of t with reset(t)) == seen ? ret : 0       (any other reset since the last scan clears it)
 *   for t in 0 .. horizon-1:  if !reset(t): R = R * gamma + (double)reward[t][i] (two roundings), d = R - shift,
 *                             S1 += d, S2 += d * d, n += 1;  if done[t][i] != 0: R = 0  (termination and truncation)
 *   ret = R, seen = begun
 * out_dev float64 [3] DEVICE receives {S1, S2, n} summed over the slice (shifted sums of several ranks add up with one
 * all-reduce SUM when every rank uses the same shift).  Start with ret = 0 and seen = -1.  Rewards of steps that no call
 * scanned (fxenv_step_many, greedy rollouts) do not enter the return; an episode that ended or was reset in between still
 * clears it, through begun.  A fxenv_set_state that rewinds an env past one of its resets clears it the same way; one
 * that does not keeps the carried return.  The summation order depends only on (horizon, env_begin, env_end): the same
 * inputs give the same bits; no atomics.  Stream-ordered, no host synchronisation.  horizon < 1, a range outside
 * [0, num_envs) or empty, gamma outside [0, 1] or NaN, a non-finite shift or a NULL pointer: FXENV_E_INVALID, nothing
 * enqueued. */
int fxenv_return_moments(FxEnv* env, const float* reward_dev, const uint8_t* done_dev, const uint8_t* prev_done_dev,
                         int32_t horizon, int32_t env_begin, int32_t env_end, double gamma, double shift,
                         double* ret_dev, int32_t* seen_dev, double* out_dev, void* stream);

/* fxenv_policy_peek `what` */
#define FXENV_PEEK_OBS16 0   /* slot 0 | 1: the bf16 observation copy the policy reads, [num_envs][k_pad] (k_pad = obs_dim
                              * rounded up to a multiple of 64, zero pad columns); a rollout's step t reads slot t % 2.
                              * With a normalizer on (fxenv_policy_set_obs_norm) it is the normalized copy. */
#define FXENV_PEEK_H1 1      /* slot 0: the layer-1 activations of the last policy evaluation (after a rollout: the
                              * bootstrap one), bf16 [num_envs rounded up to a multiple of 128][hidden]; with
                              * FXENV_POLICY_SEPARATE [...][2 hidden]: the actor's columns, then the critic's */
/* Test / debugging aid: stream-ordered copy of an internal policy buffer into caller DEVICE memory `dst` of `bytes`
 * bytes.  dst == NULL: returns the byte size needed.  Returns the bytes copied, or <0.  Reads only. */
int64_t fxenv_policy_peek(FxPolicy* pol, int what, int slot, void* dst, int64_t bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FXENV_H_ */
