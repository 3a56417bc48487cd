// fx_capi.cu -- the C-ABI of libfxenv.so (include/fxenv.h): handle management, device memory, kernel launches.
// No torch types, no exceptions across the boundary; every entry point returns a status code.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <new>
#include <string>
#include <type_traits>
#include <vector>

#include "fx_kernels.cuh"
#include "fx_policy.cuh"

namespace {

thread_local std::string g_create_error;

}  // namespace

// Instantiated CUDA graphs of launch sequences (launch_cached), one per slot, each stored with the key it was captured
// for and the handle's params_epoch at the capture: the graphs capture the kernel parameters (FxEnv::P) by value, so a
// slot of an older epoch is captured again.
template <typename Key, int Slots>
struct GraphCache {
  static_assert(std::has_unique_object_representations_v<Key>, "keys are compared bytewise: no padding");
  struct Slot {
    cudaGraphExec_t exec = nullptr;
    Key key;
    uint64_t epoch = 0, used = 0;
  } slot[Slots];
  uint64_t clock = 0;  // `used` of the last launched slot: the least recently used slot is replaced
  ~GraphCache() { for (auto& s : slot) if (s.exec) cudaGraphExecDestroy(s.exec); }
};

struct StepManyKey {
  const void* actions;
  float *obs, *reward;
  uint8_t* term;
  int32_t steps, slots;
};

struct RolloutKey {
  FxRollout io;
  uint64_t flags;  // FXENV_ROLLOUT_*, 64 bits wide so that the key has no padding
};

struct FxEnv {
  FxKernelParams P;
  int device = 0;
  unsigned char* slab = nullptr;
  size_t slab_bytes = 0;
  double* candles_dev[FXENV_MAX_PAIRS] = {};
  double* stats_dev[FXENV_MAX_PAIRS] = {};
  int64_t* minutes_dev[FXENV_MAX_PAIRS] = {};
  bool loaded[FXENV_MAX_PAIRS] = {};
  bool tame[FXENV_MAX_PAIRS] = {};
  bool was_reset = false;
  bool first_reset = true;
  int timeline_steps = 0;
  int force_engine = -1;           // FXENV_ENGINE (timing experiments): 0 graph of single steps, 1 persistent launch
  bool seq_tracked = true;         // fx_rollout_kernel's seq[] / ticket words hold (seq_base, ticket_base): no memset needed
  unsigned seq_base = 0u, ticket_base = 0u;
  int64_t launches = 0;
  std::string err;
  // fxenv_step_host staging
  static constexpr int kHostSlices = 8;
  cudaStream_t hstream = nullptr, hcopy = nullptr;
  cudaEvent_t hev[kHostSlices] = {};
  void* h_actions = nullptr;
  float* h_obs = nullptr;
  float* h_reward = nullptr;
  uint8_t* h_term = nullptr;
  // fxenv_step_many, graph engine: the two most recent launch sequences, keyed by the pointer set and sizes
  GraphCache<StepManyKey, 2> step_graphs;
  // bumped by params_changing whenever a launch parameter in P changes: every cached graph captured the old P by value
  uint64_t params_epoch = 0;
  // the deferred kernel bits (FX_V_TRUNC, FX_V_PARAMS) ever turned on: the kernel halves they cover are configured
  unsigned deferred = 0u;
  // per-env parameters (fxenv_set_env_params): the host copy of the table while it is on (the LEAN choice is made on its
  // values).  The device table lives behind the sequence words in the allocation of P.seq, at params_off (0: not yet
  // allocated); P.env_params_off is params_off while the table is on and 0 while it is off.
  std::vector<double> params_host;
  uint32_t params_off = 0;
};

namespace {

int fail(FxEnv* env, int code, const std::string& msg) {
  if (env) env->err = msg; else g_create_error = msg;
  return code;
}

int cuda_fail(FxEnv* env, cudaError_t e, const char* what) {
  return fail(env, FXENV_E_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

#define FX_CUDA(env, call)                                   \
  do {                                                       \
    cudaError_t e__ = (call);                                \
    if (e__ != cudaSuccess) return cuda_fail(env, e__, #call); \
  } while (0)

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) cudaSetDevice(dev); else prev = -1;
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

int validate(const FxConfig& c, std::string& why) {
  char buf[256];
#define BAD(...) do { snprintf(buf, sizeof buf, __VA_ARGS__); why = buf; return FXENV_E_INVALID; } while (0)
  if (c.struct_size != (int32_t)sizeof(FxConfig)) BAD("FxConfig.struct_size %d != %d (ABI mismatch)", c.struct_size, (int)sizeof(FxConfig));
  if (c.num_envs < 1) BAD("num_envs must be >= 1");
  if (c.num_pairs < 1 || c.num_pairs > FXENV_MAX_PAIRS) BAD("num_pairs must be in 1..%d", FXENV_MAX_PAIRS);
  if (c.n_cols < 5 || c.n_cols > FXENV_MAX_COLS) BAD("n_cols must be in 5..%d", FXENV_MAX_COLS);
  if (c.order_capacity < 0 || c.order_capacity > 512) BAD("order_capacity must be in 0..512");
  if (c.window_size < 1) BAD("window_size must be >= 1");
  if (c.price_col < 0 || c.price_col >= c.n_cols) BAD("price_col out of range");
  if (!(c.slippage_perc >= 0.0 && c.slippage_perc < 1.0)) BAD("slippage_perc must be in [0, 1)");
  if (!(c.leverage > 0.0)) BAD("leverage must be > 0");
  if (c.strategy < 0 || c.strategy > FX_STRATEGY_ATR_SLTP) BAD("unknown strategy %d", c.strategy);
  if (c.strategy == FX_STRATEGY_ATR_SLTP && (c.atr_period < 1 || c.atr_period > 64)) BAD("atr_period must be in 1..64");
  if (c.strategy != FX_STRATEGY_DEFAULT && c.strat_position_size == 0.0 && !c.use_rel_volume) BAD("bracket strategies need position_size != 0");
  if (c.preproc < 0 || c.preproc > FX_PREPROC_FEATURE_WINDOW) BAD("unknown preprocessor %d", c.preproc);
  if (c.preproc == FX_PREPROC_FEATURE_WINDOW) {
    if (c.n_features < 1 || c.n_features > FXENV_MAX_FEATURES) BAD("n_features must be in 1..%d", FXENV_MAX_FEATURES);
    for (int i = 0; i < c.n_features; i++)
      if (c.feature_cols[i] < 0 || c.feature_cols[i] >= c.n_cols) BAD("feature_cols[%d] out of range", i);
    if (c.scaling < 0 || c.scaling > FX_SCALING_EXPANDING) BAD("unknown feature scaling %d", c.scaling);
    if (c.scaling == FX_SCALING_ROLLING && c.scaling_window < 1) BAD("feature_scaling_window must be >= 1");
  }
  if (c.reward < 0 || c.reward > FX_REWARD_DD) BAD("unknown reward %d", c.reward);
  if (c.reward == FX_REWARD_SHARPE && (c.sharpe_window < 1 || c.sharpe_window > 4096)) BAD("sharpe window must be in 1..4096");
  if (c.reward_initial_cash == 0.0) BAD("reward_initial_cash must be non-zero (the reference substitutes 1.0)");
  if (c.episode_bars < 0) BAD("episode_bars must be >= 0");
#undef BAD
  return FXENV_OK;
}

int require_ready(FxEnv* env, bool need_reset) {
  if (!env) return FXENV_E_INVALID;
  for (int p = 0; p < env->P.cfg.num_pairs; p++)
    if (!env->loaded[p]) return fail(env, FXENV_E_STATE, "candles for pair " + std::to_string(p) + " not loaded");
  if (need_reset && !env->was_reset) return fail(env, FXENV_E_STATE, "Call reset() before step().");
  return FXENV_OK;
}

// A launch parameter in env->P is about to change: wait until no launch may still run with the old one, and bump the
// epoch, so that every cached graph (step-many and rollout), which captured the old P, is captured again on its next use
int params_changing(FxEnv* env) {
  FX_CUDA(env, cudaDeviceSynchronize());
  env->params_epoch++;
  return FXENV_OK;
}

// Runs the launch sequence enqueue(stream) through `cache`: replays the graph captured for `key` at the current
// params_epoch, or first captures and instantiates one in the least recently used slot.  Inside someone else's capture
// (e.g. a torch CUDA graph), on the legacy stream, or with `direct`, the sequence is launched as it is.
template <typename Key, int Slots, typename Enqueue>
int launch_cached(FxEnv* env, GraphCache<Key, Slots>& cache, const Key& key, bool direct, cudaStream_t stream,
                  const Enqueue& enqueue, const char* what) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (stream != nullptr) cudaStreamIsCapturing(stream, &cs);
  if (direct || cs != cudaStreamCaptureStatusNone || stream == nullptr) {
    FX_CUDA(env, enqueue(stream));
    return FXENV_OK;
  }
  typename GraphCache<Key, Slots>::Slot* s = nullptr;
  for (auto& c : cache.slot)
    if (c.exec && c.epoch == env->params_epoch && memcmp(&c.key, &key, sizeof key) == 0) s = &c;
  if (!s) {
    s = &cache.slot[0];
    for (auto& c : cache.slot) if (c.used < s->used) s = &c;
    if (s->exec) { cudaGraphExecDestroy(s->exec); s->exec = nullptr; }
    cudaGraph_t graph = nullptr;
    FX_CUDA(env, cudaStreamBeginCapture(stream, cudaStreamCaptureModeThreadLocal));
    cudaError_t e = enqueue(stream);
    const cudaError_t e2 = cudaStreamEndCapture(stream, &graph);
    if (e != cudaSuccess) { if (graph) cudaGraphDestroy(graph); return cuda_fail(env, e, what); }
    if (e2 != cudaSuccess) return cuda_fail(env, e2, "cudaStreamEndCapture");
    e = cudaGraphInstantiate(&s->exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) { s->exec = nullptr; return cuda_fail(env, e, "cudaGraphInstantiate"); }
    s->key = key;
    s->epoch = env->params_epoch;
  }
  s->used = ++cache.clock;
  FX_CUDA(env, cudaGraphLaunch(s->exec, stream));
  return FXENV_OK;
}

// A setter turns the deferred kernel bit `bit` (FX_V_TRUNC or FX_V_PARAMS) on: configures every kernel half whose bits
// are now all on for the first time -- their attributes, and the persistent grid's minimum over them (every launch
// reads the grid and advances the ticket words by its own warp count)
int use_deferred(FxEnv* env, unsigned bit) {
  const unsigned on = env->deferred | bit;
  for (const unsigned half : std::initializer_list<unsigned>{FX_V_TRUNC, FX_V_PARAMS, FX_V_TRUNC | FX_V_PARAMS})
    if ((half & ~on) == 0u && (half & ~env->deferred) != 0u) FX_CUDA(env, fx_configure_half(env->P, half));
  env->deferred = on;
  return FXENV_OK;
}

// The per-env state slab, described once: every column in slab order with its element count, each column's bytes
// rounded up to 256.  Returns the slab's size; given the allocation (`base`) it also points the columns into it.  The
// order and the rounding are the layout of a snapshot blob (fxenv_get_state).
size_t slab_layout(FxKernelParams& P, unsigned char* base) {
  const size_t N = (size_t)P.cfg.num_envs, capP = (size_t)P.cap + FXO_SLACK;
  const size_t ring = (P.cfg.reward == FX_REWARD_SHARPE) ? (size_t)P.cfg.sharpe_window : 1;
  size_t off = 0;
  const auto col = [&](auto*& p, size_t n) {
    if (base) p = reinterpret_cast<std::remove_reference_t<decltype(p)>>(base + off);
    off += (n * sizeof(*p) + 255) & ~(size_t)255;
  };
  FxDeviceState& st = P.st;
  for (double** p : {&st.cash, &st.psize, &st.pprice, &st.equity, &st.prev_equity, &st.price, &st.commission_paid,
                     &st.dd_peak, &st.sub_need})
    col(*p, N);
  col(st.start, N);
  col(st.nbar, N * 6);
  col(st.rstats, N * FX_RS_N);
  for (int32_t** p : {&st.t, &st.total_bars, &st.position, &st.bar_index, &st.trades, &st.n_orders, &st.sh_len,
                      &st.sh_head, &st.sh_last_step, &st.dd_last_step, &st.n_acc})
    col(*p, N);
  col(st.flags, N);
  col(st.sh_ring, N * ring);
  col(st.welford, N * FXENV_MAX_FEATURES * 2);
  col(st.o_meta, N * capP);
  col(st.o_p0, N * capP);
  col(st.o_p1, N * capP);
  col(st.o_sz, N * capP);
  col(st.ep_lo, N);
  col(st.ep_span, N);
  col(st.ep_seed, 1);
  col(st.ep_begun, N);
  col(st.ep_done, N);
  col(st.ep_last, N * FXENV_EPISODE_STATS);
  col(P.ep_steps, N);
  return off;
}

// Whether the handle runs the LEAN kernels (fx_config_is_lean): decided once every candle table is loaded, on the costs
// of the per-env table `rows` ([N][FXENV_ENV_PARAMS] host copy) if one is on
int lean_choice(const FxEnv* env, const double* rows) {
  for (int p = 0; p < env->P.cfg.num_pairs; p++)
    if (!env->loaded[p]) return 0;
  if (getenv("FXENV_NO_LEAN")) return 0;
  return fx_config_is_lean(env->P, rows) ? 1 : 0;
}

// The check_submitted cash bound each env keeps for the orders its last strategy call submitted (FxDeviceState::sub_need)
// was computed with the costs of that call.  After the costs may have changed (a per-env table set, changed or turned
// off, or a snapshot restored on a handle that has had one), +inf makes the next env-step run the exact check instead.
int invalidate_cash_bounds(FxEnv* env) {
  const std::vector<double> inf((size_t)env->P.cfg.num_envs, INFINITY);
  FX_CUDA(env, cudaMemcpy(env->P.st.sub_need, inf.data(), inf.size() * sizeof(double), cudaMemcpyHostToDevice));
  return FXENV_OK;
}

}  // namespace

extern "C" {

int fxenv_abi_version(void) { return FXENV_ABI_VERSION; }

const char* fxenv_last_error(const FxEnv* env) { return env ? env->err.c_str() : g_create_error.c_str(); }

int fxenv_destroy(FxEnv* env);

int fxenv_create(const FxConfig* cfg, FxEnv** out) {
  if (!cfg || !out) return fail(nullptr, FXENV_E_INVALID, "null argument");
  *out = nullptr;
  std::string why;
  int rc = validate(*cfg, why);
  if (rc != FXENV_OK) return fail(nullptr, rc, why);
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0)
    return fail(nullptr, FXENV_E_CUDA, std::string("no CUDA device available (libfxenv has no CPU path): ") +
                                           (ce != cudaSuccess ? cudaGetErrorString(ce) : "device count is 0"));
  FxEnv* env = new (std::nothrow) FxEnv();
  if (!env) return fail(nullptr, FXENV_E_NOMEM, "out of host memory");
  memset(&env->P, 0, sizeof env->P);
  env->P.cfg = *cfg;
  FxConfig& c = env->P.cfg;
  if (cudaGetDevice(&env->device) != cudaSuccess) { delete env; return fail(nullptr, FXENV_E_CUDA, "cudaGetDevice failed"); }
  // FX_CUDA for what follows: frees what was allocated so far, and the message goes to fxenv_last_error(NULL)
#define FX_CREATE(call)                                                                  \
  do {                                                                                   \
    cudaError_t e__ = (call);                                                            \
    if (e__ != cudaSuccess) { fxenv_destroy(env); return cuda_fail(nullptr, e__, #call); } \
  } while (0)
  int cap = c.order_capacity == 0 ? 128 : c.order_capacity;
  cap = (cap + 31) & ~31;
  c.order_capacity = cap;
  env->P.cap = cap;
  env->P.obs_dim = (int32_t)fx_obs_dim(c);
  env->P.inv_initial_cash = 1.0 / (c.initial_cash != 0.0 ? c.initial_cash : 1.0);
  env->P.repeat = 1;  // no action repeat (fxenv_set_action_repeat)
  if (const char* dv = getenv("FXENV_DEBUG")) env->P.debug = atoi(dv);  // timing experiments only
  if (const char* tv = getenv("FXENV_TIMING")) {
    if (atoi(tv)) {
      FX_CREATE(cudaMalloc(&env->P.timing, (size_t)c.num_envs * 2 * FX_NSTAMP * sizeof(long long)));
      FX_CREATE(cudaMemset(env->P.timing, 0, (size_t)c.num_envs * 2 * FX_NSTAMP * sizeof(long long)));
    }
  }
  env->P.fast_features = 0;
  if (c.preproc == FX_PREPROC_FEATURE_WINDOW && c.n_features == 5 && c.n_cols == 5) {
    env->P.fast_features = 5;
    for (int i = 0; i < 5; i++) if (c.feature_cols[i] != i) env->P.fast_features = 0;
  }
  if (const char* tl = getenv("FXENV_TIMELINE")) {  // debug, timing build: per-ticket start / end stamps of fxenv_step_many
    if (atoi(tl) > 0) {
      env->timeline_steps = atoi(tl);
      const size_t nb = (size_t)env->timeline_steps * c.num_envs * 2 * sizeof(long long);
      FX_CREATE(cudaMalloc(&env->P.timeline, nb));
      FX_CREATE(cudaMemset(env->P.timeline, 0, nb));
    }
  }
  if (const char* fe = getenv("FXENV_ENGINE")) env->force_engine = (fe[0] == 'p') ? 1 : (fe[0] == 'g' ? 0 : -1);
  env->P.any_binary = 0;
  for (int i = 0; i < c.n_features; i++) if (c.feature_binary[i]) env->P.any_binary = 1;
  if (c.preproc != FX_PREPROC_FEATURE_WINDOW) env->P.any_binary = 0;
  env->P.lean = 0;  // decided in fxenv_load_candles (needs to know that the data are finite)
  ce = fx_configure_kernels(env->P);
  if (const char* rb = getenv("FXENV_ROLLOUT_BLOCKS"))  // timing experiments only: grid of the persistent launch
    if (atoi(rb) > 0 && atoi(rb) < env->P.resident_blocks) env->P.resident_blocks = atoi(rb);
  if (ce != cudaSuccess) { fxenv_destroy(env); return cuda_fail(nullptr, ce, "window_size * n_cols too large for shared memory"); }
  // one slab for the whole per-env state (snapshot == one memcpy)
  env->slab_bytes = slab_layout(env->P, nullptr);
  FX_CREATE(cudaMalloc(&env->slab, env->slab_bytes));
  FX_CREATE(cudaMemset(env->slab, 0, env->slab_bytes));
  slab_layout(env->P, env->slab);
  const size_t N = (size_t)c.num_envs;
  FX_CREATE(cudaMalloc(&env->P.seq, (N + 1) * sizeof(int32_t)));
  FX_CREATE(cudaMemset(env->P.seq, 0, (N + 1) * sizeof(int32_t)));
#undef FX_CREATE
  *out = env;
  return FXENV_OK;
}

int fxenv_destroy(FxEnv* env) {
  if (!env) return FXENV_OK;
  DeviceGuard g(env->device);
  for (int p = 0; p < FXENV_MAX_PAIRS; p++) {
    cudaFree(env->candles_dev[p]); cudaFree(env->stats_dev[p]); cudaFree(env->minutes_dev[p]);
  }
  cudaFree(env->slab);
  cudaFree(env->P.seq);
  cudaFree(env->P.timing);
  cudaFree(env->P.timeline);
  cudaFree(env->P.audit); cudaFree(env->P.audit_written);
  cudaFree(env->h_actions); cudaFree(env->h_obs); cudaFree(env->h_reward); cudaFree(env->h_term);
  if (env->hstream) cudaStreamDestroy(env->hstream);
  if (env->hcopy) cudaStreamDestroy(env->hcopy);
  for (auto& ev : env->hev) if (ev) cudaEventDestroy(ev);
  delete env;
  return FXENV_OK;
}

int fxenv_load_candles(FxEnv* env, int pair_id, const double* candles_host, int64_t T, const int64_t* minutes_host) {
  if (!env) return FXENV_E_INVALID;
  const FxConfig& c = env->P.cfg;
  if (pair_id < 0 || pair_id >= c.num_pairs) return fail(env, FXENV_E_INVALID, "pair_id out of range");
  if (!candles_host) return fail(env, FXENV_E_INVALID, "candles_host is null");
  // app/env.py:64-65: the data must be longer than the window
  if (T < (int64_t)c.window_size + 2) return fail(env, FXENV_E_INVALID, "input data is empty or too short for the configured window");
  DeviceGuard g(env->device);
  if (const int rc = params_changing(env)) return rc;  // the table's pointers, tame_data and the LEAN choice change
  cudaFree(env->candles_dev[pair_id]); cudaFree(env->stats_dev[pair_id]); cudaFree(env->minutes_dev[pair_id]);
  env->candles_dev[pair_id] = nullptr; env->stats_dev[pair_id] = nullptr; env->minutes_dev[pair_id] = nullptr;
  env->loaded[pair_id] = false;
  const size_t bytes = (size_t)T * c.n_cols * 8;
  FX_CUDA(env, cudaMalloc(&env->candles_dev[pair_id], bytes + 32));  // tail padding: TMA bulk copies are 16-B granular
  FX_CUDA(env, cudaMemset(reinterpret_cast<char*>(env->candles_dev[pair_id]) + bytes, 0, 32));
  FX_CUDA(env, cudaMemcpy(env->candles_dev[pair_id], candles_host, bytes, cudaMemcpyHostToDevice));
  if (minutes_host) {
    FX_CUDA(env, cudaMalloc(&env->minutes_dev[pair_id], (size_t)T * 8));
    FX_CUDA(env, cudaMemcpy(env->minutes_dev[pair_id], minutes_host, (size_t)T * 8, cudaMemcpyHostToDevice));
  }
  if (c.preproc == FX_PREPROC_FEATURE_WINDOW && c.scaling == FX_SCALING_ROLLING) {
    FX_CUDA(env, cudaMalloc(&env->stats_dev[pair_id], (size_t)T * c.n_features * 16));
    FX_CUDA(env, fx_launch_stats(c, env->candles_dev[pair_id], env->stats_dev[pair_id], T, 0));
    env->launches++;
    FX_CUDA(env, cudaDeviceSynchronize());
  }
  FxPairTable& tb = env->P.pair[pair_id];
  tb.candles = env->candles_dev[pair_id];
  tb.stats = env->stats_dev[pair_id];
  tb.minutes = env->minutes_dev[pair_id];
  tb.T = T;
  env->loaded[pair_id] = true;
  // finite and far from overflow => the observation code may skip its NaN fix-up (FxKernelParams::tame_data)
  bool tame = true;
  for (size_t i = 0, n = (size_t)T * c.n_cols; i < n && tame; i++) tame = fabs(candles_host[i]) < 1e100;  // false for NaN / inf
  env->tame[pair_id] = tame;
  env->P.tame_data = 1;
  for (int p = 0; p < c.num_pairs; p++) if (env->loaded[p] && !env->tame[p]) env->P.tame_data = 0;
  env->P.lean = lean_choice(env, env->P.env_params_off ? env->params_host.data() : nullptr);
  return FXENV_OK;
}

int64_t fxenv_obs_dim(const FxEnv* env) { return env ? env->P.obs_dim : -1; }

int fxenv_reset(FxEnv* env, const int64_t* start_bar_dev, const uint8_t* mask_dev, void* stream) {
  int rc = require_ready(env, false);
  if (rc) return rc;
  DeviceGuard g(env->device);
  FX_CUDA(env, fx_launch_reset(env->P, start_bar_dev, env->first_reset ? nullptr : mask_dev, env->first_reset ? 1 : 0,
                               (cudaStream_t)stream));
  env->launches++;
  env->first_reset = false;
  env->was_reset = true;
  return FXENV_OK;
}

int fxenv_observe(FxEnv* env, float* obs_dev, void* stream) {
  int rc = require_ready(env, true);
  if (rc) return rc;
  if (!obs_dev) return fail(env, FXENV_E_INVALID, "obs_dev is null");
  DeviceGuard g(env->device);
  FX_CUDA(env, fx_launch_observe(env->P, obs_dev, (cudaStream_t)stream));
  env->launches++;
  return FXENV_OK;
}

int fxenv_step(FxEnv* env, const void* actions_dev, float* obs_dev, float* reward_dev, uint8_t* terminated_dev,
               double* reward64_dev, void* stream) {
  int rc = require_ready(env, true);
  if (rc) return rc;
  if (!actions_dev || !obs_dev || !reward_dev || !terminated_dev) return fail(env, FXENV_E_INVALID, "null I/O pointer");
  DeviceGuard g(env->device);
  FX_CUDA(env, fx_launch_step(env->P, actions_dev, obs_dev, reward_dev, reward64_dev, terminated_dev, (cudaStream_t)stream));
  env->launches++;
  return FXENV_OK;
}

static bool batch_uses_rollout(const FxEnv* env, int n_steps) {
  // measured (one H100 SXM, 700 W, bench.py --steps 1000 --warmup 100, us/step persistent vs graph of single steps): cfg2
  // 4096 envs 9.1 vs 20.3; cfg3 (16384 envs, 7.2 KB rows) 64.7 vs 88.5; cfg5 (8192 envs, 14 KB rows) 91.3 vs 117.8 -- every
  // batch of more than one step uses it
  bool rollout = n_steps > 1;
  if (env->force_engine == 0) rollout = false;             // FXENV_ENGINE=graph / persistent: A/B of the engines
  if (env->force_engine == 1 && n_steps > 1) rollout = true;
  if (env->P.debug & (4 | 8)) rollout = false;             // FXENV_DEBUG: force the graph of single steps (A/B timing)
  if ((env->P.debug & 16) && n_steps > 1) rollout = true;  // FXENV_DEBUG & 16: force the persistent launch
  return rollout;
}

int fxenv_step_many_engine(const FxEnv* env, int n_steps) {
  if (!env) return FXENV_E_INVALID;
  return batch_uses_rollout(env, n_steps) ? 1 : 0;
}

int fxenv_step_many(FxEnv* env, int n_steps, const void* actions_dev, float* obs_dev, int obs_slots, float* reward_dev,
                    uint8_t* terminated_dev, void* stream_) {
  int rc = require_ready(env, true);
  if (rc) return rc;
  if (n_steps < 1 || obs_slots < 1) return fail(env, FXENV_E_INVALID, "n_steps and obs_slots must be >= 1");
  if (!actions_dev || !obs_dev || !reward_dev || !terminated_dev) return fail(env, FXENV_E_INVALID, "null I/O pointer");
  DeviceGuard g(env->device);
  cudaStream_t stream = (cudaStream_t)stream_;
  const size_t N = (size_t)env->P.cfg.num_envs, D = (size_t)env->P.obs_dim;
  auto enqueue = [&](cudaStream_t s) -> cudaError_t {
    for (int k = 0; k < n_steps; k++) {
      const char* a = reinterpret_cast<const char*>(actions_dev) + (size_t)k * N * 4;
      cudaError_t e = fx_launch_step(env->P, a, obs_dev + (size_t)(k % obs_slots) * N * D, reward_dev + (size_t)k * N,
                                     nullptr, terminated_dev + (size_t)k * N, s);
      if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
  };
  // Two ways to run a batch: (a) ONE persistent launch whose warps pull (step, env) tickets and honour per-env
  // dependencies (fx_rollout_kernel) -- the tail of a step (envs with many fills) overlaps the next step; (b) a CUDA graph
  // of K single-step launches -- wins for large observation rows once the device is saturated (see batch_uses_rollout).
  const bool rollout = batch_uses_rollout(env, n_steps);
  if (rollout) {
    if ((unsigned long long)N * (unsigned long long)n_steps >= (1ull << 31))
      return fail(env, FXENV_E_INVALID, "num_envs * n_steps must be < 2^31 per fxenv_step_many call");
    // the per-env sequence words and the ticket counter are epoch-based: the host knows what they hold after every
    // launch, so no memset is needed between batches.  Inside a stream capture (the launch may be replayed any number
    // of times) that knowledge is lost: such launches, and every launch after one, zero the words first.
    cudaStreamCaptureStatus rcs = cudaStreamCaptureStatusNone;
    if (stream != nullptr) cudaStreamIsCapturing(stream, &rcs);
    if (rcs != cudaStreamCaptureStatusNone) env->seq_tracked = false;
    const bool tracked = env->seq_tracked;
    if (env->P.timeline && n_steps > env->timeline_steps) return fail(env, FXENV_E_INVALID, "FXENV_TIMELINE smaller than n_steps");
    const FxChunkPlan plan = fx_rollout_plan(env->P, n_steps);
    FX_CUDA(env, fx_launch_rollout(env->P, actions_dev, obs_dev, obs_slots, reward_dev, terminated_dev, plan,
                                   tracked ? env->seq_base : 0u, tracked ? env->ticket_base : 0u, !tracked, stream));
    if (tracked) {
      env->seq_base += (unsigned)n_steps;
      env->ticket_base += (unsigned)(N * (size_t)plan.n_rounds) + (unsigned)fx_rollout_warps(env->P);
    }
    env->launches += 1;
    return FXENV_OK;
  }
  // a single step has nothing to amortise: a plain launch
  const StepManyKey key = {actions_dev, obs_dev, reward_dev, terminated_dev, n_steps, obs_slots};
  rc = launch_cached(env, env->step_graphs, key, n_steps == 1, stream, enqueue, "capture: fx_launch_step");
  if (rc) return rc;
  env->launches += n_steps;
  return FXENV_OK;
}

int fxenv_step_host(FxEnv* env, const void* actions_host, float* obs_host, float* reward_host, uint8_t* terminated_host) {
  int rc = require_ready(env, true);
  if (rc) return rc;
  if (!actions_host || !obs_host || !reward_host || !terminated_host) return fail(env, FXENV_E_INVALID, "null I/O pointer");
  DeviceGuard g(env->device);
  const size_t N = (size_t)env->P.cfg.num_envs, D = (size_t)env->P.obs_dim;
  if (!env->hstream) {
    FX_CUDA(env, cudaStreamCreateWithFlags(&env->hstream, cudaStreamNonBlocking));
    FX_CUDA(env, cudaStreamCreateWithFlags(&env->hcopy, cudaStreamNonBlocking));
    for (auto& ev : env->hev) FX_CUDA(env, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    FX_CUDA(env, cudaMalloc(&env->h_actions, N * 4));
    FX_CUDA(env, cudaMalloc(&env->h_obs, N * D * 4));
    FX_CUDA(env, cudaMalloc(&env->h_reward, N * 4));
    FX_CUDA(env, cudaMalloc(&env->h_term, N));
  }
  // The call is PCIe-bound (the observation rows: 3.6 KB per env).  The envs are stepped in up to 8 slices, slice i's
  // rows travelling to the host (copy engine, second stream) while slice i + 1 is being computed, so that only the
  // first slice's kernel time is exposed in front of the transfer.
  cudaStream_t s = env->hstream, sc = env->hcopy;
  int slices = (int)(N / 1024);
  if (slices > 2) slices = 2;  // measured (H100 SXM, cfg2, 4096 envs): 1 slice 12.3-12.7 M env-steps/s, 2: 12.8 M, 4: 12.8-12.9 M
  if (const char* hs = getenv("FXENV_HOST_SLICES")) slices = atoi(hs);  // timing experiments only
  if (slices < 1) slices = 1;
  if (slices > FxEnv::kHostSlices) slices = FxEnv::kHostSlices;
  const size_t per = ((N + slices - 1) / slices + 31) & ~(size_t)31;
  FX_CUDA(env, cudaMemcpyAsync(env->h_actions, actions_host, N * 4, cudaMemcpyHostToDevice, s));
  for (int i = 0; i < slices; i++) {
    const size_t e0 = (size_t)i * per, e1 = (e0 + per < N) ? e0 + per : N;
    if (e0 >= e1) break;
    FX_CUDA(env, fx_launch_step(env->P, env->h_actions, env->h_obs, env->h_reward, nullptr, env->h_term, s, (int)e0, (int)e1));
    env->launches++;
    FX_CUDA(env, cudaEventRecord(env->hev[i], s));
    FX_CUDA(env, cudaStreamWaitEvent(sc, env->hev[i], 0));
    FX_CUDA(env, cudaMemcpyAsync(obs_host + e0 * D, env->h_obs + e0 * D, (e1 - e0) * D * 4, cudaMemcpyDeviceToHost, sc));
  }
  FX_CUDA(env, cudaMemcpyAsync(reward_host, env->h_reward, N * 4, cudaMemcpyDeviceToHost, sc));
  FX_CUDA(env, cudaMemcpyAsync(terminated_host, env->h_term, N, cudaMemcpyDeviceToHost, sc));
  FX_CUDA(env, cudaStreamSynchronize(sc));  // sc's last copy waited for the last slice's kernel: s is idle too
  return FXENV_OK;
}

int fxenv_get_info(FxEnv* env, FxInfoPtrs* out) {
  if (!env || !out) return FXENV_E_INVALID;
  const FxDeviceState& st = env->P.st;
  out->equity = st.equity; out->prev_equity = st.prev_equity; out->price = st.price; out->cash = st.cash;
  out->position_size = st.psize; out->position_price = st.pprice; out->commission_paid = st.commission_paid;
  out->position = st.position; out->bar_index = st.bar_index; out->total_bars = st.total_bars;
  out->trades = st.trades; out->n_orders = st.n_orders; out->flags = st.flags;
  out->run_stats = st.rstats;
  return FXENV_OK;
}

// A snapshot = header + the raw state slab.  The header pins what the slab's layout depends on, so that a blob taken
// from a different configuration / order capacity / candle table length / library version is refused instead of being
// reinterpreted.
struct FxStateHeader {
  uint32_t magic, abi, config_bytes, order_capacity;
  uint64_t slab_bytes, config_hash;
  int64_t table_rows[FXENV_MAX_PAIRS];
};

static FxStateHeader state_header(const FxEnv* env) {
  FxStateHeader h;
  memset(&h, 0, sizeof h);
  h.magic = 0x32535846u;  // "FXS2"
  h.abi = FXENV_ABI_VERSION;
  h.config_bytes = (uint32_t)sizeof(FxConfig);
  h.order_capacity = (uint32_t)env->P.cap;
  h.slab_bytes = env->slab_bytes;
  uint64_t x = 1469598103934665603ull;  // FNV-1a over the resolved config
  const unsigned char* b = reinterpret_cast<const unsigned char*>(&env->P.cfg);
  for (size_t i = 0; i < sizeof(FxConfig); i++) { x ^= b[i]; x *= 1099511628211ull; }
  h.config_hash = x;
  for (int p = 0; p < FXENV_MAX_PAIRS; p++) h.table_rows[p] = env->P.pair[p].T;
  return h;
}

int64_t fxenv_state_bytes(const FxEnv* env) { return env ? (int64_t)(sizeof(FxStateHeader) + env->slab_bytes) : -1; }

int fxenv_get_state(FxEnv* env, void* buf_host, int64_t nbytes) {
  if (!env || !buf_host) return FXENV_E_INVALID;
  if (nbytes != fxenv_state_bytes(env)) return fail(env, FXENV_E_INVALID, "state buffer size mismatch");
  DeviceGuard g(env->device);
  FX_CUDA(env, cudaDeviceSynchronize());
  const FxStateHeader h = state_header(env);
  memcpy(buf_host, &h, sizeof h);
  FX_CUDA(env, cudaMemcpy(static_cast<char*>(buf_host) + sizeof h, env->slab, env->slab_bytes, cudaMemcpyDeviceToHost));
  return FXENV_OK;
}

int fxenv_set_state(FxEnv* env, const void* buf_host, int64_t nbytes) {
  if (!env || !buf_host) return FXENV_E_INVALID;
  if (nbytes != fxenv_state_bytes(env)) return fail(env, FXENV_E_INVALID, "state buffer size mismatch");
  FxStateHeader got;
  memcpy(&got, buf_host, sizeof got);
  const FxStateHeader want = state_header(env);
  if (got.magic != want.magic || got.abi != want.abi) return fail(env, FXENV_E_INVALID, "not a state blob of this library version");
  if (memcmp(&got, &want, sizeof got) != 0)
    return fail(env, FXENV_E_INVALID, "state blob was taken from a different configuration (config / order capacity / candle tables differ)");
  DeviceGuard g(env->device);
  FX_CUDA(env, cudaDeviceSynchronize());
  FX_CUDA(env, cudaMemcpy(env->slab, static_cast<const char*>(buf_host) + sizeof got, env->slab_bytes, cudaMemcpyHostToDevice));
  if (env->deferred & FX_V_PARAMS) {  // the handle has had a table: the blob's cash bounds may stem from other costs
    if (const int rc = invalidate_cash_bounds(env)) return rc;
  }
  env->was_reset = true;
  env->first_reset = false;
  return FXENV_OK;
}

int64_t fxenv_launch_count(const FxEnv* env) { return env ? env->launches : -1; }

int fxenv_set_reset_starts(FxEnv* env, const int64_t* lo_host, const int64_t* hi_host, uint64_t seed) {
  if (!env) return FXENV_E_INVALID;
  if ((lo_host == nullptr) != (hi_host == nullptr)) return fail(env, FXENV_E_INVALID, "lo_host and hi_host must both be given or both be NULL");
  int rc = require_ready(env, false);
  if (rc) return rc;
  const FxConfig& c = env->P.cfg;
  const size_t N = (size_t)c.num_envs;
  std::vector<int64_t> lo(N, 0);
  std::vector<uint64_t> span(N, 0);
  if (lo_host) {
    for (size_t i = 0; i < N; i++) {
      const int64_t T = env->P.pair[i % c.num_pairs].T;
      if (!(0 <= lo_host[i] && lo_host[i] <= hi_host[i] && hi_host[i] <= T - 1)) {
        char buf[160];
        snprintf(buf, sizeof buf, "start range of env %zu is [%lld, %lld]; it must satisfy 0 <= lo <= hi <= %lld", i,
                 (long long)lo_host[i], (long long)hi_host[i], (long long)(T - 1));
        return fail(env, FXENV_E_INVALID, buf);
      }
      lo[i] = lo_host[i];
      span[i] = (uint64_t)(hi_host[i] - lo_host[i]) + 1u;
    }
  } else {
    seed = 0;  // cleared: the state is what it was before any range was set
  }
  DeviceGuard g(env->device);
  FX_CUDA(env, cudaDeviceSynchronize());
  const FxDeviceState& st = env->P.st;
  FX_CUDA(env, cudaMemcpy(st.ep_lo, lo.data(), N * 8, cudaMemcpyHostToDevice));
  FX_CUDA(env, cudaMemcpy(st.ep_span, span.data(), N * 8, cudaMemcpyHostToDevice));
  FX_CUDA(env, cudaMemcpy(st.ep_seed, &seed, 8, cudaMemcpyHostToDevice));
  return FXENV_OK;
}

int fxenv_get_episode_info(FxEnv* env, FxEpisodePtrs* out) {
  if (!env || !out) return FXENV_E_INVALID;
  const FxDeviceState& st = env->P.st;
  out->start = st.start; out->episodes_done = st.ep_done; out->last_episode = st.ep_last;
  return FXENV_OK;
}

int fxenv_set_bracket_audit(FxEnv* env, int32_t capacity) {
  if (!env) return FXENV_E_INVALID;
  if (capacity < 0) return fail(env, FXENV_E_INVALID, "bracket audit capacity must be >= 0");
  const uint64_t N = (uint64_t)env->P.cfg.num_envs;
  const uint64_t records = N * (uint64_t)capacity;
  if (capacity > 0 && records > (uint64_t)INT64_MAX / (FXENV_AU_FIELDS * sizeof(double)))
    return fail(env, FXENV_E_INVALID, "bracket audit capacity too large");
  DeviceGuard g(env->device);
  if (const int rc = params_changing(env)) return rc;  // also: kernels in flight may still write the old ring
  cudaFree(env->P.audit); cudaFree(env->P.audit_written);
  env->P.audit = nullptr; env->P.audit_written = nullptr; env->P.audit_cap = 0;
  if (capacity == 0) return FXENV_OK;
  double* ring = nullptr;
  int64_t* written = nullptr;
  cudaError_t e = cudaMalloc(&ring, records * FXENV_AU_FIELDS * sizeof(double));
  if (e == cudaSuccess) e = cudaMalloc(&written, N * sizeof(int64_t));
  if (e == cudaSuccess) e = cudaMemset(ring, 0, records * FXENV_AU_FIELDS * sizeof(double));
  if (e == cudaSuccess) e = cudaMemset(written, 0, N * sizeof(int64_t));
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) { cudaFree(ring); cudaFree(written); return cuda_fail(env, e, "bracket audit ring"); }
  env->P.audit = ring; env->P.audit_written = written; env->P.audit_cap = capacity;
  return FXENV_OK;
}

int fxenv_get_bracket_audit(FxEnv* env, FxAuditPtrs* out) {
  if (!env || !out) return FXENV_E_INVALID;
  out->records = env->P.audit; out->written = env->P.audit_written; out->capacity = env->P.audit_cap;
  return FXENV_OK;
}

int fxenv_set_action_repeat(FxEnv* env, int32_t repeat, uint32_t flags) {
  if (!env) return FXENV_E_INVALID;
  if (repeat < 1 || repeat > FXENV_MAX_REPEAT)
    return fail(env, FXENV_E_INVALID, "action repeat must be in 1.." + std::to_string(FXENV_MAX_REPEAT) + ", got " + std::to_string(repeat));
  if (flags & ~FXENV_REPEAT_HOLD) return fail(env, FXENV_E_INVALID, "unknown action repeat flags " + std::to_string(flags));
  if (repeat == env->P.repeat && flags == env->P.repeat_flags) return FXENV_OK;
  DeviceGuard g(env->device);
  if (const int rc = params_changing(env)) return rc;
  env->P.repeat = repeat;
  env->P.repeat_flags = flags;
  return FXENV_OK;
}

int fxenv_set_time_limit(FxEnv* env, int32_t max_steps, uint32_t flags) {
  if (!env) return FXENV_E_INVALID;
  if (max_steps < 0) return fail(env, FXENV_E_INVALID, "time limit must be >= 0 decisions, got " + std::to_string(max_steps));
  if (flags & ~FXENV_TIME_LIMIT_WINDOW) return fail(env, FXENV_E_INVALID, "unknown time limit flags " + std::to_string(flags));
  DeviceGuard g(env->device);
  if (const int rc = params_changing(env)) return rc;  // also: no count is zeroed while a launch may run
  if (max_steps > 0 || flags != 0u) {
    if (const int rc = use_deferred(env, FX_V_TRUNC)) return rc;
  }
  env->P.max_steps = max_steps;
  env->P.trunc_flags = flags;
  // every running episode starts counting from here
  FX_CUDA(env, cudaMemset(env->P.ep_steps, 0, (size_t)env->P.cfg.num_envs * sizeof(int32_t)));
  FX_CUDA(env, cudaDeviceSynchronize());
  return FXENV_OK;
}

int fxenv_set_env_params(FxEnv* env, const double* params_host) {
  if (!env) return FXENV_E_INVALID;
  const size_t N = (size_t)env->P.cfg.num_envs;
  if (params_host) {  // every row first: a bad one leaves the table in force as it was
    static const char* const names[FXENV_ENV_PARAMS] = {"commission", "leverage", "slippage", "sl_pips", "tp_pips", "k_sl", "k_tp"};
    for (size_t i = 0; i < N; i++) {
      const double* r = params_host + i * FXENV_ENV_PARAMS;
      char buf[160];
      for (int j = 0; j < FXENV_ENV_PARAMS; j++)
        if (!isfinite(r[j])) {
          snprintf(buf, sizeof buf, "env params: env %zu: %s is %g; every field must be finite", i, names[j], r[j]);
          return fail(env, FXENV_E_INVALID, buf);
        }
      if (!(r[FXENV_PARAM_LEVERAGE] > 0.0)) {
        snprintf(buf, sizeof buf, "env params: env %zu: leverage is %g; it must be > 0", i, r[FXENV_PARAM_LEVERAGE]);
        return fail(env, FXENV_E_INVALID, buf);
      }
      if (!(r[FXENV_PARAM_SLIPPAGE] >= 0.0 && r[FXENV_PARAM_SLIPPAGE] < 1.0)) {
        snprintf(buf, sizeof buf, "env params: env %zu: slippage is %g; it must be in [0, 1)", i, r[FXENV_PARAM_SLIPPAGE]);
        return fail(env, FXENV_E_INVALID, buf);
      }
    }
  }
  DeviceGuard g(env->device);
  const bool was_on = env->P.env_params_off != 0u;
  // the kernel choice under the new table: a change of it (or of on / off) changes P
  const int lean = lean_choice(env, params_host);
  if (was_on != (params_host != nullptr) || lean != env->P.lean) {
    if (const int rc = params_changing(env)) return rc;
  } else {
    FX_CUDA(env, cudaDeviceSynchronize());  // no launch may still read the old values
  }
  if (params_host) {
    if (const int rc = use_deferred(env, FX_V_PARAMS)) return rc;
    if (!env->params_off) {
      // the first table: the allocation of the sequence words grows by the table (fx_env_params); the words move along
      // (no launch is running: params_changing synchronised)
      const size_t words = (N + 1) * sizeof(int32_t), off = (words + 255) & ~(size_t)255;
      int32_t* seq = nullptr;
      FX_CUDA(env, cudaMalloc(&seq, off + N * FXENV_ENV_PARAMS * sizeof(double)));
      const cudaError_t e = cudaMemcpy(seq, env->P.seq, words, cudaMemcpyDeviceToDevice);
      if (e != cudaSuccess) { cudaFree(seq); return cuda_fail(env, e, "cudaMemcpy(seq)"); }
      cudaFree(env->P.seq);
      env->P.seq = seq;
      env->params_off = (uint32_t)off;
    }
    env->P.env_params_off = env->params_off;
    FX_CUDA(env, cudaMemcpy(const_cast<double*>(fx_env_params(env->P)), params_host, N * FXENV_ENV_PARAMS * sizeof(double),
                            cudaMemcpyHostToDevice));
    env->params_host.assign(params_host, params_host + N * FXENV_ENV_PARAMS);
  } else {
    env->P.env_params_off = 0u;
    env->params_host.clear();
  }
  env->P.lean = lean;
  return invalidate_cash_bounds(env);
}

/* debug (FXENV_TIMELINE=K, timing build): copies the [K][num_envs][2] ticket start / end stamps; returns K or <0 */
int fxenv_debug_timeline(FxEnv* env, long long* out_host) {
  if (!env || !out_host || !env->P.timeline) return FXENV_E_STATE;
  DeviceGuard g(env->device);
  cudaDeviceSynchronize();
  if (cudaMemcpy(out_host, env->P.timeline, (size_t)env->timeline_steps * env->P.cfg.num_envs * 2 * sizeof(long long),
                 cudaMemcpyDeviceToHost) != cudaSuccess) return FXENV_E_CUDA;
  return env->timeline_steps;
}

/* debug / tests (pure host arithmetic, no CUDA call): how fxenv_step_many would cut n_steps into ticket rounds for
 * num_envs envs on a device holding resident_warps warps of the rollout kernel.  starts[0..rounds] receives the first
 * step of every round (starts[rounds] = n_steps); returns the number of rounds, or <0 if `cap` entries are not enough. */
int fxenv_debug_rollout_plan(int num_envs, int resident_warps, int n_steps, int* starts, int cap) {
  if (num_envs < 1 || resident_warps < 1 || n_steps < 1 || !starts) return FXENV_E_INVALID;
  FxKernelParams P = {};
  P.cfg.num_envs = num_envs;
  P.resident_blocks = (resident_warps + FX_WARPS - 1) / FX_WARPS;
  const FxChunkPlan pl = fx_rollout_plan(P, n_steps);
  if (pl.n_rounds + 1 > cap) return FXENV_E_INVALID;
  int r = 0;
  for (; r < pl.n_uniform; r++) starts[r] = r * pl.chunk;
  for (int t = 0; r <= pl.n_rounds; r++, t++) starts[r] = pl.tail_start[t];
  return pl.n_rounds;
}

/* debug / tests (pure host arithmetic, no CUDA call): whether fxenv_step_many keeps each ticket's order table in shared
 * memory for a configuration of this window / column count / Sharpe ring (0 unless sharpe_reward) / order capacity;
 * force = FXENV_ORDER_SMEM (0 or 1) or -1.  Returns 1 (resident) or 0 (global). */
int fxenv_debug_order_smem(int window_size, int n_cols, int ring_len, int order_capacity, int force) {
  if (window_size < 1 || n_cols < 1 || ring_len < 0 || order_capacity < 1) return FXENV_E_INVALID;
  FxKernelParams P = {};
  P.cfg.window_size = window_size;
  P.cfg.n_cols = n_cols;
  P.cfg.reward = ring_len > 0 ? FX_REWARD_SHARPE : FX_REWARD_PNL;
  P.cfg.sharpe_window = ring_len;
  P.cap = (order_capacity + 31) & ~31;
  return fx_order_smem_choice(P, force);
}

/* debug / tests: 1 if the env runs the specialised (LEAN) kernels (fx_config_is_lean, decided once every candle table is
 * loaded; FXENV_NO_LEAN turns them off), 0 if the general ones, <0 on error. */
int fxenv_debug_lean(const FxEnv* env) { return env ? env->P.lean : FXENV_E_INVALID; }

/* debug / tests: the variant key (FX_V_* bits, fx_kernels.cuh) of the kernels the handle's next step, step-many or rollout
 * launch runs (the step kernels ignore FX_V_RESIDENT), <0 on error. */
int fxenv_debug_variant_key(const FxEnv* env) { return env ? (int)fx_debug_variant_key(env->P) : FXENV_E_INVALID; }

/* debug / tests (no CUDA call): 1 if the library has a step, a step-norm and a rollout kernel for this strategy, reward
 * and variant key, 0 if it has none, <0 for a strategy, reward or key out of range. */
int fxenv_debug_variant_exists(int strategy, int reward, uint32_t key) {
  if (strategy < 0 || strategy >= FX_N_STRATEGIES || reward < 0 || reward >= FX_N_REWARDS || key >= FX_V_KEYS)
    return FXENV_E_INVALID;
  return fx_debug_variant_exists(strategy, reward, key) ? 1 : 0;
}

/* debug (FXENV_TIMING=1): copies the [num_envs][FX_NSTAMP] phase stamps of the last step; returns FX_NSTAMP or <0 */
int fxenv_debug_timings(FxEnv* env, long long* out_host) {
  if (!env || !out_host || !env->P.timing) return FXENV_E_STATE;
  DeviceGuard g(env->device);
  cudaDeviceSynchronize();
  if (cudaMemcpy(out_host, env->P.timing, (size_t)env->P.cfg.num_envs * 2 * FX_NSTAMP * sizeof(long long), cudaMemcpyDeviceToHost) != cudaSuccess)
    return FXENV_E_CUDA;
  return FX_NSTAMP;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------- closed loop (policy)
struct FxPolicy {
  FxEnv* env = nullptr;
  int k_pad = 0;                       // obs_dim padded to a multiple of 64 (bf16 row stride of the observation copy)
  int hidden = FX_POLICY_HIDDEN;       // width of both hidden layers: 64, 128, 256 or 512 (fxenv_policy_create_ex)
  bool separate = false;               // FXENV_POLICY_SEPARATE: actor and critic trunks, stacked (nets = 2) below
  int nets = 1;                        // trunks: 1 (shared body) or 2 (actor, critic)
  int members = 1;                     // population members (fxenv_policy_create_ex3), each num_envs / members envs
  uint16_t* w1 = nullptr;              // bf16 [members][nets][hidden][k_pad]
  uint16_t* w2 = nullptr;              // bf16 [members][nets][hidden][hidden]
  float* fparams = nullptr;            // b1[members][nets][hidden] | b2[members][nets][hidden] | head_w[members][4][hidden] | head_b[members][4]
  uint16_t* obs16[2] = {nullptr, nullptr};  // bf16 [num_envs][k_pad], double buffered
  uint16_t* h1 = nullptr;              // bf16 [num_envs padded to whole tiles][nets * hidden]: where the halves meet
  float* head_part = nullptr;          // float4 [num_envs padded][nets]: partial head sums of the second CTA of a pair
  int32_t* sync = nullptr;             // act_flag[tiles] | done_cnt[tiles] | timeouts[1] (FxTileSync), zeroed per rollout
  int tiles = 0;
  int32_t* scratch_act = nullptr;      // bootstrap evaluation: action / logp are discarded
  float* scratch_logp = nullptr;
  static constexpr int kGroups = 4;     // env groups of a rollout (see enqueue_rollout)
  cudaStream_t side[kGroups - 1] = {};
  cudaEvent_t ev_fork = nullptr, ev_join[kGroups - 1] = {};
  CUtensorMap map_obs[2], map_w1, map_w2, map_h1;
  FxPolicyDev dev;
  std::vector<bool> has_weights;       // [members]: set by fxenv_policy_set_member_weights
  int missing_weights = 0;             // members without weights: a rollout needs 0
  bool continuous = false;             // FX_ACTION_CONTINUOUS: Gaussian head, float32 actions (fx_policy_kernel<true>)
  // observation normalizer (fxenv_policy_set_obs_norm), allocated by its first use: mean [members][num_pairs][k_pad] |
  // rstd [same] | clip [members], the pad columns zero
  float* norm = nullptr;
  std::vector<bool> norm_on;           // [members]
  int norm_members = 0;                // members with a normalizer: a rollout needs 0 or all
  GraphCache<RolloutKey, 1> graph;     // fxenv_rollout_ex: the last launch sequence, keyed by the FxRollout and the flags
};

namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 2-D bf16 [rows][cols] row-major tensor, box = 64 columns (128 bytes) x box_rows rows, 128-byte swizzle, OOB -> 0
int make_map(FxEnv* env, CUtensorMap* map, void* base, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  static EncodeTiledFn encode = nullptr;
  if (!encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn)
      return fail(env, FXENV_E_CUDA, "cuTensorMapEncodeTiled is not available in this driver");
    encode = reinterpret_cast<EncodeTiledFn>(fn);
  }
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t strides[1] = {cols * 2};
  const cuuint32_t box[2] = {64, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(env, FXENV_E_CUDA, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
  return FXENV_OK;
}

// The envs are independent, so a rollout is run as up to 4 env GROUPS, each its own chain
//   policy(group, t) -> step(group, t) -> policy(group, t + 1) -> ...
// on its own stream (forked from / joined into the caller's stream; inside a capture this becomes parallel branches of
// the graph).  While one group's 128-row policy tiles occupy a few SMs, the other groups' env steps use the rest of the
// device, and a group of ~2048 envs steps in a single wave instead of the two of a 4096-env launch.  More, smaller groups
// do not pay: every group adds two kernel nodes per step to the graph, and a group's policy tiles need SMs of their own.
cudaError_t enqueue_rollout(FxEnv* env, FxPolicy* pol, const FxRollout& io, uint32_t flags, cudaStream_t s) {
  const size_t N = (size_t)env->P.cfg.num_envs, D = (size_t)env->P.obs_dim;
  const int H = io.horizon, slots = io.obs_slots;
  const bool greedy = (flags & FXENV_ROLLOUT_GREEDY) != 0;
  const size_t noise_per_env = pol->continuous ? 1 : 3;  // N(0,1) draws / Gumbel(0,1) draws per env and step
  // int32 or float32 actions: 4 bytes either way
  uint32_t* const actions = static_cast<uint32_t*>(io.actions);
  static const int skip = [] { const char* v = getenv("FXENV_ROLLOUT_SKIP"); return v ? atoi(v) : 0; }();  // timing experiments:
                                                                          // 1 = no env steps, 2 = no policy evaluations
  // FXENV_TILE_SYNC=1: per-tile hand-over between the two kernels (FxTileSync) instead of whole-kernel dependencies.
  // Off by default: bit-identical results, but the kernel boundary it removes is paid back by the polling warps.
  // A separate actor and critic always runs in kernel order: the actor pair's flag does not cover the critic pair.
  const char* tsv = getenv("FXENV_TILE_SYNC");
  const bool tile_sync = !skip && !pol->separate && tsv && atoi(tsv) != 0;
  cudaError_t e = cudaMemsetAsync(pol->sync, 0, (2 * (size_t)pol->tiles + 1) * sizeof(int32_t), s);
  if (e != cudaSuccess) return e;
  // with a normalizer on, the bf16 copies are the normalized ones (fx_observe_norm_kernel, fx_step_norm_kernel)
  const size_t MPK = (size_t)pol->members * (size_t)env->P.cfg.num_pairs * (size_t)pol->k_pad;
  const FxObsNorm norm = {pol->norm, pol->norm + MPK, pol->norm + 2 * MPK, (int32_t)(N / (size_t)pol->members),
                          env->P.cfg.num_pairs};
  const FxObsNorm* nm = pol->norm_members > 0 ? &norm : nullptr;
  e = fx_launch_observe(env->P, io.obs, s, pol->obs16[0], pol->k_pad, nm);  // the current observation, both copies
  if (e != cudaSuccess) return e;
  int groups = (int)(N / 2048);  // measured (H100 SXM, 4096 envs, cfg4 shape), us/step: 46.6 with 1 group, 44.8 with 2, 46.4 with 4
  if (groups > FxPolicy::kGroups) groups = FxPolicy::kGroups;
  if (const char* ge = getenv("FXENV_ROLLOUT_GROUPS")) { const int g = atoi(ge); if (g >= 1 && g <= FxPolicy::kGroups) groups = g; }  // measurements
  if (groups < 1 || (env->P.debug & 64)) groups = 1;
  const size_t per = ((N + groups - 1) / groups + FX_POLICY_TILE_M - 1) / FX_POLICY_TILE_M * FX_POLICY_TILE_M;
  if (groups > 1) {
    e = cudaEventRecord(pol->ev_fork, s);
    if (e != cudaSuccess) return e;
  }
  for (int g = 0; g < groups; g++) {
    const size_t e0 = (size_t)g * per, e1 = (e0 + per < N) ? e0 + per : N;
    if (e0 >= e1) break;
    cudaStream_t sg = (g == 0) ? s : pol->side[g - 1];
    if (g > 0) {
      e = cudaStreamWaitEvent(sg, pol->ev_fork, 0);
      if (e != cudaSuccess) return e;
    }
    for (int t = 0; t <= H; t++) {
      const bool last = (t == H);  // the bootstrap evaluation: value only
      if (!(skip & 2))
      e = fx_launch_policy(pol->map_obs[t & 1], pol->map_w1, pol->map_w2, pol->map_h1, pol->dev, pol->hidden, (int)N, pol->k_pad,
                           (!last && io.gumbel) ? io.gumbel + (size_t)t * N * noise_per_env : nullptr, io.seed, (unsigned)t,
                           last ? static_cast<void*>(pol->scratch_act) : actions + (size_t)t * N,
                           last ? pol->scratch_logp : io.logp + (size_t)t * N, io.value + (size_t)t * N, sg, (int)e0, (int)e1,
                           tile_sync, pol->continuous, greedy, pol->separate, pol->tiles / pol->members);
      if (e != cudaSuccess) return e;
      if (last) break;
      const FxTileSync ts = {pol->dev.act_flag, pol->sync + pol->tiles, pol->dev.timeouts, t + 1};
      if (!(skip & 1))
      e = fx_launch_step(env->P, actions + (size_t)t * N, io.obs + (size_t)((t + 1) % slots) * N * D, io.reward + (size_t)t * N,
                         nullptr, io.done + (size_t)t * N, sg, (int)e0, (int)e1, pol->obs16[(t + 1) & 1], pol->k_pad,
                         tile_sync ? &ts : nullptr, nm);
      if (e != cudaSuccess) return e;
    }
    if (g > 0) {
      e = cudaEventRecord(pol->ev_join[g - 1], sg);
      if (e != cudaSuccess) return e;
      e = cudaStreamWaitEvent(s, pol->ev_join[g - 1], 0);
      if (e != cudaSuccess) return e;
    }
  }
  return cudaSuccess;
}

}  // namespace

extern "C" {

int fxenv_policy_destroy(FxPolicy* pol) {
  if (!pol) return FXENV_OK;
  DeviceGuard g(pol->env->device);
  cudaFree(pol->w1); cudaFree(pol->w2); cudaFree(pol->fparams); cudaFree(pol->obs16[0]); cudaFree(pol->obs16[1]);
  cudaFree(pol->h1); cudaFree(pol->head_part); cudaFree(pol->sync);
  cudaFree(pol->scratch_act); cudaFree(pol->scratch_logp); cudaFree(pol->norm);
  for (auto& st : pol->side) if (st) cudaStreamDestroy(st);
  if (pol->ev_fork) cudaEventDestroy(pol->ev_fork);
  for (auto& ev : pol->ev_join) if (ev) cudaEventDestroy(ev);
  delete pol;
  return FXENV_OK;
}

/* polls of the last fxenv_rollout's per-tile hand-over that gave up (0 unless something is broken); synchronises */
int fxenv_policy_sync_timeouts(FxPolicy* pol) {
  if (!pol) return FXENV_E_INVALID;
  DeviceGuard g(pol->env->device);
  int32_t v = 0;
  if (cudaDeviceSynchronize() != cudaSuccess ||
      cudaMemcpy(&v, pol->sync + 2 * pol->tiles, sizeof(v), cudaMemcpyDeviceToHost) != cudaSuccess) return FXENV_E_CUDA;
  return (int)v;
}

int64_t fxenv_policy_peek(FxPolicy* pol, int what, int slot, void* dst, int64_t bytes, void* stream) {
  if (!pol) return FXENV_E_INVALID;
  FxEnv* env = pol->env;
  const void* src = nullptr;
  int64_t n = 0;
  if (what == FXENV_PEEK_OBS16 && (slot == 0 || slot == 1)) {
    src = pol->obs16[slot];
    n = (int64_t)env->P.cfg.num_envs * pol->k_pad * 2;
  } else if (what == FXENV_PEEK_H1 && slot == 0) {
    src = pol->h1;
    n = (int64_t)pol->tiles * FX_POLICY_TILE_M * pol->nets * pol->hidden * 2;
  } else {
    return fail(env, FXENV_E_INVALID, "fxenv_policy_peek: unknown buffer or slot");
  }
  if (!dst) return n;
  if (bytes < n) return fail(env, FXENV_E_INVALID, "fxenv_policy_peek: destination too small");
  DeviceGuard g(env->device);
  FX_CUDA(env, cudaMemcpyAsync(dst, src, (size_t)n, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return n;
}

int fxenv_policy_create(FxEnv* env, FxPolicy** out) {
  return fxenv_policy_create_ex(env, FX_POLICY_HIDDEN, out);
}

int fxenv_policy_create_ex(FxEnv* env, int32_t hidden, FxPolicy** out) {
  return fxenv_policy_create_ex2(env, hidden, 0u, out);
}

int fxenv_policy_create_ex2(FxEnv* env, int32_t hidden, uint32_t flags, FxPolicy** out) {
  return fxenv_policy_create_ex3(env, hidden, flags, 1, out);
}

int fxenv_policy_create_ex3(FxEnv* env, int32_t hidden, uint32_t flags, int32_t members, FxPolicy** out) {
  if (!env || !out) return FXENV_E_INVALID;
  *out = nullptr;
  if (flags & ~(uint32_t)FXENV_POLICY_SEPARATE) return fail(env, FXENV_E_INVALID, "unknown policy flags");
  if (env->P.cfg.action_mode != FX_ACTION_DISCRETE && env->P.cfg.action_mode != FX_ACTION_CONTINUOUS)
    return fail(env, FXENV_E_INVALID, "unknown action mode");
  if (!fx_policy_width_ok(hidden))
    return fail(env, FXENV_E_INVALID, "policy width must be 64, 128, 256 or 512, got " + std::to_string(hidden));
  if (members < 1) return fail(env, FXENV_E_INVALID, "policy members must be >= 1, got " + std::to_string(members));
  if (members > 1 && (int64_t)env->P.cfg.num_envs % ((int64_t)FX_POLICY_TILE_M * members) != 0)
    return fail(env, FXENV_E_INVALID, "num_envs (" + std::to_string(env->P.cfg.num_envs) + ") must be a multiple of " +
                                      std::to_string(FX_POLICY_TILE_M) + " x members (" + std::to_string(members) +
                                      "): each member owns whole 128-env tiles");
  DeviceGuard g(env->device);
  FxPolicy* pol = new (std::nothrow) FxPolicy();
  if (!pol) return fail(env, FXENV_E_NOMEM, "out of host memory");
  pol->env = env;
  pol->continuous = env->P.cfg.action_mode == FX_ACTION_CONTINUOUS;
  pol->hidden = hidden;
  pol->separate = (flags & FXENV_POLICY_SEPARATE) != 0;
  pol->nets = pol->separate ? 2 : 1;
  pol->members = members;
  pol->has_weights.assign((size_t)members, false);
  pol->norm_on.assign((size_t)members, false);
  pol->missing_weights = members;
  const size_t N = (size_t)env->P.cfg.num_envs, D = (size_t)env->P.obs_dim, M = (size_t)members;
  pol->k_pad = (int)((D + 63) / 64 * 64);
  const size_t KP = (size_t)pol->k_pad, Hd = (size_t)hidden, Hn = (size_t)pol->nets * Hd;  // Hn: stacked trunk rows
  bool ok = cudaMalloc(&pol->w1, M * Hn * KP * 2) == cudaSuccess && cudaMalloc(&pol->w2, M * Hn * Hd * 2) == cudaSuccess &&
            cudaMalloc(&pol->fparams, M * (2 * Hn + 4 * Hd + 4) * sizeof(float)) == cudaSuccess &&
            cudaMalloc(&pol->obs16[0], N * KP * 2) == cudaSuccess && cudaMalloc(&pol->obs16[1], N * KP * 2) == cudaSuccess &&
            cudaMalloc(&pol->scratch_act, N * 4) == cudaSuccess && cudaMalloc(&pol->scratch_logp, N * 4) == cudaSuccess;
  const size_t NP = (N + FX_POLICY_TILE_M - 1) / FX_POLICY_TILE_M * FX_POLICY_TILE_M;  // whole 128-env tiles
  ok = ok && cudaMalloc(&pol->h1, NP * Hn * 2) == cudaSuccess &&
       cudaMalloc(&pol->head_part, NP * pol->nets * 4 * sizeof(float)) == cudaSuccess;
  pol->tiles = (int)(NP / FX_POLICY_TILE_M);
  ok = ok && cudaMalloc(&pol->sync, (2 * (size_t)pol->tiles + 1) * sizeof(int32_t)) == cudaSuccess;
  if (!ok) { fxenv_policy_destroy(pol); return fail(env, FXENV_E_CUDA, "cudaMalloc(policy buffers) failed"); }
  // the K padding of the observation copies is never written by the env kernels: zero it once
  cudaMemset(pol->obs16[0], 0, N * KP * 2);
  cudaMemset(pol->obs16[1], 0, N * KP * 2);
  pol->dev.b1 = pol->fparams; pol->dev.b2 = pol->fparams + M * Hn; pol->dev.head_w = pol->fparams + 2 * M * Hn;
  pol->dev.head_b = pol->fparams + 2 * M * Hn + 4 * M * Hd;
  pol->dev.h1 = pol->h1; pol->dev.head_part = reinterpret_cast<float4*>(pol->head_part);
  pol->dev.dbg = env->P.timeline;  // (nullptr unless FXENV_TIMELINE is set; only the timing build looks at it)
  pol->dev.act_flag = pol->sync; pol->dev.done_cnt = pol->sync + pol->tiles; pol->dev.timeouts = pol->sync + 2 * pol->tiles;
  cudaMemset(pol->sync, 0, (2 * (size_t)pol->tiles + 1) * sizeof(int32_t));
  int rc = make_map(env, &pol->map_obs[0], pol->obs16[0], N, KP, FX_POLICY_TILE_M);
  if (!rc) rc = make_map(env, &pol->map_obs[1], pol->obs16[1], N, KP, FX_POLICY_TILE_M);
  // over every member's rows; a CTA loads its half of one network's units
  if (!rc) rc = make_map(env, &pol->map_w1, pol->w1, M * Hn, KP, (uint32_t)Hd / 2);
  if (!rc) rc = make_map(env, &pol->map_w2, pol->w2, M * Hn, Hd, (uint32_t)Hd / 2);
  if (!rc) rc = make_map(env, &pol->map_h1, pol->h1, NP, Hn, FX_POLICY_TILE_M);
  if (rc) { fxenv_policy_destroy(pol); return rc; }
  cudaError_t ce = fx_policy_configure();
  for (auto& st : pol->side) if (ce == cudaSuccess) ce = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
  if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&pol->ev_fork, cudaEventDisableTiming);
  for (auto& ev : pol->ev_join) if (ce == cudaSuccess) ce = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
  if (ce != cudaSuccess) { fxenv_policy_destroy(pol); return cuda_fail(env, ce, "fx_policy_configure / streams"); }
  *out = pol;
  return FXENV_OK;
}

int fxenv_policy_set_weights(FxPolicy* pol, const FxPolicyWeights* w, void* stream_) {
  return fxenv_policy_set_member_weights(pol, 0, w, stream_);
}

int fxenv_policy_set_member_weights(FxPolicy* pol, int32_t member, const FxPolicyWeights* w, void* stream_) {
  if (!pol || !w) return FXENV_E_INVALID;
  FxEnv* env = pol->env;
  if (member < 0 || member >= pol->members)
    return fail(env, FXENV_E_INVALID, "policy member " + std::to_string(member) + " out of range [0, " +
                                      std::to_string(pol->members) + ")");
  if (!w->w1 || !w->b1 || !w->w2 || !w->b2 || !w->w_pi || !w->b_pi || !w->w_v || !w->b_v) return fail(env, FXENV_E_INVALID, "null weight pointer");
  DeviceGuard g(env->device);
  cudaStream_t s = (cudaStream_t)stream_;
  const int D = env->P.obs_dim, Hd = pol->hidden, Hn = pol->nets * Hd;  // Hn: stacked trunk rows
  const size_t m = (size_t)member, M = (size_t)pol->members;
  FX_CUDA(env, fx_policy_pack(w->w1, pol->w1 + m * Hn * pol->k_pad, Hn, D, pol->k_pad, s));
  FX_CUDA(env, fx_policy_pack(w->w2, pol->w2 + m * Hn * Hd, Hn, Hd, Hd, s));
  float* f = pol->fparams;
  float* b1 = f + m * Hn;                         // the member's b1 [Hn]
  float* b2 = f + (M + m) * Hn;                   // its b2 [Hn]
  float* hw = f + 2 * M * Hn + m * 4 * Hd;        // its head rows [4][Hd]
  float* hb = f + 2 * M * Hn + 4 * M * Hd + m * 4;  // its head bias [4]
  FX_CUDA(env, cudaMemcpyAsync(b1, w->b1, Hn * 4, cudaMemcpyDeviceToDevice, s));
  FX_CUDA(env, cudaMemcpyAsync(b2, w->b2, Hn * 4, cudaMemcpyDeviceToDevice, s));
  if (pol->continuous) {  // head rows {w_mu, 0, 0, w_v}, head bias {b_mu, log sigma, 0, b_v}
    FX_CUDA(env, cudaMemcpyAsync(hw, w->w_pi, Hd * 4, cudaMemcpyDeviceToDevice, s));
    FX_CUDA(env, cudaMemsetAsync(hw + Hd, 0, 2 * Hd * 4, s));
    FX_CUDA(env, cudaMemcpyAsync(hb, w->b_pi, 2 * 4, cudaMemcpyDeviceToDevice, s));
    FX_CUDA(env, cudaMemsetAsync(hb + 2, 0, 4, s));
  } else {
    FX_CUDA(env, cudaMemcpyAsync(hw, w->w_pi, 3 * Hd * 4, cudaMemcpyDeviceToDevice, s));
    FX_CUDA(env, cudaMemcpyAsync(hb, w->b_pi, 3 * 4, cudaMemcpyDeviceToDevice, s));
  }
  FX_CUDA(env, cudaMemcpyAsync(hw + 3 * Hd, w->w_v, Hd * 4, cudaMemcpyDeviceToDevice, s));
  FX_CUDA(env, cudaMemcpyAsync(hb + 3, w->b_v, 4, cudaMemcpyDeviceToDevice, s));
  env->launches += 2;
  if (!pol->has_weights[m]) { pol->has_weights[m] = true; pol->missing_weights--; }
  return FXENV_OK;
}

int fxenv_policy_set_obs_norm(FxPolicy* pol, int32_t member, const float* mean_dev, const float* rstd_dev, float clip,
                              void* stream_) {
  if (!pol) return FXENV_E_INVALID;
  FxEnv* env = pol->env;
  if (member < 0 || member >= pol->members)
    return fail(env, FXENV_E_INVALID, "policy member " + std::to_string(member) + " out of range [0, " +
                                      std::to_string(pol->members) + ")");
  if ((mean_dev == nullptr) != (rstd_dev == nullptr))
    return fail(env, FXENV_E_INVALID, "fxenv_policy_set_obs_norm: mean and rstd must both be given or both be NULL");
  const size_t m = (size_t)member;
  const bool on = mean_dev != nullptr;
  if (on && !(clip > 0.0f))  // also NaN
    return fail(env, FXENV_E_INVALID, "fxenv_policy_set_obs_norm: clip must be > 0 (+inf allowed), got " + std::to_string(clip));
  DeviceGuard g(env->device);
  cudaStream_t s = (cudaStream_t)stream_;
  const size_t P = (size_t)env->P.cfg.num_pairs, D = (size_t)env->P.obs_dim, KP = (size_t)pol->k_pad;
  const size_t MPK = (size_t)pol->members * P * KP;
  if (on && !pol->norm) {  // zeroed once: the pad columns stay 0
    FX_CUDA(env, cudaMalloc(&pol->norm, (2 * MPK + (size_t)pol->members) * sizeof(float)));
    FX_CUDA(env, cudaMemset(pol->norm, 0, (2 * MPK + (size_t)pol->members) * sizeof(float)));
  }
  if (on != pol->norm_on[m]) {  // another kernel variant: the cached rollout graph is captured again
    if (const int rc = params_changing(env)) return rc;
  }
  if (on) {
    float* mean = pol->norm + m * P * KP;
    FX_CUDA(env, cudaMemcpy2DAsync(mean, KP * 4, mean_dev, D * 4, D * 4, P, cudaMemcpyDeviceToDevice, s));
    FX_CUDA(env, cudaMemcpy2DAsync(mean + MPK, KP * 4, rstd_dev, D * 4, D * 4, P, cudaMemcpyDeviceToDevice, s));
    FX_CUDA(env, cudaMemcpyAsync(pol->norm + 2 * MPK + m, &clip, sizeof(float), cudaMemcpyHostToDevice, s));
  }
  if (on != pol->norm_on[m]) {
    pol->norm_on[m] = on;
    pol->norm_members += on ? 1 : -1;
  }
  return FXENV_OK;
}

int fxenv_obs_moments(FxEnv* env, const float* obs_dev, int32_t slots, int32_t env_begin, int32_t env_end,
                      const float* shift_dev, double* out_dev, void* stream_) {
  if (!env) return FXENV_E_INVALID;
  if (!obs_dev || !shift_dev || !out_dev) return fail(env, FXENV_E_INVALID, "fxenv_obs_moments: null pointer");
  const int N = env->P.cfg.num_envs;
  if (slots < 1) return fail(env, FXENV_E_INVALID, "fxenv_obs_moments: slots must be >= 1, got " + std::to_string(slots));
  if (env_begin < 0 || env_end > N || env_begin >= env_end)
    return fail(env, FXENV_E_INVALID, "fxenv_obs_moments: env range [" + std::to_string(env_begin) + ", " +
                                      std::to_string(env_end) + ") is empty or outside [0, " + std::to_string(N) + ")");
  DeviceGuard g(env->device);
  FX_CUDA(env, fx_launch_obs_moments(obs_dev, slots, N, env->P.obs_dim, env->P.cfg.num_pairs, env_begin, env_end, shift_dev,
                                     out_dev, (cudaStream_t)stream_));
  env->launches += 2;
  return FXENV_OK;
}

int fxenv_return_moments(FxEnv* env, const float* reward_dev, const uint8_t* done_dev, const uint8_t* prev_done_dev,
                         int32_t horizon, int32_t env_begin, int32_t env_end, double gamma, double shift,
                         double* ret_dev, int32_t* seen_dev, double* out_dev, void* stream_) {
  if (!env) return FXENV_E_INVALID;
  if (!reward_dev || !done_dev || !prev_done_dev || !ret_dev || !seen_dev || !out_dev)
    return fail(env, FXENV_E_INVALID, "fxenv_return_moments: null pointer");
  const int N = env->P.cfg.num_envs;
  if (horizon < 1)
    return fail(env, FXENV_E_INVALID, "fxenv_return_moments: horizon must be >= 1, got " + std::to_string(horizon));
  if (env_begin < 0 || env_end > N || env_begin >= env_end)
    return fail(env, FXENV_E_INVALID, "fxenv_return_moments: env range [" + std::to_string(env_begin) + ", " +
                                      std::to_string(env_end) + ") is empty or outside [0, " + std::to_string(N) + ")");
  if (!(gamma >= 0.0 && gamma <= 1.0))  // also NaN
    return fail(env, FXENV_E_INVALID, "fxenv_return_moments: gamma must be in [0, 1], got " + std::to_string(gamma));
  if (!isfinite(shift))
    return fail(env, FXENV_E_INVALID, "fxenv_return_moments: shift must be finite, got " + std::to_string(shift));
  DeviceGuard g(env->device);
  FX_CUDA(env, fx_launch_return_moments(reward_dev, done_dev, prev_done_dev, env->P.st.ep_begun, N, horizon, env_begin,
                                        env_end, gamma, shift, ret_dev, seen_dev, out_dev, (cudaStream_t)stream_));
  env->launches += 2;
  return FXENV_OK;
}

int fxenv_rollout(FxEnv* env, FxPolicy* pol, const FxRollout* io, void* stream_) {
  return fxenv_rollout_ex(env, pol, io, 0u, stream_);
}

int fxenv_rollout_ex(FxEnv* env, FxPolicy* pol, const FxRollout* io, uint32_t flags, void* stream_) {
  int rc = require_ready(env, true);
  if (rc) return rc;
  if (!pol || !io || pol->env != env) return fail(env, FXENV_E_INVALID, "policy does not belong to this env");
  if (flags & ~(uint32_t)FXENV_ROLLOUT_GREEDY) return fail(env, FXENV_E_INVALID, "unknown rollout flags");
  if (pol->missing_weights > 0) {
    if (pol->members == 1) return fail(env, FXENV_E_STATE, "fxenv_policy_set_weights has not been called");
    int first = 0;
    while (pol->has_weights[first]) first++;
    return fail(env, FXENV_E_STATE, std::to_string(pol->missing_weights) + " of " + std::to_string(pol->members) +
                                    " policy members have no weights yet (first: member " + std::to_string(first) + ")");
  }
  if (pol->norm_members > 0 && pol->norm_members < pol->members)
    return fail(env, FXENV_E_STATE, std::to_string(pol->norm_members) + " of " + std::to_string(pol->members) +
                                    " policy members have an observation normalizer: every member or none");
  if (io->horizon < 1 || io->obs_slots < 2) return fail(env, FXENV_E_INVALID, "horizon must be >= 1 and obs_slots >= 2");
  if (!io->obs || !io->actions || !io->logp || !io->value || !io->reward || !io->done) return fail(env, FXENV_E_INVALID, "null I/O pointer");
  DeviceGuard g(env->device);
  cudaStream_t stream = (cudaStream_t)stream_;
  // the graph bakes in the buffers, the seed, the flags (greedy or sampling) and the env's kernel parameters (P, by
  // value); FXENV_DEBUG & 32: plain launches (timing experiments)
  const RolloutKey key = {*io, flags};
  const auto enqueue = [&](cudaStream_t s) { return enqueue_rollout(env, pol, *io, flags, s); };
  rc = launch_cached(env, pol->graph, key, (env->P.debug & 32) != 0, stream, enqueue, "capture: rollout");
  if (rc) return rc;
  env->launches += 2 * (int64_t)io->horizon + 2;
  return FXENV_OK;
}

}  // extern "C"
