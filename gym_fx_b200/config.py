"""
Host-side lowering of the reference's "dict of everything" configuration into the FxConfig POD of
include/fxenv.h.

The reference reads its config dict at CALL time inside every plugin, each with its own precedence rule
(SURVEY.md section 5 "Config / flags"):

  * env                 config.get(key, default)                              app/env.py:56-80
  * default_broker      config.get(key, plugin.params[key])                   broker_plugins/default_broker.py:36-45
  * direct_*_sltp       plugin.params, overridden by non-None config values   strategy_plugins/direct_fixed_sltp.py:79-84,
                        for the plugin's own keys only                        strategy_plugins/direct_atr_sltp.py:226-231
  * preprocessors       config.get(key, plugin.params[key])                   preprocessor_plugins/*.py
  * rewards             config.get(key, plugin.params[key]); sharpe's deque   reward_plugins/*.py
                        length comes from plugin.params["window"] only        reward_plugins/sharpe_reward.py:24-32

`lower_config` applies exactly those rules ONCE and returns a ctypes struct that is passed by pointer to
fxenv_create().  Plugins are recognised by the name of the module their class lives in (the same names the
reference registers as entry points, setup.py:11-35), so reference plugin instances and this package's mirrors
lower identically.
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Dict, Optional, Sequence

FXENV_MAX_PAIRS = 8
FXENV_MAX_FEATURES = 16
FXENV_MAX_COLS = 16

ACTION_DISCRETE, ACTION_CONTINUOUS = 0, 1
STRATEGY_DEFAULT, STRATEGY_FIXED_SLTP, STRATEGY_ATR_SLTP = 0, 1, 2
PREPROC_DEFAULT, PREPROC_FEATURE_WINDOW = 0, 1
SCALING_NONE, SCALING_ROLLING, SCALING_EXPANDING = 0, 1, 2
REWARD_PNL, REWARD_SHARPE, REWARD_DD = 0, 1, 2
SIZE_FX_UNITS, SIZE_NOTIONAL = 0, 1

FLAG_STARTED, FLAG_TERMINATED, FLAG_EXHAUSTED, FLAG_BROKE, FLAG_ORDER_OVERFLOW = 1, 2, 4, 8, 16

BASE_COLUMNS = ("OPEN", "HIGH", "LOW", "CLOSE", "VOLUME")


class FxConfig(C.Structure):
    """ctypes mirror of `struct FxConfig` (include/fxenv.h) -- field order and types must match."""

    _fields_ = [
        ("struct_size", C.c_int32),
        ("num_envs", C.c_int32),
        ("num_pairs", C.c_int32),
        ("n_cols", C.c_int32),
        ("order_capacity", C.c_int32),
        ("auto_reset", C.c_int32),
        ("episode_bars", C.c_int64),
        ("initial_cash", C.c_double),
        ("position_size", C.c_double),
        ("min_equity", C.c_double),
        ("action_mode", C.c_int32),
        ("_pad0", C.c_int32),
        ("continuous_action_threshold", C.c_double),
        ("commission", C.c_double),
        ("leverage", C.c_double),
        ("slippage_perc", C.c_double),
        ("children_same_bar", C.c_int32),
        ("strategy", C.c_int32),
        ("strat_position_size", C.c_double),
        ("sl_pips", C.c_double),
        ("tp_pips", C.c_double),
        ("pip_size", C.c_double),
        ("pair_pip_size", C.c_double * FXENV_MAX_PAIRS),
        ("atr_period", C.c_int32),
        ("use_rel_volume", C.c_int32),
        ("k_sl", C.c_double),
        ("k_tp", C.c_double),
        ("rel_volume", C.c_double),
        ("strat_leverage", C.c_double),
        ("min_order_volume", C.c_double),
        ("max_order_volume", C.c_double),
        ("size_mode", C.c_int32),
        ("use_min_frac", C.c_int32),
        ("use_max_frac", C.c_int32),
        ("session_filter", C.c_int32),
        ("min_sltp_frac", C.c_double),
        ("max_sltp_frac", C.c_double),
        ("entry_dow_start", C.c_int32),
        ("entry_hour_start", C.c_int32),
        ("force_close_dow", C.c_int32),
        ("force_close_hour", C.c_int32),
        ("preproc", C.c_int32),
        ("window_size", C.c_int32),
        ("price_col", C.c_int32),
        ("n_features", C.c_int32),
        ("feature_cols", C.c_int32 * FXENV_MAX_FEATURES),
        ("feature_binary", C.c_int32 * FXENV_MAX_FEATURES),
        ("scaling", C.c_int32),
        ("scaling_window", C.c_int32),
        ("include_price_window", C.c_int32),
        ("include_agent_state", C.c_int32),
        ("feature_clip", C.c_double),
        ("obs_position_size", C.c_double),
        ("reward", C.c_int32),
        ("sharpe_window", C.c_int32),
        ("reward_initial_cash", C.c_double),
        ("reward_scale", C.c_double),
        ("annualization_factor", C.c_double),
        ("penalty_lambda", C.c_double),
    ]


def plugin_kind(plugin: Any) -> str:
    """Entry-point style name of a plugin instance: the last component of its class's module
    (e.g. 'direct_fixed_sltp'), or its explicit `plugin_kind` attribute."""
    k = getattr(plugin, "plugin_kind", None)
    if k:
        return str(k)
    return type(plugin).__module__.split(".")[-1]


def _params(plugin: Any) -> Dict[str, Any]:
    p = getattr(plugin, "params", None)
    if p is None:
        p = getattr(plugin, "plugin_params", {})
    return dict(p)


def _cfg_or_param(config: Dict[str, Any], params: Dict[str, Any], key: str, default: Any = None) -> Any:
    """config.get(key, plugin.params[key]) -- the broker / preprocessor / reward rule."""
    if key in config:
        return config[key]
    return params.get(key, default)


def _resolve_known(config: Dict[str, Any], plugin: Any) -> Dict[str, Any]:
    """direct_*_sltp `_resolve`: plugin.params, overridden by NON-None config values of the plugin's own keys."""
    merged = _params(plugin)
    for k in getattr(type(plugin), "plugin_params", {}):
        if k in config and config[k] is not None:
            merged[k] = config[k]
    return merged


def lower_config(
    config: Dict[str, Any],
    *,
    broker_plugin: Any,
    strategy_plugin: Any,
    preprocessor_plugin: Any,
    reward_plugin: Any,
    columns: Sequence[str] = BASE_COLUMNS,
    num_envs: int = 1,
    num_pairs: int = 1,
    order_capacity: int = 0,
    auto_reset: bool = False,
    episode_bars: int = 0,
    children_same_bar: bool = False,
    pair_pip_size: Optional[Sequence[float]] = None,
) -> FxConfig:
    columns = [str(c) for c in columns]
    if tuple(columns[:5]) != BASE_COLUMNS:
        raise ValueError(f"candle table columns must start with {BASE_COLUMNS}; got {columns[:5]}")
    if len(columns) > FXENV_MAX_COLS:
        raise ValueError(f"at most {FXENV_MAX_COLS} candle columns are supported")
    if not (1 <= num_pairs <= FXENV_MAX_PAIRS):
        raise ValueError(f"num_pairs must be in 1..{FXENV_MAX_PAIRS}")
    c = FxConfig()
    c.struct_size = C.sizeof(FxConfig)
    c.num_envs = int(num_envs)
    c.num_pairs = int(num_pairs)
    c.n_cols = len(columns)
    c.order_capacity = int(order_capacity)
    c.auto_reset = int(bool(auto_reset))
    c.episode_bars = int(episode_bars)
    c.children_same_bar = int(bool(children_same_bar))

    # ---- GymFxEnv (app/env.py:56-80)
    c.initial_cash = float(config.get("initial_cash", 10000.0))
    c.position_size = float(config.get("position_size", 1.0))
    window_size = int(config.get("window_size", 32))
    price_column = config.get("price_column", "CLOSE")
    c.min_equity = float(config.get("min_equity", c.initial_cash * 0.01))
    mode = str(config.get("action_space_mode", "discrete")).lower()
    c.action_mode = ACTION_CONTINUOUS if mode == "continuous" else ACTION_DISCRETE
    c.continuous_action_threshold = float(config.get("continuous_action_threshold", 0.33))
    if price_column not in columns:
        raise ValueError(f"price_column '{price_column}' not found in data")

    # ---- broker (broker_plugins/default_broker.py:35-53)
    bk = plugin_kind(broker_plugin)
    if bk != "default_broker":
        raise ValueError(f"broker plugin '{bk}' cannot be lowered to the GPU env (only default_broker)")
    bp = _params(broker_plugin)
    broker_cash = float(_cfg_or_param(config, bp, "initial_cash", 10000.0))
    if broker_cash != c.initial_cash:
        raise ValueError("broker initial_cash differs from env initial_cash; unsupported")
    c.commission = float(_cfg_or_param(config, bp, "commission", 0.0))
    c.slippage_perc = float(config.get("slippage_perc", config.get("slippage", bp.get("slippage_perc", 0.0))))
    c.leverage = float(_cfg_or_param(config, bp, "leverage", 1.0))

    # ---- strategy
    sk = plugin_kind(strategy_plugin)
    c.pip_size = 1e-4
    c.sl_pips, c.tp_pips = 20.0, 40.0
    c.strat_position_size = c.position_size
    c.atr_period, c.k_sl, c.k_tp = 14, 2.0, 3.0
    c.strat_leverage, c.max_order_volume = 1.0, 1e12
    if sk == "default_strategy" or not callable(getattr(strategy_plugin, "apply_action", None)):
        c.strategy = STRATEGY_DEFAULT  # app/bt_bridge.py:171-190
    elif sk == "direct_fixed_sltp":
        c.strategy = STRATEGY_FIXED_SLTP
        p = _resolve_known(config, strategy_plugin)
        c.strat_position_size = float(p["position_size"])
        c.pip_size = float(p["pip_size"])
        c.sl_pips = float(p["sl_pips"])
        c.tp_pips = float(p["tp_pips"])
    elif sk == "direct_atr_sltp":
        c.strategy = STRATEGY_ATR_SLTP
        p = _resolve_known(config, strategy_plugin)
        c.atr_period = int(p["atr_period"])
        c.k_sl = float(p["k_sl"])
        c.k_tp = float(p["k_tp"])
        c.strat_position_size = float(p["position_size"])
        rel = p.get("rel_volume")
        c.use_rel_volume = int(rel is not None)
        c.rel_volume = float(rel) if rel is not None else 0.0
        c.strat_leverage = float(p.get("leverage", 1.0))
        c.min_order_volume = float(p.get("min_order_volume", 0.0))
        c.max_order_volume = float(p.get("max_order_volume", 1e12))
        c.size_mode = SIZE_NOTIONAL if str(p.get("size_mode", "fx_units")).lower() == "notional" else SIZE_FX_UNITS
        mn, mx = p.get("min_sltp_frac"), p.get("max_sltp_frac")
        c.use_min_frac, c.use_max_frac = int(mn is not None), int(mx is not None)
        c.min_sltp_frac = float(mn) if mn is not None else 0.0
        c.max_sltp_frac = float(mx) if mx is not None else 0.0
        c.session_filter = int(bool(p.get("session_filter")))
        c.entry_dow_start = int(p["entry_dow_start"])
        c.entry_hour_start = int(p["entry_hour_start"])
        c.force_close_dow = int(p["force_close_dow"])
        c.force_close_hour = int(p["force_close_hour"])
        if not (1 <= c.atr_period <= 64):
            raise ValueError("atr_period must be in 1..64")
    else:
        raise ValueError(f"strategy plugin '{sk}' has a custom apply_action and cannot be lowered to the GPU env")
    for i in range(FXENV_MAX_PAIRS):
        c.pair_pip_size[i] = float(pair_pip_size[i]) if pair_pip_size is not None and i < len(pair_pip_size) else 0.0

    # ---- preprocessor
    pk = plugin_kind(preprocessor_plugin)
    pp = _params(preprocessor_plugin)
    c.window_size = int(_cfg_or_param(config, pp, "window_size", 32))
    if c.window_size != window_size:
        # env.window_size only sizes the (inaccurate) observation_space of the reference; the plugin value rules
        pass
    pc = _cfg_or_param(config, pp, "price_column", "CLOSE")
    if pc not in columns:
        raise ValueError(f"price_column '{pc}' not found in data")
    c.price_col = columns.index(pc)
    c.obs_position_size = float(config.get("position_size", 1.0))
    c.include_price_window = 1
    c.include_agent_state = 1
    c.feature_clip = 10.0
    c.scaling_window = 256
    if pk == "default_preprocessor":
        c.preproc = PREPROC_DEFAULT
    elif pk == "feature_window_preprocessor":
        c.preproc = PREPROC_FEATURE_WINDOW
        cols = config.get("feature_columns") or pp.get("feature_columns") or []
        if not cols:
            raise ValueError("feature_window_preprocessor requires non-empty 'feature_columns'.")
        missing = [x for x in cols if x not in columns]
        if missing:
            raise ValueError(
                "feature_window_preprocessor: configured feature_columns "
                f"missing from dataframe: {missing[:5]}{'...' if len(missing) > 5 else ''}"
            )
        if len(cols) > FXENV_MAX_FEATURES:
            raise ValueError(f"at most {FXENV_MAX_FEATURES} feature columns are supported")
        binary = set(config.get("feature_binary_columns") or pp.get("feature_binary_columns") or [])
        c.n_features = len(cols)
        for i, name in enumerate(cols):
            c.feature_cols[i] = columns.index(name)
            c.feature_binary[i] = int(name in binary)
        sm = str(_cfg_or_param(config, pp, "feature_scaling", "rolling_zscore")).lower()
        valid = {"none": SCALING_NONE, "rolling_zscore": SCALING_ROLLING, "expanding_zscore": SCALING_EXPANDING}
        if sm not in valid:
            raise ValueError(f"feature_scaling must be one of {tuple(valid)}; got {sm!r}")
        c.scaling = valid[sm]
        c.scaling_window = int(_cfg_or_param(config, pp, "feature_scaling_window", 256))
        c.feature_clip = float(_cfg_or_param(config, pp, "feature_clip", 10.0))
        c.include_price_window = int(bool(_cfg_or_param(config, pp, "include_price_window", True)))
        c.include_agent_state = int(bool(_cfg_or_param(config, pp, "include_agent_state", True)))
    else:
        raise ValueError(f"preprocessor plugin '{pk}' cannot be lowered to the GPU env")
    if c.window_size < 1:
        raise ValueError("window_size must be >= 1")

    # ---- reward
    rk = plugin_kind(reward_plugin)
    rp = _params(reward_plugin)
    c.reward_initial_cash = float(_cfg_or_param(config, rp, "initial_cash", 10000.0)) or 1.0
    c.reward_scale, c.sharpe_window, c.annualization_factor, c.penalty_lambda = 1.0, 64, 252.0, 1.0
    if rk == "pnl_reward":
        c.reward = REWARD_PNL
        c.reward_scale = float(_cfg_or_param(config, rp, "reward_scale", 1.0))
    elif rk == "sharpe_reward":
        c.reward = REWARD_SHARPE
        c.sharpe_window = int(rp.get("window", 64))  # deque(maxlen=params["window"]); config is not consulted
        c.annualization_factor = float(_cfg_or_param(config, rp, "annualization_factor", 252.0))
        if not (1 <= c.sharpe_window <= 4096):
            raise ValueError("sharpe window must be in 1..4096")
    elif rk == "dd_penalized_reward":
        c.reward = REWARD_DD
        c.penalty_lambda = float(_cfg_or_param(config, rp, "penalty_lambda", 1.0))
    else:
        raise ValueError(f"reward plugin '{rk}' cannot be lowered to the GPU env")
    return c


# The columns of a per-env parameter row (include/fxenv.h FXENV_PARAM_*) and the FxConfig field each one replaces
ENV_PARAM_FIELDS = ("commission", "leverage", "slippage", "sl_pips", "tp_pips", "k_sl", "k_tp")
_ENV_PARAM_CFG = ("commission", "leverage", "slippage_perc", "sl_pips", "tp_pips", "k_sl", "k_tp")


def env_params_table(cfg: FxConfig, **fields) -> "np.ndarray":
    """The float64 [num_envs, 7] table of fxenv_set_env_params (VecFxEnv.set_env_params).  Each keyword of
    ENV_PARAM_FIELDS is None (the config's value for every env), a scalar (every env) or num_envs values (a sequence, numpy
    array or tensor).  Raises TypeError for an unknown field or a non-numeric value, ValueError for a wrong length, a value
    that is not finite, leverage <= 0 or slippage outside [0, 1) (the rules fxenv_create applies to the config)."""
    import numpy as np

    unknown = sorted(set(fields) - set(ENV_PARAM_FIELDS))
    if unknown:
        raise TypeError(f"unknown env parameter(s) {unknown}; expected some of {ENV_PARAM_FIELDS}")
    n = int(cfg.num_envs)
    table = np.empty((n, len(ENV_PARAM_FIELDS)), np.float64)
    for j, (name, cname) in enumerate(zip(ENV_PARAM_FIELDS, _ENV_PARAM_CFG)):
        v = fields.get(name)
        if v is None:
            table[:, j] = getattr(cfg, cname)
            continue
        if hasattr(v, "detach"):  # torch tensor, on any device
            v = v.detach().cpu().numpy()
        a = np.asarray(v)
        if a.dtype.kind not in "iuf":
            raise TypeError(f"{name} must be numeric, got {a.dtype} ({v!r:.60})")
        if a.ndim == 0 or a.shape == (n,):
            table[:, j] = a.astype(np.float64)
        else:
            raise ValueError(f"{name} must be a scalar or {n} values (one per env), got shape {a.shape}")
    for j, name in enumerate(ENV_PARAM_FIELDS):
        col = table[:, j]
        bad = ~np.isfinite(col)
        if name == "leverage":
            bad |= ~(col > 0.0)
        elif name == "slippage":
            bad |= ~((col >= 0.0) & (col < 1.0))
        if bad.any():
            i = int(np.flatnonzero(bad)[0])
            rule = {"leverage": "finite and > 0", "slippage": "in [0, 1)"}.get(name, "finite")
            raise ValueError(f"env {i}: {name} = {col[i]!r} must be {rule}")
    return table


def obs_dim(cfg: FxConfig) -> int:
    """Flat observation width (SURVEY A.2): features W*F | prices W | returns W | 4 agent scalars."""
    W = cfg.window_size
    if cfg.preproc == PREPROC_DEFAULT:
        return 2 * W + 4
    return W * cfg.n_features + (2 * W if cfg.include_price_window else 0) + (4 if cfg.include_agent_state else 0)


def obs_layout(cfg: FxConfig) -> Dict[str, tuple]:
    """name -> (offset, shape) of each part of a flat observation row."""
    W, out, off = cfg.window_size, {}, 0
    if cfg.preproc == PREPROC_FEATURE_WINDOW:
        out["features"] = (off, (W, cfg.n_features))
        off += W * cfg.n_features
    if cfg.preproc == PREPROC_DEFAULT or cfg.include_price_window:
        out["prices"] = (off, (W,))
        out["returns"] = (off + W, (W,))
        off += 2 * W
    if cfg.preproc == PREPROC_DEFAULT or cfg.include_agent_state:
        for k in ("position", "equity_norm", "unrealized_pnl_norm", "steps_remaining_norm"):
            out[k] = (off, (1,))
            off += 1
    return out
