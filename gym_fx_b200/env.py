"""
GymFxEnv -- the reference's single-env Gym API (app/env.py:31-271) on top of the GPU step kernel.

Same constructor signature, same reset/step/render/close/summary surface, same Dict observation (numpy) and info
dict, same error behaviour (ValueError for short/missing data at construction, RuntimeError for step-before-reset,
malformed actions coerced to hold).  The per-tick work is one launch of the fused kernel for a 1-env VecFxEnv 
(device tensors in, results copied back for the numpy-facing API); there is no CPU implementation behind this class.

Differences, all deliberate (SURVEY.md App. B):
  * `observation_space` is derived from the preprocessor's real layout (the reference omits `features` and
    ignores include_price_window/include_agent_state, App. B #9);
  * there is no backtrader: `summary()` passes an empty analyzers dict to the metrics plugin, which is what the
    reference effectively does on the live path (App. B #12).

With the config key `max_episode_steps` (Gymnasium's name; not a reference key) an episode is cut after that many steps:
step() then returns terminated=False, truncated=True, and keeps answering so until reset(), as after a termination.
Without the key, truncated is always False as in the reference.

With direct_atr_sltp and GYMFX_BRACKET_AUDIT set (read at import of the strategy module, as in the reference), every
step() appends the decisions the step kernel logged to that file, in the reference's line format.
"""
from __future__ import annotations

from typing import Any, Dict, Optional

import numpy as np
import torch

from . import spaces
from .config import STRATEGY_ATR_SLTP, lower_config, obs_layout
from .strategy_plugins import direct_atr_sltp as _atr
from .vec_env import VecFxEnv


class GymFxEnv(spaces.EnvBase):
    metadata = {"render_modes": []}

    def __init__(self, config: Dict[str, Any], data_feed_plugin, broker_plugin, strategy_plugin, preprocessor_plugin,
                 reward_plugin, metrics_plugin):
        self.config = dict(config)
        self.data_feed_plugin = data_feed_plugin
        self.broker_plugin = broker_plugin
        self.strategy_plugin = strategy_plugin
        self.preprocessor_plugin = preprocessor_plugin
        self.reward_plugin = reward_plugin
        self.metrics_plugin = metrics_plugin

        cfg = self.config
        self.initial_cash = float(cfg.get("initial_cash", 10000.0))
        self.position_size = float(cfg.get("position_size", 1.0))
        self.window_size = int(cfg.get("window_size", 32))
        self.price_column = cfg.get("price_column", "CLOSE")
        self.min_equity = float(cfg.get("min_equity", self.initial_cash * 0.01))

        self.dataframe = self.data_feed_plugin.load_data(cfg)
        if self.dataframe is None or len(self.dataframe) < self.window_size + 2:
            raise ValueError("input data is empty or too short for the configured window")
        if self.price_column not in self.dataframe.columns:
            raise ValueError(f"price_column '{self.price_column}' not found in data")
        self.total_bars = int(len(self.dataframe))

        want = list(cfg.get("feature_columns") or getattr(preprocessor_plugin, "params", {}).get("feature_columns") or [])
        extra = [c for c in want if c in self.dataframe.columns]
        if self.price_column not in extra:
            extra.append(self.price_column)
        build_table = getattr(type(data_feed_plugin), "build_table", None)
        if build_table is None:
            from .data_feed_plugins.default_data_feed import Plugin as _Feed
            build_table = _Feed.build_table
        self._table, self._columns, self._minutes = build_table(self.dataframe, extra_columns=extra)
        self._fxcfg = lower_config(cfg, broker_plugin=broker_plugin, strategy_plugin=strategy_plugin,
                                   preprocessor_plugin=preprocessor_plugin, reward_plugin=reward_plugin,
                                   columns=self._columns, num_envs=1,
                                   order_capacity=int(cfg.get("order_capacity", 256)))

        mes = cfg.get("max_episode_steps")
        if mes is not None and (isinstance(mes, bool) or int(mes) != mes or int(mes) < 1):
            raise ValueError(f"max_episode_steps must be a positive integer, got {mes!r}")
        self.max_episode_steps = None if mes is None else int(mes)

        self.action_space_mode = str(cfg.get("action_space_mode", "discrete")).lower()
        if self.action_space_mode == "continuous":
            self.action_space = spaces.Box(low=-1.0, high=1.0, shape=(1,), dtype=np.float32)
            self.continuous_action_threshold = float(cfg.get("continuous_action_threshold", 0.33))
        else:
            self.action_space = spaces.Discrete(3)
            self.continuous_action_threshold = None
        self._layout = obs_layout(self._fxcfg)
        box = {}
        for k, (_, shape) in self._layout.items():
            lo, hi = (-1.0, 1.0) if k == "position" else ((0.0, 1.0) if k == "steps_remaining_norm" else (-np.inf, np.inf))
            box[k] = spaces.Box(low=lo, high=hi, shape=tuple(shape), dtype=np.float32)
        self.observation_space = spaces.Dict(box)

        self._vec: Optional[VecFxEnv] = None
        self._started = False
        self._terminated = False
        self._closed_analyzers = None
        self._last_equity = self.initial_cash   # bridge.equity survives close() in the reference (app/env.py:258-262)
        self._np_random = np.random.default_rng()

    # ------------------------------------------------------------------ Gymnasium API
    def reset(self, *, seed: Optional[int] = None, options: Optional[Dict[str, Any]] = None):
        try:
            super().reset(seed=seed)
        except TypeError:  # pragma: no cover
            pass
        if seed is not None:
            self._np_random = np.random.default_rng(seed)  # unused by the dynamics, as in the reference
        if self._vec is None:
            self._vec = VecFxEnv(self._fxcfg, [self._table], [self._minutes])
            if _atr._AUDIT_PATH and self._fxcfg.strategy == STRATEGY_ATR_SLTP:
                self._vec.set_bracket_audit(4)  # at most one record per step, drained after every step
            if self.max_episode_steps is not None:
                self._vec.set_time_limit(self.max_episode_steps)
        obs, _ = self._vec.reset(torch.zeros(1, dtype=torch.int64))
        self._started = True
        self._terminated = False
        info = self._make_info()
        info.pop("_pnl")
        self._last_equity = info["equity"]
        return self._split(obs.cpu().numpy()[0]), info

    def step(self, action):
        if not self._started:
            raise RuntimeError("Call reset() before step().")
        was_terminated = self._terminated
        a = torch.tensor([self._host_action(action)], dtype=self._vec.action_dtype, device=self._vec.device)
        obs, _, term, trunc, _ = self._vec.step(a)
        if self._vec._audit is not None:
            self._emit_audit()
        reward = float(self._vec.reward64[0])          # fp64, like the reference's Python float
        terminated, truncated = bool(term[0]), bool(trunc[0])
        self._terminated = terminated or truncated  # the episode is over either way
        info = self._make_info()
        pnl = info.pop("_pnl")
        self._last_equity = info["equity"]
        if not was_terminated:  # a step on an already terminated env returns the bare _make_info() (app/env.py:137-138)
            info.update(reward=reward, pnl=pnl, trade_cost=0.0)  # trade_cost is always 0.0 (App. B #7)
        return self._split(obs[0].cpu().numpy()), reward, terminated, truncated, info

    def render(self):
        return None

    def close(self):
        if self._vec is not None:
            if self._started:
                self._closed_analyzers = self._vec.analyzers(0)  # run over: the analyzers become visible (see summary())
            self._vec.close()
            self._vec = None
        self._started = False

    # ------------------------------------------------------------------ helpers
    def _host_action(self, action):
        """Only makes the value representable; the {0,1,2} coercion itself happens in the kernel (fx_core.cuh)."""
        if self.action_space_mode == "continuous":
            try:
                return float(np.asarray(action).reshape(-1)[0])
            except Exception:
                return 0.0
        try:
            a = int(action)
        except Exception:
            a = 0
        return a if -2**31 <= a < 2**31 else 0

    def _emit_audit(self):
        """_audit_emit (strategy_plugins/direct_atr_sltp.py:35-45) for the records of the last step."""
        r = self._vec.bracket_audit()
        if r["kind"].numel() and _atr._AUDIT_PATH:
            cols = [r[k].tolist() for k in ("kind", "entry", "stop", "limit", "size", "atr")]
            _atr.audit_append(_atr._AUDIT_PATH, "".join(_atr.audit_line(*rec) for rec in zip(*cols)))

    def _split(self, row: np.ndarray) -> Dict[str, np.ndarray]:
        return {k: row[off:off + int(np.prod(shape))].reshape(shape).copy() for k, (off, shape) in self._layout.items()}

    def _make_info(self) -> Dict[str, Any]:
        i = self._vec.info()
        eq, prev = float(i["equity"][0]), float(i["prev_equity"][0])
        return {"equity": eq, "position": int(i["position"][0]), "price": float(i["price"][0]),
                "bar_index": int(i["bar_index"][0]), "total_bars": self.total_bars, "trades": int(i["trades"][0]),
                "commission_paid": float(i["commission_paid"][0]), "_pnl": eq - prev}

    def summary(self) -> Dict[str, Any]:
        """app/env.py:256-271.  The reference sees its analyzers only once cerebro.run() has returned -- i.e. after the
        episode terminated (data exhausted / broke) or after close() -- and an empty dict before (SURVEY App. B #12);
        the same rule is kept here (an episode cut by max_episode_steps counts as ended), with the analyzer results coming from the step kernel's per-env statistics."""
        final = float(self._vec.info()["equity"][0]) if self._vec is not None else self._last_equity
        analyzers: Dict[str, Any] = {}
        if self._vec is not None and self._terminated:
            analyzers = self._vec.analyzers(0)
        elif self._vec is None and self._closed_analyzers is not None:
            analyzers = self._closed_analyzers
        return self.metrics_plugin.summarize(initial_cash=self.initial_cash, final_equity=final, analyzers=analyzers,
                                             config=self.config)
