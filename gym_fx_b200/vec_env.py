"""
VecFxEnv -- N lock-stepped gym-fx environments on one GPU, torch tensors in and out, no host round trip.

Semantics per env are those of the reference's GymFxEnv.reset/step (app/env.py:102-172); a step of all N envs is ONE
launch of the fused sm_90a kernel in libfxenv.so, a batch of K steps with known actions ONE persistent launch.  torch is used only for device memory and streams.
"""
from __future__ import annotations

import ctypes as C
from typing import Any, Dict, Optional, Sequence

import numpy as np
import torch

from . import _native
from .config import FxConfig, env_params_table, obs_dim, obs_layout


class VecFxEnv:
    """
    cfg      FxConfig from gym_fx_b200.config.lower_config (num_envs, plugin selection and parameters)
    candles  one float64 [T, n_cols] array per currency pair (env i trades pair i % num_pairs)
    minutes  optional int64 [T] minutes-since-epoch per pair (ATR session filter)
    """

    def __init__(self, cfg: FxConfig, candles: Sequence[np.ndarray], minutes: Optional[Sequence[np.ndarray]] = None,
                 device: Optional[torch.device | str | int] = None):
        if not torch.cuda.is_available():
            raise _native.FxEnvError("VecFxEnv needs a CUDA device (libfxenv.so has no CPU path)")
        self.L = _native.load()
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if self.device.type != "cuda":
            raise _native.FxEnvError("VecFxEnv device must be a CUDA device")
        self.cfg = cfg
        self.num_envs = int(cfg.num_envs)
        self.obs_dim = int(obs_dim(cfg))
        self.layout = obs_layout(cfg)
        if len(candles) != cfg.num_pairs:
            raise ValueError(f"expected {cfg.num_pairs} candle tables, got {len(candles)}")
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            rc = self.L.fxenv_create(C.byref(cfg), C.byref(self._h))
            _native.check(self.L, None, rc, "fxenv_create")
            assert self.L.fxenv_obs_dim(self._h) == self.obs_dim
            self.total_rows = []
            for p, tab in enumerate(candles):
                tab = np.ascontiguousarray(tab, dtype=np.float64)
                if tab.ndim != 2 or tab.shape[1] != cfg.n_cols:
                    raise ValueError(f"candle table {p} must be [T, {cfg.n_cols}]")
                m = None if minutes is None or minutes[p] is None else np.ascontiguousarray(minutes[p], np.int64)
                rc = self.L.fxenv_load_candles(self._h, p, tab.ctypes.data, tab.shape[0],
                                               None if m is None else m.ctypes.data)
                _native.check(self.L, self._h, rc, "fxenv_load_candles")
                self.total_rows.append(tab.shape[0])
        N, D, dev = self.num_envs, self.obs_dim, self.device
        self.obs = torch.empty((N, D), dtype=torch.float32, device=dev)
        self.reward = torch.empty(N, dtype=torch.float32, device=dev)
        self.reward64 = torch.empty(N, dtype=torch.float64, device=dev)
        self.terminated = torch.empty(N, dtype=torch.uint8, device=dev)
        self.truncated = torch.zeros(N, dtype=torch.bool, device=dev)  # always False (app/env.py:158) without a time limit
        self._term_bool = None  # bool [N] split of the codes while truncation is on (set_time_limit)
        self._info_ptrs = _native.FxInfoPtrs()
        self.L.fxenv_get_info(self._h, C.byref(self._info_ptrs))
        self._info_views: Dict[str, torch.Tensor] = {}
        self.action_dtype = torch.float32 if cfg.action_mode == 1 else torch.int32
        self._policies: list = []
        self._audit = None  # (ring [N, capacity, 8], written [N], read cursor [N]) while the bracket audit is on
        self.action_repeat = (1, False)  # (k, hold): set_action_repeat
        self.time_limit = (0, False)  # (max_steps, truncate_window): set_time_limit
        self.env_params: Optional[np.ndarray] = None  # float64 [N, 7] host copy of the per-env table (set_env_params)

    # ------------------------------------------------------------------ lifecycle
    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            # the info tensors are zero-copy views of the library's state slab, which fxenv_destroy frees: drop the cached
            # ones (views a caller still holds become invalid, like any tensor handed out by info() -- clone to keep)
            self._info_views.clear()
            self._audit = None
            for pol in list(getattr(self, "_policies", [])):   # policies hold device buffers tied to this handle
                pol.close()
            self.L.fxenv_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _set(self, fn: str, *args):
        """Call the handle setter `fn` of the library on the handle's device: ValueError with the library's message when
        it rejects the arguments (FXENV_E_INVALID), FxEnvError on any other failure."""
        with torch.cuda.device(self.device):
            rc = getattr(self.L, fn)(self._h, *args)
        if rc == -1:
            raise ValueError(self.L.fxenv_last_error(self._h).decode())
        _native.check(self.L, self._h, rc, fn)

    # ------------------------------------------------------------------ Gym-style API
    def reset(self, start_bars: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None):
        """-> (obs [N, D] float32, info).  start_bars: int64 [N] first table row of each env's episode window."""
        sb = mk = None
        if start_bars is not None:
            sb = torch.as_tensor(start_bars, dtype=torch.int64, device=self.device).contiguous().reshape(-1)
            if sb.numel() != self.num_envs:
                raise ValueError(f"start_bars must have {self.num_envs} elements, got {sb.numel()}")
        if mask is not None:
            mk = torch.as_tensor(mask, device=self.device).to(torch.uint8).contiguous().reshape(-1)
            if mk.numel() != self.num_envs:
                raise ValueError(f"mask must have {self.num_envs} elements, got {mk.numel()}")
        rc = self.L.fxenv_reset(self._h, None if sb is None else sb.data_ptr(), None if mk is None else mk.data_ptr(),
                                self._stream())
        _native.check(self.L, self._h, rc, "fxenv_reset")
        rc = self.L.fxenv_observe(self._h, self.obs.data_ptr(), self._stream())
        _native.check(self.L, self._h, rc, "fxenv_observe")
        return self.obs, self.info()

    def step(self, actions: torch.Tensor, out_obs: Optional[torch.Tensor] = None):
        """-> (obs, reward float32 [N], terminated bool [N], truncated bool [N], info).
        One step is one decision: with an action repeat k > 1 (set_action_repeat) it runs up to k bars.
        truncated is all False unless a time limit is set (set_time_limit); terminated and truncated are never both True.
        The returned tensors are views of buffers that the next step() overwrites."""
        a = actions
        if a.dtype != self.action_dtype or a.device != self.device or not a.is_contiguous():
            a = a.to(device=self.device, dtype=self.action_dtype).contiguous()
        a = a.reshape(-1)
        if a.numel() != self.num_envs:
            raise ValueError(f"expected {self.num_envs} actions")
        obs = self.obs
        if out_obs is not None:
            self._check("out_obs", out_obs, torch.float32, (self.num_envs, self.obs_dim))
            obs = out_obs
        rc = self.L.fxenv_step(self._h, a.data_ptr(), obs.data_ptr(), self.reward.data_ptr(),
                               self.terminated.data_ptr(), self.reward64.data_ptr(), self._stream())
        _native.check(self.L, self._h, rc, "fxenv_step")
        if self._term_bool is None:
            return obs, self.reward, self.terminated.view(torch.bool), self.truncated, self.info()
        # truncation on: self.terminated holds the FXENV_DONE_* codes
        torch.eq(self.terminated, _native.DONE_TERMINATED, out=self._term_bool)
        torch.eq(self.terminated, _native.DONE_TRUNCATED, out=self.truncated)
        return obs, self.reward, self._term_bool, self.truncated, self.info()

    # ---- argument checks of the raw-pointer calls: a wrong dtype / shape / device would be read as garbage or fault
    def _check(self, name: str, t: torch.Tensor, dtype: torch.dtype, shape, host: bool = False):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f"{name} must be a torch.Tensor")
        if t.dtype != dtype:
            raise ValueError(f"{name} must be {dtype}, got {t.dtype}")
        if tuple(t.shape) != tuple(shape):
            raise ValueError(f"{name} must have shape {tuple(shape)}, got {tuple(t.shape)}")
        if not t.is_contiguous():
            raise ValueError(f"{name} must be contiguous")
        if host:
            if t.device.type != "cpu":
                raise ValueError(f"{name} must be a host (ideally pinned) tensor")
        elif t.device != self.device:
            raise ValueError(f"{name} must live on {self.device}, got {t.device}")

    def _check_batch(self, actions, obs_ring, rewards, terminated):
        if actions.dim() != 2:
            raise ValueError("actions must be [K, num_envs]")
        K, N, D = int(actions.shape[0]), self.num_envs, self.obs_dim
        if K < 1:
            raise ValueError("step_many needs at least one step")
        self._check("actions", actions, self.action_dtype, (K, N))
        if obs_ring.dim() != 3 or obs_ring.shape[0] < 1:
            raise ValueError("obs_ring must be [slots, num_envs, obs_dim] with slots >= 1")
        self._check("obs_ring", obs_ring, torch.float32, (int(obs_ring.shape[0]), N, D))
        self._check("rewards", rewards, torch.float32, (K, N))
        self._check("terminated", terminated, torch.uint8, (K, N))
        return K

    def step_many(self, actions: torch.Tensor, obs_ring: torch.Tensor, rewards: torch.Tensor, terminated: torch.Tensor):
        """K consecutive steps with all actions supplied up front (replay / random / scripted drivers); identical results
        to K calls of step().  A step is a decision (up to k bars with set_action_repeat).  actions [K, N] (int32, or float32 in continuous mode); obs_ring float32 [slots, N, D]
        (step k writes slot k % slots); rewards float32 [K, N]; terminated uint8 [K, N]: 0 / 1, or with a time limit
        (set_time_limit) the codes 0, 1 = terminated, 2 = truncated.  The library runs the batch as one
        persistent launch or as a cached CUDA graph of single steps (`step_many_engine`)."""
        K = self._check_batch(actions, obs_ring, rewards, terminated)
        rc = self.L.fxenv_step_many(self._h, K, actions.data_ptr(), obs_ring.data_ptr(), int(obs_ring.shape[0]),
                                    rewards.data_ptr(), terminated.data_ptr(), self._stream())
        _native.check(self.L, self._h, rc, "fxenv_step_many")

    def plan_step_many(self, actions: torch.Tensor, obs_ring: torch.Tensor, rewards: torch.Tensor,
                       terminated: torch.Tensor):
        """Validate a step_many argument set ONCE and return a zero-argument callable that enqueues the batch on the
        current stream with a single C call (for loops that replay the same buffers: the checks and the Python attribute
        lookups stay out of the hot loop).  The tensors must stay alive and unchanged in place while the plan is used."""
        K = self._check_batch(actions, obs_ring, rewards, terminated)
        fn, h, check = self.L.fxenv_step_many, self._h, _native.check
        args = (K, actions.data_ptr(), obs_ring.data_ptr(), int(obs_ring.shape[0]), rewards.data_ptr(),
                terminated.data_ptr())
        keep = (actions, obs_ring, rewards, terminated)
        stream_of = self._stream

        def launch(_keep=keep):
            rc = fn(h, *args, stream_of())
            if rc:
                check(self.L, h, rc, "fxenv_step_many")

        return launch

    def step_host(self, actions_host: torch.Tensor, obs_host: torch.Tensor, reward_host: torch.Tensor,
                  terminated_host: torch.Tensor):
        """Reference-facing call with (pinned) HOST tensors: H2D actions, one step (one decision: up to k bars with
        set_action_repeat), D2H results, synchronous."""
        N, D = self.num_envs, self.obs_dim
        self._check("actions_host", actions_host, self.action_dtype, (N,), host=True)
        self._check("obs_host", obs_host, torch.float32, (N, D), host=True)
        self._check("reward_host", reward_host, torch.float32, (N,), host=True)
        self._check("terminated_host", terminated_host, torch.uint8, (N,), host=True)
        rc = self.L.fxenv_step_host(self._h, actions_host.data_ptr(), obs_host.data_ptr(), reward_host.data_ptr(),
                                    terminated_host.data_ptr())
        _native.check(self.L, self._h, rc, "fxenv_step_host")

    # ------------------------------------------------------------------ info / state
    def _view(self, name: str) -> torch.Tensor:
        v = self._info_views.get(name)
        if v is None:
            ptr = getattr(self._info_ptrs, name)
            dt = getattr(torch, _native.INFO_DTYPES[name])
            v = _tensor_from_ptr(ptr, self.num_envs, dt, self.device)
            self._info_views[name] = v
        return v

    def info(self) -> Dict[str, torch.Tensor]:
        """Zero-copy views of the device-side info columns (app/env.py:244-254,162-166)."""
        return _LazyInfo(self)

    def obs_dict(self, obs: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
        """Split flat rows into the reference's Dict observation (views)."""
        o = self.obs if obs is None else obs
        return {k: o[:, off:off + int(np.prod(shape))].reshape((o.shape[0],) + tuple(shape))
                for k, (off, shape) in self.layout.items()}

    def run_stats(self) -> torch.Tensor:
        """float64 [N, 12] view of the per-env analyzer state (include/fxenv.h FXENV_RS_*)."""
        v = self._info_views.get("run_stats")
        if v is None:
            v = _tensor_from_ptr(self._info_ptrs.run_stats, self.num_envs * _native.RUN_STATS, torch.float64, self.device)
            v = v.view(self.num_envs, _native.RUN_STATS)
            self._info_views["run_stats"] = v
        return v

    def summary(self) -> Dict[str, Any]:
        """Per-env end-of-run summary as device tensors, plus fleet aggregates: the fields of GymFxEnv.summary()
        (app/env.py:256-271 -> metrics_plugins/default_metrics.py:48-60).  The analyzer-derived ones (max drawdown,
        trades won / lost, average trade pnl, SQN) are tracked inside the step kernel -- what backtrader's DrawDown /
        TradeAnalyzer / SQN analyzers would report if the run ended now; NaN where the reference reports None.
        `sharpe_ratio` (SharpeRatio over calendar days) is not tracked and stays None."""
        i = self.info()
        R = _native.RS
        rs = self.run_stats()
        ic = float(self.cfg.initial_cash)
        eq = i["equity"]
        ret = eq / ic - 1.0 if ic else torch.zeros_like(eq)
        closed = i["trades"].double()
        nan = torch.full_like(closed, float("nan"))
        avg = torch.where(closed > 0, rs[:, R["pnl_net"]] / closed.clamp(min=1.0), nan)
        sqn = self._sqn(rs[:, R["pnl_net"]], rs[:, R["pnl_sq"]], closed)
        return {
            "initial_cash": ic, "final_equity": eq, "total_return": ret,
            "max_drawdown_pct": rs[:, R["dd_max_pct"]], "max_drawdown_money": rs[:, R["dd_max_money"]],
            "sharpe_ratio": None, "sqn": sqn,
            "trades_total": rs[:, R["opened"]].to(torch.int64), "trades_won": rs[:, R["won"]].to(torch.int64),
            "trades_lost": rs[:, R["lost"]].to(torch.int64), "trades_closed": i["trades"], "avg_trade_pnl": avg,
            "commission_paid": i["commission_paid"], "position": i["position"], "bar_index": i["bar_index"],
            "mean_total_return": float(ret.mean()), "min_total_return": float(ret.min()),
            "max_total_return": float(ret.max()), "mean_trades": float(closed.mean()),
            "worst_max_drawdown_pct": float(rs[:, R["dd_max_pct"]].max()),
            "fleet_win_rate": float(rs[:, R["won"]].sum() / closed.sum().clamp(min=1.0)),
            "order_overflow_envs": int((i["flags"] & 16).ne(0).sum()),
        }

    @staticmethod
    def _sqn(s1: torch.Tensor, s2: torch.Tensor, n: torch.Tensor) -> torch.Tensor:
        """backtrader's SQN = sqrt(n) * mean / population std of the closed trades' net pnl, from their sum and sum of
        squares; 0 for n <= 1 and NaN (the reference's None) when all trades had the same pnl (std == 0)."""
        nn = n.clamp(min=1.0)
        mean = s1 / nn
        ex2 = s2 / nn
        var = ex2 - mean * mean
        degenerate = var <= 1e-12 * ex2          # rounding noise of the subtraction, not a variance
        sd = torch.sqrt(var.clamp(min=0.0))
        sqn = torch.sqrt(nn) * mean / torch.where(degenerate, torch.ones_like(sd), sd)
        sqn = torch.where(degenerate, torch.full_like(sqn, float("nan")), sqn)
        return torch.where(n > 1, sqn, torch.zeros_like(sqn))

    def analyzers(self, env: int = 0) -> Dict[str, Any]:
        """The analyzer results of ONE env in the shape of backtrader's get_analysis() dicts, as GymFxEnv.summary()
        hands them to the metrics plugin (app/env.py:258-265): trades / drawdown / sqn / sharpe / time_return."""
        R = _native.RS
        rs = self.run_stats()[env].cpu().numpy()
        closed = int(self.info()["trades"][env])
        trades: Dict[str, Any] = {"total": {"total": int(rs[R["opened"]]), "open": int(rs[R["opened"]]) - closed,
                                            "closed": closed}}
        if closed:
            trades.update(won={"total": int(rs[R["won"]])}, lost={"total": int(rs[R["lost"]])},
                          pnl={"net": {"total": float(rs[R["pnl_net"]]), "average": float(rs[R["pnl_net"]]) / closed}})
        if closed > 1:
            v = float(self._sqn(torch.tensor([rs[R["pnl_net"]]], dtype=torch.float64), torch.tensor([rs[R["pnl_sq"]]], dtype=torch.float64),
                                torch.tensor([float(closed)], dtype=torch.float64))[0])
            sqn = None if v != v else v
        else:
            sqn = 0
        return {"trades": trades, "sqn": {"sqn": sqn, "trades": closed}, "sharpe": {}, "time_return": {},
                "drawdown": {"max": {"drawdown": float(rs[R["dd_max_pct"]]), "moneydown": float(rs[R["dd_max_money"]])}}}

    # ------------------------------------------------------------------ episode starts / records
    def set_episode_starts(self, lo, hi=None, seed: int = 0):
        """Draw the start bar of every new episode -- each auto-reset, and reset() without start_bars -- uniformly from the
        inclusive range [lo_i, hi_i] of rows of env i's table, by a counter-based rule of (seed, env, episode number):
        reproducible, and the same in snapshots (include/fxenv.h fxenv_set_reset_starts).  lo / hi: ints (every env) or
        int [N] arrays; with several pairs of different lengths use arrays.  set_episode_starts(None) clears the ranges:
        an episode then restarts at its current start, as without them."""
        N = self.num_envs
        if lo is None:
            if hi is not None:
                raise ValueError("hi must be None when lo is None")
            lo_a = hi_a = None
        else:
            if hi is None:
                raise ValueError("hi is required with lo")
            lo_a, hi_a = (np.ascontiguousarray(np.broadcast_to(np.asarray(v), (N,)), dtype=np.int64) if np.ndim(v) == 0
                          else np.ascontiguousarray(np.asarray(v), dtype=np.int64) for v in (lo, hi))
            for name, v, a in (("lo", lo, lo_a), ("hi", hi, hi_a)):
                if a.shape != (N,):
                    raise ValueError(f"{name} must be a scalar or have {N} elements, got shape {np.shape(v)}")
                if not np.array_equal(a, np.broadcast_to(np.asarray(v), (N,))):
                    raise ValueError(f"{name} must hold integers")
            T = np.asarray([self.total_rows[i % len(self.total_rows)] for i in range(N)], np.int64)
            bad = np.nonzero((lo_a < 0) | (lo_a > hi_a) | (hi_a > T - 1))[0]
            if bad.size:
                i = int(bad[0])
                raise ValueError(f"start range of env {i} is [{lo_a[i]}, {hi_a[i]}]; it must satisfy 0 <= lo <= hi <= "
                                 f"{T[i] - 1} (rows of its table - 1)")
        seed = int(seed)
        if not 0 <= seed < 2**64:
            raise ValueError("seed must be in [0, 2**64)")
        self._set("fxenv_set_reset_starts", None if lo_a is None else lo_a.ctypes.data,
                  None if hi_a is None else hi_a.ctypes.data, seed)

    def _episode_views(self):
        v = self._info_views.get("episodes")
        if v is None:
            p = _native.FxEpisodePtrs()
            _native.check(self.L, self._h, self.L.fxenv_get_episode_info(self._h, C.byref(p)), "fxenv_get_episode_info")
            N, E = self.num_envs, _native.EPISODE_STATS
            v = (_tensor_from_ptr(p.start, N, torch.int64, self.device), _tensor_from_ptr(p.episodes_done, N, torch.int32, self.device),
                 _tensor_from_ptr(p.last_episode, N * E, torch.float64, self.device).view(N, E))
            self._info_views["episodes"] = v
        return v

    def episode_stats(self) -> Dict[str, Any]:
        """The record of each env's last finished episode (latched when a reset -- auto or explicit -- ended it), as device
        tensors: what RecordEpisodeStatistics / GymFxEnv.summary() would report for it.  `episodes_done` counts the
        records (0: nothing recorded yet, the fields are then 0); `start` is the first bar of the CURRENT episode,
        `episode_start` that of the recorded one.  end_flags: FX_FLAG_TERMINATED (2) | EXHAUSTED (4) | BROKE (8) |
        TRUNCATED (64) bits, 0 = cut short by a reset.  total_return, avg_trade_pnl (NaN without closed trades) and sqn are derived as in summary()."""
        start, done, last = self._episode_views()
        E = _native.EP
        col = {k: last[:, j] for k, j in E.items()}
        ic = float(self.cfg.initial_cash)
        closed = col["closed"]
        nan = torch.full_like(closed, float("nan"))
        return {
            "start": start, "episodes_done": done, "episode_start": col["start"].to(torch.int64),
            "bars": col["bars"].to(torch.int32), "final_equity": col["equity"],
            "total_return": col["equity"] / ic - 1.0 if ic else torch.zeros_like(col["equity"]),
            "commission_paid": col["commission"], "end_flags": col["end_flags"].to(torch.int32),
            "max_drawdown_pct": col["dd_max_pct"], "max_drawdown_money": col["dd_max_money"],
            "pnl_net": col["pnl_net"], "pnl_sq": col["pnl_sq"],
            "trades_total": col["opened"].to(torch.int64), "trades_closed": closed.to(torch.int64),
            "trades_won": col["won"].to(torch.int64), "trades_lost": col["lost"].to(torch.int64),
            "avg_trade_pnl": torch.where(closed > 0, col["pnl_net"] / closed.clamp(min=1.0), nan),
            "sqn": self._sqn(col["pnl_net"], col["pnl_sq"], closed), "episode_index": col["index"].to(torch.int64),
        }

    # ------------------------------------------------------------------ bracket audit
    def set_bracket_audit(self, capacity: int):
        """Turn the ATR strategy's bracket audit on with a ring of `capacity` records per env (the counters and the read
        cursors restart at 0), or off with 0 (include/fxenv.h fxenv_set_bracket_audit).  Accepted for every strategy;
        only direct_atr_sltp writes records.  Synchronous."""
        capacity = int(capacity)
        if not 0 <= capacity < 2**31:
            raise ValueError(f"bracket audit capacity must be in [0, 2**31), got {capacity}")
        self._set("fxenv_set_bracket_audit", capacity)
        self._audit = None
        if capacity:
            p = _native.FxAuditPtrs()
            _native.check(self.L, self._h, self.L.fxenv_get_bracket_audit(self._h, C.byref(p)), "fxenv_get_bracket_audit")
            N, F = self.num_envs, _native.AU_FIELDS
            ring = _tensor_from_ptr(p.records, N * p.capacity * F, torch.float64, self.device).view(N, p.capacity, F)
            written = _tensor_from_ptr(p.written, N, torch.int64, self.device)
            self._audit = (ring, written, torch.zeros(N, dtype=torch.int64, device=self.device))

    def bracket_audit(self) -> Dict[str, torch.Tensor]:
        """Drain the audit rings: every record written since the last drain, as device tensors ordered by env and then
        by record -- env, bar (table row of the signal bar), episode (the episode's k), kind (1 long_bracket, 2
        short_bracket, 3 session_force_close), entry, stop, limit, size, atr (NaN stop / limit / atr for a force-close) --
        plus dropped [N]: records overwritten in the ring before they could be drained.  Ordered on the current stream
        (torch ops; sizing the result waits for the counters).  The log must be on (set_bracket_audit)."""
        if getattr(self, "_audit", None) is None:
            raise _native.FxEnvError("the bracket audit is off: call set_bracket_audit(capacity) first")
        ring, written, cursor = self._audit
        N, cap = self.num_envs, ring.shape[1]
        w = written.clone()
        first = torch.maximum(cursor, w - cap)
        dropped = first - cursor
        count = w - first
        env = torch.repeat_interleave(torch.arange(N, device=self.device), count)
        offset = torch.cumsum(count, 0) - count
        idx = first[env] + (torch.arange(env.numel(), device=self.device) - offset[env])
        rec = ring[env, idx % cap]
        cursor.copy_(w)
        A = _native.AU
        out = {"env": env, "bar": rec[:, A["bar"]].to(torch.int64), "episode": rec[:, A["episode"]].to(torch.int64),
               "kind": rec[:, A["kind"]].to(torch.int32)}
        for k in ("entry", "stop", "limit", "size", "atr"):
            out[k] = rec[:, A[k]]
        out["dropped"] = dropped
        return out

    # ------------------------------------------------------------------ action repeat
    def set_action_repeat(self, k: int, hold: bool = False):
        """One decision per k bars (1 <= k <= 256; 1 = off, the default): every later step(), step_many() decision,
        step_host() and rollout() decision runs up to k bars.  hold=False applies the action on each of the k bars
        (frame skip); hold=True applies it on the first bar only and holds (action 0) on the others.  A step stops early
        at a bar that terminates the episode, and a terminated env's step is its auto-reset step alone.  The observation
        is that after the step's last bar, the reward the float64 sum of the bars' rewards (include/fxenv.h
        fxenv_set_action_repeat).  A setting of the handle, not of the env state: snapshots and reset() keep it."""
        if isinstance(k, bool) or int(k) != k:
            raise ValueError(f"action repeat must be an integer, got {k!r}")
        k = int(k)
        if not 1 <= k <= _native.MAX_REPEAT:
            raise ValueError(f"action repeat must be in [1, {_native.MAX_REPEAT}], got {k}")
        self._set("fxenv_set_action_repeat", k, _native.REPEAT_HOLD if hold else 0)
        self.action_repeat = (k, bool(hold))

    # ------------------------------------------------------------------ time limit / truncation
    def set_time_limit(self, max_steps: int, truncate_window: bool = False):
        """End every episode after `max_steps` decisions as a truncation (Gymnasium's max_episode_steps; 0 = no limit,
        the default), and with truncate_window=True report the end of the episode window (episode_bars or the end of the
        table) as a truncation instead of a termination.  A decision is one step(), step_many() decision or rollout()
        decision; the first step of an episode is decision 1, an auto-reset step does not count.  A step that terminates
        (broke) reports a termination only.  While either is set, step() returns real truncated flags and the uint8
        outputs of step_many / step_host / rollout (done) carry codes 0, 1 = terminated, 2 = truncated.  Every running
        episode starts counting afresh.  A setting of the handle (include/fxenv.h fxenv_set_time_limit): snapshots and
        reset() keep it; each env's decision count is env state.  Synchronous."""
        if isinstance(max_steps, bool) or int(max_steps) != max_steps:
            raise ValueError(f"time limit must be an integer, got {max_steps!r}")
        max_steps = int(max_steps)
        if not 0 <= max_steps < 2**31:
            raise ValueError(f"time limit must be in [0, 2**31), got {max_steps}")
        if not isinstance(truncate_window, bool):
            raise ValueError(f"truncate_window must be a bool, got {truncate_window!r}")
        self._set("fxenv_set_time_limit", max_steps, _native.TIME_LIMIT_WINDOW if truncate_window else 0)
        self.time_limit = (max_steps, truncate_window)
        if max_steps > 0 or truncate_window:
            if self._term_bool is None:
                self._term_bool = torch.zeros(self.num_envs, dtype=torch.bool, device=self.device)
        else:   # off: back to the zero-overhead views of the 0 / 1 buffer
            self._term_bool = None
            self.truncated.zero_()

    # ------------------------------------------------------------------ per-env broker / strategy parameters
    def set_env_params(self, commission=None, leverage=None, slippage=None, sl_pips=None, tp_pips=None, k_sl=None,
                       k_tp=None):
        """Give each env its own broker costs and bracket settings (include/fxenv.h fxenv_set_env_params): commission,
        leverage and slippage of the broker, sl_pips / tp_pips of direct_fixed_sltp, k_sl / k_tp of direct_atr_sltp.  Each
        argument is a scalar (every env) or an [N] array / tensor; a field left as None keeps the config's value.  With
        every field None (set_env_params(None)) the table is turned off and every env uses the config again.  Fields
        the strategy does not use are ignored.  A setting of the handle: snapshots and reset() keep it.  New values apply
        from the next step on; updating the values while the table stays on keeps the cached step_many / rollout graphs.
        Synchronous.  Bad values (not finite, leverage <= 0, slippage outside [0, 1), a wrong length) raise ValueError
        and leave the table in force as it was.  The host copy of the table in force is `env_params` (None when off)."""
        fields = dict(commission=commission, leverage=leverage, slippage=slippage, sl_pips=sl_pips, tp_pips=tp_pips,
                      k_sl=k_sl, k_tp=k_tp)
        table = None if all(v is None for v in fields.values()) else env_params_table(self.cfg, **fields)
        self._set("fxenv_set_env_params", None if table is None else table.ctypes.data)
        self.env_params = table

    # ------------------------------------------------------------------ closed loop (policy on the device)
    def make_policy(self, weights=None, hidden: Optional[int] = None, separate: Optional[bool] = None,
                    members: Optional[int] = None) -> "FusedPolicy":
        """An actor-critic MLP(obs_dim, hidden, hidden) evaluated by the fused tensor-core kernel (fxenv.h: FxPolicy).
        hidden: 64, 128, 256 or 512; None takes it from the weights (the rows of w1), or 256 without weights.
        separate: separate actor and critic networks instead of one shared body; None takes it from the weights (a
        module with a critic_body, or a dict with w1_v, b1_v, w2_v, b2_v), or False without weights.
        members: a population of that many independent networks of one width and layout, member m acting for the
        envs `policy.member_envs(m)` (num_envs must then be a multiple of 128 * members); `weights` is then a list or
        tuple with one module or dict per member.  None takes len(weights) for a list or tuple, else 1."""
        return FusedPolicy(self, weights, hidden, separate, members)

    def rollout(self, policy: "FusedPolicy", horizon: int, buffers: Optional[Dict[str, torch.Tensor]] = None,
                gumbel: Optional[torch.Tensor] = None, seed: int = 0, noise: Optional[torch.Tensor] = None,
                deterministic: bool = False) -> Dict[str, torch.Tensor]:
        """`horizon` closed-loop steps (policy -> sample -> env.step) from the current state, all on the device: the
        loop of the reference's driver (app/main.py:57-65) with a learned policy.  A step is one policy decision: with an
        action repeat k > 1 (set_action_repeat) the env runs up to k bars between two evaluations.  Returns / fills `buffers`:
        obs [H+1, N, D] (obs[t] is what the policy saw at step t), actions [H, N] (int32, or float32 in continuous mode),
        logp [H, N], value [H+1, N] (value[H] bootstraps), reward [H, N], done uint8 [H, N] (0 / 1, or with a time limit
        the codes 0, 1 = terminated, 2 = truncated: after a truncation at t, obs[t+1] is the final observation of the
        cut episode, value[t+1] its value, and step t+1 the reset step with auto_reset).
        Sampling noise for reproducible rollouts -- discrete mode: gumbel, float32 [H, N, 3] Gumbel(0,1); continuous
        mode: noise, float32 [H, N] standard normal; default: the kernel's counter-based generator seeded with `seed`.
        deterministic: greedy evaluation, the most likely action (argmax of the logits / the Gaussian mean)."""
        H, N, D, dev = int(horizon), self.num_envs, self.obs_dim, self.device
        continuous = self.action_dtype == torch.float32
        b = buffers if buffers is not None else {}
        want = {"obs": ((H + 1, N, D), torch.float32), "actions": ((H, N), self.action_dtype), "logp": ((H, N), torch.float32),
                "value": ((H + 1, N), torch.float32), "reward": ((H, N), torch.float32), "done": ((H, N), torch.uint8)}
        for k, (shape, dt) in want.items():
            if k not in b:
                b[k] = torch.empty(shape, dtype=dt, device=dev)
            elif k == "obs":
                if b[k].dim() != 3 or b[k].shape[0] < 2:
                    raise ValueError("obs must be [slots >= 2, num_envs, obs_dim]")
                self._check("obs", b[k], dt, (int(b[k].shape[0]), N, D))
            else:
                self._check(k, b[k], dt, shape)
        if continuous and gumbel is not None:
            raise ValueError("gumbel noise is for discrete action mode; continuous mode takes `noise` [H, N]")
        if not continuous and noise is not None:
            raise ValueError("noise is for continuous action mode; discrete mode takes `gumbel` [H, N, 3]")
        if gumbel is not None:
            self._check("gumbel", gumbel, torch.float32, (H, N, 3))
        if noise is not None:
            self._check("noise", noise, torch.float32, (H, N))
        eps = noise if continuous else gumbel
        io = _native.FxRollout(H, int(b["obs"].shape[0]), b["obs"].data_ptr(), b["actions"].data_ptr(), b["logp"].data_ptr(),
                               b["value"].data_ptr(), b["reward"].data_ptr(), b["done"].data_ptr(),
                               0 if eps is None else eps.data_ptr(), int(seed) & (2**64 - 1))
        flags = _native.ROLLOUT_GREEDY if deterministic else 0
        rc = self.L.fxenv_rollout_ex(self._h, policy._p, C.byref(io), flags, self._stream())
        _native.check(self.L, self._h, rc, "fxenv_rollout_ex")
        policy._keep = (b, eps)
        return b

    def obs_moments(self, obs: torch.Tensor, shift: torch.Tensor, envs: slice = slice(None)) -> torch.Tensor:
        """Shifted column moments of rollout observations for an observation normalizer (include/fxenv.h
        fxenv_obs_moments): obs float32 [slots, N, D] (a rollout's obs, or a prefix of it), shift float32 [num_pairs, D]
        (the running mean).  Over every slot and the envs of `envs` (a contiguous slice, e.g. a population member's
        policy.member_envs(m)), grouped by pair p = env % num_pairs: float64 [num_pairs, 2, D] with [p, 0] = sum (x -
        shift[p]) and [p, 1] = sum (x - shift[p])^2.  The order of summation depends on the shapes only, so the same
        inputs give the same bits.  Ordered on the current stream."""
        P, N, D = int(self.cfg.num_pairs), self.num_envs, self.obs_dim
        if not isinstance(obs, torch.Tensor) or obs.dim() != 3 or obs.shape[0] < 1:
            raise ValueError(f"obs must be a [slots >= 1, {N}, {D}] tensor")
        self._check("obs", obs, torch.float32, (int(obs.shape[0]), N, D))
        self._check("shift", shift, torch.float32, (P, D))
        if not isinstance(envs, slice) or envs.step not in (None, 1):
            raise ValueError(f"envs must be a contiguous slice, got {envs!r}")
        e0, e1, _ = envs.indices(N)
        out = torch.empty((P, 2, D), dtype=torch.float64, device=self.device)
        self._set("fxenv_obs_moments", obs.data_ptr(), int(obs.shape[0]), e0, e1, shift.data_ptr(), out.data_ptr(),
                  self._stream())
        return out

    def return_moments(self, reward: torch.Tensor, done: torch.Tensor, prev_done: torch.Tensor, ret: torch.Tensor,
                       seen: torch.Tensor, gamma: float, shift: float, envs: slice = slice(None)) -> torch.Tensor:
        """Moments of the discounted returns of a rollout for a reward normalizer (include/fxenv.h
        fxenv_return_moments): reward float32 [H, N] and done uint8 [H, N] (a rollout's buffers), prev_done uint8 [N] (the
        done of the step before it).  Over the envs of `envs` (a contiguous slice, e.g. a population member's
        policy.member_envs(m)), whose returns carry over from call to call in ret float64 [W] and seen int32 [W] (W = the
        slice's width; start from zeros and -1), updated in place.  Reset steps are skipped, any done ends the return,
        and an episode begun outside this rollout's reset steps clears it.  Returns float64 [3] = (sum (R - shift),
        sum (R - shift)^2, count) over the slice's scanned steps, in an order that depends on the shapes only.  Ordered on
        the current stream."""
        N = self.num_envs
        if not isinstance(reward, torch.Tensor) or reward.dim() != 2 or reward.shape[0] < 1:
            raise ValueError(f"reward must be a [H >= 1, {N}] tensor")
        H = int(reward.shape[0])
        self._check("reward", reward, torch.float32, (H, N))
        self._check("done", done, torch.uint8, (H, N))
        self._check("prev_done", prev_done, torch.uint8, (N,))
        if not isinstance(envs, slice) or envs.step not in (None, 1):
            raise ValueError(f"envs must be a contiguous slice, got {envs!r}")
        e0, e1, _ = envs.indices(N)
        W = max(e1 - e0, 0)
        self._check("ret", ret, torch.float64, (W,))
        self._check("seen", seen, torch.int32, (W,))
        out = torch.empty(3, dtype=torch.float64, device=self.device)
        self._set("fxenv_return_moments", reward.data_ptr(), done.data_ptr(), prev_done.data_ptr(), H, e0, e1,
                  float(gamma), float(shift), ret.data_ptr(), seen.data_ptr(), out.data_ptr(), self._stream())
        return out

    def launch_count(self) -> int:
        return int(self.L.fxenv_launch_count(self._h))

    def step_many_engine(self, n_steps: int) -> str:
        """'persistent' (one launch, per-env dependencies) or 'graph' (CUDA graph of single steps) -- see fxenv.h."""
        return "persistent" if int(self.L.fxenv_step_many_engine(self._h, int(n_steps))) == 1 else "graph"

    def get_state(self) -> bytes:
        n = self.L.fxenv_state_bytes(self._h)
        buf = (C.c_char * n)()
        _native.check(self.L, self._h, self.L.fxenv_get_state(self._h, buf, n), "fxenv_get_state")
        return bytes(buf)

    def set_state(self, blob: bytes):
        _native.check(self.L, self._h, self.L.fxenv_set_state(self._h, blob, len(blob)), "fxenv_set_state")


class _LazyInfo(dict):
    """dict of info tensors materialised on first access (keeps step() free of Python overhead)."""

    KEYS = tuple(_native.INFO_DTYPES)

    def __init__(self, env: VecFxEnv):
        super().__init__()
        self._env = env

    def __missing__(self, key):
        if key == "pnl":
            v = self._env._view("equity") - self._env._view("prev_equity")
        elif key == "reward":
            v = self._env.reward
        elif key in self.KEYS:
            v = self._env._view(key)
        else:
            raise KeyError(key)
        self[key] = v
        return v

    def keys(self):
        return list(self.KEYS) + ["pnl", "reward"]

    def __contains__(self, key):
        return key in self.KEYS or key in ("pnl", "reward")


class _CudaArrayView:
    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (int(ptr), False), "version": 3}


def _tensor_from_ptr(ptr: int, n: int, dtype: torch.dtype, device: torch.device) -> torch.Tensor:
    typestr = {torch.float64: "<f8", torch.int32: "<i4", torch.int64: "<i8", torch.uint8: "|u1"}[dtype]
    with torch.cuda.device(device):
        return torch.as_tensor(_CudaArrayView(ptr, n, typestr), device=device)


class FusedPolicy:
    """Device-resident actor-critic MLP(obs_dim, hidden, hidden) -> 3 logits + value, evaluated between env steps by the
    fused wgmma kernel (gym_fx_b200/csrc/fx_policy.cu).  `set_weights` takes float32 CUDA tensors in torch.nn.Linear
    layout (or a module with .body[0], .body[2], .pi, .v like gym_fx_b200.learner.ActorCritic).
    In continuous action mode the actor is a Gaussian: `pi` is Linear(hidden, 1) (the mean) and a `log_std` tensor of
    shape [1] (dict key "log_std", or the module's .log_std parameter) gives the state-independent log sigma.
    hidden (both layers): 64, 128, 256 or 512.  None takes the width from `weights` (module.body[0].out_features, or the
    rows of weights["w1"]), or HIDDEN = 256 without weights; an explicit width that disagrees with the weights is a
    ValueError.  The width is fixed for the life of the policy (`self.hidden`).
    separate (`self.separate`, fixed too): separate actor and critic networks of the same width (fxenv.h:
    FXENV_POLICY_SEPARATE) -- `body` feeds `pi` and a second trunk `critic_body` feeds `v` (ActorCritic(separate=True));
    a weight dict adds the critic trunk as w1_v, b1_v, w2_v, b2_v.  None takes it from `weights`, or False without
    weights; an explicit value that disagrees with the weights is a ValueError.
    members (`self.members`, fixed too): a population of independent networks of that one width and layout (fxenv.h:
    fxenv_policy_create_ex3); member m acts for the envs `member_envs(m)` and gives there exactly what a single policy
    with its weights gives.  Weights come as a list or tuple of one module or dict per member (`set_weights`), or one
    member at a time (`set_member_weights`); members whose weights disagree on the width or layout are a ValueError.
    Observation normalizer (fxenv.h: fxenv_policy_set_obs_norm): weights with one -- a module whose `obs_norm` is a
    learner.ObsNormalizer (ActorCritic(obs_norm=True)), or a dict with obs_mean and obs_rstd float32 [num_pairs,
    obs_dim] and obs_clip -- make the kernel normalize the bf16 observation it reads, with the statistics of each env's
    pair; weights without one turn it off.  Every member has one or none."""

    HIDDEN = 256
    CRITIC_KEYS = ("w1_v", "b1_v", "w2_v", "b2_v")   # the critic trunk in a weight dict of a separate policy

    def __init__(self, env: VecFxEnv, weights=None, hidden: Optional[int] = None, separate: Optional[bool] = None,
                 members: Optional[int] = None):
        listed = isinstance(weights, (list, tuple))
        if members is None:
            members = len(weights) if listed else 1
        if isinstance(members, bool) or not isinstance(members, (int, np.integer)) or members < 1:
            raise ValueError(f"members must be an integer >= 1, got {members!r}")
        members = int(members)
        if listed and len(weights) != members:
            raise ValueError(f"{len(weights)} weight sets for a population of {members} members")
        if weights is not None and not listed and members != 1:
            raise ValueError(f"a population of {members} members takes a list of {members} weight sets")
        if members > 1 and env.num_envs % (128 * members):
            raise ValueError(f"num_envs ({env.num_envs}) must be a multiple of 128 x members ({members}): each member "
                             "owns whole 128-env tiles")
        each = None if weights is None else (list(weights) if listed else [weights])
        inferred = None if each is None else self._common(each, self._width_of, "width")
        if hidden is None:
            hidden = self.HIDDEN if inferred is None else inferred
        elif inferred is not None and int(hidden) != inferred:
            raise ValueError(f"hidden={hidden} disagrees with the weights, which are {inferred} wide")
        if int(hidden) not in _native.POLICY_WIDTHS:
            raise ValueError(f"policy width must be one of {_native.POLICY_WIDTHS}, got {hidden}")
        sep = None if each is None else self._common(each, self._separate_of, "layout (shared body or separate trunks)")
        if separate is None:
            separate = bool(sep)
        elif sep is not None and bool(separate) != sep:
            raise ValueError(f"separate={separate} disagrees with the weights, which have "
                             f"{'separate actor and critic trunks' if sep else 'one shared body'}")
        self.env = env
        self.hidden = int(hidden)
        self.separate = bool(separate)
        self.members = members
        self.continuous = env.action_dtype == torch.float32
        self._p = C.c_void_p()
        flags = _native.POLICY_SEPARATE if self.separate else 0
        rc = env.L.fxenv_policy_create_ex3(env._h, self.hidden, flags, self.members, C.byref(self._p))
        _native.check(env.L, env._h, rc, "fxenv_policy_create_ex3")
        self._keep = None
        self._w: Dict[int, Dict[str, torch.Tensor]] = {}
        self._norm_on = [False] * members  # which members' weights came with an observation normalizer
        env._policies.append(self)
        if weights is not None:
            self.set_weights(weights)

    @staticmethod
    def _common(each, of, what):
        """the value `of` gives for every member's weights; members that disagree are a ValueError"""
        vals = [of(w) for w in each]
        if any(v != vals[0] for v in vals):
            raise ValueError(f"the members' weights disagree on the {what}: {vals}")
        return vals[0]

    @staticmethod
    def _width_of(weights) -> int:
        """hidden width of an ActorCritic-like module or a weight dict (the rows of w1)"""
        if isinstance(weights, dict):
            return int(weights["w1"].shape[0])
        return int(weights.body[0].out_features)

    @classmethod
    def _separate_of(cls, weights) -> bool:
        """whether weights hold separate actor and critic trunks (a critic_body, or the w1_v ... keys of a dict)"""
        if isinstance(weights, dict):
            return any(k in weights for k in cls.CRITIC_KEYS)
        return getattr(weights, "critic_body", None) is not None

    def sync_timeouts(self) -> int:
        """Polls of the last rollout's tile hand-over that gave up (0 unless something is broken); synchronises."""
        rc = int(self.env.L.fxenv_policy_sync_timeouts(self._p))
        if rc < 0:
            _native.check(self.env.L, self.env._h, rc, "fxenv_policy_sync_timeouts")
        return rc

    def peek(self, what: str, slot: int = 0) -> torch.Tensor:
        """Copy of an internal device buffer of the policy, for tests and debugging (fxenv_policy_peek), ordered on the
        current stream.  what = "obs16": the bf16 observation copy of `slot` (0 or 1) that the kernel reads,
        [num_envs, k_pad]; "h1": the layer-1 activations of the last evaluation, [num_envs rounded up to 128, hidden]
        (separate: [..., 2 * hidden], the actor's columns first)."""
        code = {"obs16": _native.PEEK_OBS16, "h1": _native.PEEK_H1}.get(what)
        if code is None:
            raise ValueError(f"what must be 'obs16' or 'h1', got {what!r}")
        L, s = self.env.L, self.env._stream()
        n = int(L.fxenv_policy_peek(self._p, code, int(slot), None, 0, s))
        if n < 0:
            _native.check(L, self.env._h, n, "fxenv_policy_peek")
        cols = self.hidden * (2 if self.separate else 1) if what == "h1" else (self.env.obs_dim + 63) // 64 * 64
        out = torch.empty((n // (2 * cols), cols), dtype=torch.int16, device=self.env.device)
        rc = int(L.fxenv_policy_peek(self._p, code, int(slot), out.data_ptr(), n, s))
        if rc < 0:
            _native.check(L, self.env._h, rc, "fxenv_policy_peek")
        return out.view(torch.bfloat16)

    def member_envs(self, m: int) -> slice:
        """The envs member m acts for: [m N / members, (m + 1) N / members) of the handle's N envs."""
        self._check_member(m)
        n = self.env.num_envs // self.members
        return slice(int(m) * n, (int(m) + 1) * n)

    def _check_member(self, m):
        if isinstance(m, bool) or not isinstance(m, (int, np.integer)) or not 0 <= m < self.members:
            raise ValueError(f"member must be an integer in [0, {self.members}), got {m!r}")

    def set_weights(self, weights):
        """New parameters for every member: one module or weight dict, or for a population a list or tuple of one per
        member.  Every set is checked before any is written."""
        each = list(weights) if isinstance(weights, (list, tuple)) else [weights]
        if len(each) != self.members:
            raise ValueError(f"{len(each)} weight sets for a policy of {self.members} member(s)")
        sets = [self._tensors(w) for w in each]
        self._common(sets, lambda ts: "obs_mean" in ts, "observation normalizer (every member has one or none)")
        for m, ts in enumerate(sets):
            self._upload(m, ts)

    def set_member_weights(self, m: int, weights):
        """New parameters for member m only (a module or weight dict of this policy's width and layout); the other
        members keep theirs, and the cached rollout graph stays."""
        self._check_member(m)
        ts = self._tensors(weights)
        on = "obs_mean" in ts
        others = [self._norm_on[k] for k in self._w if k != int(m)]
        if any(o != on for o in others):
            raise ValueError(f"member {m}'s weights {'have an' if on else 'have no'} observation normalizer, unlike the "
                             "other members': every member has one or none")
        self._upload(int(m), ts)

    def _upload(self, m: int, ts: Dict[str, torch.Tensor]):
        w = _native.FxPolicyWeights(*[ts[k].data_ptr() for k in ("w1", "b1", "w2", "b2", "w_pi", "b_pi", "w_v", "b_v")])
        L, s = self.env.L, self.env._stream()
        rc = L.fxenv_policy_set_member_weights(self._p, m, C.byref(w), s)
        _native.check(L, self.env._h, rc, "fxenv_policy_set_member_weights")
        on = "obs_mean" in ts
        rc = L.fxenv_policy_set_obs_norm(self._p, m, ts["obs_mean"].data_ptr() if on else None,
                                         ts["obs_rstd"].data_ptr() if on else None, float(ts["obs_clip"]) if on else 0.0, s)
        _native.check(L, self.env._h, rc, "fxenv_policy_set_obs_norm")
        self._norm_on[m] = on
        self._w[m] = ts  # keep the sources alive until the stream-ordered copies have run

    def _tensors(self, weights) -> Dict[str, torch.Tensor]:
        """float32 device tensors in the FxPolicyWeights layout of this policy, checked against its width and layout"""
        sep = self._separate_of(weights)
        if sep != self.separate:
            raise ValueError("this policy has " + ("separate actor and critic trunks" if self.separate else "one shared body")
                             + ", the weights " + ("have separate trunks" if sep else "have one shared body"))
        if not isinstance(weights, dict):
            m = weights
            weights = {"w1": m.body[0].weight, "b1": m.body[0].bias, "w2": m.body[2].weight, "b2": m.body[2].bias,
                       "w_pi": m.pi.weight, "b_pi": m.pi.bias, "w_v": m.v.weight, "b_v": m.v.bias}
            if self.separate:
                c = m.critic_body
                weights.update({"w1_v": c[0].weight, "b1_v": c[0].bias, "w2_v": c[2].weight, "b2_v": c[2].bias})
            if self.continuous:
                if getattr(m, "log_std", None) is None:
                    raise ValueError("continuous action mode needs a log_std parameter of shape [1] on the module")
                weights["log_std"] = m.log_std
            nm = getattr(m, "obs_norm", None)
            if nm is not None:  # learner.ObsNormalizer: the float32 statistics its forward() uses
                weights.update({"obs_mean": nm.mean32(), "obs_rstd": nm.rstd32(), "obs_clip": nm.clip})
        D, Hd = self.env.obs_dim, self.hidden
        n_pi = 1 if self.continuous else 3
        shapes = {"w1": (Hd, D), "b1": (Hd,), "w2": (Hd, Hd), "b2": (Hd,), "w_pi": (n_pi, Hd), "b_pi": (n_pi,), "w_v": (Hd,),
                  "b_v": (1,)}
        if self.separate:
            shapes.update({"w1_v": (Hd, D), "b1_v": (Hd,), "w2_v": (Hd, Hd), "b2_v": (Hd,)})
        if self.continuous:
            if "log_std" not in weights:
                raise ValueError("continuous action mode needs weights['log_std'] of shape [1]")
            shapes["log_std"] = (1,)
        ts = {}
        for k, shape in shapes.items():
            t = weights[k].detach()
            if k == "w_v":
                t = t.reshape(-1)
            t = t.to(device=self.env.device, dtype=torch.float32).contiguous()
            if tuple(t.shape) != shape:
                raise ValueError(f"{k} must have shape {shape} for this {Hd}-wide policy, got {tuple(t.shape)}")
            ts[k] = t
        if self.continuous:  # FxPolicyWeights.b_pi in continuous mode: {b_mu, log sigma}
            ts["b_pi"] = torch.cat([ts["b_pi"], ts.pop("log_std")])
        if self.separate:  # FxPolicyWeights under FXENV_POLICY_SEPARATE: both trunks stacked, the actor's first
            for k in ("w1", "b1", "w2", "b2"):
                ts[k] = torch.cat([ts[k], ts.pop(k + "_v")])
        given = [k for k in ("obs_mean", "obs_rstd", "obs_clip") if weights.get(k) is not None]
        if given and len(given) != 3:
            raise ValueError(f"an observation normalizer needs obs_mean, obs_rstd and obs_clip, got only {given}")
        if given:
            P = int(self.env.cfg.num_pairs)
            for k in ("obs_mean", "obs_rstd"):
                t = torch.as_tensor(weights[k]).detach().to(device=self.env.device, dtype=torch.float32).contiguous()
                if tuple(t.shape) != (P, D):
                    raise ValueError(f"{k} must have shape {(P, D)} (num_pairs, obs_dim), got {tuple(t.shape)}")
                ts[k] = t
            clip = float(weights["obs_clip"])
            if not clip > 0.0:
                raise ValueError(f"obs_clip must be > 0 (inf allowed), got {clip}")
            ts["obs_clip"] = clip
        return ts

    def close(self):
        if self._p:
            self.env.L.fxenv_policy_destroy(self._p)
            self._p = C.c_void_p()
            if self in self.env._policies:
                self.env._policies.remove(self)

    def __del__(self):
        try:
            if self.env._h:
                self.close()
        except Exception:
            pass
