"""
tests/time_limit_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

TimeLimitOracle: the time limit and truncation of include/fxenv.h (fxenv_set_time_limit) restated around RepeatOracle
(which itself wraps the unchanged C oracle).  The wrapped oracle knows nothing of truncation; this wrapper
  * counts the decisions of each env's episode (a step of an env whose episode is running, whatever number of substeps
    it ran); an auto-reset step does not count, a reset zeroes the count, and so does set_time_limit;
  * after a decision that did not terminate, cuts the episode once the count reaches max_steps (code 2);
  * with the WINDOW rule, reports the oracle's data exhaustion (terminated, EXHAUSTED and not BROKE) as a truncation;
  * treats a cut env as the library treats a terminated one: with auto-reset its next step is the reset step (reward 0,
    code 0), without it every later step gives the observation of the current state, reward 0 and code 2 (1 once
    truncation has been turned off: the outputs are 0 / 1 then, and the cut episode stays over);
  * returns the codes 0 / 1 = terminated / 2 = truncated (0 / 1 only, as the library, while truncation is off), and
    shows FX_FLAG_TRUNCATED in the flags of info() and in the end flags of the episode records.
"""
from __future__ import annotations

import numpy as np

from repeat_oracle import RepeatOracle

FLAG_TERMINATED, FLAG_EXHAUSTED, FLAG_BROKE, FLAG_TRUNCATED = 2, 4, 8, 64
DONE_TERMINATED, DONE_TRUNCATED = 1, 2
CUT_LIMIT, CUT_WINDOW = 1, 2   # how a cut env's episode ended
EP_END_FLAGS = 4               # FXENV_EP_END_FLAGS


class TimeLimitOracle:
    """N oracle envs with an action repeat and a time limit; the surface of RepeatOracle plus set_time_limit."""

    def __init__(self, cfg, candles, minutes=None, k=1, hold=False, audit=False, max_steps=0, window=False):
        self.r = RepeatOracle(cfg, candles, minutes, k=k, hold=hold, audit=audit)
        self.o = self.r.o
        self.cfg, self.N, self.D = cfg, self.r.N, self.r.D
        self.count = np.zeros(self.N, np.int64)   # decisions of the current episode
        self.cut = np.zeros(self.N, np.int8)      # 0, CUT_LIMIT or CUT_WINDOW
        self.set_time_limit(max_steps, window)

    @property
    def substeps(self):
        return self.r.substeps

    def set_action_repeat(self, k, hold=False):
        self.r.set_action_repeat(k, hold)

    @property
    def on(self):
        return self.max_steps > 0 or self.window

    def set_time_limit(self, max_steps, window=False):
        self.max_steps, self.window = int(max_steps), bool(window)
        self.count[:] = 0

    def _begin(self, i, start):
        """A reset of env i (the wrapped oracle's), with the record of a cut episode showing how it was cut."""
        before = int(self.o.done[i])
        self.o._begin(i, start)
        if int(self.o.done[i]) != before and self.cut[i]:
            f = int(self.o.last[i, EP_END_FLAGS])
            if self.cut[i] == CUT_WINDOW:
                f &= ~FLAG_TERMINATED
            self.o.last[i, EP_END_FLAGS] = float(f | FLAG_TRUNCATED)
        self.cut[i] = 0
        self.count[i] = 0

    def step(self, actions, want_obs=True):
        a = np.asarray(actions)
        obs = np.empty((self.N, self.D), np.float32)
        rew64 = np.empty(self.N, np.float64)
        code = np.empty(self.N, np.uint8)
        L = self.o.vec.L
        for i in range(self.N):
            row = obs[i].ctypes.data
            h = self.o.vec.envs[i]
            if self.cut[i] or (self.r._flags(i) & FLAG_TERMINATED):   # the episode is over
                if self.cfg.auto_reset:
                    self._begin(i, None)
                    L.fxo_observe(h, row)
                    rew64[i], code[i] = 0.0, 0
                elif self.cut[i] == CUT_LIMIT:   # the oracle's env is still running: its observation, untouched
                    L.fxo_observe(h, row)
                    rew64[i], code[i] = 0.0, DONE_TRUNCATED if self.on else DONE_TERMINATED
                else:
                    r, t = self.r._substep(i, a[i], row)   # (obs, 0.0, True) of a terminated oracle env
                    rew64[i], code[i] = r, DONE_TRUNCATED if (self.cut[i] and self.on) else t
                self.r.substeps[i] = 1
                continue
            acc = 0.0
            for j in range(self.r.k):
                r, t = self.r._substep(i, a[i] if j == 0 or not self.r.hold else 0, row)
                acc = r if j == 0 else acc + r
                if t:
                    break
            self.r.substeps[i] = j + 1
            self.count[i] += 1
            c = 0
            if t:
                f = self.r._flags(i)
                if self.window and (f & FLAG_EXHAUSTED) and not (f & FLAG_BROKE):
                    c, self.cut[i] = DONE_TRUNCATED, CUT_WINDOW
                else:
                    c = DONE_TERMINATED
            elif self.max_steps > 0 and self.count[i] >= self.max_steps:
                c, self.cut[i] = DONE_TRUNCATED, CUT_LIMIT
            rew64[i], code[i] = acc, c
        return (obs if want_obs else None), rew64.astype(np.float32), rew64, code

    def reset(self, start_bars=None, mask=None):
        for i in range(self.N):
            if mask is None or mask[i]:
                self._begin(i, None if start_bars is None else int(start_bars[i]))
        return self.o.observe()

    def info(self):
        d = dict(self.o.info())
        f = np.asarray(d["flags"]).astype(np.int64).copy()
        for i in np.nonzero(self.cut)[0]:
            if self.cut[i] == CUT_WINDOW:
                f[i] &= ~FLAG_TERMINATED
            f[i] |= FLAG_TRUNCATED
        d["flags"] = f.astype(np.asarray(d["flags"]).dtype)
        return d

    # ---- the rest is the wrapped oracle's
    def set_episode_starts(self, lo=None, hi=None, seed=0):
        self.r.set_episode_starts(lo, hi, seed)

    def episodes(self):
        return self.r.episodes()

    def env_records(self, i):
        return self.r.env_records(i)

    def observe(self):
        return self.r.observe()

    def summary(self):
        return self.r.summary()

    def close(self):
        self.r.close()
