"""
tests/repeat_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

RepeatOracle: the action repeat of include/fxenv.h (fxenv_set_action_repeat) restated around the C oracle.  It wraps an
EpisodeOracle (episode starts and records), or an AuditOracle when the bracket audit is wanted, and steps each env
through its own substeps, each of them exactly one step of the wrapped oracle for that env:
  * an env that is terminated when the step begins runs one substep (with auto-reset: the reset step);
  * otherwise substeps run until k have run or one terminates;
  * repeat mode passes the step's action to every substep, hold mode passes it to the first one and 0 to the others
    (a raw 0 coerces to the hold action 0 in both action modes for every threshold >= 0);
  * the observation and the terminated flag are those of the last substep, the reward the float64 sum of the substep
    rewards in substep order, starting from the first one.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from audit_ref import EPISODE, AuditOracle
from episode_oracle import FLAG_TERMINATED, EpisodeOracle
from oracle.c_oracle import FxoInfo


class RepeatOracle:
    """N oracle envs with an action repeat k and a mode; the surface of EpisodeOracle (AuditOracle with audit=True)."""

    def __init__(self, cfg, candles, minutes=None, k=1, hold=False, audit=False):
        self.o = (AuditOracle if audit else EpisodeOracle)(cfg, candles, minutes)
        self.audit = audit
        self.cfg, self.N, self.D = cfg, self.o.N, self.o.D
        self.set_action_repeat(k, hold)
        self.substeps = np.zeros(self.N, np.int32)  # substeps each env ran in the last step
        self._inf = FxoInfo()

    def set_action_repeat(self, k, hold=False):
        self.k, self.hold = int(k), bool(hold)

    def _flags(self, i):
        self.o.vec.L.fxo_info(self.o.vec.envs[i], C.byref(self._inf))
        return int(self._inf.flags)

    def _substep(self, i, action, row):
        """One step of env i, as the wrapped oracle's step() runs it -> (reward64, terminated)."""
        o, h = self.o, self.o.vec.envs[i]
        if self.cfg.auto_reset and (self._flags(i) & FLAG_TERMINATED):
            o._begin(i, None)
            o.vec.L.fxo_observe(h, row)
            return 0.0, 0
        r, t = C.c_double(), C.c_uint8()
        if self.audit:
            rec = np.zeros(8, np.float64)
            if o.A.fxa_step(h, float(action), row, C.byref(r), C.byref(t), rec.ctypes.data):
                rec[EPISODE] = float(o.begun[i] - 1)
                o.records[i].append(rec)
        else:
            o.vec.L.fxo_step(h, float(action), row, C.byref(r), C.byref(t))
        return r.value, t.value

    def step(self, actions, want_obs=True):
        a = np.asarray(actions)
        obs = np.empty((self.N, self.D), np.float32)
        rew64 = np.empty(self.N, np.float64)
        term = np.empty(self.N, np.uint8)
        for i in range(self.N):
            row = obs[i].ctypes.data
            was_terminated = (self._flags(i) & FLAG_TERMINATED) != 0
            acc = 0.0
            for j in range(self.k):
                r, t = self._substep(i, a[i] if j == 0 or not self.hold else 0, row)
                acc = r if j == 0 else acc + r
                if was_terminated or t:
                    break
            rew64[i], term[i] = acc, t
            self.substeps[i] = j + 1
        return (obs if want_obs else None), rew64.astype(np.float32), rew64, term

    # ---- the rest is the wrapped oracle's
    def set_episode_starts(self, lo=None, hi=None, seed=0):
        self.o.set_episode_starts(lo, hi, seed)

    def reset(self, start_bars=None, mask=None):
        return self.o.reset(start_bars, mask)

    def episodes(self):
        return self.o.episodes()

    def env_records(self, i):
        return self.o.env_records(i)

    def observe(self):
        return self.o.observe()

    def info(self):
        return self.o.info()

    def summary(self):
        return self.o.summary()

    def close(self):
        self.o.close()
