"""
tests/episode_oracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

EpisodeOracle: the C oracle (oracle.c_oracle.OracleVec, unchanged) with the episode starts and records of
include/fxenv.h restated around it -- per-env start ranges and a seed (fxenv_set_reset_starts), the episode counters and
the record of the last finished episode (fxenv_get_episode_info, FXENV_EP_*).  Resets, including the auto-reset step
after a termination, are driven from here, so that the new episode can start at a drawn bar; every other step is the
oracle's own fxo_step.  The record is read from the oracle's analyzer state by tests/episode_oracle.c, compiled with the
oracle's flags into a temporary directory on first use.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle.c_oracle import OracleVec

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_lib = None

FLAG_STARTED, FLAG_TERMINATED = 1, 2


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "episode_oracle.c"), os.path.join(_ROOT, "oracle", "fxenv_oracle.c"),
                os.path.join(_ROOT, "include", "fxenv.h")]
        tag = hashlib.sha256(b"".join(open(p, "rb").read() for p in srcs)).hexdigest()[:16]
        out = os.path.join(tempfile.gettempdir(), f"gymfx_episode_oracle_{os.getuid()}_{tag}.so")
        if not os.path.exists(out):
            tmp = out + f".{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-O2", "-pthread", "-fPIC", "-std=gnu11", "-ffp-contract=off", "-fno-fast-math",
                                   "-shared", "-o", tmp, srcs[0], "-lm"])
            os.replace(tmp, out)
        L = C.CDLL(out)
        L.fxe_draw_start.restype = C.c_int64
        L.fxe_draw_start.argtypes = [C.c_uint64, C.c_int32, C.c_int32, C.c_int64, C.c_uint64]
        L.fxe_started.argtypes = [C.c_void_p]
        L.fxe_record.argtypes = [C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


class EpisodeOracle:
    """N oracle envs with start ranges and episode records; the surface of OracleVec plus set_episode_starts / episodes."""

    EPISODE_FIELDS = ("start", "bars", "equity", "commission", "end_flags", "dd_max_pct", "dd_max_money", "pnl_net",
                      "pnl_sq", "opened", "closed", "won", "lost", "index")   # FXENV_EP_*

    def __init__(self, cfg, candles, minutes=None):
        self.vec = OracleVec(cfg, candles, minutes)
        self.E = lib()
        self.cfg, self.N, self.D = cfg, self.vec.N, self.vec.D
        self.T = np.asarray([self.vec.candles[i % cfg.num_pairs].shape[0] for i in range(self.N)], np.int64)
        self.lo = np.zeros(self.N, np.int64)
        self.span = np.zeros(self.N, np.uint64)      # 0 = no range
        self.seed = 0
        self.start = np.zeros(self.N, np.int64)      # first bar of the current episode
        self.begun = np.zeros(self.N, np.int64)      # episodes begun (the k of the next draw)
        self.done = np.zeros(self.N, np.int32)
        self.last = np.zeros((self.N, len(self.EPISODE_FIELDS)), np.float64)

    @staticmethod
    def draw_start(seed, env, k, lo, hi):
        return int(lib().fxe_draw_start(int(seed) & (2**64 - 1), int(env), int(k), int(lo), int(hi) - int(lo) + 1))

    def set_episode_starts(self, lo=None, hi=None, seed=0):
        """Inclusive ranges [lo_i, hi_i] (int64 [N]) and the seed; lo = None clears them."""
        if lo is None:
            self.lo[:], self.span[:], self.seed = 0, 0, 0
        else:
            self.lo = np.asarray(lo, np.int64).copy()
            self.span = (np.asarray(hi, np.int64) - self.lo + 1).astype(np.uint64)
            self.seed = int(seed) & (2**64 - 1)

    def _begin(self, i, start):
        """A reset of env i: record the episode it ends (if it took a step), then start the next one at `start`, or at a
        drawn bar when start is None and a range is set, else at the current start."""
        h = self.vec.envs[i]
        k = int(self.begun[i])
        if self.E.fxe_started(h):
            self.E.fxe_record(h, self.last[i].ctypes.data)
            self.last[i, 0] = float(self.start[i])
            self.last[i, 13] = float(k - 1)
            self.done[i] += 1
        self.begun[i] = k + 1
        if start is None:
            start = (self.E.fxe_draw_start(self.seed, i, k, int(self.lo[i]), int(self.span[i])) if self.span[i]
                     else int(self.start[i]))
        start = min(max(int(start), 0), int(self.T[i]) - 1)
        self.start[i] = start
        self.vec.L.fxo_reset(h, start)

    def reset(self, start_bars=None, mask=None):
        for i in range(self.N):
            if mask is None or mask[i]:
                self._begin(i, None if start_bars is None else int(start_bars[i]))
        return self.vec.observe()

    def step(self, actions, want_obs=True):
        """One step of every env: the oracle's fxo_step, except that a terminated env with auto_reset begins its next
        episode here (what fxo_step would do at the old start: reset, observation of the new episode, reward 0, not done)."""
        a = np.asarray(actions)
        obs = np.empty((self.N, self.D), np.float32)
        rew64 = np.empty(self.N, np.float64)
        term = np.empty(self.N, np.uint8)
        flags = self.vec.info()["flags"]
        L = self.vec.L
        r, t = C.c_double(), C.c_uint8()
        for i, h in enumerate(self.vec.envs):
            row = obs[i].ctypes.data
            if self.cfg.auto_reset and (int(flags[i]) & FLAG_TERMINATED):
                self._begin(i, None)
                L.fxo_observe(h, row)
                rew64[i], term[i] = 0.0, 0
            else:
                L.fxo_step(h, float(a[i]), row, C.byref(r), C.byref(t))
                rew64[i], term[i] = r.value, t.value
        return (obs if want_obs else None), rew64.astype(np.float32), rew64, term

    def episodes(self):
        """-> (start int64 [N] of the current episodes, episodes_done int32 [N], last_episode float64 [N, 14])."""
        return self.start.copy(), self.done.copy(), self.last.copy()

    def observe(self):
        return self.vec.observe()

    def info(self):
        return self.vec.info()

    def summary(self):
        return self.vec.summary()

    def close(self):
        self.vec.close()
