"""
tests/audit_ref.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Reference records for the bracket audit (include/fxenv.h FXENV_AU_*), as float64 [n, 8] arrays in the product's field
order:
  * AuditOracle: EpisodeOracle (the C oracle, unchanged, with episode starts) whose steps go through tests/audit_oracle.c,
    which reads each step's record off the orders the oracle's strategy call created; episode = the env's k.
  * HostAuditEnv: the g++ build of the product core (tests/hostsim) with the FxAudit out-parameter, tests/audit_hostsim.cpp.
  * audit_text: records -> the reference's file content, through the product's formatter.
Both libraries are compiled into a temporary directory on first use.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from episode_oracle import FLAG_TERMINATED, EpisodeOracle
from gym_fx_b200.strategy_plugins.direct_atr_sltp import audit_line
from hostsim.hostsim import HostSimEnv
from hostsim.hostsim import lib as _hostsim_lib

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
F = 8  # FXENV_AU_FIELDS
KIND, BAR, EPISODE, ENTRY, STOP, LIMIT, SIZE, ATR = range(F)
_libs = {}


def _compile(name, cmd, srcs):
    if name not in _libs:
        tag = hashlib.sha256(b"".join(open(p, "rb").read() for p in srcs)).hexdigest()[:16]
        out = os.path.join(tempfile.gettempdir(), f"gymfx_{name}_{os.getuid()}_{tag}.so")
        if not os.path.exists(out):
            tmp = out + f".{os.getpid()}.tmp"
            subprocess.check_call(cmd + ["-o", tmp, srcs[0], "-lm"])
            os.replace(tmp, out)
        _libs[name] = C.CDLL(out)
    return _libs[name]


def oracle_lib():
    srcs = [os.path.join(_HERE, "audit_oracle.c"), os.path.join(_ROOT, "oracle", "fxenv_oracle.c"),
            os.path.join(_ROOT, "include", "fxenv.h")]
    L = _compile("audit_oracle", ["gcc", "-O2", "-pthread", "-fPIC", "-std=gnu11", "-ffp-contract=off", "-fno-fast-math",
                                  "-shared"], srcs)
    L.fxa_step.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_uint8), C.c_void_p]
    return L


def hostsim_lib():
    srcs = [os.path.join(_HERE, "audit_hostsim.cpp"), os.path.join(_HERE, "hostsim", "fx_hostsim.cpp"),
            os.path.join(_ROOT, "gym_fx_b200", "csrc", "fx_core.cuh"), os.path.join(_ROOT, "include", "fxenv.h")]
    L = _compile("audit_hostsim", ["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared"],
                 srcs)
    H = _hostsim_lib()
    for f in ("hs_create", "hs_destroy", "hs_reset", "hs_step", "hs_scalars", "hs_info", "hs_stats"):
        getattr(L, f).argtypes = getattr(H, f).argtypes
        getattr(L, f).restype = getattr(H, f).restype
    L.hsa_records.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.hsa_forget.argtypes = [C.c_void_p]
    return L


class AuditOracle(EpisodeOracle):
    """EpisodeOracle that also keeps every env's audit records (list of float64 [8] per env)."""

    def __init__(self, cfg, candles, minutes=None):
        super().__init__(cfg, candles, minutes)
        self.A = oracle_lib()
        self.records = [[] for _ in range(self.N)]

    def step(self, actions, want_obs=True):
        a = np.asarray(actions)
        obs = np.empty((self.N, self.D), np.float32)
        rew64 = np.empty(self.N, np.float64)
        term = np.empty(self.N, np.uint8)
        flags = self.vec.info()["flags"]
        r, t = C.c_double(), C.c_uint8()
        rec = np.zeros(F, np.float64)
        for i, h in enumerate(self.vec.envs):
            row = obs[i].ctypes.data
            if self.cfg.auto_reset and (int(flags[i]) & FLAG_TERMINATED):
                self._begin(i, None)
                self.vec.L.fxo_observe(h, row)
                rew64[i], term[i] = 0.0, 0
                continue
            if self.A.fxa_step(h, float(a[i]), row, C.byref(r), C.byref(t), rec.ctypes.data):
                rec[EPISODE] = float(self.begun[i] - 1)
                self.records[i].append(rec.copy())
            rew64[i], term[i] = r.value, t.value
        return (obs if want_obs else None), rew64.astype(np.float32), rew64, term

    def env_records(self, i):
        return np.asarray(self.records[i], np.float64).reshape(-1, F)


class HostAuditEnv(HostSimEnv):
    """One env of the product core's host build, with its audit records."""

    def __init__(self, cfg, candles, minutes=None):
        self.L = hostsim_lib()
        self.candles = np.ascontiguousarray(candles, np.float64)
        self.minutes = None if minutes is None else np.ascontiguousarray(minutes, np.int64)
        self.h = self.L.hs_create(C.byref(cfg), 0, self.candles.ctypes.data, self.candles.shape[0],
                                  None if self.minutes is None else self.minutes.ctypes.data)

    def __del__(self):
        try:
            self.L.hsa_forget(self.h)
            self.L.hs_destroy(self.h)
        except Exception:
            pass

    def records(self):
        n = self.L.hsa_records(self.h, None, 0)
        out = np.zeros((n, F), np.float64)
        self.L.hsa_records(self.h, out.ctypes.data, n)
        return out


def audit_text(records) -> str:
    """float64 [n, 8] records -> what the reference appends to GYMFX_BRACKET_AUDIT for them."""
    return "".join(audit_line(int(r[KIND]), r[ENTRY], r[STOP], r[LIMIT], r[SIZE], r[ATR]) for r in np.asarray(records))
