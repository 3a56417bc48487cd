"""tests/env_params_hostsim.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

ParamsHostEnv: one env of the g++ build of the product core (tests/hostsim) that takes commission, leverage, slippage,
sl_pips, tp_pips, k_sl and k_tp from a per-env parameter row (include/fxenv.h FXENV_PARAM_* order) instead of the config,
through tests/params_hostsim.cpp.  The library is compiled into a temporary directory on first use."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from hostsim.hostsim import HostSimEnv
from hostsim.hostsim import lib as _hostsim_lib

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_lib = None


def params_hostsim_lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_HERE, "params_hostsim.cpp"), os.path.join(_HERE, "hostsim", "fx_hostsim.cpp"),
                os.path.join(_ROOT, "gym_fx_b200", "csrc", "fx_core.cuh"), os.path.join(_ROOT, "include", "fxenv.h")]
        tag = hashlib.sha256(b"".join(open(p, "rb").read() for p in srcs)).hexdigest()[:16]
        out = os.path.join(tempfile.gettempdir(), f"gymfx_params_hostsim_{os.getuid()}_{tag}.so")
        if not os.path.exists(out):
            tmp = out + f".{os.getpid()}.tmp"
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared",
                                   "-o", tmp, srcs[0], "-lm"])
            os.replace(tmp, out)
        L = C.CDLL(out)
        H = _hostsim_lib()
        for f in ("hs_create", "hs_destroy", "hs_reset", "hs_step", "hs_scalars", "hs_info", "hs_stats"):
            getattr(L, f).argtypes = getattr(H, f).argtypes
            getattr(L, f).restype = getattr(H, f).restype
        L.hsp_set_params.argtypes = [C.c_void_p, C.c_void_p]
        _lib = L
    return _lib


class ParamsHostEnv(HostSimEnv):
    """One env of the product core's host build, stepping with a parameter row (None: the config's values)."""

    def __init__(self, cfg, candles, minutes=None, row=None):
        self.L = params_hostsim_lib()
        self.candles = np.ascontiguousarray(candles, np.float64)
        self.minutes = None if minutes is None else np.ascontiguousarray(minutes, np.int64)
        self.h = self.L.hs_create(C.byref(cfg), 0, self.candles.ctypes.data, self.candles.shape[0],
                                  None if self.minutes is None else self.minutes.ctypes.data)
        self.set_params(row)

    def set_params(self, row=None):
        r = None if row is None else np.ascontiguousarray(row, np.float64)
        if r is not None and r.shape != (7,):
            raise ValueError(f"a parameter row has 7 values, got shape {r.shape}")
        self.L.hsp_set_params(self.h, None if r is None else r.ctypes.data)

    def __del__(self):
        try:
            self.L.hsp_set_params(self.h, None)
            self.L.hs_destroy(self.h)
        except Exception:
            pass
