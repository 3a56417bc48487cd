"""
ctypes binding of libfxenv.so (include/fxenv.h).  The library is built in-tree by `build()` (nvcc, sm_90a);
there is NO fallback: if the shared object is missing or no CUDA device is present the import of the env classes
succeeds but any attempt to create an env raises `FxEnvError`.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

from .config import FxConfig

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, os.environ.get("FXENV_LIB", "libfxenv.so"))  # FXENV_LIB: experiment builds
CSRC = os.path.join(_HERE, "csrc")

class FxPolicyWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("w1", "b1", "w2", "b2", "w_pi", "b_pi", "w_v", "b_v")]


class FxRollout(C.Structure):
    _fields_ = [("horizon", C.c_int32), ("obs_slots", C.c_int32), ("obs", C.c_void_p), ("actions", C.c_void_p),
                ("logp", C.c_void_p), ("value", C.c_void_p), ("reward", C.c_void_p), ("done", C.c_void_p),
                ("gumbel", C.c_void_p), ("seed", C.c_uint64)]


EXPORTS = [
    "fxenv_abi_version", "fxenv_create", "fxenv_destroy", "fxenv_last_error", "fxenv_load_candles", "fxenv_obs_dim",
    "fxenv_reset", "fxenv_observe", "fxenv_step", "fxenv_step_many", "fxenv_step_host", "fxenv_get_info",
    "fxenv_state_bytes", "fxenv_get_state", "fxenv_set_state", "fxenv_launch_count", "fxenv_step_many_engine",
    "fxenv_policy_create", "fxenv_policy_set_weights", "fxenv_policy_destroy", "fxenv_rollout", "fxenv_policy_sync_timeouts",
    "fxenv_rollout_ex", "fxenv_policy_peek", "fxenv_set_reset_starts", "fxenv_get_episode_info",
    "fxenv_set_bracket_audit", "fxenv_get_bracket_audit", "fxenv_set_action_repeat", "fxenv_policy_create_ex",
    "fxenv_set_time_limit", "fxenv_set_env_params", "fxenv_policy_create_ex2", "fxenv_policy_create_ex3",
    "fxenv_policy_set_member_weights", "fxenv_policy_set_obs_norm", "fxenv_obs_moments",
    "fxenv_return_moments",
]

ROLLOUT_GREEDY = 1  # FXENV_ROLLOUT_GREEDY
PEEK_OBS16, PEEK_H1 = 0, 1  # FXENV_PEEK_*
MAX_REPEAT, REPEAT_HOLD = 256, 1  # FXENV_MAX_REPEAT, FXENV_REPEAT_HOLD
POLICY_WIDTHS = (64, 128, 256, 512)  # the hidden widths fxenv_policy_create_ex accepts
POLICY_SEPARATE = 1  # FXENV_POLICY_SEPARATE (fxenv_policy_create_ex2 flags)
FLAG_TRUNCATED, TIME_LIMIT_WINDOW = 64, 1  # FX_FLAG_TRUNCATED, FXENV_TIME_LIMIT_WINDOW
DONE_TERMINATED, DONE_TRUNCATED = 1, 2  # FXENV_DONE_* codes of the terminated / done outputs while truncation is on
# FXENV_ENV_PARAMS and the FXENV_PARAM_* columns of a per-env parameter row (fxenv_set_env_params)
ENV_PARAMS = 7
PARAM_COMMISSION, PARAM_LEVERAGE, PARAM_SLIPPAGE, PARAM_SL_PIPS, PARAM_TP_PIPS, PARAM_K_SL, PARAM_K_TP = range(7)


class FxEnvError(RuntimeError):
    pass


class FxInfoPtrs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "equity", "prev_equity", "price", "cash", "position_size", "position_price", "commission_paid",
        "position", "bar_index", "total_bars", "trades", "n_orders", "flags", "run_stats")]

RUN_STATS = 12  # FXENV_RUN_STATS
RS = {"dd_maxvalue": 0, "dd_max_money": 1, "dd_max_pct": 2, "tr_pnl": 3, "tr_comm": 4, "tr_price": 5, "pnl_net": 6,
      "pnl_sq": 7, "spare": 8, "opened": 9, "won": 10, "lost": 11}  # FXENV_RS_*


class FxEpisodePtrs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("start", "episodes_done", "last_episode")]


EPISODE_STATS = 14  # FXENV_EPISODE_STATS
EP = {"start": 0, "bars": 1, "equity": 2, "commission": 3, "end_flags": 4, "dd_max_pct": 5, "dd_max_money": 6,
      "pnl_net": 7, "pnl_sq": 8, "opened": 9, "closed": 10, "won": 11, "lost": 12, "index": 13}  # FXENV_EP_*


class FxAuditPtrs(C.Structure):
    _fields_ = [("records", C.c_void_p), ("written", C.c_void_p), ("capacity", C.c_int32)]


AU_FIELDS = 8  # FXENV_AU_FIELDS
AU = {"kind": 0, "bar": 1, "episode": 2, "entry": 3, "stop": 4, "limit": 5, "size": 6, "atr": 7}  # FXENV_AU_*
AU_KIND_LONG, AU_KIND_SHORT, AU_KIND_FORCE_CLOSE = 1, 2, 3  # FXENV_AU_KIND_*


INFO_DTYPES = {
    "equity": "float64", "prev_equity": "float64", "price": "float64", "cash": "float64", "position_size": "float64",
    "position_price": "float64", "commission_paid": "float64", "position": "int32", "bar_index": "int32",
    "total_bars": "int32", "trades": "int32", "n_orders": "int32", "flags": "int32",
}


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile gym_fx_b200/csrc/*.cu into gym_fx_b200/libfxenv.so with nvcc for sm_90a (works without a GPU)."""
    srcs = [os.path.join(CSRC, f) for f in ("fx_capi.cu", "fx_kernels.cu", "fx_kernels_trunc.cu", "fx_kernels_params.cu",
                                            "fx_kernels_params_trunc.cu", "fx_policy.cu", "fx_obs_stats.cu", "fx_return_stats.cu",
                                            "fx_core.cuh", "fx_kernels.cuh", "fx_env_step.cuh", "fx_policy.cuh", "Makefile")]
    srcs.append(os.path.join(_HERE, "..", "include", "fxenv.h"))
    stale = (not os.path.exists(LIB_PATH)) or any(os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in srcs)
    if force or stale:
        cmd = ["make", "-j6", "-C", CSRC] + (["-B"] if force else [])  # the sources compile in parallel
        out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if verbose or out.returncode != 0:
            print(out.stdout)
        if out.returncode != 0:
            raise FxEnvError("building libfxenv.so failed (nvcc required)")
    return LIB_PATH


_lib = None


def load():
    """dlopen libfxenv.so and declare the prototypes of include/fxenv.h."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FxEnvError(f"{LIB_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                         "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, i64, i32 = C.c_void_p, C.c_int64, C.c_int
    L.fxenv_abi_version.restype = i32
    L.fxenv_create.argtypes = [C.POINTER(FxConfig), C.POINTER(vp)]
    L.fxenv_destroy.argtypes = [vp]
    L.fxenv_last_error.restype = C.c_char_p
    L.fxenv_last_error.argtypes = [vp]
    L.fxenv_load_candles.argtypes = [vp, i32, vp, i64, vp]
    L.fxenv_obs_dim.restype = i64
    L.fxenv_obs_dim.argtypes = [vp]
    L.fxenv_reset.argtypes = [vp, vp, vp, vp]
    L.fxenv_observe.argtypes = [vp, vp, vp]
    L.fxenv_step.argtypes = [vp, vp, vp, vp, vp, vp, vp]
    L.fxenv_step_many.argtypes = [vp, i32, vp, vp, i32, vp, vp, vp]
    L.fxenv_step_host.argtypes = [vp, vp, vp, vp, vp]
    L.fxenv_get_info.argtypes = [vp, C.POINTER(FxInfoPtrs)]
    L.fxenv_state_bytes.restype = i64
    L.fxenv_state_bytes.argtypes = [vp]
    L.fxenv_get_state.argtypes = [vp, vp, i64]
    L.fxenv_set_state.argtypes = [vp, vp, i64]
    L.fxenv_launch_count.restype = i64
    L.fxenv_launch_count.argtypes = [vp]
    L.fxenv_step_many_engine.restype = C.c_int
    L.fxenv_step_many_engine.argtypes = [vp, C.c_int]
    L.fxenv_policy_create.argtypes = [vp, C.POINTER(vp)]
    L.fxenv_policy_create_ex.argtypes = [vp, C.c_int32, C.POINTER(vp)]
    L.fxenv_policy_create_ex2.argtypes = [vp, C.c_int32, C.c_uint32, C.POINTER(vp)]
    L.fxenv_policy_create_ex3.argtypes = [vp, C.c_int32, C.c_uint32, C.c_int32, C.POINTER(vp)]
    L.fxenv_policy_set_weights.argtypes = [vp, C.POINTER(FxPolicyWeights), vp]
    L.fxenv_policy_set_member_weights.argtypes = [vp, C.c_int32, C.POINTER(FxPolicyWeights), vp]
    L.fxenv_policy_destroy.argtypes = [vp]
    L.fxenv_rollout.argtypes = [vp, vp, C.POINTER(FxRollout), vp]
    L.fxenv_rollout_ex.argtypes = [vp, vp, C.POINTER(FxRollout), C.c_uint32, vp]
    L.fxenv_policy_sync_timeouts.argtypes = [vp]
    L.fxenv_policy_peek.restype = i64
    L.fxenv_policy_peek.argtypes = [vp, i32, i32, vp, i64, vp]
    L.fxenv_set_reset_starts.argtypes = [vp, vp, vp, C.c_uint64]
    L.fxenv_get_episode_info.argtypes = [vp, C.POINTER(FxEpisodePtrs)]
    L.fxenv_set_bracket_audit.argtypes = [vp, C.c_int32]
    L.fxenv_get_bracket_audit.argtypes = [vp, C.POINTER(FxAuditPtrs)]
    L.fxenv_set_action_repeat.argtypes = [vp, C.c_int32, C.c_uint32]
    L.fxenv_set_time_limit.argtypes = [vp, C.c_int32, C.c_uint32]
    L.fxenv_set_env_params.argtypes = [vp, vp]
    L.fxenv_policy_set_obs_norm.argtypes = [vp, C.c_int32, vp, vp, C.c_float, vp]
    L.fxenv_obs_moments.argtypes = [vp, vp, C.c_int32, C.c_int32, C.c_int32, vp, vp, vp]
    L.fxenv_return_moments.argtypes = [vp, vp, vp, vp, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_double, vp, vp,
                                       vp, vp]
    if L.fxenv_abi_version() != 2:
        raise FxEnvError("libfxenv.so ABI version mismatch")
    _lib = L
    return L


def check(L, handle, rc: int, what: str):
    if rc != 0:
        msg = L.fxenv_last_error(handle)
        raise FxEnvError(f"{what} failed ({rc}): {msg.decode() if msg else '?'}")
