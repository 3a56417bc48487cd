"""direct_atr_sltp mirror (reference: strategy_plugins/direct_atr_sltp.py:48-263): ATR-sized SL/TP brackets
(simple-mean ATR over `atr_period` true ranges), optional cash-relative sizing and a week-session filter.
Parameters are lowered to FxConfig; TR/ATR, sizing, clamps and order placement run in the step kernel.

Bracket audit: as in the reference module (:35-45), GYMFX_BRACKET_AUDIT is read once, at import.  When it names a file,
GymFxEnv keeps the step kernel's audit log on for its env and appends one line per decision to that file
(`audit_line`); VecFxEnv.set_bracket_audit / bracket_audit give the same records for any number of envs."""
import json
import os

from ..plugin_base import PluginBase, kernel_resident

_AUDIT_PATH = os.environ.get("GYMFX_BRACKET_AUDIT")

AUDIT_KINDS = {1: "long_bracket", 2: "short_bracket", 3: "session_force_close"}  # FXENV_AU_KIND_*


def audit_line(kind: int, entry: float, stop: float, limit: float, size: float, atr: float) -> str:
    """One audit record as the reference writes it (direct_atr_sltp.py:138-142, :188-191, :199-202): json.dumps of the
    dict in the reference's key order, plus a newline.  A force-close line has no stop, limit or atr."""
    name = AUDIT_KINDS[int(kind)]
    if name == "session_force_close":
        rec = {"kind": name, "entry": float(entry), "size": float(size)}
    else:
        rec = {"kind": name, "entry": float(entry), "stop": float(stop), "limit": float(limit), "size": float(size),
               "atr": float(atr)}
    return json.dumps(rec) + "\n"


def audit_append(path: str, text: str) -> None:
    """_audit_emit's file handling: append, and swallow I/O errors."""
    try:
        with open(path, "a", encoding="utf-8") as fh:
            fh.write(text)
    except Exception:
        pass


class Plugin(PluginBase):
    plugin_kind = "direct_atr_sltp"
    strict_keys = True
    plugin_params = {
        "atr_period": 14, "k_sl": 2.0, "k_tp": 3.0, "position_size": 1.0,
        "rel_volume": None, "leverage": 1.0, "min_order_volume": 0.0, "max_order_volume": 1e12,
        "size_mode": "fx_units", "min_sltp_frac": 0.001, "max_sltp_frac": 0.20,
        "session_filter": False, "entry_dow_start": 0, "entry_hour_start": 12,
        "force_close_dow": 4, "force_close_hour": 20,
    }

    def decide_action(self, obs, info, step: int) -> int:
        return 0

    def on_reset(self, bt_strategy, config) -> None:
        return None

    def apply_action(self, bt_strategy, action, config) -> None:
        kernel_resident("direct_atr_sltp.apply_action")

    def hparam_schema(self):
        return [("atr_period", 7, 30, "int"), ("k_sl", 1.0, 4.0, "float"), ("k_tp", 1.5, 6.0, "float")]
