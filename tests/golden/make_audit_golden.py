#!/usr/bin/env python3
"""
tests/golden/make_audit_golden.py -- regenerates tests/golden/audit/ (the bracket audit fixtures).

Runs the UNMODIFIED reference over oracle/bt_shim with GYMFX_BRACKET_AUDIT set, through make_golden.generate, and
stores the file that direct_atr_sltp._audit_emit wrote:
  * tests/golden/audit/<name>.jsonl for every direct_atr_sltp scenario of scenarios.py.  The run's rewards and equity
    must equal the committed tests/golden/<name>.npz bit for bit (so the audit belongs to that trajectory); the
    committed .npz files are never written.
  * AUDIT_SCENARIOS below (clamps that the golden scenarios never reach): tests/golden/audit/<name>.npz (inputs and
    trajectory, the make_golden format) plus <name>.jsonl.  They live in the subdirectory so that the *.npz glob of
    tests/common.py does not pick them up.
The reference module reads GYMFX_BRACKET_AUDIT at import, so every scenario runs in a fresh subprocess with the
variable set before the plugin import.

Usage:  GYMFX_REFERENCE_ROOT=<checkout of harveybc/gym-fx> python tests/golden/make_audit_golden.py [scenario_name ...]
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "audit")
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import scenarios as S  # noqa: E402

_ATR = S._pl(strategy="direct_atr_sltp")

AUDIT_SCENARIOS = [
    # max_sltp_frac * close (~4.4e-4) below both k * ATR distances: stop and limit are both clamped to it
    dict(name="atr_max_frac_clamp", data=("synth", 400, 0, 91),
         cfg={"max_sltp_frac": 0.0004, "min_sltp_frac": 0.0001, "atr_period": 8},
         plugins=_ATR, actions=("sticky", 31, 0.6), steps=360),
    # no ceiling and k_tp * ATR >= close: the take-profit distance is halved to close * 0.5
    dict(name="atr_tp_halving", data=("synth", 400, 2, 92),
         cfg={"max_sltp_frac": None, "k_tp": 5000.0, "atr_period": 4},
         plugins=_ATR, actions=("random", 32), steps=360),
]


def atr_golden_scenarios():
    return [sc for sc in S.SCENARIOS if sc["plugins"]["strategy"] == "direct_atr_sltp"]


def _child(name, outdir):
    """In the subprocess: GYMFX_BRACKET_AUDIT is already set; run the reference on one scenario."""
    import make_golden as M

    sc = next(s for s in atr_golden_scenarios() + AUDIT_SCENARIOS if s["name"] == name)
    M.generate(sc, outdir)


def _run(sc, tmp):
    audit = os.path.join(tmp, sc["name"] + ".jsonl")
    env = dict(os.environ, GYMFX_BRACKET_AUDIT=audit)
    subprocess.check_call([sys.executable, os.path.abspath(__file__), "--child", sc["name"], tmp], env=env)
    if not os.path.exists(audit):  # a run that placed no bracket leaves no file
        open(audit, "w").close()
    return audit, os.path.join(tmp, sc["name"] + ".npz")


def main(names):
    os.makedirs(OUT, exist_ok=True)
    for sc in atr_golden_scenarios() + AUDIT_SCENARIOS:
        if names and sc["name"] not in names:
            continue
        with tempfile.TemporaryDirectory() as tmp:
            audit, npz = _run(sc, tmp)
            if sc in AUDIT_SCENARIOS:
                shutil.copyfile(npz, os.path.join(OUT, sc["name"] + ".npz"))
            else:
                new, old = np.load(npz), np.load(os.path.join(HERE, sc["name"] + ".npz"))
                for key in ("reward", "equity"):
                    if new[key].tobytes() != old[key].tobytes():
                        raise SystemExit(f"{sc['name']}: the reference's {key} differs from the committed golden")
            shutil.copyfile(audit, os.path.join(OUT, sc["name"] + ".jsonl"))
            with open(audit) as fh:
                lines = fh.read().splitlines()
        kinds = {k: sum(f'"kind": "{k}"' in ln for ln in lines)
                 for k in ("long_bracket", "short_bracket", "session_force_close")}
        print(f"{sc['name']:24s} records={len(lines):4d} {kinds}")


if __name__ == "__main__":
    if len(sys.argv) == 4 and sys.argv[1] == "--child":
        _child(sys.argv[2], sys.argv[3])
    else:
        main(set(sys.argv[1:]))
