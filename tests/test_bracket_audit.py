"""CPU (-m "not gpu"): the bracket audit of direct_atr_sltp (GYMFX_BRACKET_AUDIT, include/fxenv.h FXENV_AU_*).

  * tests/golden/audit/*.jsonl were written by the UNMODIFIED reference (tests/golden/make_audit_golden.py).  The C
    oracle's records and those of the product core's host build, formatted by the product's formatter, equal each file
    byte for byte; deliberately wrong records (one ulp off in any field, stop and limit swapped, a force-close emitted one
    bar early or late) do not.
  * A decision whose orders find the order table full is still recorded.
  * The product core's records equal the oracle's on the ATR members of the seeded random configurations (session
    filter, rel-volume in both size modes, leverage, commission, slippage, per-pair pip sizes).
  * With the reference tree available (GYMFX_REFERENCE_ROOT), the fixtures regenerate unchanged and the committed
    goldens stay byte-identical."""
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import scenarios as S
from audit_ref import ATR, BAR, ENTRY, KIND, LIMIT, SIZE, STOP, AuditOracle, HostAuditEnv, audit_text
from common import GOLDEN_DIR, config_from_meta
from gym_fx_b200.config import lower_config
from gym_fx_b200.synth import synth_candles, synth_minutes
from gym_fx_b200.strategy_plugins.direct_atr_sltp import audit_line
from test_core_vs_oracle_random import _random_case

AUDIT_DIR = os.path.join(GOLDEN_DIR, "audit")


def audit_names():
    return sorted(os.path.basename(p)[:-6] for p in glob.glob(os.path.join(AUDIT_DIR, "*.jsonl")))


def load_audit_case(name):
    """(golden dict, expected file text): the trajectory next to the goldens, or the audit-only one under audit/."""
    path = os.path.join(GOLDEN_DIR, name + ".npz")
    if not os.path.exists(path):
        path = os.path.join(AUDIT_DIR, name + ".npz")
    z = np.load(path)
    g = {k: z[k] for k in z.files}
    g["meta"] = json.loads(bytes(g["meta"]).decode())
    with open(os.path.join(AUDIT_DIR, name + ".jsonl"), encoding="utf-8") as fh:
        return g, fh.read()


def _replay(env, g, oracle):
    n = g["reward"].shape[0]
    for a in g["actions"][:n - 1]:
        env.step(np.array([a]) if oracle else a)
    return env.env_records(0) if oracle else env.records()


def oracle_records(g):
    cfg = config_from_meta(g["meta"], order_capacity=512)
    o = AuditOracle(cfg, [g["candles"]], [g["minutes"]])
    o.reset(np.zeros(1, np.int64))
    return _replay(o, g, True)


def test_fixture_set_is_complete():
    assert audit_names() == sorted(["atr_fw32_dd", "atr_relvol_lev_sharpe", "atr_notional_jpy", "atr_session_filter",
                                    "slip_atr_lev_sharpe", "atr_max_frac_clamp", "atr_tp_halving"])


@pytest.mark.parametrize("name", audit_names())
def test_oracle_records_equal_reference_file(name):
    g, want = load_audit_case(name)
    assert audit_text(oracle_records(g)) == want


@pytest.mark.parametrize("name", audit_names())
def test_product_core_records_equal_reference_file(name):
    g, want = load_audit_case(name)
    cfg = config_from_meta(g["meta"], order_capacity=512)
    env = HostAuditEnv(cfg, g["candles"], g["minutes"])
    env.reset(0)
    rec = _replay(env, g, False)
    assert audit_text(rec) == want
    np.testing.assert_array_equal(rec, oracle_records(g))   # bar and the NaN fields too


def test_fixtures_reach_every_branch():
    """Force-closes of both signs, the min-fraction clamp, the max-fraction clamp of both distances, tp halving."""
    recs = {n: oracle_records(load_audit_case(n)[0]) for n in ("atr_session_filter", "atr_fw32_dd", "atr_max_frac_clamp",
                                                              "atr_tp_halving")}
    fc = recs["atr_session_filter"][recs["atr_session_filter"][:, KIND] == 3]
    assert len(fc) == 4 and (fc[:, SIZE] > 0).sum() == 2 and (fc[:, SIZE] < 0).sum() == 2
    r = recs["atr_fw32_dd"][0]   # a short bracket whose stop distance is the min-fraction floor
    assert r[KIND] == 2 and r[STOP] == r[ENTRY] + 0.001 * r[ENTRY]
    m = recs["atr_max_frac_clamp"]   # both distances at the max-fraction ceiling
    ceil = 0.0004 * m[:, ENTRY]
    sign = np.where(m[:, KIND] == 1, 1.0, -1.0)
    assert np.array_equal(m[:, STOP], m[:, ENTRY] - sign * ceil) and np.array_equal(m[:, LIMIT], m[:, ENTRY] + sign * ceil)
    h = recs["atr_tp_halving"]   # take-profit distance halved to close * 0.5
    sign = np.where(h[:, KIND] == 1, 1.0, -1.0)
    assert np.array_equal(h[:, LIMIT], h[:, ENTRY] + sign * (h[:, ENTRY] * 0.5))


def test_negative_controls_fail_the_comparison():
    g, want = load_audit_case("atr_session_filter")
    rec = oracle_records(g)
    assert audit_text(rec) == want
    br = int(np.nonzero(rec[:, KIND] != 3)[0][0])
    for f in (ENTRY, STOP, LIMIT, SIZE, ATR):
        bad = rec.copy()
        bad[br, f] = np.nextafter(bad[br, f], np.inf)
        assert audit_text(bad) != want, f"one ulp in field {f} went unnoticed"
    bad = rec.copy()
    bad[br, [STOP, LIMIT]] = bad[br, [LIMIT, STOP]]
    assert audit_text(bad) != want
    closes = g["candles"][:, 3]
    shifted = 0
    for fc in np.nonzero(rec[:, KIND] == 3)[0]:   # each force-close emitted one bar early / late: the entry of that bar
        bar = int(rec[fc, BAR])
        for other in (bar - 1, bar + 1):
            if closes[other] != closes[bar]:
                bad = rec.copy()
                bad[fc, [BAR, ENTRY]] = other, closes[other]
                assert audit_text(bad) != want, (fc, other)
                shifted += 1
    assert shifted >= 4
    assert audit_line(3, 1.1, np.nan, np.nan, -1.0, np.nan) == '{"kind": "session_force_close", "entry": 1.1, "size": -1.0}\n'


def _atr_random_cases():
    """The direct_atr_sltp members of test_core_vs_oracle_random's seeded configurations, each also with the session
    filter (close zone every day from 20:00) and with the per-pair pip size of its pair."""
    out = []
    for seed in range(2, 36, 3):
        cfg, candles, minutes, acts = _random_case(seed)
        out.append((f"seed{seed}", cfg, candles, minutes, acts))
    for seed in range(2, 36, 9):
        cfg, candles, minutes, acts = _random_case(seed)
        cfg.session_filter, cfg.entry_dow_start, cfg.entry_hour_start = 1, 0, 2
        cfg.force_close_dow, cfg.force_close_hour = 4, 20
        out.append((f"seed{seed}_session", cfg, candles, minutes, acts))
    return out


@pytest.mark.parametrize("case", _atr_random_cases(), ids=lambda c: c[0])
def test_product_core_records_equal_oracle_on_random_configs(case):
    _, cfg, candles, minutes, acts = case
    assert cfg.strategy == 2
    core = HostAuditEnv(cfg, candles, minutes)
    orc = AuditOracle(cfg, [candles], [minutes])
    core.reset(0)
    orc.reset(np.zeros(1, np.int64))
    for a in acts:
        _, t = core.step(a)
        orc.step(np.array([a], np.int32))
        if t:
            break
    got, ref = core.records(), orc.env_records(0)
    assert len(ref) > 10
    np.testing.assert_array_equal(got[:, :BAR + 1], ref[:, :BAR + 1])
    assert got[:, ENTRY:].tobytes() == ref[:, ENTRY:].tobytes()


def overflow_case(n_envs):
    """direct_atr_sltp with an order table of 32 entries that runs full: stops and limits so far away that no child ever
    triggers (k_sl = k_tp = 3000 ATR, no ceiling, tp halved to close * 0.5), so every bracket leaves a live pair behind."""
    cfgd = {**S.DEFAULTS, "window_size": 16, "atr_period": 6, "k_sl": 3000.0, "k_tp": 3000.0, "max_sltp_frac": None}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, "strategy": "direct_atr_sltp"})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"], preprocessor_plugin=pl["preprocessor"],
                       reward_plugin=pl["reward"], columns=S.OHLCV, num_envs=n_envs, order_capacity=32)
    return cfg, synth_candles(1200, 0, 3), synth_minutes(1200)


def test_record_is_written_when_the_order_table_overflows():
    """The product drops the orders of a decision that finds the table full (FX_FLAG_ORDER_OVERFLOW); the reference's list
    is unbounded.  Up to and including the step that overflows, the records equal the oracle's, and that step has one."""
    cfg, candles, minutes = overflow_case(1)
    core = HostAuditEnv(cfg, candles, minutes)
    orc = AuditOracle(cfg, [candles], [minutes])
    core.reset(0)
    orc.reset(np.zeros(1, np.int64))
    for k, a in enumerate(S.make_actions(("sticky", 5, 0.3), 400)):
        before = len(core.records())
        core.step(a)
        orc.step(np.array([a], np.int32))
        assert core.records().tobytes() == orc.env_records(0).tobytes(), k
        if core.info()["flags"] & 16:
            assert len(core.records()) == before + 1
            break
    else:
        pytest.fail("the order table never overflowed")


@pytest.mark.skipif(not os.path.isdir(os.environ.get("GYMFX_REFERENCE_ROOT", "")),
                    reason="needs the reference tree (GYMFX_REFERENCE_ROOT)")
def test_make_audit_golden_reruns_and_leaves_goldens_unchanged():
    paths = sorted(glob.glob(os.path.join(GOLDEN_DIR, "*.npz")) + glob.glob(os.path.join(AUDIT_DIR, "*")))
    before = {p: open(p, "rb").read() for p in paths}
    subprocess.check_call([sys.executable, os.path.join(GOLDEN_DIR, "make_audit_golden.py")])
    for p in paths:
        if p.endswith(".npz") and os.path.dirname(p) == AUDIT_DIR:
            continue   # the audit-only trajectories carry the generating tool versions; their jsonl must not change
        assert open(p, "rb").read() == before[p], p
