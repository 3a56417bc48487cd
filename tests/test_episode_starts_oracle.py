"""CPU (-m "not gpu"): the start-range draw and the episode record restated around the C oracle
(tests/episode_oracle.py; include/fxenv.h fxenv_set_reset_starts / FXENV_EP_*).  The draw must equal a plain-Python-integer replica of the documented rule; the
record latched at a reset must equal what the oracle's own info() / summary() reported at the step that ended the
episode; the episode counter rises once per finished episode."""
import numpy as np
import pytest

import scenarios as S
from gym_fx_b200.config import lower_config
from gym_fx_b200.synth import synth_candles, synth_minutes
from episode_oracle import EpisodeOracle

M64 = (1 << 64) - 1


def splitmix64(z):
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def draw(seed, env, k, lo, hi):
    """start = lo + umulhi64(splitmix64(seed ^ (env << 32 | k)), hi - lo + 1), in Python integers."""
    seed, env, k, lo, hi = (int(x) for x in (seed, env, k, lo, hi))
    h = splitmix64((seed ^ ((env << 32) | (k & 0xFFFFFFFF))) & M64)
    return lo + ((h * (hi - lo + 1)) >> 64)


def test_splitmix64_replica_known_values():
    # the first outputs of the reference SplitMix64 generator seeded with 0 (state += golden gamma, then the finaliser)
    assert splitmix64(0) == 0xE220A8397B1DCDAF
    assert splitmix64(0x9E3779B97F4A7C15) == 0x6E789E6AA1B965F4


@pytest.mark.parametrize("lo,hi", [(0, 0), (17, 17), (5, 6), (0, 1), (100, 101), (3, 5), (0, 999),
                                   (12345, 12345 + (1 << 20) + 7), (0, (1 << 40) + 3)])
def test_oracle_draw_equals_python_replica(lo, hi):
    rng = np.random.default_rng(lo ^ hi)
    seeds = [0, 1, M64, 0xDEADBEEFCAFEF00D] + [int(x) for x in rng.integers(0, 2**63, 6, dtype=np.int64)]
    seen = set()
    for seed in seeds:
        for env in (0, 1, 7, 4095, 65535, 2**31 - 1):
            for k in (0, 1, 2, 3, 1000, 2**31 - 1):
                got = EpisodeOracle.draw_start(seed, env, k, lo, hi)
                assert got == draw(seed, env, k, lo, hi), (seed, env, k, lo, hi)
                assert lo <= got <= hi
                seen.add(got)
    if hi - lo <= 2:
        assert seen == set(range(lo, hi + 1))   # every bar of a small range occurs


def _mk(cfgd, plugins, N, T, **kw):
    cfgd = {**S.DEFAULTS, **cfgd}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, **plugins})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"],
                       preprocessor_plugin=pl["preprocessor"], reward_plugin=pl["reward"], columns=S.OHLCV,
                       num_envs=N, **kw)
    return cfg, [synth_candles(T, 0)], [synth_minutes(T)]


CASES = {
    # equity below min_equity (FX_FLAG_BROKE), mixed with exhausted episode windows
    "broke": (dict(window_size=8, position_size=2.0e5, leverage=400.0, min_equity=9900.0), {}, dict(episode_bars=60)),
    # episode_bars: data exhaustion of the episode window
    "exhausted": (dict(window_size=8, sl_pips=3.0, tp_pips=4.0, commission=2e-5),
                  dict(strategy="direct_fixed_sltp", reward="sharpe_reward"), dict(episode_bars=40)),
}


def _record_from_step(orc, i, info, summ, start, k):
    """What the record of env i must hold, from info() / summary() taken right after the episode's last step."""
    rec = dict(start=start, bars=info["bar_index"][i], equity=info["equity"][i], commission=info["commission_paid"][i],
               end_flags=int(info["flags"][i]) & 14, dd_max_pct=summ["max_drawdown_pct"][i],
               dd_max_money=summ["max_drawdown_money"][i], opened=summ["trades_total"][i], closed=summ["trades_closed"][i],
               won=summ["trades_won"][i], lost=summ["trades_lost"][i], index=k)
    if summ["trades_closed"][i] > 0:
        rec["pnl_net"] = summ["avg_trade_pnl"][i] * summ["trades_closed"][i]
    return rec


def _check_record(last, want, tag):
    F = EpisodeOracle.EPISODE_FIELDS
    for key, v in want.items():
        got = last[F.index(key)]
        if key == "pnl_net":   # avg * n rounds: compare the average instead
            assert got / want["closed"] == pytest.approx(v / want["closed"], rel=1e-12, abs=1e-12), f"{tag}: {key}"
        else:
            assert got == v, f"{tag}: {key} {got!r} vs {v!r}"


@pytest.mark.parametrize("case", sorted(CASES))
def test_record_equals_info_and_summary_at_the_terminating_step(case):
    cfgd, plugins, kw = CASES[case]
    N, T, steps = 24, 900, 260
    cfg, candles, minutes = _mk(cfgd, plugins, N, T, auto_reset=1, **kw)
    orc = EpisodeOracle(cfg, candles, minutes)
    lo, hi = np.arange(N) * 3, np.arange(N) * 3 + 400
    orc.set_episode_starts(lo, hi, seed=99)
    orc.reset()
    begun = np.ones(N, np.int64)                        # the first reset began episode 0
    start0, done0, _ = orc.episodes()
    assert np.all(done0 == 0)
    for i in range(N):
        assert start0[i] == draw(99, i, 0, lo[i], hi[i])
    pending = {}
    rng = np.random.default_rng(3)
    ends, kinds = 0, set()
    for k in range(steps):
        _, _, _, term = orc.step(rng.integers(0, 3, N).astype(np.int32))
        start, done, last = orc.episodes()
        for i in list(pending):                         # this step auto-reset env i: its record is the pending one
            want, idx = pending.pop(i)
            assert done[i] == idx + 1, f"{case} step {k} env {i}: episodes_done"
            _check_record(last[i], want, f"{case} step {k} env {i}")
            assert start[i] == draw(99, i, begun[i], lo[i], hi[i]), "new start drawn with the next k"
            begun[i] += 1
        if term.any():
            info, summ = orc.info(), orc.summary()
            for i in np.nonzero(term)[0]:
                pending[int(i)] = (_record_from_step(orc, i, info, summ, start[i], begun[i] - 1), int(done[i]))
                ends += 1
                kinds.add(pending[int(i)][0]["end_flags"])
        assert np.all(done == begun - 1), f"{case} step {k}: one record per finished episode"
    assert ends >= N, f"{case}: only {ends} episodes ended"
    assert kinds == ({2 | 8, 2 | 4} if case == "broke" else {2 | 4}), kinds
    orc.close()


def test_record_of_an_explicitly_cut_episode_and_counters():
    cfgd, plugins, kw = CASES["exhausted"]
    N, T = 16, 700
    cfg, candles, minutes = _mk(cfgd, plugins, N, T, **kw)    # no auto-reset
    orc = EpisodeOracle(cfg, candles, minutes)
    starts = np.arange(N) * 11
    orc.reset(starts)
    assert np.all(orc.episodes()[1] == 0), "the first reset after create records nothing"
    orc.reset(starts)                                         # nothing stepped: still nothing to record
    assert np.all(orc.episodes()[1] == 0)
    rng = np.random.default_rng(8)
    for _ in range(25):
        orc.step(rng.integers(0, 3, N).astype(np.int32))
    info, summ = orc.info(), orc.summary()
    mask = (np.arange(N) % 2).astype(np.uint8)
    orc.reset(None, mask)                                     # cut short: end flags 0
    start, done, last = orc.episodes()
    np.testing.assert_array_equal(done, mask.astype(np.int32))
    for i in np.nonzero(mask)[0]:
        want = _record_from_step(orc, i, info, summ, starts[i], 1)   # the second episode begun (index 1)
        assert want["end_flags"] == 0
        _check_record(last[i], want, f"cut env {i}")
    # ranges cleared again: reset() without start bars restarts at the current start
    orc.set_episode_starts(np.zeros(N, np.int64), np.full(N, 300), seed=5)
    orc.set_episode_starts(None)
    orc.reset()
    np.testing.assert_array_equal(orc.episodes()[0], starts)
    orc.close()
