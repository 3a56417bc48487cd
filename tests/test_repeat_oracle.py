"""CPU (-m "not gpu"): the action repeat of include/fxenv.h (fxenv_set_action_repeat) restated around the C oracle
(tests/repeat_oracle.py).
  * k = 1 is the unrepeated library: bit for bit EpisodeOracle, with auto-reset and episode start ranges;
  * for k in {2, 3, 8} and both modes, every step equals env i of a plain EpisodeOracle driven through env i's expanded
    action stream: its outputs at the step's last substep, its rewards summed in order;
  * the hand-checkable cases: the first decision of an episode covers k - 1 bars, a step stops at its terminating
    substep, a terminated env with auto-reset runs the reset step only, hold with threshold 0 holds, and reward64 is the
    in-order float64 sum."""
import numpy as np
import pytest

import scenarios as S
from episode_oracle import FLAG_TERMINATED, EpisodeOracle
from gym_fx_b200.config import lower_config
from gym_fx_b200.synth import synth_candles, synth_minutes
from repeat_oracle import RepeatOracle


def _mk(cfgd, plugins, N, T, **kw):
    cfgd = {**S.DEFAULTS, **cfgd}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, **plugins})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"],
                       preprocessor_plugin=pl["preprocessor"], reward_plugin=pl["reward"], columns=S.OHLCV,
                       num_envs=N, **kw)
    return cfg, [synth_candles(T, 0)], [synth_minutes(T)]


# brackets on short episodes with auto-reset: terminations fall inside steps
FIXED = (dict(window_size=8, sl_pips=3.0, tp_pips=4.0), dict(strategy="direct_fixed_sltp"))
# the default strategy with a huge position against a high floor: envs go broke
BROKE = (dict(window_size=8, position_size=2.0e5, leverage=400.0, min_equity=9900.0), {})


def _same(tag, a, b):
    assert a.shape == b.shape and a.tobytes() == b.tobytes(), tag


def _starts(o, N, T):
    lo = (np.arange(N) * 37) % (T // 2)
    o.set_episode_starts(lo, lo + 150, seed=1234)


@pytest.mark.parametrize("case", ["fixed", "broke"])
def test_k1_is_the_episode_oracle(case):
    cfgd, plugins = {"fixed": FIXED, "broke": BROKE}[case]
    N, T = 12, 900
    cfg, candles, minutes = _mk(cfgd, plugins, N, T, auto_reset=1, episode_bars=23)
    rep, ref = RepeatOracle(cfg, candles, minutes), EpisodeOracle(cfg, candles, minutes)
    for o in (rep, ref):
        _starts(o, N, T)
    _same("reset", rep.reset(), ref.reset())
    rng = np.random.default_rng(5)
    ends = 0
    for s in range(300):
        a = rng.integers(0, 3, N).astype(np.int32)
        g, w = rep.step(a), ref.step(a)
        for name, x, y in zip(("obs", "rew32", "rew64", "term"), g, w):
            _same(f"step {s}: {name}", x, y)
        ends += int(w[3].sum())
    for name, x, y in zip(("start", "done", "last"), rep.episodes(), ref.episodes()):
        _same(name, x, y)
    assert ends > N, "no terminations"


def _expanded(cfg, candles, minutes, N, T, k, hold, steps, actions):
    """Env i of its own N-env EpisodeOracle, driven through env i's expanded stream (every env of that oracle gets the
    same actions; only env i is read).  -> per step (obs [N, D], rew64 [N], term [N]) and the final episode state."""
    D = None
    outs = []
    for i in range(N):
        o = EpisodeOracle(cfg, candles, minutes)
        _starts(o, N, T)
        o.reset()
        D = o.D
        rows = []
        for s in range(steps):
            began_terminated = (int(o.info()["flags"][i]) & FLAG_TERMINATED) != 0
            acc = None
            for j in range(k):
                a = actions[s, i] if (j == 0 or not hold) else 0
                obs, _, r64, t = o.step(np.full(N, a, actions.dtype))
                acc = r64[i] if j == 0 else acc + r64[i]
                if began_terminated or t[i]:
                    break
            rows.append((obs[i].copy(), acc, t[i]))
        outs.append((rows, tuple(x[i].copy() for x in o.episodes())))
        o.close()
    per_step = []
    for s in range(steps):
        per_step.append((np.stack([outs[i][0][s][0] for i in range(N)]).reshape(N, D),
                         np.asarray([outs[i][0][s][1] for i in range(N)], np.float64),
                         np.asarray([outs[i][0][s][2] for i in range(N)], np.uint8)))
    return per_step, [outs[i][1] for i in range(N)]


@pytest.mark.parametrize("k", [2, 3, 8])
@pytest.mark.parametrize("hold", [False, True])
def test_steps_equal_the_expanded_action_stream(k, hold):
    N, T, steps = 6, 700, 40
    cfg, candles, minutes = _mk(*FIXED, N, T, auto_reset=1, episode_bars=19)
    rng = np.random.default_rng(100 * k + hold)
    actions = rng.integers(0, 3, (steps, N)).astype(np.int32)
    want, eps = _expanded(cfg, candles, minutes, N, T, k, hold, steps, actions)
    rep = RepeatOracle(cfg, candles, minutes, k=k, hold=hold)
    _starts(rep, N, T)
    rep.reset()
    multi = 0
    for s in range(steps):
        obs, r32, r64, term = rep.step(actions[s])
        _same(f"step {s}: obs", obs, want[s][0])
        _same(f"step {s}: reward64", r64, want[s][1])
        _same(f"step {s}: reward", r32, want[s][1].astype(np.float32))
        _same(f"step {s}: terminated", term, want[s][2])
        multi += int((rep.substeps > 1).sum())
    for i in range(N):
        for name, x, y in zip(("start", "done", "last"), (v[i] for v in rep.episodes()), eps[i]):
            _same(f"env {i}: {name}", np.asarray(x), np.asarray(y))
    assert multi > 0


def test_first_decision_covers_k_minus_1_bars_and_stops_at_termination():
    N, T, k = 4, 600, 5
    cfg, candles, minutes = _mk(*FIXED, N, T, auto_reset=0, episode_bars=13)
    rep = RepeatOracle(cfg, candles, minutes, k=k)
    rep.reset(np.zeros(N, np.int64))
    rep.step(np.zeros(N, np.int32))
    assert (rep.info()["bar_index"] == k).all()          # substep 0 stays on bar 0, then k - 1 bars
    assert (rep.substeps == k).all()
    rep.step(np.zeros(N, np.int32))
    assert (rep.info()["bar_index"] == 2 * k).all()
    _, _, _, term = rep.step(np.zeros(N, np.int32))       # bars 10..12 of 13; the next substep exhausts the data
    assert term.all() and (rep.substeps == 4).all() and (rep.info()["bar_index"] == 13).all()
    _, r32, r64, term = rep.step(np.zeros(N, np.int32))  # terminated without auto-reset: (obs, 0.0, True), one substep
    assert term.all() and (rep.substeps == 1).all() and (r64 == 0.0).all()


def test_terminated_env_with_auto_reset_runs_the_reset_step_only():
    N, T, k = 3, 600, 4
    cfg, candles, minutes = _mk(*FIXED, N, T, auto_reset=1, episode_bars=6)
    rep = RepeatOracle(cfg, candles, minutes, k=k)
    rep.reset(np.zeros(N, np.int64))
    rep.step(np.zeros(N, np.int32))                        # bars 0..3
    _, _, _, term = rep.step(np.zeros(N, np.int32))       # bars 4, 5, then exhausted
    assert term.all() and (rep.substeps == 3).all()
    _, _, r64, term = rep.step(np.ones(N, np.int32))      # the reset step alone: reward 0, not done, bar 1 of the new one
    assert (rep.substeps == 1).all() and not term.any() and (r64 == 0.0).all()
    assert (rep.info()["bar_index"] == 1).all() and (rep.info()["position"] == 0).all()
    assert (rep.episodes()[1] == 1).all()


def test_hold_with_threshold_zero_holds_in_continuous_mode():
    N, T, k = 2, 600, 4
    cfg, candles, minutes = _mk({"window_size": 8, "action_space_mode": "continuous", "continuous_action_threshold": 0.0},
                                {}, N, T)
    assert cfg.continuous_action_threshold == 0.0
    hold = RepeatOracle(cfg, candles, minutes, k=k, hold=True)
    ref = EpisodeOracle(cfg, candles, minutes)
    for o in (hold, ref):
        o.reset(np.zeros(N, np.int64))
    a = np.asarray([0.9, -0.9], np.float32)
    for _ in range(2):   # the first decision's action is placed on bar 0 and fills on bar 1
        hold.step(a)
        for j in range(k):
            ref.step(a if j == 0 else np.zeros(N, np.float32))
    for name in ("position_size", "cash", "equity", "trades", "position"):
        _same(name, hold.info()[name], ref.info()[name])
    assert (ref.info()["position"] == [1, -1]).all()


def test_reward64_is_the_in_order_float64_sum():
    N, T, k = 5, 800, 6
    cfg, candles, minutes = _mk(*FIXED, N, T)
    rep, ref = RepeatOracle(cfg, candles, minutes, k=k), EpisodeOracle(cfg, candles, minutes)
    for o in (rep, ref):
        o.reset(np.arange(N) * 11)
    rng = np.random.default_rng(9)
    nonzero = 0
    for s in range(12):
        a = rng.integers(0, 3, N).astype(np.int32)
        _, r32, r64, _ = rep.step(a)
        assert (rep.substeps == k).all()   # no termination inside: the reference steps k times in lock step
        parts = [ref.step(a)[2] for _ in range(k)]
        want = parts[0].copy()
        for p in parts[1:]:
            want = want + p
        _same(f"step {s}", r64, want)
        _same(f"step {s} (float32)", r32, want.astype(np.float32))
        nonzero += int((want != 0).sum())
    assert nonzero > 0
