"""CPU (-m "not gpu"): the time limit and truncation of include/fxenv.h (fxenv_set_time_limit) restated around the C
oracle (tests/time_limit_oracle.py), and the learner's GAE on the done codes.
  * the wrapper on hand-counted cases: limit 1, a limit that lands on the broke step, the limit with k = 3 in repeat and
    hold mode, the WINDOW rule with episode_bars, a limit set in the middle of an episode, and no truncation at all;
  * gae: bit-identical to the formula before the codes on random 0 / 1 buffers; a three-step hand-computed case where a
    truncation bootstraps value[t + 1] and a termination does not; the masks of the step after each kind of end."""
import numpy as np
import pytest
import torch

import scenarios as S
from gym_fx_b200.config import lower_config
from gym_fx_b200.learner import gae
from gym_fx_b200.synth import synth_candles, synth_minutes
from repeat_oracle import RepeatOracle
from time_limit_oracle import FLAG_TRUNCATED, TimeLimitOracle

FIXED = (dict(window_size=8, sl_pips=3.0, tp_pips=4.0), dict(strategy="direct_fixed_sltp"))
BROKE = (dict(window_size=8, position_size=2.0e5, leverage=400.0, min_equity=9900.0), {})


def _mk(cfgd, plugins, N, T, **kw):
    cfgd = {**S.DEFAULTS, **cfgd}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, **plugins})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"],
                       preprocessor_plugin=pl["preprocessor"], reward_plugin=pl["reward"], columns=S.OHLCV,
                       num_envs=N, **kw)
    return cfg, [synth_candles(T, 0)], [synth_minutes(T)]


def _codes(o, acts):
    return np.stack([o.step(a)[3] for a in acts])


def test_limit_1_cuts_every_first_decision():
    N, T = 4, 400
    cfg, candles, minutes = _mk(*FIXED, N, T, auto_reset=1)
    o = TimeLimitOracle(cfg, candles, minutes, max_steps=1)
    o.reset(np.zeros(N, np.int64))
    c = _codes(o, np.ones((6, N), np.int32))
    # decision 1 is cut, the next step is the reset step (code 0, not counted), then decision 1 of the next episode
    assert (c == np.array([[2], [0], [2], [0], [2], [0]])).all()
    _, done, last = o.episodes()
    assert (done == 3).all() and (last[:, 4].astype(int) == FLAG_TRUNCATED).all()
    assert (last[:, 1] == 1).all(), "a cut first decision does not advance the bar"
    o.close()


def test_limit_on_the_broke_step_is_a_termination():
    N, T = 8, 400
    cfg, candles, minutes = _mk(*BROKE, N, T, auto_reset=0)
    acts = np.random.default_rng(2).integers(0, 3, (80, N)).astype(np.int32)
    probe = TimeLimitOracle(cfg, candles, minutes)
    probe.reset(np.zeros(N, np.int64))
    c0 = _codes(probe, acts)
    probe.close()
    ends = [(int(np.nonzero(c0[:, i] == 1)[0][0]) + 1, i) for i in range(N) if (c0[:, i] == 1).any()]
    broke, i = min(e for e in ends if e[0] > 2)    # decisions up to and including env i's broke one
    for limit, want in ((broke, 1), (broke - 1, 2)):
        o = TimeLimitOracle(cfg, candles, minutes, max_steps=limit)
        o.reset(np.zeros(N, np.int64))
        c = _codes(o, acts[:broke + 3])[:, i]
        assert (c[:limit - 1] == 0).all() and c[limit - 1] == want
        assert (c[limit:] == want).all(), "without auto-reset an ended env keeps answering its code"
        flags = int(o.info()["flags"][i])
        assert bool(flags & FLAG_TRUNCATED) == (want == 2) and bool(flags & 2) == (want == 1) and bool(flags & 8) == (want == 1)
        o.close()


@pytest.mark.parametrize("hold", [False, True], ids=["repeat", "hold"])
def test_limit_counts_decisions_with_repeat(hold):
    N, T, k, M = 3, 600, 3, 4
    cfg, candles, minutes = _mk(*FIXED, N, T, auto_reset=1)
    o = TimeLimitOracle(cfg, candles, minutes, k=k, hold=hold, max_steps=M)
    o.reset(np.zeros(N, np.int64))
    c = _codes(o, np.ones((2 * (M + 1), N), np.int32))
    assert (c[M - 1] == 2).all() and (c[2 * M] == 2).all()
    assert (c[:M - 1] == 0).all() and (c[M] == 0).all()
    # the cut episode ran M decisions of k bars each, the first of which covers k - 1 bars
    _, done, last = o.episodes()
    assert (done == 2).all() and (last[:, 1] == 1 + M * k - 1).all()
    o.close()


def test_window_rule_with_episode_bars():
    N, T, B = 2, 500, 7
    for window, want in ((False, 1), (True, 2)):
        cfg, candles, minutes = _mk(*FIXED, N, T, auto_reset=1, episode_bars=B)
        o = TimeLimitOracle(cfg, candles, minutes, window=window)
        o.reset(np.zeros(N, np.int64))
        c = _codes(o, np.zeros((2 * (B + 2), N), np.int32))
        # decisions 1..B reach the window's last bar; decision B + 1 finds it exhausted; the next step is the reset step
        assert (c[:B] == 0).all() and (c[B] == want).all() and (c[B + 1] == 0).all() and (c[2 * B + 2] == want).all()
        last = o.episodes()[2]
        assert (last[:, 4].astype(int) == (4 | 64 if window else 4 | 2)).all()
        o.close()


def test_limit_set_in_the_middle_of_an_episode():
    N, T = 2, 500
    cfg, candles, minutes = _mk(*FIXED, N, T, auto_reset=1)
    o = TimeLimitOracle(cfg, candles, minutes)
    o.reset(np.zeros(N, np.int64))
    acts = np.zeros((20, N), np.int32)
    assert (_codes(o, acts[:5]) == 0).all()
    o.set_time_limit(3)   # the running episode gets 3 more decisions
    c = _codes(o, acts[5:12])
    assert (c[:2] == 0).all() and (c[2] == 2).all() and (c[3] == 0).all() and (c[6] == 2).all()
    assert (o.episodes()[2][:, 1] == 8).all(), "5 + 3 decisions: the first one does not advance"
    o.close()


def test_off_is_the_repeat_oracle():
    N, T = 6, 700
    cfg, candles, minutes = _mk(*BROKE, N, T, auto_reset=1, episode_bars=31)
    a, b = TimeLimitOracle(cfg, candles, minutes, k=2), RepeatOracle(cfg, candles, minutes, k=2)
    for o in (a, b):
        o.reset(np.zeros(N, np.int64))
    rng = np.random.default_rng(3)
    for s in range(120):
        act = rng.integers(0, 3, N).astype(np.int32)
        for x, y in zip(a.step(act), b.step(act)):
            assert x.tobytes() == y.tobytes(), s
    for x, y in zip(a.episodes(), b.episodes()):
        assert x.tobytes() == y.tobytes()
    a.close(), b.close()


# ------------------------------------------------------------------------------------------------------------ GAE
def _gae_before(reward, value, done, prev_done, gamma=0.99, lam=0.95):
    """learner.gae as it was before the done codes (0 / 1 flags only)."""
    H = reward.shape[0]
    adv = torch.zeros_like(reward)
    last = torch.zeros_like(reward[0])
    donef = done.to(reward.dtype)
    for t in reversed(range(H)):
        nd = 1.0 - donef[t]
        delta = reward[t] + gamma * value[t + 1] * nd - value[t]
        last = delta + gamma * lam * nd * last
        adv[t] = last
    valid = torch.ones_like(reward)
    valid[0] = 1.0 - prev_done.to(reward.dtype)
    valid[1:] = 1.0 - donef[:-1]
    return adv, adv + value[:H], valid


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_gae_is_bit_identical_on_flags(dtype):
    g = torch.Generator().manual_seed(0)
    H, N = 40, 257
    reward = torch.randn((H, N), generator=g, dtype=dtype)
    value = torch.randn((H + 1, N), generator=g, dtype=dtype)
    done = (torch.rand((H, N), generator=g) < 0.1).to(torch.uint8)
    prev = (torch.rand(N, generator=g) < 0.3).to(torch.uint8)
    for x, y in zip(gae(reward, value, done, prev, 0.97, 0.9), _gae_before(reward, value, done, prev, 0.97, 0.9)):
        assert x.dtype == y.dtype and x.numpy().tobytes() == y.numpy().tobytes()


def test_gae_truncation_bootstraps_and_termination_does_not():
    gamma, lam = 0.5, 0.5
    r = torch.tensor([[1.0, 1.0], [2.0, 2.0], [4.0, 4.0]], dtype=torch.float64)
    v = torch.tensor([[10.0, 10.0], [20.0, 20.0], [30.0, 30.0], [40.0, 40.0]], dtype=torch.float64)
    # env 0: step 1 truncates (value[2] = 30 is the cut episode's final value); env 1: step 1 terminates
    done = torch.tensor([[0, 0], [2, 1], [0, 0]], dtype=torch.uint8)
    adv, ret, valid = gae(r, v, done, torch.zeros(2, dtype=torch.uint8), gamma, lam)
    d2 = 4.0 + 0.5 * 40.0 - 30.0                     # -6 (step 2: the reset step, masked below)
    d1_trunc = 2.0 + 0.5 * 30.0 - 20.0               # -3: bootstraps from value[2]
    d1_term = 2.0 - 20.0                             # -18
    d0 = 1.0 + 0.5 * 20.0 - 10.0                     # 1
    want = torch.tensor([[d0 + 0.25 * d1_trunc, d0 + 0.25 * d1_term], [d1_trunc, d1_term], [d2, d2]], dtype=torch.float64)
    assert torch.equal(adv, want)
    assert torch.equal(ret, want + v[:3])
    assert torch.equal(valid, torch.tensor([[1.0, 1.0], [1.0, 1.0], [0.0, 0.0]], dtype=torch.float64))


def test_gae_masks_the_step_after_each_kind_of_end():
    H, N = 4, 3
    r, v = torch.zeros((H, N)), torch.zeros((H + 1, N))
    done = torch.tensor([[0, 1, 2], [0, 0, 0], [2, 0, 1], [0, 0, 0]], dtype=torch.uint8)
    prev = torch.tensor([0, 1, 2], dtype=torch.uint8)
    _, _, valid = gae(r, v, done, prev)
    want = torch.tensor([[1, 0, 0], [1, 0, 0], [1, 1, 1], [0, 1, 0]], dtype=torch.float32)
    assert torch.equal(valid, want)
