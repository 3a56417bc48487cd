"""GPU (-m gpu): a candle table reloaded through the C-ABI (fxenv_load_candles on a handle that has already run) reaches
every cached graph.  The graphs capture the kernel parameters by value: the table's pointers, tame_data and the LEAN
choice all change with a reload.

  * The closed loop: a rollout graph cached on a non-default stream, then a reload of pair 0 (same length, other values,
    with or without NaN), a reset to the same start bars and a rollout on the same buffers and seed.  A twin handle given
    the same loads and resets and stepped with the rollouts' actions by step() gives the same observations, rewards and
    state, bit for bit.  A LEAN and a general configuration.
  * The step-many graph engine (FXENV_ENGINE=graph) across a reload, against single steps on a twin."""
import numpy as np
import pytest
import torch

import scenarios as S
from gym_fx_b200.config import lower_config
from gym_fx_b200.synth import synth_candles, synth_minutes
from gym_fx_b200.vec_env import VecFxEnv

pytestmark = pytest.mark.gpu

# name -> (config, plugins, pairs)
CONFIGS = {
    # the cfg2 shape: the LEAN kernels while every table is finite
    "lean": (dict(window_size=32, sl_pips=3.0, tp_pips=4.0, feature_scaling_window=16, feature_columns=list(S.OHLCV)),
             dict(strategy="direct_fixed_sltp", preprocessor="feature_window_preprocessor"), 1),
    # the general kernels: ATR brackets, the drawdown-penalised reward, two pairs
    "general": (dict(window_size=16, atr_period=6), dict(strategy="direct_atr_sltp", reward="dd_penalized_reward"), 2),
}
T0 = 900  # rows of pair 0's table, before and after the reload


def _handle(name, N):
    cfgd, plugins, pairs = CONFIGS[name]
    cfgd = {**S.DEFAULTS, **cfgd}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, **plugins})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"],
                       preprocessor_plugin=pl["preprocessor"], reward_plugin=pl["reward"], columns=S.OHLCV,
                       num_envs=N, num_pairs=pairs, order_capacity=256, episode_bars=37)
    cfg.auto_reset = 1
    Ts = [T0 + 130 * p for p in range(pairs)]
    env = VecFxEnv(cfg, [synth_candles(T, p) for p, T in enumerate(Ts)], [synth_minutes(T) for T in Ts])
    env.set_episode_starts(40, T0 - 80, seed=21)   # auto-resets draw starts all over the reloaded table
    return env


def _reload(env, nan):
    """Pair 0's table replaced by one of the same length with other values; with `nan` every 41st volume is NaN."""
    tab = synth_candles(T0, 0, seed=7)
    if nan:
        tab[::41, 4] = np.nan
    minutes = synth_minutes(T0)
    with torch.cuda.device(env.device):
        rc = env.L.fxenv_load_candles(env._h, 0, tab.ctypes.data, T0, minutes.ctypes.data)
    assert rc == 0, env.L.fxenv_last_error(env._h).decode()


def _same(x, y):
    return x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes()


def _starts(N):
    return (torch.arange(N, dtype=torch.int64, device="cuda") * 7) % 400 + 40


@pytest.mark.parametrize("nan", [False, True], ids=["finite", "nan"])
@pytest.mark.parametrize("name", ["lean", "general"])
def test_rollout_after_a_reload_replays_through_step_on_a_twin(name, nan):
    from gym_fx_b200.learner import ActorCritic
    N, H = 128, 12
    a, b = _handle(name, N), _handle(name, N)
    assert a.L.fxenv_debug_lean(a._h) == (1 if name == "lean" else 0)
    torch.manual_seed(3)
    pol = a.make_policy(ActorCritic(a.obs_dim).cuda())
    bufs = None
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):   # a non-default stream: the rollout graph is captured and cached
        starts = _starts(N)
        for reload in (False, True):
            if reload:
                _reload(a, nan)
                _reload(b, nan)
                assert a.L.fxenv_debug_lean(a._h) == (1 if name == "lean" and not nan else 0)
            a.reset(starts)
            o0 = b.reset(starts)[0].clone()
            bufs = a.rollout(pol, H, buffers=bufs, seed=11)
            s.synchronize()
            assert _same(o0, bufs["obs"][0]), reload
            for t in range(H):
                o, r, _, _, _ = b.step(bufs["actions"][t])
                s.synchronize()
                assert _same(o, bufs["obs"][t + 1]) and _same(r, bufs["reward"][t]), (reload, t)
            assert a.get_state() == b.get_state(), reload
    a.close(), b.close()


@pytest.mark.parametrize("name", ["lean", "general"])
def test_step_many_graph_engine_across_a_reload(name, monkeypatch):
    N, K = 64, 12
    monkeypatch.setenv("FXENV_ENGINE", "graph")
    a = _handle(name, N)
    monkeypatch.delenv("FXENV_ENGINE")
    b = _handle(name, N)
    assert a.step_many_engine(K) == "graph"
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):   # a non-default stream: the graph engine captures and caches
        acts = torch.as_tensor(np.random.default_rng(2).integers(0, 3, (K, N)).astype(np.int32)).cuda()
        ring = torch.empty((K, N, a.obs_dim), dtype=torch.float32, device="cuda")
        rew = torch.empty((K, N), dtype=torch.float32, device="cuda")
        term = torch.empty((K, N), dtype=torch.uint8, device="cuda")
        starts = _starts(N)
        for reload in (False, True):
            if reload:
                _reload(a, True)
                _reload(b, True)
            a.reset(starts)
            b.reset(starts)
            a.step_many(acts, ring, rew, term)
            s.synchronize()
            for j in range(K):
                o, r, t, _, _ = b.step(acts[j])
                s.synchronize()
                assert _same(o, ring[j]) and _same(r, rew[j]) and _same(t.to(torch.uint8), term[j]), (reload, j)
            assert a.get_state() == b.get_state(), reload
    a.close(), b.close()
