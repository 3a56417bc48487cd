"""GPU (-m gpu): episode start ranges and episode records (include/fxenv.h fxenv_set_reset_starts,
fxenv_get_episode_info; VecFxEnv.set_episode_starts / episode_stats).

  * lockstep against the C oracle with ranges set: several pairs of different lengths, auto-reset, short episode
    windows and a broke-prone account; every step's outputs, info and summary, and the current start, the episode
    counters and the record (integers and fp64 bit for bit);
  * both step_many engines against single steps, with many resets inside a batch: identical state blobs;
  * the closed loop (fxenv_rollout) against a twin env stepped with the recorded actions: identical outputs and blobs;
  * a snapshot restored into a fresh env continues with the same draws;
  * the draws are uniform (chi-square, p = 1e-4);
  * with the ranges cleared the state is bit-identical to an env that never had them; bad ranges and calls before the
    candles are loaded are errors."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import scenarios as S
from common_gpu import GpuVec, compare_info, compare_step, compare_summary, gpu_summary
from gym_fx_b200 import _native
from gym_fx_b200.config import lower_config
from gym_fx_b200.synth import start_offsets, synth_candles, synth_minutes
from gym_fx_b200.vec_env import VecFxEnv
from episode_oracle import EpisodeOracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    assert torch.cuda.is_available(), "GPU tests selected but no CUDA device is visible"


def _cfg(cfgd, plugins, N, pairs=1, **kw):
    cfgd = {**S.DEFAULTS, **cfgd}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, **plugins})
    return lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"],
                        preprocessor_plugin=pl["preprocessor"], reward_plugin=pl["reward"], columns=S.OHLCV,
                        num_envs=N, num_pairs=pairs, **kw)


FW = {"feature_columns": list(S.OHLCV)}
LOCKSTEP = {
    # default strategy, huge position against a high floor: many envs go broke, the rest exhaust their window
    "broke_default": (dict(window_size=8, position_size=2.0e5, leverage=400.0, min_equity=9900.0), {}),
    # brackets, commission, rolling z-score features, Sharpe ring
    "fixed_fw_sharpe": (dict(window_size=16, sl_pips=3.0, tp_pips=4.0, commission=2e-5, **FW),
                        dict(strategy="direct_fixed_sltp", preprocessor="feature_window_preprocessor",
                             reward="sharpe_reward")),
}


def _ranges(N, Ts):
    """Per-env ranges over the env's own table: wide ones, a single bar (lo == hi) and spans of 2 and 3."""
    lo, hi = np.zeros(N, np.int64), np.zeros(N, np.int64)
    for i in range(N):
        T = Ts[i % len(Ts)]
        kind = i % 4
        lo[i] = (7 * i) % 200
        hi[i] = {0: T - 1, 1: lo[i], 2: lo[i] + 1, 3: lo[i] + 2}[kind]
    return lo, hi


def _compare_summary(tag, gpu_env, osum):
    """compare_summary, with sqn checked where it is well conditioned: the device evaluates it from the running sum and sum
    of squares, the oracle from the list of trades, and when the closed trades' results are nearly equal the variance
    E[x^2] - mean^2 cancels to far fewer digits than 1e-9 (SQN values of 50 and more).  Its inputs, the sum and sum of
    squares, are compared bit for bit through the episode records."""
    gs = gpu_summary(gpu_env)
    compare_summary(tag, {**gs, "sqn": np.full_like(gs["sqn"], np.nan)}, {**osum, "sqn": np.full_like(osum["sqn"], np.nan)})
    a, b = gs["sqn"], osum["sqn"]
    assert np.array_equal(np.isnan(a), np.isnan(b)), f"{tag}: sqn NaN pattern"
    rs = gpu_env.run_stats().cpu().numpy()
    n = np.maximum(gpu_env.info()["trades"].cpu().numpy().astype(np.float64), 1.0)
    ex2, mean = rs[:, _native.RS["pnl_sq"]] / n, rs[:, _native.RS["pnl_net"]] / n
    ok = ~np.isnan(a) & (ex2 - mean * mean > 1e-4 * ex2)
    np.testing.assert_allclose(a[ok], b[ok], rtol=1e-9, atol=1e-12, err_msg=f"{tag}: sqn")


def _gpu_episodes(env):
    start, done, last = env._episode_views()
    return start.cpu().numpy(), done.cpu().numpy(), last.cpu().numpy()


def _compare_episodes(tag, gpu_env, orc):
    gs, gd, gl = _gpu_episodes(gpu_env)
    os_, od, ol = orc.episodes()
    np.testing.assert_array_equal(gs, os_, err_msg=f"{tag}: start")
    np.testing.assert_array_equal(gd, od, err_msg=f"{tag}: episodes_done")
    bad = np.argwhere(gl.view(np.uint64) != ol.view(np.uint64))
    assert bad.size == 0, f"{tag}: record not bit-exact at env {bad[0][0]} field {EpisodeOracle.EPISODE_FIELDS[bad[0][1]]}: " \
                          f"{gl[tuple(bad[0])]!r} vs {ol[tuple(bad[0])]!r}"


@pytest.mark.parametrize("case", sorted(LOCKSTEP))
def test_lockstep_with_oracle_auto_reset_and_ranges(case):
    cfgd, plugins = LOCKSTEP[case]
    N, Ts, steps, seed = 96, (700, 950, 1300), 170, 0xC0FFEE1234
    cfg = _cfg(cfgd, plugins, N, pairs=3, order_capacity=512, auto_reset=1, episode_bars=40)
    candles = [synth_candles(T, p) for p, T in enumerate(Ts)]
    minutes = [synth_minutes(T) for T in Ts]
    gpu, orc = GpuVec(cfg, candles, minutes), EpisodeOracle(cfg, candles, minutes)
    lo, hi = _ranges(N, Ts)
    gpu.env.set_episode_starts(lo, hi, seed)
    orc.set_episode_starts(lo, hi, seed)
    np.testing.assert_allclose(gpu.reset(), orc.reset(), rtol=1e-5, atol=2e-6, err_msg="reset obs")
    _compare_episodes(f"{case} reset", gpu.env, orc)
    rng = np.random.default_rng(17)
    ends, kinds = 0, set()
    for k in range(steps):
        a = rng.integers(0, 3, N).astype(np.int32)
        go, oo = gpu.step(a), orc.step(a)
        compare_step(f"{case} step {k}", go, oo)
        compare_info(f"{case} step {k}", gpu.info(), orc.info())
        _compare_summary(f"{case} step {k}", gpu.env, orc.summary())
        _compare_episodes(f"{case} step {k}", gpu.env, orc)
        ends += int(oo[3].sum())
        kinds |= set((orc.info()["flags"][oo[3] == 1] & 14).tolist())
        if k == 90:      # explicit reset of a third of the envs without start bars: drawn, the episodes cut short
            mask = (np.arange(N) % 3 == 0).astype(np.uint8)
            np.testing.assert_allclose(gpu.reset(None, mask), orc.reset(None, mask), rtol=1e-5, atol=2e-6)
            _compare_episodes(f"{case} masked reset", gpu.env, orc)
        if k == 130:     # explicit start bars win over the ranges
            starts = (np.arange(N) * 5) % 600
            np.testing.assert_allclose(gpu.reset(starts), orc.reset(starts), rtol=1e-5, atol=2e-6)
            _compare_episodes(f"{case} explicit reset", gpu.env, orc)
            np.testing.assert_array_equal(_gpu_episodes(gpu.env)[0], starts)
    assert ends >= 2 * N, f"{case}: only {ends} episodes ended"
    if case == "broke_default":
        assert 10 in kinds and 6 in kinds, kinds   # broke and exhausted episodes both occurred
    st = gpu.env.episode_stats()
    assert int(st["episodes_done"].min()) >= 2
    gpu.close(); orc.close()


def _engine_env(eng, cfg, candles, minutes):
    os.environ["FXENV_ENGINE"] = eng
    try:
        return VecFxEnv(cfg, candles, minutes)
    finally:
        del os.environ["FXENV_ENGINE"]


@pytest.mark.parametrize("case", ["cfg2_lean", "atr_dd_2pairs"])
def test_step_many_engines_match_single_steps_with_draws(case):
    if case == "cfg2_lean":   # the BASELINE cfg2 shape: the specialised (LEAN) kernels
        cfg = _cfg(dict(window_size=128, **FW), dict(strategy="direct_fixed_sltp", preprocessor="feature_window_preprocessor"),
                   700, order_capacity=256, auto_reset=1, episode_bars=9)
        Ts = (3000,)
    else:
        cfg = _cfg(dict(window_size=32, commission=1e-5, **FW), dict(strategy="direct_atr_sltp",
                   preprocessor="feature_window_preprocessor", reward="dd_penalized_reward"), 700, pairs=2,
                   order_capacity=256, auto_reset=1, episode_bars=9)
        Ts = (3000, 2100)
    N, K = cfg.num_envs, 40
    candles, minutes = [synth_candles(T, p) for p, T in enumerate(Ts)], [synth_minutes(T) for T in Ts]
    lo, hi = _ranges(N, Ts)
    acts = torch.randint(0, 3, (2, K, N), dtype=torch.int32, generator=torch.Generator().manual_seed(4)).cuda()
    blobs, outs = [], []
    for eng in ("persistent", "graph", "single"):
        env = _engine_env("graph" if eng == "single" else eng, cfg, candles, minutes)
        env.set_episode_starts(lo, hi, seed=2**64 - 5)
        env.reset()
        ring = torch.zeros((2, N, env.obs_dim), dtype=torch.float32, device="cuda")
        rews = torch.zeros((2, K, N), dtype=torch.float32, device="cuda")
        terms = torch.zeros((2, K, N), dtype=torch.uint8, device="cuda")
        for b in range(2):
            if eng == "single":
                for k in range(K):
                    env.step(acts[b, k], out_obs=ring[k % 2])
                    rews[b, k] = env.reward
                    terms[b, k] = env.terminated
            else:
                assert env.step_many_engine(K) == eng
                env.step_many(acts[b], ring, rews[b], terms[b])
        torch.cuda.synchronize()
        blobs.append(env.get_state())
        outs.append((ring, rews, terms))
        done = env.episode_stats()["episodes_done"]
        assert int(done.min()) >= 6, "several resets per env inside the batches"
        env.close()
    for o in outs[1:]:
        assert all(torch.equal(x, y) for x, y in zip(outs[0], o))
    assert blobs[0] == blobs[1] == blobs[2]


def test_closed_loop_rollout_matches_twin_with_draws():
    from gym_fx_b200.learner import ActorCritic
    N, H, T = 600, 24, 4000
    cfg = _cfg(dict(window_size=128, **FW), dict(strategy="direct_fixed_sltp", preprocessor="feature_window_preprocessor",
                                                 reward="sharpe_reward"), N, order_capacity=256, auto_reset=1, episode_bars=7)
    candles, minutes = [synth_candles(T, 0)], [synth_minutes(T)]
    env, twin = VecFxEnv(cfg, candles, minutes), VecFxEnv(cfg, candles, minutes)
    lo, hi = _ranges(N, (T,))
    for e in (env, twin):
        e.set_episode_starts(lo, hi, seed=31337)
        e.reset()
    torch.manual_seed(0)
    pol = env.make_policy(ActorCritic(env.obs_dim).cuda())
    for rep in range(2):        # the second rollout replays the cached graph after more draws
        out = env.rollout(pol, H, seed=11 + rep)
        torch.cuda.synchronize()
        for t in range(H):
            o, r, term, _, _ = twin.step(out["actions"][t])
            assert torch.equal(o, out["obs"][t + 1]) and torch.equal(r, out["reward"][t]), (rep, t)
            assert torch.equal(term.to(torch.uint8), out["done"][t]), (rep, t)
        assert env.get_state() == twin.get_state(), rep
    assert int(env.episode_stats()["episodes_done"].min()) >= 4
    env.close(); twin.close()


def test_snapshot_continues_with_the_same_draws():
    N, T, K = 256, 2500, 60
    cfg = _cfg(dict(window_size=16, sl_pips=3.0, tp_pips=4.0), dict(strategy="direct_fixed_sltp"), N, order_capacity=256,
               auto_reset=1, episode_bars=11)
    candles, minutes = [synth_candles(T, 0)], [synth_minutes(T)]
    a = VecFxEnv(cfg, candles, minutes)
    a.set_episode_starts(100, 2000, seed=77)
    a.reset()
    acts = torch.randint(0, 3, (2 * K, N), dtype=torch.int32, generator=torch.Generator().manual_seed(9)).cuda()
    for k in range(K):
        a.step(acts[k])
    blob = a.get_state()
    b = VecFxEnv(cfg, candles, minutes)      # never had ranges: the snapshot carries them, the seed and the counters
    b.set_state(blob)
    for k in range(K, 2 * K):
        oa, ra, _, _, _ = a.step(acts[k])
        ob, rb, _, _, _ = b.step(acts[k])
        assert torch.equal(oa, ob) and torch.equal(ra, rb), k
    a.reset(); b.reset()                      # explicit draws, too
    assert a.get_state() == b.get_state()
    sa, sb = a.episode_stats(), b.episode_stats()
    assert torch.equal(sa["start"], sb["start"]) and int(sa["episodes_done"].min()) >= 6
    assert bool(((sa["start"] >= 100) & (sa["start"] <= 2000)).all())
    a.close(); b.close()


def test_draws_are_uniform():
    from scipy.stats import chisquare
    N, T = 4096, 5000
    cfg = _cfg(dict(window_size=8), {}, N)
    env = VecFxEnv(cfg, [synth_candles(T, 0)], [synth_minutes(T)])
    for lo, hi, resets in ((40, 49, 8), (0, T - 1, 25)):
        env.set_episode_starts(lo, hi, seed=123456789)
        draws = []
        for _ in range(resets):
            env.reset()
            draws.append(env.episode_stats()["start"].cpu().numpy().copy())
        d = np.concatenate(draws)
        assert d.min() >= lo and d.max() <= hi
        bins = 10 if hi - lo + 1 == 10 else 50
        counts = np.bincount((d - lo) * bins // (hi - lo + 1), minlength=bins)
        p = chisquare(counts).pvalue
        assert p > 1e-4, (lo, hi, p, counts)
        assert len(np.unique(np.stack(draws)[:, :64], axis=0)) == resets   # new draws at every reset
    env.close()


def test_cleared_ranges_are_the_default_and_errors():
    N, T, K = 128, 1500, 50
    cfg = _cfg(dict(window_size=8), dict(strategy="direct_fixed_sltp"), N, order_capacity=128, auto_reset=1, episode_bars=13)
    candles, minutes = [synth_candles(T, 0)], [synth_minutes(T)]
    plain, cleared = VecFxEnv(cfg, candles, minutes), VecFxEnv(cfg, candles, minutes)
    cleared.set_episode_starts(0, T - 1, seed=5)
    cleared.set_episode_starts(None)
    starts = torch.as_tensor(start_offsets(N, T, 100, 300))
    acts = torch.randint(0, 3, (K, N), dtype=torch.int32, generator=torch.Generator().manual_seed(1)).cuda()
    for e in (plain, cleared):
        e.reset(starts)
        for k in range(K):
            e.step(acts[k])
        e.reset()
    torch.cuda.synchronize()
    assert plain.get_state() == cleared.get_state()
    st = plain.episode_stats()
    assert torch.equal(st["start"].cpu(), starts), "without ranges an episode restarts at its start"
    # argument errors (VecFxEnv) and the library's own checks
    for lo, hi in ((-1, 5), (6, 5), (0, T), (np.zeros(N + 1, np.int64), np.ones(N + 1, np.int64)), (1.5, 3), (0, None)):
        with pytest.raises(ValueError):
            plain.set_episode_starts(lo, hi)
    with pytest.raises(ValueError):
        plain.set_episode_starts(0, 5, seed=-1)
    L = plain.L
    lo_bad, hi_bad = np.zeros(N, np.int64), np.full(N, T, np.int64)
    assert L.fxenv_set_reset_starts(plain._h, lo_bad.ctypes.data, hi_bad.ctypes.data, 0) == -1
    assert L.fxenv_set_reset_starts(plain._h, lo_bad.ctypes.data, None, 0) == -1
    h = C.c_void_p()
    assert L.fxenv_create(C.byref(cfg), C.byref(h)) == 0
    try:
        lo_ok = np.zeros(N, np.int64)
        assert L.fxenv_set_reset_starts(h, lo_ok.ctypes.data, lo_ok.ctypes.data, 0) == -3   # FXENV_E_STATE
        assert b"not loaded" in L.fxenv_last_error(h)
    finally:
        L.fxenv_destroy(h)
    plain.close(); cleared.close()
