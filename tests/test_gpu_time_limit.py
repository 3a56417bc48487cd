"""GPU (-m gpu): the time limit and truncation (include/fxenv.h fxenv_set_time_limit; VecFxEnv.set_time_limit).

  * Lock step with tests/time_limit_oracle.py: fixed and ATR strategies; pnl, Sharpe and drawdown rewards; discrete and
    continuous actions; 1 and 3 pairs; a broke-prone account; auto_reset 0 and 1; k = 1 and k = 3 in repeat and hold
    mode; the limit only, the WINDOW rule only, and both.  Codes, integer and fp64 state, the flags (TRUNCATED
    included) and the episode records bit for bit; rewards and observations at the usual tolerances.
  * The engines agree bit for bit: step, step_many persistent (shared-memory and global order table, tickets that end
    mid-episode) and graph, and step_host.
  * A rollout replays through step() on a twin handle; at every code-2 step t, obs[t + 1] is the cut episode's final
    observation and step t + 1 is the reset step.
  * Switching: set_time_limit(0) equals a handle never set; a new limit between two step_many calls and between two
    rollouts on the same buffers takes effect; a snapshot continues identically on a fresh handle with the same limit;
    bad arguments raise; GymFxEnv with max_episode_steps returns (..., False, True, ...) exactly at the cut."""
import numpy as np
import pytest
import torch

import scenarios as S
from common_gpu import GpuVec, compare_info, compare_step
from gym_fx_b200.config import lower_config
from gym_fx_b200.synth import synth_candles, synth_minutes
from gym_fx_b200.vec_env import VecFxEnv
from time_limit_oracle import FLAG_TRUNCATED, TimeLimitOracle

pytestmark = pytest.mark.gpu

FW = {"feature_columns": list(S.OHLCV)}
FWP = {"preprocessor": "feature_window_preprocessor"}
END_BITS = 2 | 4 | 8 | FLAG_TRUNCATED

# name -> (config, plugins, pairs)
CONFIGS = {
    "fixed_pnl": (dict(window_size=32, sl_pips=3.0, tp_pips=4.0, feature_scaling_window=16, **FW),
                  dict(strategy="direct_fixed_sltp", **FWP), 1),
    "atr_dd": (dict(window_size=16, atr_period=6), dict(strategy="direct_atr_sltp", reward="dd_penalized_reward"), 1),
    "sharpe_3pairs": (dict(window_size=16, sl_pips=3.0, tp_pips=4.0, window=12, **FW),
                      dict(strategy="direct_fixed_sltp", reward="sharpe_reward", **FWP), 3),
    "continuous": (dict(window_size=12, action_space_mode="continuous", continuous_action_threshold=0.0), {}, 1),
    "broke": (dict(window_size=8, position_size=2.0e5, leverage=400.0, min_equity=9900.0), {}, 1),
}
# mode -> (max_steps, window)
MODES = {"limit": (9, False), "window": (0, True), "both": (13, True)}


def _cfg(name, N, episode_bars=23, auto_reset=1):
    """episode_bars: bars of an episode window (the lock step scales it with k)."""
    cfgd, plugins, pairs = CONFIGS[name]
    cfgd = {**S.DEFAULTS, **cfgd}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, **plugins})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"],
                       preprocessor_plugin=pl["preprocessor"], reward_plugin=pl["reward"], columns=S.OHLCV,
                       num_envs=N, num_pairs=pairs, order_capacity=256, episode_bars=episode_bars)
    cfg.auto_reset = auto_reset
    Ts = [900 + 130 * p for p in range(pairs)]
    return cfg, [synth_candles(T, p) for p, T in enumerate(Ts)], [synth_minutes(T) for T in Ts], Ts


def _ranges(N, Ts, tail=0):
    """Start ranges; tail > 0: every 8th env starts inside the last tail bars of its table (a short window)."""
    lo = np.asarray([(29 * i) % (Ts[i % len(Ts)] // 2) for i in range(N)], np.int64)
    hi = lo + np.asarray([[0, 1, 90, 300][i % 4] for i in range(N)], np.int64)
    if tail:
        for i in range(7, N, 8):
            T = Ts[i % len(Ts)]
            lo[i], hi[i] = T - tail, T - tail // 2
    return lo, hi


def _actions(cfg, rng, shape):
    if cfg.action_mode == 1:
        return rng.uniform(-1.0, 1.0, shape).astype(np.float32)
    return rng.integers(0, 3, shape).astype(np.int32)


def _gpu_step(env, a):
    """-> (obs, rew32, rew64, code) of VecFxEnv.step, checking its bool split against the codes."""
    obs, rew, term, trunc, _ = env.step(torch.as_tensor(np.ascontiguousarray(a)))
    code = env.terminated.cpu().numpy().copy()
    assert np.array_equal(term.cpu().numpy(), code == 1) and np.array_equal(trunc.cpu().numpy(), code == 2)
    return obs.cpu().numpy(), rew.cpu().numpy(), env.reward64.cpu().numpy(), code


# ---------------------------------------------------------------------------------------------- lock step with oracle
@pytest.mark.parametrize("rep", ["k1", "k3repeat", "k3hold"])
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("auto_reset", [0, 1])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_lockstep_with_the_time_limit_oracle(name, auto_reset, mode, rep):
    N, steps = 32, 45
    k, hold = (1, False) if rep == "k1" else (3, rep == "k3hold")
    max_steps, window = MODES[mode]
    cfg, candles, minutes, Ts = _cfg(name, N, episode_bars=23 * k, auto_reset=auto_reset)
    gpu = GpuVec(cfg, candles, minutes)
    orc = TimeLimitOracle(cfg, candles, minutes, k=k, hold=hold, max_steps=max_steps, window=window)
    lo, hi = _ranges(N, Ts, tail=10 * k)   # windows shorter than the limit: both kinds of cut in one run
    gpu.env.set_episode_starts(lo, hi, seed=77)
    orc.set_episode_starts(lo, hi, seed=77)
    if k > 1:
        gpu.env.set_action_repeat(k, hold=hold)
    gpu.env.set_time_limit(max_steps, truncate_window=window)
    assert gpu.env.time_limit == (max_steps, window)
    np.testing.assert_allclose(gpu.reset(), orc.reset(), rtol=1e-5, atol=2e-6, err_msg="reset obs")
    rng = np.random.default_rng(len(name) * 1000 + 10 * k + hold + auto_reset)
    counts = np.zeros(3, np.int64)
    for s in range(steps):
        a = _actions(cfg, rng, N)
        go, oo = _gpu_step(gpu.env, a), orc.step(a)
        tag = f"{name} auto_reset={auto_reset} {mode} {rep} step {s}"
        compare_step(tag, go, oo)
        gi, oi = gpu.info(), orc.info()
        compare_info(tag, gi, oi)
        assert np.array_equal(gi["flags"].astype(np.int64) & END_BITS, oi["flags"].astype(np.int64) & END_BITS), tag
        counts += np.bincount(oo[3], minlength=3)[:3]
    start, done, last = (x.cpu().numpy() for x in gpu.env._episode_views())
    for what, g, o in zip(("start", "episodes_done", "last_episode"), (start, done, last), orc.episodes()):
        assert g.tobytes() == o.tobytes(), f"{name} {mode} {rep}: {what}"
    assert counts[2] > 0, "no truncation"
    gpu.close()
    orc.close()


# ---------------------------------------------------------------------------------------------------- engines agree
def _run(name, how, acts, monkeypatch, N, k=1, limit=(7, True)):
    for v in ("FXENV_ORDER_SMEM", "FXENV_ENGINE", "FXENV_CHUNK"):
        monkeypatch.delenv(v, raising=False)
    if how.startswith("smem"):
        monkeypatch.setenv("FXENV_ORDER_SMEM", how[4])
        monkeypatch.setenv("FXENV_ENGINE", "persistent")
        if how.endswith("chunk"):
            monkeypatch.setenv("FXENV_CHUNK", "3")   # tickets end inside episodes
    elif how == "graph":
        monkeypatch.setenv("FXENV_ENGINE", "graph")
    cfg, candles, minutes, Ts = _cfg(name, N)
    env = VecFxEnv(cfg, candles, minutes)
    env.set_episode_starts(*_ranges(N, Ts), seed=5)
    env.set_action_repeat(k)
    env.set_time_limit(*limit)
    env.reset()
    K, D = acts.shape[0], env.obs_dim
    obs = torch.empty((K, N, D), dtype=torch.float32, device="cuda")
    rew = torch.empty((K, N), dtype=torch.float32, device="cuda")
    term = torch.empty((K, N), dtype=torch.uint8, device="cuda")
    a_dev = torch.as_tensor(acts).cuda().contiguous()
    if how == "single":
        for s in range(K):
            o, r, _, _, _ = env.step(a_dev[s])
            obs[s].copy_(o); rew[s].copy_(r); term[s].copy_(env.terminated)
    elif how == "host":
        for s in range(K):
            oh = torch.empty((N, D), dtype=torch.float32).pin_memory()
            rh = torch.empty(N, dtype=torch.float32).pin_memory()
            th = torch.empty(N, dtype=torch.uint8).pin_memory()
            env.step_host(torch.as_tensor(acts[s]).contiguous(), oh, rh, th)
            obs[s].copy_(oh); rew[s].copy_(rh); term[s].copy_(th)
    else:
        for s0 in range(0, K, 20):   # batches of 20 decisions on the same buffers
            env.step_many(a_dev[s0:s0 + 20], obs[s0:s0 + 20], rew[s0:s0 + 20], term[s0:s0 + 20])
    torch.cuda.synchronize()
    out = (obs.cpu().numpy(), rew.cpu().numpy(), term.cpu().numpy(), env.get_state())
    env.close()
    return out


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("name", ["fixed_pnl", "atr_dd", "sharpe_3pairs"])
def test_engines_agree_bit_for_bit(name, k, monkeypatch):
    N, K = 48, 60
    cfg, _, _, _ = _cfg(name, N)
    acts = _actions(cfg, np.random.default_rng(3), (K, N))
    base = _run(name, "single", acts, monkeypatch, N, k)
    assert (base[2] == 2).sum() > 0
    for how in ("smem1", "smem0", "smem1chunk", "smem0chunk", "graph", "host"):
        other = _run(name, how, acts, monkeypatch, N, k)
        for what, x, y in zip(("obs", "reward", "codes"), other[:3], base[:3]):
            assert x.tobytes() == y.tobytes(), f"{name} k={k} {how}: {what}"
        assert other[3] == base[3], f"{name} k={k} {how}: state"


# ------------------------------------------------------------------------------------------------------ closed loop
def _policy_net(env, continuous):
    from gym_fx_b200.learner import ActorCritic
    torch.manual_seed(3)
    return ActorCritic(env.obs_dim, continuous=continuous).cuda()


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("name", ["fixed_pnl", "continuous"])
def test_rollout_replays_through_step_on_a_twin(name, k):
    N, H = 256, 30
    cfg, candles, minutes, Ts = _cfg(name, N)
    envs = [VecFxEnv(cfg, candles, minutes) for _ in range(2)]
    for e in envs:
        e.set_episode_starts(*_ranges(N, Ts), seed=8)
        e.set_action_repeat(k)
        e.set_time_limit(6, truncate_window=True)
        e.reset()
    cont = cfg.action_mode == 1
    pol = envs[0].make_policy(_policy_net(envs[0], cont))
    out = envs[0].rollout(pol, H, seed=12)
    torch.cuda.synchronize()
    assert pol.sync_timeouts() == 0
    twin = envs[1]
    done = out["done"].cpu().numpy()
    for t in range(H):
        o, r, _, _, _ = twin.step(out["actions"][t])
        torch.cuda.synchronize()
        assert torch.equal(o, out["obs"][t + 1]), f"step {t}: obs"
        assert torch.equal(r, out["reward"][t]), f"step {t}: reward"
        assert torch.equal(twin.terminated, out["done"][t]), f"step {t}: done"
        if t + 1 < H:   # after a truncation: the reset step (reward 0, code 0, a fresh episode)
            cut = done[t] == 2
            assert (done[t + 1][cut] == 0).all() and (out["reward"][t + 1].cpu().numpy()[cut] == 0).all()
    assert (done == 2).sum() > 0
    assert envs[0].get_state() == twin.get_state()
    for e in envs:
        e.close()


def test_cut_episode_final_observation_is_kept():
    """At a code-2 step t, obs[t + 1] is the cut episode's last row: equal to what a handle without auto-reset keeps
    answering after the cut."""
    N, H = 64, 12
    cfg_a, candles, minutes, Ts = _cfg("fixed_pnl", N, auto_reset=1)
    cfg_b, _, _, _ = _cfg("fixed_pnl", N, auto_reset=0)
    a, b = VecFxEnv(cfg_a, candles, minutes), VecFxEnv(cfg_b, candles, minutes)
    starts = torch.as_tensor(_ranges(N, Ts)[0])
    for e in (a, b):
        e.set_time_limit(5)
        e.reset(starts)
    pol = a.make_policy(_policy_net(a, False))
    out = a.rollout(pol, H, deterministic=True)
    torch.cuda.synchronize()
    done = out["done"].cpu().numpy()
    assert (done[4] == 2).all() and (done[:4] == 0).all() and (done[5] == 0).all()
    for t in range(H):
        o, _, _, trunc, _ = b.step(out["actions"][t])
        if t <= 4:
            assert torch.equal(o, out["obs"][t + 1]), t
    assert torch.equal(b.obs, out["obs"][5]) and bool(trunc.all())   # b keeps answering the cut episode's row
    assert (b.terminated.cpu().numpy() == 2).all()
    a.close(), b.close()


def test_episode_records_carry_the_truncated_flag():
    N = 32
    cfg, candles, minutes, Ts = _cfg("fixed_pnl", N, episode_bars=11)
    env = VecFxEnv(cfg, candles, minutes)
    env.set_time_limit(0, truncate_window=True)
    env.reset(torch.zeros(N, dtype=torch.int64))
    for _ in range(13):
        env.step(torch.zeros(N, dtype=torch.int32, device="cuda"))
    ep = env.episode_stats()
    assert (ep["episodes_done"] == 1).all()
    assert (ep["end_flags"] == (4 | FLAG_TRUNCATED)).all()
    env.close()


# ------------------------------------------------------------------------------------- a cut outlives its setting
@pytest.mark.parametrize("auto_reset", [0, 1])
@pytest.mark.parametrize("window", [False, True], ids=["limit", "window"])
def test_limit_off_right_after_a_cut(window, auto_reset):
    """A cut env whose reset step is still pending when truncation is turned off: with auto-reset its next step is the
    reset step, without it the episode stays over (code 1 now that the outputs are 0 / 1); no episode record ever holds
    TERMINATED and TRUNCATED together.  In lock step with the oracle through the switch and back."""
    N, M = 32, 6
    cfg, candles, minutes, Ts = _cfg("fixed_pnl", N, episode_bars=M - 1 if window else 23, auto_reset=auto_reset)
    gpu = GpuVec(cfg, candles, minutes)
    orc = TimeLimitOracle(cfg, candles, minutes)
    lo, hi = _ranges(N, Ts)
    for o in (gpu.env, orc):
        o.set_episode_starts(lo, hi, seed=3)
    limit = (0, True) if window else (M, False)
    gpu.env.set_time_limit(*limit)
    orc.set_time_limit(*limit)
    gpu.reset(), orc.reset()
    rng = np.random.default_rng(9)
    records = []
    for s in range(3 * M + 4):
        if s == M:            # every env was cut at decision M (limit) / M (window of M - 1 bars): turn truncation off
            gpu.env.set_time_limit(0)
            orc.set_time_limit(0)
        if s == 2 * M + 2:    # and on again
            gpu.env.set_time_limit(*limit)
            orc.set_time_limit(*limit)
        a = _actions(cfg, rng, N)
        go, oo = _gpu_step(gpu.env, a), orc.step(a)
        compare_step(f"window={window} auto_reset={auto_reset} step {s}", go, oo)
        gi, oi = gpu.info(), orc.info()
        compare_info(f"step {s}", gi, oi)
        assert np.array_equal(gi["flags"].astype(np.int64) & END_BITS, oi["flags"].astype(np.int64) & END_BITS), s
        if s == M - 1:
            assert (go[3] == 2).all(), "every env is cut at decision M"
        if s == M:
            assert (go[3] == (0 if auto_reset else 1)).all() and (go[2] == 0).all()
        records.append(gpu.env.episode_stats()["end_flags"].cpu().numpy().copy())
    start, done, last = (x.cpu().numpy() for x in gpu.env._episode_views())
    for what, g, o in zip(("start", "episodes_done", "last_episode"), (start, done, last), orc.episodes()):
        assert g.tobytes() == o.tobytes(), what
    rec = np.stack(records)
    assert not ((rec & 2) & ((rec & 64) >> 5)).any(), "an episode record with TERMINATED and TRUNCATED"
    if auto_reset:
        assert (done >= 1).all() and (rec[M] == (4 | 64 if window else 64)).all()
    gpu.close()
    orc.close()


def test_snapshot_of_a_cut_env_restored_without_a_limit():
    N, M = 32, 5
    acts = np.random.default_rng(6).integers(0, 3, (M + 3, N)).astype(np.int32)
    a = _fresh("fixed_pnl", N, limit=(M, False))
    ra = _steps(a, acts[:M])
    assert (ra[-1][2] == 2).all()
    blob = a.get_state()
    b = _fresh("fixed_pnl", N)          # no time limit
    b.set_state(blob)
    rb = _steps(b, acts[M:])
    assert (rb[0][2] == 0).all() and (rb[0][1] == 0).all(), "the restored cut env takes its reset step"
    ep = b.episode_stats()
    assert (ep["end_flags"] == FLAG_TRUNCATED).all()
    a.set_time_limit(0)                 # the same through the switch on the original handle
    assert all(x.tobytes() == y.tobytes() for p, q in zip(_steps(a, acts[M:]), rb) for x, y in zip(p, q))
    assert a.get_state() == b.get_state()
    a.close(), b.close()


# ------------------------------------------------------------------------------------------------------ switching
def _fresh(name, N, limit=None, k=1):
    cfg, candles, minutes, Ts = _cfg(name, N)
    env = VecFxEnv(cfg, candles, minutes)
    env.set_episode_starts(*_ranges(N, Ts), seed=21)
    env.set_action_repeat(k)
    if limit is not None:
        env.set_time_limit(*limit)
    env.reset()
    return env


def _steps(env, acts):
    outs = []
    for a in acts:
        o, r, _, _, _ = env.step(torch.as_tensor(a).cuda())
        outs.append((o.cpu().numpy().copy(), r.cpu().numpy().copy(), env.terminated.cpu().numpy().copy()))
    return outs


def test_limit_0_equals_a_handle_never_set():
    N, name = 64, "fixed_pnl"
    acts = np.random.default_rng(1).integers(0, 3, (40, N)).astype(np.int32)
    a = _fresh(name, N, limit=(4, True))
    a.set_time_limit(0)
    b = _fresh(name, N)
    for x, y in zip(_steps(a, acts), _steps(b, acts)):
        assert all(p.tobytes() == q.tobytes() for p, q in zip(x, y))
    assert a.get_state() == b.get_state()
    o, _, t, tr, _ = a.step(torch.zeros(N, dtype=torch.int32, device="cuda"))
    assert t.data_ptr() == a.terminated.data_ptr() and not bool(tr.any())
    a.close(), b.close()


@pytest.mark.parametrize("engine", ["persistent", "graph"])
def test_new_limit_between_step_many_calls_on_the_same_buffers(engine, monkeypatch):
    monkeypatch.setenv("FXENV_ENGINE", engine)
    N, K, name = 64, 12, "fixed_pnl"
    acts = np.random.default_rng(2).integers(0, 3, (K, N)).astype(np.int32)
    a = _fresh(name, N)
    monkeypatch.delenv("FXENV_ENGINE")
    b = _fresh(name, N)
    D = a.obs_dim
    ring = torch.empty((K, N, D), dtype=torch.float32, device="cuda")
    rew = torch.empty((K, N), dtype=torch.float32, device="cuda")
    term = torch.empty((K, N), dtype=torch.uint8, device="cuda")
    a_dev = torch.as_tensor(acts).cuda()
    s = torch.cuda.Stream()
    seen = 0
    with torch.cuda.stream(s):   # a non-default stream: the graph engine captures and caches
        for limit in ((0, False), (5, False), (3, True), (0, False)):
            a.set_time_limit(*limit)
            b.set_time_limit(*limit)
            a.step_many(a_dev, ring, rew, term)
            s.synchronize()
            want = _steps(b, acts)
            for j in range(K):
                assert ring[j].cpu().numpy().tobytes() == want[j][0].tobytes(), (limit, j)
                assert rew[j].cpu().numpy().tobytes() == want[j][1].tobytes(), (limit, j)
                assert term[j].cpu().numpy().tobytes() == want[j][2].tobytes(), (limit, j)
            seen += int((term == 2).sum())
            assert a.get_state() == b.get_state(), limit
    assert seen > 0
    a.close(), b.close()


def test_new_limit_between_two_rollouts_on_the_same_buffers():
    N, H, name = 128, 10, "fixed_pnl"
    a, b = _fresh(name, N), _fresh(name, N)
    pol = a.make_policy(_policy_net(a, False))
    bufs = None
    s = torch.cuda.Stream()
    cuts = []
    with torch.cuda.stream(s):   # a non-default stream: the rollout graph is captured and cached
        for limit in (4, 3, 0):
            a.set_time_limit(limit)
            b.set_time_limit(limit)
            bufs = a.rollout(pol, H, buffers=bufs, seed=11)
            s.synchronize()
            for t in range(H):
                o, r, _, _, _ = b.step(bufs["actions"][t])
                s.synchronize()
                assert torch.equal(o, bufs["obs"][t + 1]) and torch.equal(r, bufs["reward"][t]), (limit, t)
                assert torch.equal(b.terminated, bufs["done"][t]), (limit, t)
            cuts.append(int((bufs["done"] == 2).sum()))
            assert a.get_state() == b.get_state(), limit
    assert cuts[0] > 0 and cuts[1] > 0 and cuts[2] == 0
    a.close(), b.close()


def test_snapshot_mid_episode_continues_on_a_fresh_handle():
    N, name = 64, "atr_dd"
    acts = np.random.default_rng(4).integers(0, 3, (30, N)).astype(np.int32)
    a = _fresh(name, N, limit=(8, True), k=3)
    _steps(a, acts[:5])
    blob = a.get_state()
    b = _fresh(name, N, limit=(8, True), k=3)
    b.set_state(blob)
    assert b.time_limit == (8, True)
    ra, rb = _steps(a, acts[5:]), _steps(b, acts[5:])
    for x, y in zip(ra, rb):
        assert all(p.tobytes() == q.tobytes() for p, q in zip(x, y))
    assert sum(int((x[2] == 2).sum()) for x in ra) > 0
    assert a.get_state() == b.get_state()
    a.close(), b.close()


def test_bad_arguments_raise():
    env = _fresh("fixed_pnl", 8)
    for bad in (-1, 2.5, True, 2**31):
        with pytest.raises(ValueError):
            env.set_time_limit(bad)
    with pytest.raises(ValueError):
        env.set_time_limit(3, truncate_window=1)
    assert env.time_limit == (0, False)
    assert env.L.fxenv_set_time_limit(env._h, 4, 2) == -1           # unknown flag bit
    assert b"flags" in env.L.fxenv_last_error(env._h)
    assert env.L.fxenv_set_time_limit(env._h, -5, 0) == -1
    assert env.L.fxenv_set_time_limit(None, 2, 0) == -1
    env.close()


def test_gym_env_max_episode_steps(tmp_path):
    from gym_fx_b200 import GymFxEnv
    from gym_fx_b200.synth import write_csv
    T, M = 300, 7
    csv = tmp_path / "data.csv"
    write_csv(str(csv), synth_candles(T, 0), synth_minutes(T))
    config = {**S.DEFAULTS, "window_size": 8, "input_data_file": str(csv), "max_episode_steps": M}
    pl = S.build_mirror_plugins(config, dict(S.DEFAULT_PLUGINS))
    env = GymFxEnv(config, pl["data_feed"], pl["broker"], pl["strategy"], pl["preprocessor"], pl["reward"], pl["metrics"])
    env.reset()
    for s in range(M + 2):
        _, reward, term, trunc, _ = env.step(1)
        assert term is False and trunc == (s >= M - 1), s
        if s >= M:
            assert reward == 0.0
    env.close()
    plain = GymFxEnv({k: v for k, v in config.items() if k != "max_episode_steps"}, pl["data_feed"], pl["broker"],
                     pl["strategy"], pl["preprocessor"], pl["reward"], pl["metrics"])
    plain.reset()
    for s in range(M + 2):
        assert plain.step(1)[3] is False
    plain.close()
