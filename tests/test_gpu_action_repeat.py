"""GPU (-m gpu): the action repeat (include/fxenv.h fxenv_set_action_repeat; VecFxEnv.set_action_repeat).

  * Lock step with tests/repeat_oracle.py for k in {2, 3, 8}, both modes, over configurations that reach every kernel
    family: the cfg2 shape (LEAN), ATR + dd_penalized with the bracket audit, Sharpe over 4 pairs, continuous actions,
    default_preprocessor, commission / leverage / slippage, expanding z-score through its warm-up, and a broke-prone
    account; all with auto-reset, short episodes and start ranges, so that terminations fall inside steps.  Integer and
    fp64 state and the summary bit for bit, reward64 1e-9, observations at the usual tolerances, episode records and
    audit records equal.
  * The engines agree bit for bit: single steps, step_many (persistent with the shared-memory and the global order
    table, several ticket rounds; graph of single steps) and step_host.
  * The closed loop: a rollout replayed through step() on a twin handle gives identical outputs and state; the bf16 row
    copy is the round-to-nearest-even of the float32 row; greedy rollouts are reproducible.
  * Switching: back to k = 1 equals a handle never set; a new k between two step_many calls or two rollouts on the same
    buffers takes effect (the cached graphs were dropped); a snapshot continues identically on a fresh handle with the
    same setting; bad arguments raise."""
import numpy as np
import pytest
import torch

import scenarios as S
from common_gpu import GpuVec, compare_info, compare_step, compare_summary, gpu_summary
from gym_fx_b200.config import lower_config
from gym_fx_b200.synth import synth_candles, synth_minutes
from gym_fx_b200.vec_env import VecFxEnv
from repeat_oracle import RepeatOracle

pytestmark = pytest.mark.gpu

FIELDS = ("kind", "bar", "episode", "entry", "stop", "limit", "size", "atr")
FW = {"feature_columns": list(S.OHLCV)}
FWP = {"preprocessor": "feature_window_preprocessor"}

# name -> (config, plugins, pairs, extra lower_config arguments)
CONFIGS = {
    # the cfg2 shape: LEAN kernels (W % 4 == 0, OHLCV features, rolling z-score), fixed brackets, pnl
    "lean_fixed_pnl": (dict(window_size=32, sl_pips=3.0, tp_pips=4.0, feature_scaling_window=16, **FW),
                       dict(strategy="direct_fixed_sltp", **FWP), 1, {}),
    "atr_dd_audit": (dict(window_size=16, atr_period=6), dict(strategy="direct_atr_sltp", reward="dd_penalized_reward"), 1, {}),
    "sharpe_4pairs": (dict(window_size=16, sl_pips=3.0, tp_pips=4.0, window=12, **FW),
                      dict(strategy="direct_fixed_sltp", reward="sharpe_reward", **FWP), 4, {}),
    "continuous": (dict(window_size=12, action_space_mode="continuous", continuous_action_threshold=0.0), {}, 1, {}),
    "default_preproc": (dict(window_size=24, sl_pips=5.0, tp_pips=5.0), dict(strategy="direct_fixed_sltp"), 1, {}),
    "comm_lev_slip": (dict(window_size=16, sl_pips=3.0, tp_pips=6.0, commission=2e-5, leverage=20.0, slippage_perc=5e-5,
                           **FW), dict(strategy="direct_fixed_sltp", **FWP), 1, {}),
    "expanding_zscore": (dict(window_size=20, feature_scaling="expanding_zscore", **FW), FWP, 1, {}),
    "broke": (dict(window_size=8, position_size=2.0e5, leverage=400.0, min_equity=9900.0), {}, 1, {}),
}


def _cfg(name, N, episode_bars=37, auto_reset=1):
    cfgd, plugins, pairs, kw = CONFIGS[name]
    cfgd = {**S.DEFAULTS, **cfgd}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, **plugins})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"],
                       preprocessor_plugin=pl["preprocessor"], reward_plugin=pl["reward"], columns=S.OHLCV,
                       num_envs=N, num_pairs=pairs, order_capacity=256, episode_bars=episode_bars, **kw)
    cfg.auto_reset = auto_reset
    Ts = [900 + 130 * p for p in range(pairs)]
    return cfg, [synth_candles(T, p) for p, T in enumerate(Ts)], [synth_minutes(T) for T in Ts], Ts


def _ranges(N, Ts):
    lo = np.asarray([(29 * i) % (Ts[i % len(Ts)] // 2) for i in range(N)], np.int64)
    return lo, lo + np.asarray([[0, 1, 90, 300][i % 4] for i in range(N)], np.int64)


def _actions(cfg, rng, shape):
    if cfg.action_mode == 1:
        return rng.uniform(-1.0, 1.0, shape).astype(np.float32)
    return rng.integers(0, 3, shape).astype(np.int32)


def _per_env(r, n):
    env = r["env"].cpu().numpy()
    cols = np.stack([r[k].double().cpu().numpy() for k in FIELDS], axis=1) if env.size else np.zeros((0, 8))
    return [cols[env == i] for i in range(n)]


def _episodes(env):
    start, done, last = env._episode_views()
    return start.cpu().numpy(), done.cpu().numpy(), last.cpu().numpy()


# ---------------------------------------------------------------------------------------------- lock step with oracle
@pytest.mark.parametrize("hold", [False, True], ids=["repeat", "hold"])
@pytest.mark.parametrize("k", [2, 3, 8])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_lockstep_with_the_repeat_oracle(name, k, hold):
    N, steps = 32, 48 if k < 8 else 30
    cfg, candles, minutes, Ts = _cfg(name, N)
    audit = name.startswith("atr")
    gpu = GpuVec(cfg, candles, minutes)
    orc = RepeatOracle(cfg, candles, minutes, k=k, hold=hold, audit=audit)
    lo, hi = _ranges(N, Ts)
    gpu.env.set_episode_starts(lo, hi, seed=99)
    orc.set_episode_starts(lo, hi, seed=99)
    gpu.env.set_action_repeat(k, hold=hold)
    assert gpu.env.action_repeat == (k, hold)
    if audit:
        gpu.env.set_bracket_audit(4096)
    np.testing.assert_allclose(gpu.reset(), orc.reset(), rtol=1e-5, atol=2e-6, err_msg="reset obs")
    if name == "lean_fixed_pnl":
        assert gpu.env.L.fxenv_debug_lean(gpu.env._h) == 1, "the configuration no longer selects the LEAN kernels"
    rng = np.random.default_rng(1000 * k + 7 * hold + len(name))
    ends, inside = 0, 0
    for s in range(steps):
        a = _actions(cfg, rng, N)
        go, oo = gpu.step(a), orc.step(a)
        tag = f"{name} k={k} hold={hold} step {s}"
        compare_step(tag, go, oo)
        compare_info(tag, gpu.info(), orc.info())
        ends += int(oo[3].sum())
        inside += int(((oo[3] == 1) & (orc.substeps < k) & (orc.substeps > 1)).sum())
    gs, osum = gpu_summary(gpu.env), orc.summary()
    compare_summary(f"{name} k={k}: summary", {**gs, "sqn": np.full_like(gs["sqn"], np.nan)},
                    {**osum, "sqn": np.full_like(osum["sqn"], np.nan)})
    for what, g, o in zip(("start", "episodes_done", "last_episode"), _episodes(gpu.env), orc.episodes()):
        assert g.tobytes() == o.tobytes(), f"{name} k={k}: {what}"
    assert ends > 0, "no episode ended"
    if k > 2:
        assert inside > 0, "no termination inside a step"
    if audit:
        got = _per_env(gpu.env.bracket_audit(), N)
        n = 0
        for i in range(N):
            ref = orc.env_records(i)
            assert got[i].shape == ref.shape and got[i].tobytes() == ref.tobytes(), (name, i)
            n += len(ref)
        assert n > N
    gpu.close()
    orc.close()


# ---------------------------------------------------------------------------------------------------- engines agree
def _run(name, how, acts, k, hold, monkeypatch, N):
    for v in ("FXENV_ORDER_SMEM", "FXENV_ENGINE", "FXENV_CHUNK"):
        monkeypatch.delenv(v, raising=False)
    if how.startswith("smem"):
        monkeypatch.setenv("FXENV_ORDER_SMEM", how[4])
        monkeypatch.setenv("FXENV_ENGINE", "persistent")
        if how.endswith("chunk"):
            monkeypatch.setenv("FXENV_CHUNK", "5")
    elif how == "graph":
        monkeypatch.setenv("FXENV_ENGINE", "graph")
    cfg, candles, minutes, Ts = _cfg(name, N)
    env = VecFxEnv(cfg, candles, minutes)
    env.set_episode_starts(*_ranges(N, Ts), seed=5)
    env.set_action_repeat(k, hold=hold)
    if name.startswith("atr"):
        env.set_bracket_audit(4096)
    env.reset()
    K, D = acts.shape[0], env.obs_dim
    obs = torch.empty((K, N, D), dtype=torch.float32, device="cuda")
    rew = torch.empty((K, N), dtype=torch.float32, device="cuda")
    term = torch.empty((K, N), dtype=torch.uint8, device="cuda")
    a_dev = torch.as_tensor(acts).cuda().contiguous()
    if how == "single":
        for s in range(K):
            o, r, t, _, _ = env.step(a_dev[s])
            obs[s].copy_(o); rew[s].copy_(r); term[s].copy_(t.to(torch.uint8))
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
    audit = env._audit[0].cpu().numpy().copy() if env._audit else None
    out = (obs.cpu().numpy(), rew.cpu().numpy(), term.cpu().numpy(), env.get_state(), audit)
    env.close()
    return out


@pytest.mark.parametrize("hold", [False, True], ids=["repeat", "hold"])
@pytest.mark.parametrize("name", ["lean_fixed_pnl", "atr_dd_audit", "sharpe_4pairs", "continuous"])
def test_engines_agree_bit_for_bit(name, hold, monkeypatch):
    N, K, k = 48, 60, 3
    cfg, _, _, _ = _cfg(name, N)
    acts = _actions(cfg, np.random.default_rng(3), (K, N))
    base = _run(name, "single", acts, k, hold, monkeypatch, N)
    assert base[2].sum() > 0
    for how in ("smem1", "smem0", "smem1chunk", "smem0chunk", "graph", "host"):
        other = _run(name, how, acts, k, hold, monkeypatch, N)
        for what, x, y in zip(("obs", "reward", "terminated"), other[:3], base[:3]):
            assert x.tobytes() == y.tobytes(), f"{name} {how}: {what}"
        assert other[3] == base[3], f"{name} {how}: state"
        if base[4] is not None:
            assert other[4].tobytes() == base[4].tobytes(), f"{name} {how}: audit"


# ------------------------------------------------------------------------------------------------------ closed loop
def _policy_net(env, continuous):
    from gym_fx_b200.learner import ActorCritic
    torch.manual_seed(3)
    return ActorCritic(env.obs_dim, continuous=continuous).cuda()


@pytest.mark.parametrize("hold", [False, True], ids=["repeat", "hold"])
@pytest.mark.parametrize("name", ["lean_fixed_pnl", "continuous"])
def test_rollout_replays_through_step_on_a_twin(name, hold):
    N, H, k = 256, 24, 4
    cfg, candles, minutes, Ts = _cfg(name, N)
    envs = [VecFxEnv(cfg, candles, minutes) for _ in range(2)]
    for e in envs:
        e.set_episode_starts(*_ranges(N, Ts), seed=8)
        e.set_action_repeat(k, hold=hold)
        e.reset()
    cont = cfg.action_mode == 1
    net = _policy_net(envs[0], cont)
    pol = envs[0].make_policy(net)
    g = torch.Generator(device="cuda").manual_seed(4)
    if cont:
        noise = torch.randn((H, N), device="cuda", generator=g)
        out = envs[0].rollout(pol, H, noise=noise)
    else:
        u = torch.rand((H, N, 3), device="cuda", generator=g).clamp_(1e-7, 1 - 1e-7)
        out = envs[0].rollout(pol, H, gumbel=-torch.log(-torch.log(u)))
    torch.cuda.synchronize()
    assert pol.sync_timeouts() == 0
    twin = envs[1]
    for t in range(H):
        o, r, d, _, _ = twin.step(out["actions"][t])
        torch.cuda.synchronize()
        assert torch.equal(o, out["obs"][t + 1]), f"step {t}: obs"
        assert torch.equal(r, out["reward"][t]), f"step {t}: reward"
        assert torch.equal(d.to(torch.uint8), out["done"][t]), f"step {t}: done"
    assert int(out["done"].sum()) > 0
    assert envs[0].get_state() == twin.get_state()
    # the bf16 copy the policy reads: round-to-nearest-even of the last row
    D = envs[0].obs_dim
    row16 = pol.peek("obs16", H % 2)[:, :D]
    assert torch.equal(row16.view(torch.int16), out["obs"][H].to(torch.bfloat16).view(torch.int16))
    # greedy rollouts from the same state are reproducible
    blob = envs[0].get_state()
    g1 = {k_: v.clone() for k_, v in envs[0].rollout(pol, 8, deterministic=True).items()}
    envs[0].set_state(blob)
    g2 = envs[0].rollout(pol, 8, deterministic=True)
    torch.cuda.synchronize()
    for k_ in ("obs", "actions", "reward", "done", "value"):
        assert torch.equal(g1[k_], g2[k_]), k_
    for e in envs:
        e.close()


# ------------------------------------------------------------------------------------------------------ switching
def _fresh(name, N, k=None, hold=False):
    cfg, candles, minutes, Ts = _cfg(name, N)
    env = VecFxEnv(cfg, candles, minutes)
    env.set_episode_starts(*_ranges(N, Ts), seed=21)
    if k is not None:
        env.set_action_repeat(k, hold=hold)
    env.reset()
    return env


def _steps(env, acts):
    outs = []
    for a in acts:
        o, r, t, _, _ = env.step(torch.as_tensor(a).cuda())
        outs.append((o.cpu().numpy().copy(), r.cpu().numpy().copy(), t.cpu().numpy().copy()))
    return outs


def test_back_to_k1_equals_a_handle_never_set():
    N, name = 64, "lean_fixed_pnl"
    acts = np.random.default_rng(1).integers(0, 3, (40, N)).astype(np.int32)
    a = _fresh(name, N, k=5, hold=True)
    a.set_action_repeat(1)
    b = _fresh(name, N)
    for x, y in zip(_steps(a, acts), _steps(b, acts)):
        assert all(p.tobytes() == q.tobytes() for p, q in zip(x, y))
    assert a.get_state() == b.get_state()
    a.close(), b.close()


@pytest.mark.parametrize("engine", ["persistent", "graph"])
def test_new_k_between_step_many_calls_on_the_same_buffers(engine, monkeypatch):
    monkeypatch.setenv("FXENV_ENGINE", engine)
    N, K, name = 64, 12, "lean_fixed_pnl"
    acts = np.random.default_rng(2).integers(0, 3, (K, N)).astype(np.int32)
    a = _fresh(name, N, k=2)
    monkeypatch.delenv("FXENV_ENGINE")
    b = _fresh(name, N, k=2)
    D = a.obs_dim
    ring = torch.empty((K, N, D), dtype=torch.float32, device="cuda")
    rew = torch.empty((K, N), dtype=torch.float32, device="cuda")
    term = torch.empty((K, N), dtype=torch.uint8, device="cuda")
    a_dev = torch.as_tensor(acts).cuda()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):   # a non-default stream: the graph engine captures and caches
        for k, hold in ((2, False), (3, False), (3, True), (1, False)):
            a.set_action_repeat(k, hold=hold)
            b.set_action_repeat(k, hold=hold)
            a.step_many(a_dev, ring, rew, term)
            s.synchronize()
            want = _steps(b, acts)
            for j in range(K):
                assert ring[j].cpu().numpy().tobytes() == want[j][0].tobytes(), (k, hold, j)
                assert rew[j].cpu().numpy().tobytes() == want[j][1].tobytes(), (k, hold, j)
            assert a.get_state() == b.get_state(), (k, hold)
    a.close(), b.close()


def test_new_k_between_two_rollouts_on_the_same_buffers():
    N, H, name = 128, 10, "lean_fixed_pnl"
    a, b = _fresh(name, N, k=2), _fresh(name, N, k=2)
    pol = a.make_policy(_policy_net(a, False))
    bufs = None
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):   # a non-default stream: the rollout graph is captured and cached
        for k in (2, 6, 1):
            a.set_action_repeat(k)
            b.set_action_repeat(k)
            bufs = a.rollout(pol, H, buffers=bufs, seed=11)
            s.synchronize()
            for t in range(H):
                o, r, _, _, _ = b.step(bufs["actions"][t])
                s.synchronize()
                assert torch.equal(o, bufs["obs"][t + 1]) and torch.equal(r, bufs["reward"][t]), (k, t)
            assert a.get_state() == b.get_state(), k
    a.close(), b.close()


def test_snapshot_under_repeat_continues_on_a_fresh_handle():
    N, name = 64, "atr_dd_audit"
    acts = np.random.default_rng(4).integers(0, 3, (30, N)).astype(np.int32)
    a = _fresh(name, N, k=3, hold=True)
    _steps(a, acts[:10])
    blob = a.get_state()
    b = _fresh(name, N, k=3, hold=True)
    b.set_state(blob)
    assert b.action_repeat == (3, True)
    for x, y in zip(_steps(a, acts[10:]), _steps(b, acts[10:])):
        assert all(p.tobytes() == q.tobytes() for p, q in zip(x, y))
    assert a.get_state() == b.get_state()
    a.close(), b.close()


def test_bad_arguments_raise():
    env = _fresh("lean_fixed_pnl", 8)
    for bad in (0, -1, 257, 2.5, True):
        with pytest.raises(ValueError):
            env.set_action_repeat(bad)
    assert env.action_repeat == (1, False)
    assert env.L.fxenv_set_action_repeat(env._h, 4, 2) == -1           # unknown flag bit
    assert b"flags" in env.L.fxenv_last_error(env._h)
    assert env.L.fxenv_set_action_repeat(env._h, 257, 0) == -1
    assert env.L.fxenv_set_action_repeat(None, 2, 0) == -1
    env.set_action_repeat(256, hold=True)
    assert env.action_repeat == (256, True)
    env.close()
