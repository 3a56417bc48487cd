"""GPU (-m gpu): per-env broker and strategy parameters (include/fxenv.h fxenv_set_env_params; VecFxEnv.set_env_params).

  * A table whose every row equals the config gives bit-identical outputs to no table (LEAN fixed SL/TP with pnl, ATR with
    drawdown and the bracket audit, the default strategy with Sharpe, continuous actions, action repeat 3 with a time
    limit), through step, step_many (persistent with the order table in shared / global memory, graph) and rollout.
  * A table of 8 distinct rows over 64 envs against one C oracle per row, built from a base config that differs from
    every row: all three strategies, pnl and drawdown rewards.
  * The engines agree bit for bit on such a table; a rollout replays through step() on a twin handle.
  * The LEAN choice follows the table's costs, with oracle parity either way.
  * Handle-setting contract: state size, snapshots, reset, in-place updates reaching cached graphs, rejected rows,
    turning the table off.
  * A commission set mid-episode, checked by hand on a scripted few-bar scenario."""
import numpy as np
import pytest
import torch

import scenarios as S
from common_gpu import INFO_KEYS, GpuVec, compare_info, compare_step, compare_summary, gpu_summary
from gym_fx_b200.config import ENV_PARAM_FIELDS, FxConfig, lower_config
from gym_fx_b200.synth import start_offsets, synth_candles, synth_minutes
from gym_fx_b200.vec_env import VecFxEnv
from oracle.c_oracle import OracleVec

pytestmark = pytest.mark.gpu

FW = {"feature_columns": list(S.OHLCV)}
FWP = {"preprocessor": "feature_window_preprocessor"}
CFG_FIELD = dict(zip(ENV_PARAM_FIELDS, ("commission", "leverage", "slippage_perc", "sl_pips", "tp_pips", "k_sl", "k_tp")))

# name -> (config, plugins)
CASES = {
    "lean_fixed_pnl": (dict(window_size=32, sl_pips=3.0, tp_pips=5.0, feature_scaling_window=16, **FW),
                       dict(strategy="direct_fixed_sltp", **FWP)),
    "atr_dd": (dict(window_size=16, atr_period=6, commission=2e-5, leverage=5.0, slippage=1e-4),
               dict(strategy="direct_atr_sltp", reward="dd_penalized_reward")),
    "default_sharpe": (dict(window_size=16, commission=3e-5, slippage=5e-5, window=12), dict(reward="sharpe_reward")),
    "continuous": (dict(window_size=12, action_space_mode="continuous", continuous_action_threshold=0.2, commission=1e-5), {}),
}


def _cfg(name, N, T=1500, episode_bars=0):
    cfgd, plugins = CASES[name]
    cfgd = {**S.DEFAULTS, **cfgd}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, **plugins})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"], preprocessor_plugin=pl["preprocessor"],
                       reward_plugin=pl["reward"], columns=S.OHLCV, num_envs=N, order_capacity=256, episode_bars=episode_bars)
    cfg.auto_reset = 1
    return cfg, [synth_candles(T, 0)], [synth_minutes(T)]


def _actions(cfg, rng, shape):
    if cfg.action_mode == 1:
        return rng.uniform(-1.0, 1.0, shape).astype(np.float32)
    return rng.integers(0, 3, shape).astype(np.int32)


def _uniform(cfg):
    return {f: getattr(cfg, CFG_FIELD[f]) for f in ENV_PARAM_FIELDS}


def _env(cfg, candles, minutes, monkeypatch, how):
    for v in ("FXENV_ORDER_SMEM", "FXENV_ENGINE"):
        monkeypatch.delenv(v, raising=False)
    if how.startswith("smem"):
        monkeypatch.setenv("FXENV_ORDER_SMEM", how[4])
        monkeypatch.setenv("FXENV_ENGINE", "persistent")
    elif how == "graph":
        monkeypatch.setenv("FXENV_ENGINE", "graph")
    return VecFxEnv(cfg, candles, minutes)


def _outputs(env, how, acts, audit=False, batch=6):
    """Everything a run produces: per-step obs / rewards / codes (and info columns for step()), then the statistics."""
    N, D, K = env.num_envs, env.obs_dim, acts.shape[0]
    out = {}
    if how == "step":
        for k in range(K):
            obs, rew, term, _, _ = env.step(torch.as_tensor(acts[k]))
            out[f"obs{k}"] = obs.cpu().numpy().copy()
            out[f"rew{k}"] = rew.cpu().numpy().copy()
            out[f"rew64_{k}"] = env.reward64.cpu().numpy().copy()
            out[f"term{k}"] = env.terminated.cpu().numpy().copy()
            info = env.info()
            for key in INFO_KEYS:
                out[f"{key}{k}"] = info[key].cpu().numpy().copy()
    elif how == "rollout":
        torch.manual_seed(0)
        from gym_fx_b200.learner import ActorCritic
        net = ActorCritic(D, continuous=env.cfg.action_mode == 1).cuda()
        pol = env.make_policy(net)
        r = env.rollout(pol, K, seed=11)
        for key in ("obs", "actions", "reward", "done", "value", "logp"):
            out[key] = r[key].cpu().numpy().copy()
    else:
        a = torch.as_tensor(acts).cuda()
        for k0 in range(0, K, batch):
            kb = min(batch, K - k0)
            ring = torch.empty((kb, N, D), dtype=torch.float32, device="cuda")
            rews = torch.empty((kb, N), dtype=torch.float32, device="cuda")
            terms = torch.empty((kb, N), dtype=torch.uint8, device="cuda")
            env.step_many(a[k0:k0 + kb].contiguous(), ring, rews, terms)
            out[f"ring{k0}"], out[f"rews{k0}"], out[f"terms{k0}"] = (x.cpu().numpy().copy() for x in (ring, rews, terms))
    torch.cuda.synchronize()
    out["run_stats"] = env.run_stats().cpu().numpy().copy()
    for key, v in env.episode_stats().items():
        out[f"ep_{key}"] = np.asarray(v.cpu().numpy() if hasattr(v, "cpu") else v).copy()
    info = env.info()
    for key in INFO_KEYS:
        out[f"final_{key}"] = info[key].cpu().numpy().copy()
    if audit:
        for key, v in env.bracket_audit().items():
            out[f"audit_{key}"] = v.cpu().numpy().copy()
    return out


def _same(a, b, tag):
    assert a.keys() == b.keys(), tag
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), f"{tag}: {k} differs"


# ------------------------------------------------------------------------------------------- a uniform table is a no-op
VARIANTS = ["lean_fixed_pnl", "atr_dd", "default_sharpe", "continuous", "repeat3_limit"]


@pytest.mark.parametrize("how", ["step", "smem1", "smem0", "graph", "rollout"])
@pytest.mark.parametrize("variant", VARIANTS)
def test_uniform_table_is_bit_identical_to_no_table(variant, how, monkeypatch):
    name = "lean_fixed_pnl" if variant == "repeat3_limit" else variant
    N, K = 96, 24
    cfg, candles, minutes = _cfg(name, N, episode_bars=60)
    acts = _actions(cfg, np.random.default_rng(3), (K, N))
    starts = start_offsets(N, 1500, 200, 600)
    res = []
    for table in (False, True):
        env = _env(cfg, candles, minutes, monkeypatch, how)
        if variant == "repeat3_limit":
            env.set_action_repeat(3)
            env.set_time_limit(5)
        if name == "atr_dd":
            env.set_bracket_audit(64)
        if table:
            env.set_env_params(**_uniform(cfg))
            assert env.env_params is not None and env.env_params.shape == (N, 7)
        if name == "lean_fixed_pnl":
            assert env.L.fxenv_debug_lean(env._h) == 1, "a uniform table of the config's costs keeps the LEAN kernels"
        env.reset(torch.as_tensor(starts))
        res.append(_outputs(env, how, acts, audit=name == "atr_dd"))
        env.close()
    _same(res[0], res[1], f"{variant} {how}")


# ------------------------------------------------------------------------------------- a heterogeneous table vs oracle
ROWS = np.array([  # commission, leverage, slippage, sl_pips, tp_pips, k_sl, k_tp
    [0.0, 1.0, 0.0, 2.0, 3.0, 0.5, 1.0],
    [1e-5, 2.0, 5e-5, 5.0, 8.0, 2.0, 3.0],
    [7e-5, 30.0, 3e-4, 20.0, 40.0, 0.5, 3.0],
    [7e-5, 0.5, 0.0, 2.0, 40.0, 2.0, 1.0],      # leverage < 1: the cash bound is max(1, 1 / leverage) + commission
    [0.0, 30.0, 5e-5, 20.0, 3.0, 0.5, 1.0],
    [1e-5, 1.0, 3e-4, 5.0, 3.0, 2.0, 3.0],
    [7e-5, 2.0, 0.0, 2.0, 8.0, 0.5, 3.0],
    [0.0, 2.0, 3e-4, 20.0, 8.0, 2.0, 1.0],
])
BASE = dict(commission=3e-5, leverage=4.0, slippage=2e-5, sl_pips=7.0, tp_pips=11.0, k_sl=1.5, k_tp=2.5)


def _with_row(cfg, row, n):
    out = FxConfig.from_buffer_copy(cfg)
    out.num_envs = n
    for f, v in zip(ENV_PARAM_FIELDS, row):
        setattr(out, CFG_FIELD[f], float(v))
    return out


def _hetero_cfg(strategy, reward, N, position_size):
    cfgd = {**S.DEFAULTS, "window_size": 16, "atr_period": 5, "position_size": position_size, "window": 10,
            **{("slippage" if k == "slippage" else k): v for k, v in BASE.items()}}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, "strategy": strategy, "reward": reward})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"], preprocessor_plugin=pl["preprocessor"],
                       reward_plugin=pl["reward"], columns=S.OHLCV, num_envs=N, order_capacity=256)
    for f, v in BASE.items():
        setattr(cfg, CFG_FIELD[f], v)
    assert all((ROWS[:, j] != BASE[f]).all() for j, f in enumerate(ENV_PARAM_FIELDS))
    return cfg


@pytest.mark.parametrize("reward", ["pnl_reward", "dd_penalized_reward"])
@pytest.mark.parametrize("strategy", ["default_strategy", "direct_fixed_sltp", "direct_atr_sltp"])
def test_heterogeneous_table_matches_one_oracle_per_row(strategy, reward):
    N, G, T, steps = 64, 8, 1200, 160
    cfg = _hetero_cfg(strategy, reward, N, position_size=9000.0 if strategy == "direct_atr_sltp" else 4000.0)
    candles, minutes = [synth_candles(T, 0, 4242)], [synth_minutes(T)]
    table = np.repeat(ROWS, N // G, axis=0)     # env i has row i // 8
    gpu = GpuVec(cfg, candles, minutes)
    gpu.env.set_env_params(**{f: table[:, j] for j, f in enumerate(ENV_PARAM_FIELDS)})
    assert gpu.env.L.fxenv_debug_lean(gpu.env._h) == 0
    starts = start_offsets(N, T, steps + 10, 300)
    orcs = [OracleVec(_with_row(cfg, ROWS[g], N // G), candles, minutes) for g in range(G)]
    sl = [slice(g * (N // G), (g + 1) * (N // G)) for g in range(G)]
    o0 = gpu.reset(starts)
    for g in range(G):
        np.testing.assert_allclose(o0[sl[g]], orcs[g].reset(starts[sl[g]]), rtol=1e-5, atol=2e-6)
    rng = np.random.default_rng(17)
    for k in range(steps):
        a = rng.integers(0, 3, N).astype(np.int32)
        go, gi = gpu.step(a), gpu.info()
        for g in range(G):
            tag = f"{strategy} {reward} step {k} row {g}"
            compare_step(tag, tuple(x[sl[g]] for x in go), orcs[g].step(a[sl[g]]))
            compare_info(tag, {key: v[sl[g]] for key, v in gi.items()}, orcs[g].info())
    gs = gpu_summary(gpu.env)
    for g in range(G):
        compare_summary(f"{strategy} {reward} row {g}", {key: v[sl[g]] for key, v in gs.items()}, orcs[g].summary())
    fl = gpu.info()["flags"].astype(np.int64)
    assert not (fl & 16).any(), "order table overflow"
    trading = sum(int(gpu.info()["trades"][sl[g]].sum() > 0) for g in range(G))
    assert trading >= G // 2, f"only {trading} of {G} rows trade"   # (a row whose every entry goes Margin does not)
    gpu.close()


# --------------------------------------------------------------------------------------------------- engines agree
@pytest.mark.parametrize("strategy", ["direct_fixed_sltp", "direct_atr_sltp"])
def test_engines_agree_on_a_heterogeneous_table(strategy, monkeypatch):
    N, K, T = 64, 30, 1200
    cfg = _hetero_cfg(strategy, "pnl_reward", N, position_size=4000.0)
    cfg.auto_reset = 1
    cfg.episode_bars = 40
    candles, minutes = [synth_candles(T, 0, 99)], [synth_minutes(T)]
    table = np.repeat(ROWS, N // 8, axis=0)
    starts = torch.as_tensor(start_offsets(N, T, 60, 500))
    acts = np.random.default_rng(5).integers(0, 3, (K, N)).astype(np.int32)
    res = {}
    for how in ("smem1", "smem0", "graph"):
        env = _env(cfg, candles, minutes, monkeypatch, how)
        env.set_env_params(**{f: table[:, j] for j, f in enumerate(ENV_PARAM_FIELDS)})
        env.reset(starts)
        o = _outputs(env, how, acts, batch=K)
        res[how] = o
        env.close()
    _same(res["smem1"], res["smem0"], "persistent smem / global")
    _same(res["smem1"], res["graph"], "persistent / graph")
    # step(): the same per-step rows as the batch engines
    env = _env(cfg, candles, minutes, monkeypatch, "step")
    env.set_env_params(**{f: table[:, j] for j, f in enumerate(ENV_PARAM_FIELDS)})
    env.reset(starts)
    o = _outputs(env, "step", acts)
    env.close()
    for k in range(K):
        assert o[f"obs{k}"].tobytes() == res["graph"][f"ring0"][k].tobytes(), f"step / batch obs {k}"
        assert o[f"rew{k}"].tobytes() == res["graph"][f"rews0"][k].tobytes(), f"step / batch reward {k}"
        assert o[f"term{k}"].tobytes() == res["graph"][f"terms0"][k].tobytes(), f"step / batch code {k}"
    assert o["run_stats"].tobytes() == res["graph"]["run_stats"].tobytes()
    # rollout with fixed Gumbel noise, replayed through step() on a twin handle
    from gym_fx_b200.learner import ActorCritic
    envs = []
    for _ in range(2):
        e = _env(cfg, candles, minutes, monkeypatch, "default")
        e.set_env_params(**{f: table[:, j] for j, f in enumerate(ENV_PARAM_FIELDS)})
        e.reset(starts)
        envs.append(e)
    torch.manual_seed(1)
    pol = envs[0].make_policy(ActorCritic(envs[0].obs_dim).cuda())
    gumbel = -torch.log(-torch.log(torch.rand((K, N, 3), device="cuda").clamp_(1e-9, 1 - 1e-7)))
    r = envs[0].rollout(pol, K, gumbel=gumbel)
    for k in range(K):
        obs, rew, _, _, _ = envs[1].step(r["actions"][k].to(torch.int32).contiguous())
        assert obs.cpu().numpy().tobytes() == r["obs"][k + 1].cpu().numpy().tobytes(), f"rollout obs {k}"
        assert rew.cpu().numpy().tobytes() == r["reward"][k].cpu().numpy().tobytes(), f"rollout reward {k}"
    assert envs[0].run_stats().cpu().numpy().tobytes() == envs[1].run_stats().cpu().numpy().tobytes()
    for e in envs:
        e.close()


# ------------------------------------------------------------------------------------------------------ LEAN choice
def test_lean_choice_follows_the_table():
    N, T, steps = 64, 1500, 80
    cfg, candles, minutes = _cfg("lean_fixed_pnl", N, T)
    starts = start_offsets(N, T, steps + 10, 400)
    rng = np.random.default_rng(8)
    sl, tp = rng.choice([2.0, 4.0, 9.0], N), rng.choice([3.0, 6.0, 12.0], N)
    for comm in (0.0, 5e-5):
        gpu = GpuVec(cfg, candles, minutes)
        c = np.zeros(N)
        c[5] = comm
        gpu.env.set_env_params(sl_pips=sl, tp_pips=tp, commission=c)
        assert gpu.env.L.fxenv_debug_lean(gpu.env._h) == (1 if comm == 0.0 else 0), comm
        orcs = [OracleVec(_with_row(cfg, gpu.env.env_params[i], 1), candles, minutes) for i in range(N)]
        o0 = gpu.reset(starts)
        for i in range(N):
            np.testing.assert_allclose(o0[i:i + 1], orcs[i].reset(starts[i:i + 1]), rtol=1e-5, atol=2e-6)
        for k in range(steps):
            a = rng.integers(0, 3, N).astype(np.int32)
            go, gi = gpu.step(a), gpu.info()
            for i in range(N):
                compare_step(f"comm {comm} step {k} env {i}", tuple(x[i:i + 1] for x in go), orcs[i].step(a[i:i + 1]))
                compare_info(f"comm {comm} step {k} env {i}", {key: v[i:i + 1] for key, v in gi.items()}, orcs[i].info())
        gpu.close()


# ----------------------------------------------------------------------------------------- handle-setting contract
def test_handle_setting_contract(monkeypatch):
    N, T, K = 64, 1500, 12
    monkeypatch.setenv("FXENV_ENGINE", "graph")
    cfg, candles, minutes = _cfg("atr_dd", N, T)
    starts = torch.as_tensor(start_offsets(N, T, 200, 600))
    acts = torch.as_tensor(np.random.default_rng(2).integers(0, 3, (K, N)).astype(np.int32)).cuda()
    D = None

    def batch(env, bufs):
        env.step_many(acts, *bufs)
        torch.cuda.synchronize()
        return tuple(x.cpu().numpy().copy() for x in bufs) + (env.run_stats().cpu().numpy().copy(),)

    env = VecFxEnv(cfg, candles, minutes)
    D = env.obs_dim
    bufs = (torch.empty((K, N, D), device="cuda"), torch.empty((K, N), device="cuda"),
            torch.empty((K, N), dtype=torch.uint8, device="cuda"))
    bytes0 = env.L.fxenv_state_bytes(env._h)
    t1 = np.linspace(0.0, 7e-5, N)
    env.set_env_params(commission=t1, leverage=np.linspace(0.5, 30.0, N))
    assert env.L.fxenv_state_bytes(env._h) == bytes0
    env.reset(starts)
    batch(env, bufs)                              # captures the graph with the table on
    # a rejected row leaves the table in force
    with pytest.raises(ValueError, match="leverage"):
        env.set_env_params(commission=t1, leverage=np.r_[np.ones(N - 1), 0.0])
    assert (env.env_params[:, 1] == np.linspace(0.5, 30.0, N)).all()
    blob = env.get_state()
    # an in-place value update reaches the cached graph
    t2 = dict(commission=t1[::-1].copy(), leverage=2.0, slippage=np.linspace(0, 2e-4, N), k_sl=0.7, k_tp=4.0)
    env.set_env_params(**t2)
    got = batch(env, bufs)
    fresh = VecFxEnv(cfg, candles, minutes)
    fresh.set_env_params(**t2)
    fresh.set_state(blob)
    fbufs = tuple(torch.empty_like(x) for x in bufs)
    want = batch(fresh, fbufs)
    for g, w, what in zip(got, want, ("obs", "reward", "code", "run_stats")):
        assert g.tobytes() == w.tobytes(), f"in-place update: {what}"
    # snapshots and reset() keep the table
    env.set_state(blob)
    assert env.env_params is not None and (env.env_params[:, 0] == t2["commission"]).all()
    again = batch(env, bufs)
    for g, w in zip(again, want):
        assert g.tobytes() == w.tobytes(), "set_state keeps the table"
    env.reset(starts)
    fresh.reset(starts)
    for g, w in zip(batch(env, bufs), batch(fresh, fbufs)):
        assert g.tobytes() == w.tobytes(), "reset keeps the table"
    # off: the same as a handle that never had a table
    env.set_env_params(None)
    assert env.env_params is None
    never = VecFxEnv(cfg, candles, minutes)
    env.reset(starts)
    never.reset(starts)
    for g, w in zip(batch(env, bufs), batch(never, fbufs)):
        assert g.tobytes() == w.tobytes(), "table off"
    for e in (env, fresh, never):
        e.close()


def test_rollout_graph_follows_an_in_place_update():
    from gym_fx_b200.learner import ActorCritic
    N, T, H = 64, 1500, 8
    cfg, candles, minutes = _cfg("default_sharpe", N, T)
    starts = torch.as_tensor(start_offsets(N, T, 100, 600))
    envs = []
    for _ in range(2):
        e = VecFxEnv(cfg, candles, minutes)
        e.set_env_params(commission=0.0)
        e.reset(starts)
        envs.append(e)
    torch.manual_seed(3)
    net = ActorCritic(envs[0].obs_dim).cuda()
    pols = [e.make_policy(net) for e in envs]
    g = -torch.log(-torch.log(torch.rand((H, N, 3), device="cuda").clamp_(1e-9, 1 - 1e-7)))
    bufs = envs[0].rollout(pols[0], H, gumbel=g)                # captures the rollout graph
    envs[1].rollout(pols[1], H, gumbel=g)
    new = dict(commission=np.linspace(0, 1e-4, N), slippage=3e-4)
    for e in envs:
        e.set_env_params(**new)                                 # in place: the same key
    blob = envs[1].get_state()
    a = envs[0].rollout(pols[0], H, buffers=bufs, gumbel=g)    # the same buffers and noise: the graph is replayed
    a = {k: a[k].cpu().numpy().copy() for k in ("obs", "actions", "reward", "done")}
    fresh = VecFxEnv(cfg, candles, minutes)
    fresh.set_env_params(**new)
    fresh.set_state(blob)
    b = fresh.rollout(fresh.make_policy(net), H, gumbel=g)
    for key in a:
        assert a[key].tobytes() == b[key].cpu().numpy().tobytes(), key
    for e in envs + [fresh]:
        e.close()


def test_bad_arguments_raise():
    cfg, candles, minutes = _cfg("lean_fixed_pnl", 8)
    env = VecFxEnv(cfg, candles, minutes)
    for kw, exc in ((dict(leverage=0.0), ValueError), (dict(slippage=1.0), ValueError), (dict(commission=[1.0, 2.0]), ValueError),
                    (dict(k_sl=float("nan")), ValueError), (dict(commission="x"), TypeError)):
        with pytest.raises(exc):
            env.set_env_params(**kw)
        assert env.env_params is None
    bad = np.zeros((8, 7))
    bad[:, 1] = 1.0
    bad[3, 2] = 2.0
    assert env.L.fxenv_set_env_params(env._h, bad.ctypes.data) == -1
    msg = env.L.fxenv_last_error(env._h).decode()
    assert "env 3" in msg and "slippage" in msg, msg
    env.close()


# ------------------------------------------------------------------------------------------- a mid-episode change
def test_commission_set_mid_episode():
    """Open a long at commission 0, set commission c (and new SL / TP), hold until the bracket closes it: the commission
    paid is |size| * c * fill price, and the fill is at the bracket prices placed before the change."""
    T = 400
    cfgd = {**S.DEFAULTS, "window_size": 8, "sl_pips": 3.0, "tp_pips": 4.0, "position_size": 1000.0}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, "strategy": "direct_fixed_sltp"})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"], preprocessor_plugin=pl["preprocessor"],
                       reward_plugin=pl["reward"], columns=S.OHLCV, num_envs=1, order_capacity=64)
    candles = synth_candles(T, 0, 31)
    env = VecFxEnv(cfg, [candles], [synth_minutes(T)])
    env.set_env_params(commission=0.0)
    start = 50
    env.reset(torch.as_tensor([start]))
    step = lambda a: env.step(torch.as_tensor(np.array([a], np.int32)))
    info = lambda k: env.info()[k].cpu().numpy()[0]
    step(0)                                      # the first step does not advance (bar 0)
    step(1)                                      # bar 1: buy bracket at bar 1's close
    t_sig = 1
    pclose = candles[start + t_sig, 3]
    pip, size = cfg.pip_size if cfg.pair_pip_size[0] == 0.0 else cfg.pair_pip_size[0], cfg.strat_position_size
    stop, limit = pclose - cfg.sl_pips * pip, pclose + cfg.tp_pips * pip
    t = t_sig
    while info("position_size") == 0.0:
        step(0)
        t += 1
        assert t < 20, "the parent did not fill"
    assert info("position_size") == size and info("commission_paid") == 0.0
    c = 7e-5
    env.set_env_params(commission=c, sl_pips=50.0, tp_pips=60.0)
    while info("position_size") != 0.0:
        step(0)
        t += 1
        assert t < 300, "the bracket did not close"
    o, h, l = candles[start + t, 0], candles[start + t, 1], candles[start + t, 2]
    # the children are a sell stop @stop (examined first) and a sell limit @limit (bbroker _try_exec_stop / _try_exec_limit)
    if o <= stop:
        px = o
    elif l <= stop:
        px = stop
    elif limit <= o:
        px = o
    else:
        assert limit <= h
        px = limit
    assert info("commission_paid") == abs(size) * c * px, (info("commission_paid"), abs(size) * c * px)
    assert info("trades") == 1
    env.close()
