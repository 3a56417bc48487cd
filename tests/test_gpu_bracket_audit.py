"""GPU: the bracket audit of direct_atr_sltp written by the step kernels (include/fxenv.h fxenv_set_bracket_audit).

  * GymFxEnv with GYMFX_BRACKET_AUDIT writes, for every tests/golden/audit fixture, the reference's file byte for byte.
  * 64 envs per ATR configuration (own starts, auto-reset, episode start ranges) against the C oracle: every field of
    every record, and the counters, bit for bit.
  * Single steps, step_many (persistent with the global / shared-memory order table, graph engine), LEAN and general
    kernels, and closed-loop rollouts replayed through step_many give identical rings and counters.
  * Logging changes nothing else: observations, rewards, done flags, info columns, run_stats, episode records and the
    state snapshot are bit-identical with the log on and off.
  * A decision whose orders find the order table full (FX_FLAG_ORDER_OVERFLOW) is still recorded.
  * Ring wrap-around, drain bookkeeping and the lifecycle (cached graphs, re-enable, reset / set_state, non-ATR configs,
    argument errors)."""
import os

import numpy as np
import pytest
import torch

import scenarios as S
from audit_ref import F, AuditOracle
from gym_fx_b200.config import lower_config
from gym_fx_b200.synth import synth_candles, synth_minutes
from gym_fx_b200.vec_env import VecFxEnv
from test_bracket_audit import audit_names, load_audit_case

pytestmark = pytest.mark.gpu

FIELDS = ("kind", "bar", "episode", "entry", "stop", "limit", "size", "atr")


def _cfg(n, strategy="direct_atr_sltp", reward="dd_penalized_reward", episode_bars=0, **kw):
    cfgd = {**S.DEFAULTS, "window_size": 16, "atr_period": 6, **kw}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, "strategy": strategy, "reward": reward})
    return lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"],
                        preprocessor_plugin=pl["preprocessor"], reward_plugin=pl["reward"], columns=S.OHLCV,
                        num_envs=n, order_capacity=256, episode_bars=episode_bars)


CONFIGS = {
    "plain_dd": dict(),
    "relvol_notional_lev_comm": dict(rel_volume=0.2, size_mode="notional", leverage=20.0, commission=2e-5,
                                     max_order_volume=50000.0, reward="pnl_reward"),
    "relvol_units_slip_sharpe": dict(rel_volume=0.05, slippage_perc=5e-5, reward="sharpe_reward", window=12),
    # entries only on Monday 01:00-05:00 of the synthetic week: positions still open at 05:00 are force-closed
    "session_filter": dict(session_filter=True, entry_dow_start=0, entry_hour_start=1, force_close_dow=0,
                           force_close_hour=5),
}


def _env(cfg, T=1200, pair=0, seed=3):
    candles, minutes = [synth_candles(T, pair, seed)], [synth_minutes(T)]
    return VecFxEnv(cfg, candles, minutes), candles, minutes


def _per_env(r, n):
    """bracket_audit() -> list over envs of float64 [k, 8] (FXENV_AU_* order)."""
    env = r["env"].cpu().numpy()
    cols = np.stack([r[k].double().cpu().numpy() for k in FIELDS], axis=1) if env.size else np.zeros((0, F))
    return [cols[env == i] for i in range(n)]


def _same(a, b):
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _bits(t):
    """The tensor's bits as integers (equal NaNs compare equal, different values never do)."""
    return t.view({torch.float64: torch.int64, torch.float32: torch.int32}[t.dtype]) if t.is_floating_point() else t


# ---------------------------------------------------------------------------------------------------------- GymFxEnv
@pytest.mark.parametrize("name", audit_names())
def test_gymfxenv_writes_the_reference_file(name, tmp_path, monkeypatch):
    from gym_fx_b200 import GymFxEnv
    from gym_fx_b200.strategy_plugins import direct_atr_sltp as atr
    from gym_fx_b200.synth import write_csv

    g, want = load_audit_case(name)
    path = tmp_path / "audit.jsonl"
    monkeypatch.setattr(atr, "_AUDIT_PATH", str(path))
    csv = tmp_path / "data.csv"
    write_csv(str(csv), g["candles"], g["minutes"])
    config = {**g["meta"]["config"], "input_data_file": str(csv)}
    pl = S.build_mirror_plugins(config, g["meta"]["plugins"])
    env = GymFxEnv(config, pl["data_feed"], pl["broker"], pl["strategy"], pl["preprocessor"], pl["reward"], pl["metrics"])
    env.reset()
    for a in g["actions"][:g["reward"].shape[0] - 1]:
        env.step(int(a))
    env.close()
    assert path.read_text(encoding="utf-8") == want


# ------------------------------------------------------------------------------------------------ random vs oracle
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_records_match_the_oracle_with_auto_reset_and_start_ranges(name):
    kw = dict(CONFIGS[name])
    reward = kw.pop("reward", "dd_penalized_reward")
    N, T, steps = 64, 1500, 420
    cfg = _cfg(N, reward=reward, episode_bars=150, **kw)
    cfg.auto_reset = 1
    gpu, candles, minutes = _env(cfg, T)
    orc = AuditOracle(cfg, candles, minutes)
    rng = np.random.default_rng(11)
    lo = rng.integers(0, 600, N)
    hi = lo + rng.integers(0, 500, N)
    starts = rng.integers(0, 1200, N)
    gpu.set_episode_starts(lo, hi, seed=77)
    orc.set_episode_starts(lo, hi, seed=77)
    gpu.set_bracket_audit(1024)
    gpu.reset(torch.as_tensor(starts))
    orc.reset(starts)
    for k in range(steps):
        a = rng.integers(0, 3, N).astype(np.int32)
        gpu.step(torch.as_tensor(a))
        orc.step(a, want_obs=False)
    got = _per_env(gpu.bracket_audit(), N)
    written = gpu._audit[1].cpu().numpy()
    total = 0
    for i in range(N):
        ref = orc.env_records(i)
        assert _same(got[i], ref), (name, i, got[i][:3], ref[:3])
        assert written[i] == len(ref)
        total += len(ref)
    assert total > N * 5
    assert len(np.unique(np.concatenate([orc.env_records(i)[:, 2] for i in range(N)]))) > 1, "no auto-reset happened"
    if name == "session_filter":
        assert any((orc.env_records(i)[:, 0] == 3).any() for i in range(N))
    gpu.close()


# ------------------------------------------------------------------------------------------------ engines agree
def _run_engine(cfg, acts, how, monkeypatch, starts):
    for k in ("FXENV_ORDER_SMEM", "FXENV_ENGINE", "FXENV_NO_LEAN"):
        monkeypatch.delenv(k, raising=False)
    if how.startswith("smem"):
        monkeypatch.setenv("FXENV_ORDER_SMEM", how[-1])
        monkeypatch.setenv("FXENV_ENGINE", "persistent")
    elif how == "graph":
        monkeypatch.setenv("FXENV_ENGINE", "graph")
    elif how == "nolean":
        monkeypatch.setenv("FXENV_NO_LEAN", "1")
    env, _, _ = _env(cfg, 3000)
    env.set_bracket_audit(4096)
    env.reset(torch.as_tensor(starts))
    K, N = acts.shape
    if how in ("single", "nolean"):
        for k in range(K):
            env.step(torch.as_tensor(acts[k]).cuda())
    else:
        ring = torch.empty((2, N, env.obs_dim), dtype=torch.float32, device="cuda")
        for k0 in range(0, K, 100):
            a = torch.as_tensor(acts[k0:k0 + 100]).cuda().contiguous()
            env.step_many(a, ring, torch.empty(a.shape, dtype=torch.float32, device="cuda"),
                          torch.empty(a.shape, dtype=torch.uint8, device="cuda"))
    torch.cuda.synchronize()
    ring, written, _ = env._audit
    out = (ring.cpu().numpy().copy(), written.cpu().numpy().copy(), env.get_state(), env.L.fxenv_debug_lean(env._h))
    env.close()
    return out


@pytest.mark.parametrize("lean", [True, False], ids=["cfg3_shape", "general"])
def test_engines_give_identical_rings(lean, monkeypatch):
    N, K = 96, 400
    if lean:   # the cfg3 family: feature window W=32 over OHLCV, dd reward (LEAN kernels unless FXENV_NO_LEAN)
        cfgd = {**S.DEFAULTS, "window_size": 32, "feature_columns": list(S.OHLCV), "feature_scaling_window": 64}
        pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, "strategy": "direct_atr_sltp",
                                           "preprocessor": "feature_window_preprocessor", "reward": "dd_penalized_reward"})
        cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"],
                           preprocessor_plugin=pl["preprocessor"], reward_plugin=pl["reward"], columns=S.OHLCV,
                           num_envs=N, order_capacity=256)
    else:
        cfg = _cfg(N, commission=1e-5, slippage_perc=3e-5, session_filter=True, entry_dow_start=0, entry_hour_start=2,
                   force_close_dow=4, force_close_hour=20)
    acts = np.random.default_rng(5).integers(0, 3, (K, N)).astype(np.int32)
    starts = np.random.default_rng(6).integers(0, 2400, N)
    base = _run_engine(cfg, acts, "single", monkeypatch, starts)
    assert base[1].sum() > N * 10
    assert base[3] == (1 if lean else 0), "the configuration no longer selects the kernels this case is about"
    for how in ("smem0", "smem1", "graph") + (("nolean",) if lean else ()):
        other = _run_engine(cfg, acts, how, monkeypatch, starts)
        assert _same(other[0], base[0]) and _same(other[1], base[1]), how
        assert other[2] == base[2], how
        assert other[3] == (0 if how == "nolean" else base[3]), how


def test_record_is_written_when_the_order_table_overflows():
    """64 envs with a 32-entry order table that runs full (test_bracket_audit.overflow_case), against the oracle, whose
    order list is unbounded: every env's records equal the oracle's up to and including the step at which its table
    overflowed and the orders were dropped, and that step wrote a record."""
    from test_bracket_audit import overflow_case
    N, K = 64, 400
    cfg, candles, minutes = overflow_case(N)
    gpu = VecFxEnv(cfg, [candles], [minutes])
    orc = AuditOracle(cfg, [candles], [minutes])
    starts = np.random.default_rng(12).integers(0, 700, N)
    gpu.set_bracket_audit(K)
    gpu.reset(torch.as_tensor(starts))
    orc.reset(starts)
    acts = np.stack([S.make_actions(("sticky", 100 + i, 0.3), K) for i in range(N)], axis=1)
    counts, ocounts, flags = [], [], []
    for k in range(K):
        gpu.step(torch.as_tensor(acts[k]))
        orc.step(acts[k], want_obs=False)
        counts.append(gpu._audit[1].cpu().numpy().copy())
        ocounts.append(np.array([len(r) for r in orc.records]))
        flags.append(gpu.info()["flags"].cpu().numpy().copy())
    got = _per_env(gpu.bracket_audit(), N)
    counts, ocounts, flags = np.array(counts), np.array(ocounts), np.array(flags)
    overflowed = 0
    for i in range(N):
        hit = np.nonzero(flags[:, i] & 16)[0]
        if not hit.size:
            assert _same(got[i], orc.env_records(i)), i
            continue
        k = int(hit[0])
        overflowed += 1
        assert counts[k, i] == ocounts[k, i] and counts[k, i] == (counts[k - 1, i] if k else 0) + 1, i
        n = int(counts[k, i])
        assert _same(got[i][:n], orc.env_records(i)[:n]), i
    assert overflowed >= N // 2
    gpu.close()


@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_rollout_records_equal_step_many_replay(continuous):
    """A closed-loop rollout whose graph was cached with the log off records once the log is on; replaying its actions
    through step_many on a twin env gives the same records and state."""
    from gym_fx_b200.learner import ActorCritic
    N, H = 128, 48
    cfg = _cfg(N, **({"action_space_mode": "continuous"} if continuous else {}))
    a, _, _ = _env(cfg, 2000)
    b, _, _ = _env(cfg, 2000)
    starts = torch.as_tensor(np.random.default_rng(1).integers(0, 1800, N))
    torch.manual_seed(0)
    net = ActorCritic(a.obs_dim, continuous=continuous).cuda()
    pol = a.make_policy(net)
    a.reset(starts)
    b.reset(starts)
    bufs = {}
    obs_ring = torch.empty((2, N, b.obs_dim), dtype=torch.float32, device="cuda")
    rew = torch.empty((H, N), dtype=torch.float32, device="cuda")
    term = torch.empty((H, N), dtype=torch.uint8, device="cuda")
    for on in (False, True):
        if on:
            a.set_bracket_audit(256)
            b.set_bracket_audit(256)
        out = a.rollout(pol, H, buffers=bufs, seed=5)       # same buffers and seed: the cached graph unless invalidated
        b.step_many(out["actions"].clone(), obs_ring, rew, term)
    torch.cuda.synchronize()
    ra, rb = _per_env(a.bracket_audit(), N), _per_env(b.bracket_audit(), N)
    assert sum(len(x) for x in ra) > 0
    for i in range(N):
        assert _same(ra[i], rb[i]), i
    assert a.get_state() == b.get_state()
    a.close()
    b.close()


# ------------------------------------------------------------------------------------------------ nothing disturbed
def test_log_changes_nothing_else():
    N, K = 128, 500
    cfg = _cfg(N, episode_bars=120, session_filter=True, entry_dow_start=0, entry_hour_start=2, force_close_dow=4,
               force_close_hour=20)
    cfg.auto_reset = 1
    on, _, _ = _env(cfg, 2000)
    off, _, _ = _env(cfg, 2000)
    on.set_bracket_audit(2)
    for e in (on, off):
        e.set_episode_starts(0, 1500, seed=9)
        e.reset()
    rng = np.random.default_rng(4)
    for k in range(K):
        a = torch.as_tensor(rng.integers(0, 3, N).astype(np.int32)).cuda()
        so, ro, to, _, _ = on.step(a)
        sf, rf, tf, _, _ = off.step(a)
        assert torch.equal(so, sf) and torch.equal(ro, rf) and torch.equal(to, tf), k
        if k % 50 == 0:
            on.bracket_audit()
    io, iff = on.info(), off.info()
    for key in io.keys():
        assert torch.equal(io[key], iff[key]), key
    assert torch.equal(on.run_stats(), off.run_stats())
    for x, y in zip(on._episode_views(), off._episode_views()):   # start, episodes_done, the records themselves
        assert torch.equal(_bits(x), _bits(y))
    eo, ef = on.episode_stats(), off.episode_stats()
    for key in eo:   # the derived columns too, bit for bit (NaN where there is no closed trade)
        assert torch.equal(_bits(eo[key]), _bits(ef[key])), key
    assert int(on.episode_stats()["episodes_done"].sum()) > 0
    assert on.get_state() == off.get_state()
    assert int(on._audit[1].sum()) > 0
    on.close()
    off.close()


# ------------------------------------------------------------------------------------------------ rings
@pytest.mark.parametrize("cap", [1, 3])
def test_small_rings_keep_the_last_records(cap):
    N, K = 32, 300
    cfg = _cfg(N)
    ref, _, _ = _env(cfg)
    small, _, _ = _env(cfg)
    ref.set_bracket_audit(K)
    small.set_bracket_audit(cap)
    acts = np.random.default_rng(8).integers(0, 3, (K, N)).astype(np.int32)
    for e in (ref, small):
        e.reset()
        for k in range(K):
            e.step(torch.as_tensor(acts[k]).cuda())
    full = _per_env(ref.bracket_audit(), N)
    r = small.bracket_audit()
    got = _per_env(r, N)
    written = small._audit[1].cpu().numpy()
    dropped = r["dropped"].cpu().numpy()
    for i in range(N):
        n = len(full[i])
        assert written[i] == n
        assert dropped[i] == max(0, n - cap)
        assert _same(got[i], full[i][max(0, n - cap):]), i
    assert int(small.bracket_audit()["kind"].numel()) == 0   # nothing new since the drain
    # draining after every step loses nothing: at most one record per env-step
    small.set_bracket_audit(1)
    ref.set_bracket_audit(K)
    small.reset()
    ref.reset()
    drained = [[] for _ in range(N)]
    for k in range(K):
        for e in (ref, small):
            e.step(torch.as_tensor(acts[k]).cuda())
        r = small.bracket_audit()
        assert int(r["dropped"].sum()) == 0
        for i, x in enumerate(_per_env(r, N)):
            drained[i].extend(x)
    full = _per_env(ref.bracket_audit(), N)
    for i in range(N):
        assert _same(np.asarray(drained[i]).reshape(-1, F), full[i]), i
    ref.close()
    small.close()


# ------------------------------------------------------------------------------------------------ lifecycle
def test_lifecycle():
    N, K = 64, 120
    cfg = _cfg(N)
    env, _, _ = _env(cfg)
    env.reset()
    acts = torch.as_tensor(np.random.default_rng(2).integers(0, 3, (K, N)).astype(np.int32)).cuda()
    ring = torch.empty((2, N, env.obs_dim), dtype=torch.float32, device="cuda")
    rew = torch.empty((K, N), dtype=torch.float32, device="cuda")
    term = torch.empty((K, N), dtype=torch.uint8, device="cuda")
    os.environ["FXENV_ENGINE"] = "graph"
    try:
        g, _, _ = _env(cfg)
    finally:
        del os.environ["FXENV_ENGINE"]
    g.reset()
    for e in (env, g):
        e.step_many(acts, ring, rew, term)                  # graphs cached with the log off
    for e in (env, g):
        e.set_bracket_audit(512)
        e.step_many(acts, ring, rew, term)                  # the next call records
    n_on = [int(e._audit[1].sum()) for e in (env, g)]
    assert n_on[0] > 0 and n_on[0] == n_on[1]
    blob = env.get_state()
    env.reset()                                             # reset / set_state leave the log alone
    env.set_state(blob)
    assert int(env._audit[1].sum()) == n_on[0]
    env.set_bracket_audit(0)
    with pytest.raises(Exception):
        env.bracket_audit()
    env.step_many(acts, ring, rew, term)                    # off: nothing is written anywhere
    env.set_bracket_audit(7)                                # re-enabled at another capacity: counters from 0
    assert env._audit[0].shape[1] == 7 and int(env._audit[1].sum()) == 0
    env.step_many(acts, ring, rew, term)
    assert int(env._audit[1].sum()) > 0
    with pytest.raises(ValueError):
        env.set_bracket_audit(-1)
    assert env.L.fxenv_set_bracket_audit(env._h, -5) == -1
    env.close()
    g.close()
    for strat in ("direct_fixed_sltp", "default_strategy"):   # accepted, records nothing
        e, _, _ = _env(_cfg(N, strategy=strat))
        e.set_bracket_audit(16)
        e.reset()
        e.step_many(acts, ring, rew, term)
        torch.cuda.synchronize()
        assert int(e._audit[1].sum()) == 0 and e.bracket_audit()["kind"].numel() == 0
        e.close()
