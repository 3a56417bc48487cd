"""The env kernels over their whole variant key (fx_kernels.cuh FX_V_*, DESIGN §4 "The variant key"): one cell per
(strategy, reward, step key) that has kernels, 3 x 3 x {general, FAST5, FAST5 + LEAN} x AUDIT (ATR only) x REPEAT x TRUNC
x PARAMS = 288 cells, each reaching its key through the public setters and checking that fxenv_debug_variant_key names
it.  Two tests need no device: the schedule below and the completeness of the matrix (every triple with kernels has a
cell).  The rest need one (-m gpu).  Per cell, on one seeded action stream of DECISIONS decisions:
  (a) step() in lock step with TimeLimitOracle(k, hold, audit, max_steps, window), built from the config or, with
      PARAMS, from the uniform table's row: codes, rewards, observations and info every step (compare_step,
      compare_info, the end bits of the flags), then the episode records, the audit records and the summary;
  (b) the same actions through step_many, persistent engine, FXENV_CHUNK=3, batches that end mid-episode, once with
      the order table resident in shared memory (FXENV_ORDER_SMEM=1) and once in global memory (0): obs, rewards,
      codes, get_state(), episode views and the audit ring bit for bit equal to (a) -- the 576 rollout kernels;
  (c) closed loop (HORIZON decisions), width-64 policy in the cell's action mode: a rollout without and one with an observation
      normalizer (random per-pair statistics, clip 3), each replayed through step() on a twin handle bit for bit; with
      the normalizer, the bf16 copy of the last two slots equals bf16_rn(clamp((x - mean) * rstd, -clip, clip)) --
      the 288 step and 288 step-norm kernels.
Each cell also asserts that what its bits switch on happened: a trade, a decision of more than one bar (REPEAT), a
code-2 step (TRUNC), an audit record (AUDIT), a reset step (auto_reset), a clipped element (normalizer), and no order-table
overflow.

How each bit is reached: general = default_preprocessor, or a 3-column feature window with an odd W (the first such cell
also carries a sixth candle column of NaN / +-inf); FAST5 without LEAN = OHLCV feature window with costs (commission,
leverage, slippage) or continuous actions; LEAN = OHLCV feature window, W % 4 == 0, no costs, discrete actions (with PARAMS
the config has costs and the row has none, so the LEAN choice follows the table); AUDIT = set_bracket_audit;
REPEAT = set_action_repeat(k, hold); TRUNC = set_time_limit; PARAMS = a uniform set_env_params table whose row differs
from the config in every field.

Schedule of the secondary dimensions.  i is the cell's index in the order strategy, reward, path, audit, repeat, trunc,
params; j_X is the cell's running index among the cells with property X:
  pairs        1 + i % 3
  N            (32, 33, 64)[(i // 3) % 3]
  auto_reset   (i // 9) % 2
  starts       per-env ranges [lo, lo + (0, 1, 90, 300)[env % 4]], seed 100 + i
  actions      LEAN off: continuous when j_lean_off has an odd number of 1 bits, else discrete; LEAN: discrete
  general      the 3-column feature window when j_general has an odd number of 1 bits, else default_preprocessor
  costs        general: when (i // 3) is even
  W            default_preprocessor (9, 12, 17), 3-column window (9, 13, 17), FAST5 (10, 13, 16), LEAN (8, 12, 16),
               each indexed by (j // 2) % 3 (general) or j % 3 (FAST5, LEAN) of the path's counter
  k, hold      REPEAT: k = (2, 3, 5)[j_repeat % 3], hold when (j_repeat // 3) is odd
  trunc mode   TRUNC: (limit 9 decisions, WINDOW, both: limit 13 + WINDOW)[j_trunc % 3]
Every value of every dimension meets every strategy and every reward (test_schedule_covers_every_strategy_and_reward).
Negative controls: comparisons against an oracle that is wrong in one setting must fail."""
import collections
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

import scenarios as S
from common_gpu import GpuVec, compare_info, compare_step, compare_summary, gpu_summary
from gym_fx_b200 import _native
from gym_fx_b200.config import ENV_PARAM_FIELDS, FxConfig, lower_config
from gym_fx_b200.synth import synth_candles, synth_minutes
from gym_fx_b200.vec_env import VecFxEnv
from time_limit_oracle import FLAG_TRUNCATED, TimeLimitOracle

FX_V_FAST5, FX_V_LEAN, FX_V_RESIDENT, FX_V_AUDIT, FX_V_REPEAT, FX_V_TRUNC, FX_V_PARAMS, FX_V_KEYS = 1, 2, 4, 8, 16, 32, 64, 128
STRATEGIES = {"default": "default_strategy", "fixed": "direct_fixed_sltp", "atr": "direct_atr_sltp"}   # FxConfig.strategy 0..2
REWARDS = {"pnl": "pnl_reward", "sharpe": "sharpe_reward", "dd": "dd_penalized_reward"}                # FxConfig.reward 0..2
PATHS = {"general": 0, "fast5": FX_V_FAST5, "lean": FX_V_FAST5 | FX_V_LEAN}
CFG_FIELD = dict(zip(ENV_PARAM_FIELDS, ("commission", "leverage", "slippage_perc", "sl_pips", "tp_pips", "k_sl", "k_tp")))
TRUNC_MODES = {"limit": (9, False), "window": (0, True), "both": (13, True)}
END_BITS = 2 | 4 | 8 | FLAG_TRUNCATED
AU_FIELDS = ("kind", "bar", "episode", "entry", "stop", "limit", "size", "atr")
DECISIONS = 40
BATCHES = (7, 11, 13, 9)      # step_many batches of the DECISIONS decisions: each ends inside episodes
HORIZON = 24                  # closed-loop decisions per rollout
COSTS = dict(commission=3e-5, leverage=4.0, slippage=2e-5)


# ---------------------------------------------------------------------------------------------------------- the cells
def _parity(j):
    return bin(j).count("1") % 2 == 1


def _matrix():
    cells, seen = [], collections.Counter()

    def nxt(what):
        seen[what] += 1
        return seen[what] - 1

    two = (False, True)
    for (s, strategy), (r, reward), path, audit, repeat, trunc, params in itertools.product(
            enumerate(STRATEGIES), enumerate(REWARDS), PATHS, two, two, two, two):
        if audit and strategy != "atr":
            continue
        i = len(cells)
        key = (PATHS[path] | (FX_V_AUDIT if audit else 0) | (FX_V_REPEAT if repeat else 0) | (FX_V_TRUNC if trunc else 0)
               | (FX_V_PARAMS if params else 0))
        c = dict(i=i, strategy=strategy, reward=reward, s=s, r=r, path=path, key=key, audit=audit, repeat=repeat,
                 trunc=trunc, params=params, pairs=1 + i % 3, N=(32, 33, 64)[(i // 3) % 3], auto_reset=(i // 9) % 2,
                 seed=100 + i)
        # parities of the running indices: balanced against each bit of the key
        c["continuous"] = path != "lean" and _parity(nxt("lean_off"))
        if path == "general":
            j = nxt("general")
            c["preproc"] = "fw3" if _parity(j) else "default"
            c["W"] = ((9, 13, 17) if _parity(j) else (9, 12, 17))[(j // 2) % 3]
            c["extra_col"] = j == 1
            c["costly"] = (i // 3) % 2 == 0
        else:
            c["preproc"] = "fw5"
            c["W"] = ((10, 13, 16) if path == "fast5" else (8, 12, 16))[nxt(path) % 3]
            c["extra_col"] = False
            # FAST5 off the LEAN path: costs, or continuous actions; LEAN: no costs, unless the table's cost-free row is
            # what makes it LEAN
            c["costly"] = (not c["continuous"]) if path == "fast5" else params
        c["k"], c["hold"] = 1, False
        if repeat:
            j = nxt("repeat")
            c["k"], c["hold"] = (2, 3, 5)[j % 3], (j // 3) % 2 == 1
        c["trunc_mode"] = ("limit", "window", "both")[nxt("trunc") % 3] if trunc else None
        c["id"] = "-".join([strategy, reward, path] + [b for b, on in (("audit", audit), ("repeat", repeat), ("trunc", trunc),
                                                                        ("params", params)) if on])
        cells.append(c)
    return cells


CELLS = _matrix()
CELL_BY_ID = {c["id"]: c for c in CELLS}
LAUNCHED = {"step": set(), "step_norm": set(), "rollout": set()}   # (strategy, reward, key) triples the cells ran


def _config(c):
    cfgd = {**S.DEFAULTS, "window_size": c["W"], "atr_period": 6, "sl_pips": 3.0, "tp_pips": 4.0, "k_sl": 1.5,
            "k_tp": 2.0, "window": 12}
    if c["costly"]:
        cfgd.update(commission=COSTS["commission"], leverage=COSTS["leverage"], slippage=COSTS["slippage"])
    plugins = {**S.DEFAULT_PLUGINS, "strategy": STRATEGIES[c["strategy"]], "reward": REWARDS[c["reward"]]}
    if c["preproc"] != "default":
        cfgd["feature_columns"] = list(S.OHLCV) if c["preproc"] == "fw5" else ["OPEN", "HIGH", "CLOSE"]
        cfgd["feature_scaling_window"] = 16
        plugins["preprocessor"] = "feature_window_preprocessor"
    if c["continuous"]:
        cfgd.update(action_space_mode="continuous", continuous_action_threshold=0.2)
    columns = list(S.OHLCV) + (["EXTRA"] if c["extra_col"] else [])
    pl = S.build_mirror_plugins(cfgd, plugins)
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"], preprocessor_plugin=pl["preprocessor"],
                       reward_plugin=pl["reward"], columns=columns, num_envs=c["N"], num_pairs=c["pairs"],
                       order_capacity=256, episode_bars=17 * c["k"])
    cfg.auto_reset = c["auto_reset"]
    if c["costly"]:   # every cost field set, whatever the broker plugin takes from the config
        for f, v in COSTS.items():
            setattr(cfg, CFG_FIELD[f], v)
    assert (cfg.strategy, cfg.reward) == (c["s"], c["r"])
    Ts = [1200 + 150 * p for p in range(c["pairs"])]
    candles = []
    for p, T in enumerate(Ts):
        t = synth_candles(T, p, 7 * c["i"] + p)
        if c["extra_col"]:
            x = np.linspace(-1.0, 1.0, T)
            x[::7], x[3::11], x[5::13] = np.nan, np.inf, -np.inf
            t = np.ascontiguousarray(np.concatenate([t, x[:, None]], axis=1))
        candles.append(t)
    return cfg, candles, [synth_minutes(T) for T in Ts], Ts


def _row(c, cfg):
    """The uniform table's row of a PARAMS cell: every field differs from the config; LEAN cells get a cost-free row on a
    costly config."""
    if not c["params"]:
        return None
    base = [getattr(cfg, CFG_FIELD[f]) for f in ENV_PARAM_FIELDS]
    if c["path"] == "lean":
        costs = [0.0, 1.0, 0.0]
    else:
        costs = [base[0] * 1.5 + 1e-5, base[1] * 2.0 + 1.0, base[2] * 2.0 + 3e-5]
    row = np.array(costs + [base[3] + 2.0, base[4] + 3.0, base[5] + 0.5, base[6] + 1.0])
    assert (row != np.array(base)).all()
    return row


def _with_row(cfg, row):
    out = FxConfig.from_buffer_copy(cfg)
    for f, v in zip(ENV_PARAM_FIELDS, row):
        setattr(out, CFG_FIELD[f], float(v))
    return out


def _ranges(N, Ts):
    lo = np.asarray([(29 * i) % (Ts[i % len(Ts)] // 2) for i in range(N)], np.int64)
    return lo, lo + np.asarray([[0, 1, 90, 300][i % 4] for i in range(N)], np.int64)


def _actions(c, shape):
    rng = np.random.default_rng(c["seed"])
    if c["continuous"]:
        return rng.uniform(-1.0, 1.0, shape).astype(np.float32)
    return rng.integers(0, 3, shape).astype(np.int32)


def _variant_key(env):
    f = env.L.fxenv_debug_variant_key
    f.argtypes, f.restype = [C.c_void_p], C.c_int
    return f(env._h)


def _handle(c, cfg, candles, minutes, Ts, row, env=None):
    """A handle (a new one, or `env`) with the cell's settings, reset to its first episodes; asserts that it runs the
    cell's key."""
    env = VecFxEnv(cfg, candles, minutes) if env is None else env
    env.set_episode_starts(*_ranges(c["N"], Ts), seed=c["seed"])
    if c["audit"]:
        env.set_bracket_audit(4096)
    if c["repeat"]:
        env.set_action_repeat(c["k"], hold=c["hold"])
    if c["trunc"]:
        env.set_time_limit(*TRUNC_MODES[c["trunc_mode"]])
    if c["params"]:
        env.set_env_params(**dict(zip(ENV_PARAM_FIELDS, row)))
    env.reset()
    got = _variant_key(env)
    assert got & ~FX_V_RESIDENT == c["key"], f"{c['id']}: the handle runs key {got}, not {c['key']}"
    return env


def _triple(c, key):
    return (c["s"], c["r"], key)


# ----------------------------------------------------------------------------------------------- (a) oracle lock step
def _per_env(r, n):
    env = r["env"].cpu().numpy()
    cols = np.stack([r[k].double().cpu().numpy() for k in AU_FIELDS], axis=1) if env.size else np.zeros((0, 8))
    return [cols[env == i] for i in range(n)]


def _compare_summary(tag, env, osum):
    """compare_summary, with sqn where it is well conditioned (as tests/test_gpu_episodes.py: the device evaluates it from
    running sums, the oracle from the list of trades; the sums themselves are compared bit for bit in the records)"""
    gs = gpu_summary(env)
    compare_summary(tag, {**gs, "sqn": np.full_like(gs["sqn"], np.nan)}, {**osum, "sqn": np.full_like(osum["sqn"], np.nan)})
    a, b = gs["sqn"], osum["sqn"]
    assert np.array_equal(np.isnan(a), np.isnan(b)), f"{tag}: sqn NaN pattern"
    rs = env.run_stats().cpu().numpy()
    n = np.maximum(env.info()["trades"].cpu().numpy().astype(np.float64), 1.0)
    ex2, mean = rs[:, _native.RS["pnl_sq"]] / n, rs[:, _native.RS["pnl_net"]] / n
    ok = ~np.isnan(a) & (ex2 - mean * mean > 1e-4 * ex2)
    np.testing.assert_allclose(a[ok], b[ok], rtol=1e-9, atol=1e-12, err_msg=f"{tag}: sqn")


def _lockstep(c, setup, acts, oracle_cfg=None, k=None, hold=None, max_steps=None):
    """Run (a).  The keyword arguments replace the oracle's settings (negative controls).  -> (the outputs of every step,
    the end state of the handle, what happened)"""
    cfg, candles, minutes, Ts, row = setup
    N = c["N"]
    ms, window = TRUNC_MODES[c["trunc_mode"]] if c["trunc"] else (0, False)
    if oracle_cfg is None:
        oracle_cfg = _with_row(cfg, row) if c["params"] else cfg
    orc = TimeLimitOracle(oracle_cfg, candles, minutes, k=c["k"] if k is None else k, hold=c["hold"] if hold is None else hold,
                          audit=c["audit"], max_steps=ms if max_steps is None else max_steps, window=window)
    orc.set_episode_starts(*_ranges(N, Ts), seed=c["seed"])
    gpu = GpuVec(cfg, candles, minutes)
    try:
        _handle(c, cfg, candles, minutes, Ts, row, gpu.env)
        np.testing.assert_allclose(gpu.env.obs.cpu().numpy(), orc.reset(), rtol=1e-5, atol=2e-6, err_msg=f"{c['id']}: reset obs")
        LAUNCHED["step"].add(_triple(c, c["key"]))
        steps, happened = [], collections.Counter()
        prev = np.zeros(N, np.uint8)
        for s in range(acts.shape[0]):
            tag = f"{c['id']} decision {s}"
            go, oo = gpu.step(acts[s]), orc.step(acts[s])
            code = gpu.env.terminated.cpu().numpy().copy()
            compare_step(tag, (go[0], go[1], go[2], code), oo)
            gi, oi = gpu.info(), orc.info()
            compare_info(tag, gi, oi)
            assert np.array_equal(gi["flags"].astype(np.int64) & END_BITS, oi["flags"].astype(np.int64) & END_BITS), f"{tag}: end flags"
            steps.append((go[0].copy(), go[1].copy(), code))
            happened["traded"] = max(happened["traded"], int(gi["trades"].max()))
            happened["multi_bar"] += int((orc.substeps > 1).sum())
            happened["truncated"] += int((code == 2).sum())
            happened["reset_steps"] += int(((prev != 0) & (code == 0)).sum()) if c["auto_reset"] else 0
            happened["overflow"] += int(((gi["flags"].astype(np.int64) & 16) != 0).sum())
            prev = code
        views = [x.cpu().numpy().copy() for x in gpu.env._episode_views()]
        for what, g, o in zip(("start", "episodes_done", "last_episode"), views, orc.episodes()):
            assert g.tobytes() == o.tobytes(), f"{c['id']}: episode records, {what}"
        happened["episodes"] = int(views[1].sum())
        ring = None
        if c["audit"]:
            ring = tuple(x.cpu().numpy().copy() for x in gpu.env._audit[:2])
            got = _per_env(gpu.env.bracket_audit(), N)
            for i in range(N):
                ref = orc.env_records(i)
                assert got[i].shape == ref.shape and got[i].tobytes() == ref.tobytes(), f"{c['id']}: audit records of env {i}"
                happened["audit_records"] += len(ref)
        _compare_summary(f"{c['id']}: summary", gpu.env, orc.summary())
        end = (gpu.env.get_state(), views, ring)
    finally:
        gpu.close()
        orc.close()
    return steps, end, happened


# --------------------------------------------------------------------------------------------- (b) persistent batches
def _batches(c, setup, acts, smem, monkeypatch):
    monkeypatch.setenv("FXENV_ENGINE", "persistent")
    monkeypatch.setenv("FXENV_CHUNK", "3")
    monkeypatch.setenv("FXENV_ORDER_SMEM", str(smem))
    try:
        env = _handle(c, *setup)
    finally:
        for v in ("FXENV_ENGINE", "FXENV_ORDER_SMEM"):
            monkeypatch.delenv(v)
    key = _variant_key(env)
    assert key == c["key"] | (FX_V_RESIDENT if smem else 0), f"{c['id']}: FXENV_ORDER_SMEM={smem} runs key {key}"
    LAUNCHED["rollout"].add(_triple(c, key))
    N, D = c["N"], env.obs_dim
    a_dev = torch.as_tensor(acts).cuda()
    out, s0 = [], 0
    for K in BATCHES:
        assert env.step_many_engine(K) == "persistent"
        ring = torch.empty((K, N, D), dtype=torch.float32, device="cuda")
        rew = torch.empty((K, N), dtype=torch.float32, device="cuda")
        term = torch.empty((K, N), dtype=torch.uint8, device="cuda")
        env.step_many(a_dev[s0:s0 + K].contiguous(), ring, rew, term)
        torch.cuda.synchronize()
        out += [(ring[j].cpu().numpy(), rew[j].cpu().numpy(), term[j].cpu().numpy()) for j in range(K)]
        s0 += K
    monkeypatch.delenv("FXENV_CHUNK")
    ring = tuple(x.cpu().numpy().copy() for x in env._audit[:2]) if c["audit"] else None
    end = (env.get_state(), [x.cpu().numpy().copy() for x in env._episode_views()], ring)
    env.close()
    return out, end


def _same_run(tag, got, want):
    (g_steps, g_end), (w_steps, w_end) = got, want
    assert len(g_steps) == len(w_steps)
    for s, (g, w) in enumerate(zip(g_steps, w_steps)):
        for what, x, y in zip(("obs", "reward", "code"), g, w):
            assert x.tobytes() == y.tobytes(), f"{tag}: decision {s}: {what}"
    assert g_end[0] == w_end[0], f"{tag}: state"
    for what, x, y in zip(("start", "episodes_done", "last_episode"), g_end[1], w_end[1]):
        assert x.tobytes() == y.tobytes(), f"{tag}: episode records, {what}"
    if w_end[2] is not None:
        for what, x, y in zip(("ring", "written"), g_end[2], w_end[2]):
            assert x.tobytes() == y.tobytes(), f"{tag}: audit {what}"


# -------------------------------------------------------------------------------------------------- (c) closed loop
def _bits(t):
    return t.contiguous().view(torch.int16)


def _norm_stats(obs, P, seed):
    """random per-pair statistics around the scale of the columns of obs [N, D]: mean [P, D], var [P, D] (float64)"""
    obs = obs.double().cpu()
    g = torch.Generator().manual_seed(seed)
    mean = torch.empty(P, obs.shape[1], dtype=torch.float64)
    var = torch.empty_like(mean)
    for p in range(P):
        x = obs[p::P]
        mu, sd = x.mean(0), x.std(0, unbiased=False) + 1e-3
        mean[p] = mu + sd * torch.randn(obs.shape[1], generator=g, dtype=torch.float64) * 0.5
        var[p] = (sd * (0.3 + torch.rand(obs.shape[1], generator=g, dtype=torch.float64))) ** 2
    return mean, var


def _replay(tag, twin, out):
    """step() on the twin with the rollout's actions gives the rollout's obs, rewards and codes bit for bit"""
    for t in range(out["actions"].shape[0]):
        o, r, _, _, _ = twin.step(out["actions"][t])
        torch.cuda.synchronize()
        assert torch.equal(o, out["obs"][t + 1]), f"{tag}: decision {t}: obs"
        assert torch.equal(r, out["reward"][t]), f"{tag}: decision {t}: reward"
        assert torch.equal(twin.terminated, out["done"][t]), f"{tag}: decision {t}: done"


def _closed_loop(c, setup):
    from gym_fx_b200.learner import ActorCritic
    a, b = (_handle(c, *setup) for _ in range(2))
    P, N = c["pairs"], c["N"]
    snap = a.get_state()
    assert snap == b.get_state()
    torch.manual_seed(c["seed"])
    plain = a.make_policy(ActorCritic(a.obs_dim, hidden=64, continuous=c["continuous"]).cuda())
    out = a.rollout(plain, HORIZON, seed=c["seed"])
    torch.cuda.synchronize()
    assert plain.sync_timeouts() == 0
    LAUNCHED["step"].add(_triple(c, c["key"]))
    _replay(f"{c['id']} rollout", b, out)
    assert a.get_state() == b.get_state(), f"{c['id']} rollout: state"
    mean, var = _norm_stats(out["obs"][0], P, c["seed"])
    net = ActorCritic(a.obs_dim, hidden=64, continuous=c["continuous"], obs_norm=True, num_pairs=P)
    net.obs_norm.mean.copy_(mean)
    net.obs_norm.var.copy_(var)
    net.obs_norm.clip = 3.0
    net = net.cuda()
    normed = a.make_policy(net)
    for e in (a, b):
        e.set_state(snap)
    out = a.rollout(normed, HORIZON, seed=c["seed"] + 1)
    torch.cuda.synchronize()
    assert normed.sync_timeouts() == 0
    LAUNCHED["step_norm"].add(_triple(c, _variant_key(a) & ~FX_V_RESIDENT))
    pair = torch.arange(N, device="cuda") % P
    D = a.obs_dim
    for t in (HORIZON - 1, HORIZON):
        want = _bits(net.obs_norm(out["obs"][t], pair).to(torch.bfloat16))
        o16 = normed.peek("obs16", t & 1)
        got = _bits(o16[:, :D])
        if not torch.equal(got, want):
            bad = (got != want).nonzero()[:5].tolist()
            raise AssertionError(f"{c['id']}: normalized bf16 copy of decision {t} differs at (env, column) {bad}")
        assert not bool(_bits(o16[:, D:]).any()), f"{c['id']}: pad columns of the bf16 copy are not 0"
    clipped = int((net.obs_norm(out["obs"].reshape(-1, D), pair.repeat(HORIZON + 1)).abs() == 3.0).sum())
    _replay(f"{c['id']} normalized rollout", b, out)
    assert a.get_state() == b.get_state(), f"{c['id']} normalized rollout: state"
    a.close()
    b.close()
    return clipped


# ------------------------------------------------------------------------------------------------------------ tests
def _setup(c):
    cfg, candles, minutes, Ts = _config(c)
    return cfg, candles, minutes, Ts, _row(c, cfg)


@pytest.mark.gpu
@pytest.mark.parametrize("cell", list(CELL_BY_ID))
def test_cell(cell, monkeypatch):
    for v in ("FXENV_ENGINE", "FXENV_CHUNK", "FXENV_ORDER_SMEM", "FXENV_NO_LEAN"):
        monkeypatch.delenv(v, raising=False)
    c = CELL_BY_ID[cell]
    setup = _setup(c)
    acts = _actions(c, (DECISIONS, c["N"]))
    steps, end, happened = _lockstep(c, setup, acts)
    for smem in (1, 0):
        _same_run(f"{cell} step_many FXENV_ORDER_SMEM={smem}", _batches(c, setup, acts, smem, monkeypatch), (steps, end))
    clipped = _closed_loop(c, setup)
    assert happened["traded"] > 0, f"{cell}: no env traded"
    assert happened["overflow"] == 0, f"{cell}: order table overflow"
    if c["repeat"]:
        assert happened["multi_bar"] > 0, f"{cell}: no decision ran more than one bar"
    if c["trunc"]:
        assert happened["truncated"] > 0, f"{cell}: no truncation"
    if c["audit"]:
        assert happened["audit_records"] > 0, f"{cell}: no audit record"
    if c["auto_reset"]:
        assert happened["reset_steps"] > 0, f"{cell}: no reset step"
    assert happened["episodes"] > 0 or not c["auto_reset"], f"{cell}: no episode record"
    assert clipped > 0, f"{cell}: the normalizer never clips"


def _first(**want):
    return next(c for c in CELLS if all(c[k] == v for k, v in want.items()))


# the comparison must reject an oracle that is wrong in one setting
CONTROLS = {
    "params_from_config": (dict(strategy="fixed", path="fast5", params=True, continuous=False), "oracle_cfg"),
    "limit_plus_one": (dict(strategy="default", trunc=True, trunc_mode="limit"), "max_steps"),
    "repeat_k_minus_one": (dict(strategy="atr", repeat=True, audit=True), "k"),
    "hold_as_repeat": (dict(strategy="fixed", repeat=True, hold=True, continuous=False), "hold"),
}


@pytest.mark.gpu
@pytest.mark.parametrize("control", sorted(CONTROLS))
def test_negative_control(control):
    want, what = CONTROLS[control]
    c = _first(**want)
    setup = _setup(c)
    wrong = {"oracle_cfg": setup[0], "max_steps": TRUNC_MODES[c["trunc_mode"] or "limit"][0] + 1, "k": c["k"] - 1,
             "hold": False}[what]
    acts = _actions(c, (DECISIONS, c["N"]))
    _lockstep(c, setup, acts)   # the right oracle passes
    with pytest.raises(AssertionError):
        _lockstep(c, setup, acts, **{what: wrong})


@pytest.mark.gpu
def test_every_kernel_of_the_matrix_ran():
    """After the whole matrix in this session: the distinct (strategy, reward, key) triples each kernel kind launched."""
    if len(LAUNCHED["step"]) < len(CELLS):
        pytest.skip("only part of the matrix ran in this session")
    counts = {k: len(v) for k, v in LAUNCHED.items()}
    print(f"\nlaunched triples: {counts}")
    assert counts == {"step": 288, "step_norm": 288, "rollout": 576}


# ------------------------------------------------------------------------------------------------- no device needed
def test_every_kernel_has_a_cell():
    """The library's (strategy, reward, key) triples with kernels are the cells (step and step-norm kernels: RESIDENT
    masked off), and the cells x {RESIDENT off, on} (rollout kernels).  A new FX_V_* bit fails here until the matrix
    covers it."""
    f = _native.load().fxenv_debug_variant_exists
    f.argtypes, f.restype = [C.c_int, C.c_int, C.c_uint32], C.c_int
    have = set()
    for s in range(3):
        for r in range(3):
            for key in range(FX_V_KEYS):
                e = f(s, r, key)
                assert e in (0, 1), (s, r, key, e)
                if e:
                    have.add((s, r, key))
    assert f(3, 0, 0) < 0 and f(0, 3, 0) < 0 and f(0, 0, FX_V_KEYS) < 0
    cells = {(c["s"], c["r"], c["key"]) for c in CELLS}
    assert len(cells) == len(CELLS) == 288
    assert {(s, r, key & ~FX_V_RESIDENT) for s, r, key in have} == cells
    assert have == {(s, r, key | res) for s, r, key in cells for res in (0, FX_V_RESIDENT)}


def test_schedule_covers_every_strategy_and_reward():
    """Every value of every secondary dimension meets every strategy and every reward."""
    dims = {
        "pairs": lambda c: c["pairs"], "N": lambda c: c["N"], "auto_reset": lambda c: c["auto_reset"],
        "W": lambda c: (c["preproc"], c["path"], c["W"]),
        "actions": lambda c: c["continuous"] if c["path"] != "lean" else None,
        "general": lambda c: c["preproc"] if c["path"] == "general" else None,
        "k_hold": lambda c: (c["k"], c["hold"]) if c["repeat"] else None,
        "trunc_mode": lambda c: c["trunc_mode"],
    }
    for name, f in dims.items():
        values = {f(c) for c in CELLS} - {None}
        assert len(values) > 1, name
        for v in values:
            for axis in ("strategy", "reward"):
                met = {c[axis] for c in CELLS if f(c) == v}
                assert met == set(STRATEGIES if axis == "strategy" else REWARDS), f"{name} = {v} misses a {axis}: {met}"
    for bit in ("audit", "repeat", "trunc", "params"):   # the action modes and preprocessors are not tied to a bit
        for on in (False, True):
            assert {c["continuous"] for c in CELLS if c[bit] == on and c["path"] != "lean"} == {False, True}, bit
            assert {c["preproc"] for c in CELLS if c[bit] == on and c["path"] == "general"} == {"default", "fw3"}, bit
    assert sum(c["extra_col"] for c in CELLS) == 1
    assert all(c["continuous"] or c["costly"] for c in CELLS if c["path"] == "fast5")
    assert not any(c["continuous"] or (c["costly"] and not c["params"]) for c in CELLS if c["path"] == "lean")
