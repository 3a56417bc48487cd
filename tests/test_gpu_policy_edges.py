"""GPU (-m gpu): the fused policy kernel (gym_fx_b200/csrc/fx_policy.cu) at every shape it accepts, bit for bit where
the arithmetic allows.

  a. observation widths of 1 to 5 layer-1 k-blocks (D = 30 ... 291, with and without pad columns): h1 read back from
     the library (FusedPolicy.peek) within check_h1 of the fp64 reference for every row, padded rows = the zero-row
     evaluation, value / logits / mean / log-prob against forward_ref, each comparison with negative controls;
  b. env counts and env-group splits (ragged last tiles in later groups, an empty trailing group), tile hand-over on
     and off, with every rollout buffer at the front of a sentinel-filled allocation (no write outside [0, N));
     groups 1-4 x tile hand-over 0/1 bit-identical;
  d. the bf16 observation copy (the policy's A operand) = round-to-nearest-even of the float32 row, bit for bit, pad
     columns 0, for every emitter variant of the step / observe kernels;
  e. the sampling epilogue with a zero body (logits = b_pi exactly): caller noise bit-exact, greedy ties, the in-kernel
     Gumbel noise against an exact replica of the counter-based generator (incl. draws at the top of its grid), a
     chi-square test of the sampling frequencies, continuous-mode noise;
  f. a 2-slot observation ring gives the same rollout as the full [H + 1] buffer."""
import math

import numpy as np
import pytest
import torch
import torch.nn as nn

import policy_ref as R
import scenarios as S
from gym_fx_b200.config import lower_config
from gym_fx_b200.synth import start_offsets, synth_candles, synth_minutes

pytestmark = pytest.mark.gpu

T_BARS = 3000
OHLC = ["OPEN", "HIGH", "LOW", "CLOSE"]
_DATA = {}


def _data(kind):
    """-> (candles [T, C], columns, minutes), cached per kind."""
    if kind not in _DATA:
        if kind == "synth":
            _DATA[kind] = (synth_candles(T_BARS, 0), list(S.OHLCV), synth_minutes(T_BARS))
        else:
            tab, cols, mins = S.make_data(("synth_extra", T_BARS, 68))
            if kind == "nonfinite":   # NaN / +-inf in the extra FEAT_A column (the nan_to_num / clip path)
                tab = tab.copy()
                tab[5::37, 5] = np.nan
                tab[11::53, 5] = np.inf
                tab[23::61, 5] = -np.inf
            _DATA[kind] = (np.ascontiguousarray(tab), cols, mins)
    return _DATA[kind]


def _factory(N, W, *, preproc="fw", features=tuple(S.OHLCV), data="synth", continuous=False, price=True, agent=True,
             scaling=None, binary=(), clip=None, commission=0.0, **kw):
    from gym_fx_b200.vec_env import VecFxEnv
    cfgd = {**S.DEFAULTS, "window_size": W, "commission": commission}
    plugins = {**S.DEFAULT_PLUGINS, "strategy": "direct_fixed_sltp"}
    if preproc == "fw":
        cfgd.update({"feature_columns": list(features), "include_price_window": price, "include_agent_state": agent,
                     "feature_binary_columns": list(binary)})
        if scaling:
            cfgd["feature_scaling"] = scaling
        if clip is not None:
            cfgd["feature_clip"] = clip
        plugins["preprocessor"] = "feature_window_preprocessor"
    if continuous:
        cfgd["action_space_mode"] = "continuous"
    candles, cols, mins = _data(data)
    pl = S.build_mirror_plugins(cfgd, plugins)
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"], preprocessor_plugin=pl["preprocessor"],
                       reward_plugin=pl["reward"], columns=cols, num_envs=N, order_capacity=64, **kw)
    return lambda: VecFxEnv(cfg, [candles], [mins])


class _Net(nn.Module):
    def __init__(self, D, n_pi):
        super().__init__()
        self.body = nn.Sequential(nn.Linear(D, 256), nn.Tanh(), nn.Linear(256, 256), nn.Tanh())
        self.pi = nn.Linear(256, n_pi)
        self.v = nn.Linear(256, 1)


def _weights(D, continuous, seed, log_std=-0.5):
    torch.manual_seed(seed)
    w = R.weights_of(R.scaled_init(_Net(D, 1 if continuous else 3)))
    if continuous:
        w["log_std"] = torch.tensor([log_std])
    return {k: v.cuda() for k, v in w.items()}


def _zero_body(D, b_pi, b_v=0.375, continuous=False):
    """W1 = W2 = b1 = b2 = 0: tanh.approx(0) = 0, so h2 = 0 and the logits / mean are b_pi exactly."""
    n = 1 if continuous else 3
    g = torch.Generator().manual_seed(17)
    w = {"w1": torch.zeros(256, D), "b1": torch.zeros(256), "w2": torch.zeros(256, 256), "b2": torch.zeros(256),
         "w_pi": torch.randn((n, 256), generator=g), "b_pi": torch.tensor(b_pi[:n], dtype=torch.float32),
         "w_v": torch.randn(256, generator=g), "b_v": torch.tensor([b_v])}
    if continuous:
        w["log_std"] = torch.tensor([b_pi[1]], dtype=torch.float32)
    return {k: v.cuda() for k, v in w.items()}


def _warm(envs, N, steps, continuous):
    g = torch.Generator().manual_seed(1)
    for _ in range(steps):
        a = (torch.rand(N, generator=g) * 2 - 1) if continuous else torch.randint(0, 3, (N,), generator=g, dtype=torch.int32)
        for e in envs:
            e.step(a.cuda())


def _check_env_side(env, twin, out, H):
    obs, act, rew, done = (out[k] for k in ("obs", "actions", "reward", "done"))
    o0 = torch.empty_like(obs[0])
    twin.L.fxenv_observe(twin._h, o0.data_ptr(), twin._stream())
    torch.cuda.synchronize()
    assert torch.equal(obs[0], o0), "rollout must start from the env's current observation"
    for t in range(H):
        o, r, term, _, _ = twin.step(act[t])
        assert torch.equal(o, obs[t + 1]), f"obs after step {t}"
        assert torch.equal(r, rew[t]) and torch.equal(term.to(torch.uint8), done[t]), f"reward / done at step {t}"
    for k in ("equity", "cash", "trades", "position", "n_orders", "bar_index"):
        assert torch.equal(env.info()[k], twin.info()[k]), k


def _bits16(t):
    return t.contiguous().view(torch.int16)


def _check_obs16(pol, D, obs_row, slot, tag):
    """the bf16 copy of `slot` = RNE(float32 rows) bit for bit, pad columns exactly 0"""
    o16 = pol.peek("obs16", slot)
    assert o16.shape[1] == (D + 63) // 64 * 64, tag
    got, want = _bits16(o16[:, :D]), _bits16(obs_row.to(torch.bfloat16))
    if not torch.equal(got, want):
        bad = (got != want).nonzero()[:5].tolist()
        raise AssertionError(f"{tag}: bf16 observation copy differs at (env, column) {bad}")
    assert not bool(_bits16(o16[:, D:]).any()), f"{tag}: pad columns of the bf16 copy are not 0"


H1_STATS = []   # (tag, max_ulps, frac_equal) of every h1 comparison, printed by the last test of the module


def _check_h1_and_controls(pol, w, obs, N, agent, tag):
    h1 = pol.peek("h1")
    NP = (N + 127) // 128 * 128
    assert h1.shape == (NP, 256), tag
    ref = R.forward_ref(w, obs)
    rep = R.check_h1(h1[:N], ref, obs, w)
    H1_STATS.append((tag, rep["max_ulps"], rep["max_ulps_big"], rep["frac_equal"]))
    assert rep["bad"] == 0, (tag, rep)
    # tightness floors, from the H100 runs of this file: >= 99.92% of the elements equal the rounded fp64 reference and
    # none with |h1| >= 1/16 is off by more than 1 bf16 ulp (elements near 0 may be off by more ulps, within the bound:
    # there the fp32 accumulation error exceeds a bf16 ulp).  The bound is a worst case; these catch a systematic loss.
    assert rep["max_ulps_big"] <= 1.0 and rep["frac_equal"] >= 0.998, (tag, rep)
    ctl = R.control_refs(w, obs, agent=agent)
    for name in R.H1_CONTROLS:
        if name in ctl and not (name == "rows_shifted" and N == 1):
            assert R.check_h1(h1[:N], ctl[name], obs, w)["bad"] > 0, f"{tag}: h1 check does not reject control {name}"
    if NP > N:   # rows past the env count: TMA fills the missing observation rows with 0 -> bf16(tanh.approx(b1))
        pad = h1[N:]
        assert torch.equal(_bits16(pad), _bits16(pad[:1].expand_as(pad))), f"{tag}: padded h1 rows differ"
        z = torch.zeros((1, obs.shape[1]), device=obs.device)
        assert R.check_h1(pad[:1], R.forward_ref(w, z), z, w)["bad"] == 0, f"{tag}: padded h1 rows"
    return ref


def _check_heads(out, w, noise, H, N, continuous, tag):
    """value / logits or mean / log-prob of every step against forward_ref, with the negative controls at step 0"""
    obs, act, logp, val = out["obs"], out["actions"], out["logp"], out["value"]
    controls = [c for c in R.HEAD_CONTROLS if not (c == "rows_shifted" and N == 1)]   # one row: a shift is no change
    n_flip = 0
    for t in range(H + 1):
        ref = R.forward_ref(w, obs[t])
        assert R.head_close(val[t], ref["value"]), (tag, t, R.head_err(val[t], ref["value"]))
        if t == 0:
            ctl = R.control_refs(w, obs[t], agent=False)
            for name in controls:
                assert not R.head_close(val[t], ctl[name]["value"]), f"{tag}: value check does not reject {name}"
        if t == H:
            break
        if continuous:
            sigma = math.exp(float(w["log_std"]))
            want = ref["head"][:, 0] + sigma * noise[t].double()
            assert R.head_close(act[t], want), (tag, t, R.head_err(act[t], want))
            # logp does not depend on the mean: -eps^2/2 - log sigma - log(2 pi)/2 in float32, same operation order
            eps, ls = noise[t], w["log_std"].float()
            assert torch.equal(logp[t], ((-0.5 * eps) * eps - ls) - np.float32(0.5 * math.log(2 * math.pi))), (tag, t)
            if t == 0:
                for name in controls:
                    bad = ctl[name]["head"][:, 0] + sigma * noise[t].double()
                    assert not R.head_close(act[t], bad), f"{tag}: mean check does not reject {name}"
        else:
            sc = ref["head"] + noise[t].double()
            a_ref = sc.argmax(-1)
            top2 = sc.topk(2, -1).values
            same = act[t].long() == a_ref
            assert bool((same | (top2[:, 0] - top2[:, 1] < 5e-3)).all()), (tag, t)
            n_flip += int((~same).sum())
            lp = torch.log_softmax(ref["head"], -1).gather(1, act[t].long()[:, None]).squeeze(1)
            assert R.head_close(logp[t], lp, 3e-3), (tag, t, R.head_err(logp[t], lp))
            if t == 0:
                for name in controls:
                    lpc = torch.log_softmax(ctl[name]["head"], -1).gather(1, act[t].long()[:, None]).squeeze(1)
                    assert not R.head_close(logp[t], lpc, 3e-3), f"{tag}: log-prob check does not reject {name}"
    assert n_flip <= max(2, H * N // 500), (tag, n_flip)


def _noise(H, N, continuous, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if continuous:
        return torch.randn((H, N), device="cuda", generator=g)
    return -torch.log(-torch.log(torch.rand((H, N, 3), device="cuda", generator=g).clamp(1e-9, 1 - 1e-9)))


def _rollout(env, pol, H, noise, continuous, **kw):
    return env.rollout(pol, H, **({"noise": noise} if continuous else {"gumbel": noise}), **kw)


# ----------------------------------------------------------------------------------------------------- a. obs widths
# (name, env settings, obs_dim, layer-1 k-blocks, agent scalars at the end of the row)
SHAPES = [
    ("default_w30", dict(W=30, preproc="default"), 64, 1, True),                      # no pad columns
    ("default_w13", dict(W=13, preproc="default"), 30, 1, True),
    ("ohlc_w32_noprice_noagent", dict(W=32, features=OHLC, price=False, agent=False), 128, 2, False),   # no pad
    ("ohlcv_w20", dict(W=20), 144, 3, True),                                          # LEAN fast5
    ("ohlcv_w36", dict(W=36), 256, 4, True),                                          # no pad, k-blocks = ring stages
    ("ohlcv_w41", dict(W=41), 291, 5, True),                                          # odd W: pair path + tail element
]


@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
@pytest.mark.parametrize("name,kw,D,kb,agent", SHAPES, ids=[s[0] for s in SHAPES])
def test_obs_width_matrix(name, kw, D, kb, agent, continuous):
    N, H = 300, 3
    kw = dict(kw)
    make = _factory(N, kw.pop("W"), continuous=continuous, **kw)
    env, twin = make(), make()
    assert env.obs_dim == D and (D + 63) // 64 == kb, "the config lowering moved this shape"
    starts = torch.as_tensor(start_offsets(N, T_BARS, 200, 300))
    env.reset(starts); twin.reset(starts)
    _warm((env, twin), N, 12, continuous)
    w = _weights(D, continuous, seed=kb)
    pol = env.make_policy(w)
    noise = _noise(H, N, continuous, seed=kb)
    out = _rollout(env, pol, H, noise, continuous)
    torch.cuda.synchronize()
    _check_env_side(env, twin, out, H)
    tag = f"{name}/{'cont' if continuous else 'disc'}"
    _check_h1_and_controls(pol, w, out["obs"][H], N, agent, tag)   # h1 of the bootstrap evaluation
    _check_obs16(pol, D, out["obs"][H], H % 2, tag)
    _check_heads(out, w, noise, H, N, continuous, tag)
    env.close(); twin.close()


# ------------------------------------------------------------------------------- b./c. env counts and group splits
def _sentinel_buffers(H, N, D, dtype_act):
    """rollout buffers as views at the front of larger allocations filled with a sentinel pattern"""
    spec = {"obs": ((H + 1, N, D), torch.float32), "actions": ((H, N), dtype_act), "logp": ((H, N), torch.float32),
            "value": ((H + 1, N), torch.float32), "reward": ((H, N), torch.float32), "done": ((H, N), torch.uint8)}
    bufs, backing = {}, {}
    for k, (shape, dt) in spec.items():
        n = int(np.prod(shape))
        extra = 128 * int(np.prod(shape[1:])) // N + 4096   # > one tile of rows
        raw = torch.full((n + extra,), 0x5A if dt == torch.uint8 else -0x2F2F2F2F, dtype=torch.uint8 if dt == torch.uint8 else torch.int32, device="cuda")
        backing[k] = raw
        bufs[k] = raw[:n].view(dt).view(shape) if dt != torch.uint8 else raw[:n].view(shape)
    return bufs, backing, {k: v[int(np.prod(spec[k][0])):].clone() for k, v in backing.items()}


GROUP_CASES = [(1, None), (127, None), (129, None), (2049, None), (6000, None), (8392, None), (1000, 3), (300, 4)]


@pytest.mark.parametrize("tile_sync", [0, 1])
@pytest.mark.parametrize("N,groups", GROUP_CASES, ids=[f"N{n}-g{g or 'default'}" for n, g in GROUP_CASES])
def test_env_count_and_group_matrix(N, groups, tile_sync, monkeypatch):
    monkeypatch.setenv("FXENV_TILE_SYNC", str(tile_sync))
    if groups:
        monkeypatch.setenv("FXENV_ROLLOUT_GROUPS", str(groups))
    else:
        monkeypatch.delenv("FXENV_ROLLOUT_GROUPS", raising=False)
    H, D = 3, 144
    make = _factory(N, 20)
    env, twin = make(), make()
    starts = torch.as_tensor(start_offsets(N, T_BARS, 200, 300))
    env.reset(starts); twin.reset(starts)
    _warm((env, twin), N, 8, False)
    w = _weights(D, False, seed=N)
    pol = env.make_policy(w)
    noise = _noise(H, N, False, seed=N)
    bufs, backing, tails = _sentinel_buffers(H, N, D, torch.int32)
    out = env.rollout(pol, H, buffers=bufs, gumbel=noise)
    torch.cuda.synchronize()
    assert pol.sync_timeouts() == 0
    for k, raw in backing.items():
        assert torch.equal(raw[-tails[k].numel():], tails[k]), f"N={N}: the rollout wrote past the end of `{k}`"
    tag = f"N{N}/g{groups}/ts{tile_sync}"
    _check_env_side(env, twin, out, H)
    _check_h1_and_controls(pol, w, out["obs"][H], N, True, tag)
    _check_heads(out, w, noise, H, N, False, tag)
    env.close(); twin.close()


def test_group_splits_are_bit_identical(monkeypatch):
    """N = 8392: groups 1/2/3/4 x tile hand-over 0/1 from one state and seed -> identical outputs, h1 and bf16 copies
    (tiles always start at multiples of 128, so the split changes no arithmetic).  The cached rollout graph reads these
    settings at capture time: every setting gets its own policy."""
    N, H, D = 8392, 4, 144
    env = _factory(N, 20)()
    env.reset(torch.as_tensor(start_offsets(N, T_BARS, 200, 300)))
    _warm((env,), N, 8, False)
    w = _weights(D, False, seed=3)
    snap = env.get_state()
    first = None
    for groups in (1, 2, 3, 4):
        for ts in (0, 1):
            monkeypatch.setenv("FXENV_ROLLOUT_GROUPS", str(groups))
            monkeypatch.setenv("FXENV_TILE_SYNC", str(ts))
            env.set_state(snap)
            pol = env.make_policy(w)
            out = env.rollout(pol, H, seed=5)
            got = {k: v.clone() for k, v in out.items()}
            got["h1"] = _bits16(pol.peek("h1"))
            got["obs16_0"], got["obs16_1"] = _bits16(pol.peek("obs16", 0)), _bits16(pol.peek("obs16", 1))
            torch.cuda.synchronize()
            assert pol.sync_timeouts() == 0
            pol.close()
            if first is None:
                first = got
                continue
            for k in first:
                assert torch.equal(first[k], got[k]), f"groups={groups} tile_sync={ts}: {k} differs from groups=1"
    env.close()


# ----------------------------------------------------------------------------------------- d. the bf16 A operand
# emitter variants of the step / observe kernels that write the bf16 copy
EMITTERS = [
    ("lean_fast5", dict(W=20)),
    ("general_fast5", dict(W=20, continuous=True)),
    ("general_fast5_commission", dict(W=20, commission=1e-5)),
    ("odd_w_pairs", dict(W=21)),
    ("general_binary", dict(W=12, data="extra", features=("CLOSE", "FEAT_A", "BIN_FLAG", "VOLUME"), binary=("BIN_FLAG",))),
    ("nonfinite_extra", dict(W=12, data="nonfinite", features=("CLOSE", "FEAT_A", "VOLUME"), clip=2.5)),
    ("nonfinite_noclip", dict(W=12, data="nonfinite", features=("FEAT_A", "CLOSE"), clip=0.0, scaling="none")),
    ("expanding", dict(W=20, scaling="expanding_zscore")),
    ("default_preproc", dict(W=13, preproc="default")),
    ("noprice_noagent", dict(W=9, data="extra", features=("FEAT_A", "HIGH", "BIN_FLAG"), scaling="none", price=False,
                             agent=False, clip=0.0)),
]


@pytest.mark.parametrize("auto_reset", [False, True], ids=["no_reset", "auto_reset"])
@pytest.mark.parametrize("name,kw", EMITTERS, ids=[e[0] for e in EMITTERS])
def test_bf16_observation_copy_is_exact(name, kw, auto_reset):
    """Repeated H = 1 rollouts: the observe kernel fills slot 0, the step kernel slot 1.  Half the envs start at bar 0
    (the PAD phase: episodes younger than the window), 44-bar episodes terminate inside the run."""
    N, steps = 200, 60
    kw = dict(kw)
    continuous = kw.get("continuous", False)
    make = _factory(N, kw.pop("W"), auto_reset=auto_reset, episode_bars=44, **kw)
    env = make()
    D = env.obs_dim
    starts = torch.as_tensor(start_offsets(N, T_BARS, 200, 300))
    starts[::2] = 0
    env.reset(starts)
    pol = env.make_policy(_weights(D, continuous, seed=1))
    buf = None
    n_done = 0
    for i in range(steps):
        buf = env.rollout(pol, 1, buffers=buf, seed=9)
        torch.cuda.synchronize()
        _check_obs16(pol, D, buf["obs"][0], 0, f"{name} rollout {i} slot 0")
        _check_obs16(pol, D, buf["obs"][1], 1, f"{name} rollout {i} slot 1")
        n_done += int(buf["done"].sum())
    assert n_done >= N // 2, "the run must cross episode ends"
    env.close()


# ------------------------------------------------------------------------------------------- e. exact epilogue
def _disc_env(N, W=20):
    env = _factory(N, W)()
    env.reset(torch.as_tensor(start_offsets(N, T_BARS, 200, 300)))
    return env


def test_caller_gumbel_is_exact_with_zero_body():
    N, H = 2000, 4
    env = _disc_env(N)
    b = (0.3125, -0.1, 0.2)
    w = _zero_body(env.obs_dim, b)
    pol = env.make_policy(w)
    gum = _noise(H, N, False, seed=21)
    out = env.rollout(pol, H, gumbel=gum)
    torch.cuda.synchronize()
    bpi = w["b_pi"]
    want = (bpi + gum).argmax(-1).to(torch.int32)   # first maximum of the float32 sums, no margin excuse
    assert torch.equal(out["actions"], want)
    assert torch.equal(out["value"], torch.full_like(out["value"], 0.375))
    lp = torch.log_softmax(bpi.double(), -1)[out["actions"].long()]
    assert float((out["logp"].double() - lp).abs().max()) < 1e-6
    # h1 of a zero body is exactly 0
    assert not bool(_bits16(pol.peek("h1")).any())
    env.close()


@pytest.mark.parametrize("b_pi,want", [((0.25, 0.25, -0.5), 0), ((-0.5, 0.25, 0.25), 1), ((0.25, -0.5, 0.25), 0)])
def test_greedy_ties_take_the_first_maximum(b_pi, want):
    N, H = 300, 2
    env = _disc_env(N)
    pol = env.make_policy(_zero_body(env.obs_dim, b_pi))
    out = env.rollout(pol, H, deterministic=True)
    torch.cuda.synchronize()
    assert bool((out["actions"] == want).all()), torch.bincount(out["actions"].flatten().long(), minlength=3).tolist()
    env.close()


TOP = 64   # the top 64 points of the 2^24-point uniform grid


def _find_top_grid_seeds(N, H, tries=3000, want=6):
    """Seeds whose draws (step < H, env < N, action 1 or 2) hit the top of the uniform grid: greedily, seeds that add
    24-bit values k >= 2^24 - 8 (where |log u| is below the __logf error bound) not covered yet, then the one with the
    most top-64 hits.  Action 0 is left out: a NaN Gumbel value of action 0 still wins (it is the initial best), so
    only actions 1 and 2 can expose one."""
    t, e, a = np.arange(H)[:, None, None], np.arange(N)[None, :, None], np.arange(3)[None, None, :]
    covered, seeds, best, best_n = set(), [], 0, -1
    for seed in range(tries):
        k = R.hash_bits_np(seed, t, e, a)
        m = (k >= (1 << 24) - TOP) & (a > 0)
        ks = set(int(x) for x in k[m & (k >= (1 << 24) - 8)])
        if ks - covered and len(seeds) < want - 1:
            seeds.append(seed)
            covered |= ks
        n = int(m.sum())
        if n > best_n:
            best, best_n = seed, n
    return seeds + ([best] if best not in seeds else [])


def test_in_kernel_gumbel_matches_the_exact_replica():
    N, H = 8192, 4
    env = _disc_env(N)
    b = np.array([0.1, 0.0, -0.1], dtype=np.float32)
    pol = env.make_policy(_zero_body(env.obs_dim, tuple(b.tolist())))
    seeds = _find_top_grid_seeds(N, H)
    t, e, a = np.arange(H)[:, None, None], np.arange(N)[None, :, None], np.arange(3)[None, None, :]
    wrong, n_top, n_differ = [], 0, 0
    for seed in seeds:
        out = env.rollout(pol, H, seed=seed)
        torch.cuda.synchronize()
        act = out["actions"].cpu().numpy()
        k = R.hash_bits_np(seed, t, e, a)
        u = R.uniform_of_bits(k)
        g = R.gumbel_of_uniform(u)
        s = b.astype(np.float64)[None, None, :] + g
        a_ref = np.argmax(s, -1)
        # a draw at the top of the grid decides its env's action (g >= 12.6 against two others): the replica's action,
        # with no margin excuse
        hits = np.argwhere(k >= (1 << 24) - TOP)
        n_top += len(hits)
        wrong += [(seed, int(ti), int(ei), int(ai), int(k[ti, ei, ai]), float(g[ti, ei, ai]), int(act[ti, ei]),
                   int(a_ref[ti, ei])) for ti, ei, ai in hits if act[ti, ei] != a_ref[ti, ei]]
        # everywhere else: equal unless the top-two margin is inside the __logf error of the two draws + fp32 rounding
        order = np.argsort(-s, -1, kind="stable")
        pick = lambda x, j: np.take_along_axis(x, order[..., j:j + 1], -1)[..., 0]
        s1, s2 = pick(s, 0), pick(s, 1)
        err = R.fast_gumbel_err(u)
        slack = pick(err, 0) + pick(err, 1) + np.spacing(np.abs(s1).astype(np.float32)) + np.spacing(np.abs(s2).astype(np.float32))
        differ = act != a_ref
        n_differ += int(differ.sum())
        assert not np.any(differ & ~(s1 - s2 <= slack)), f"seed {seed}: in-kernel Gumbel-max differs from the replica beyond the error bound"
    print(f"\n[gumbel] seeds {seeds}: {n_top} draws at the top {TOP} grid points, all with the replica's action; "
          f"{n_differ} actions inside the __logf error margin differ")
    assert n_top >= 8, "too few draws at the top of the uniform grid"
    assert not wrong, f"(seed, step, env, action, 24-bit k, replica g, kernel action, replica action): {wrong}"
    assert n_differ <= 4 * len(seeds), n_differ
    env.close()


def test_in_kernel_sampling_frequencies_chi_square():
    """H * N = 65536 in-kernel draws against softmax(b_pi): Pearson chi-square, 2 degrees of freedom, fails at p < 1e-4"""
    N, H = 8192, 8
    env = _disc_env(N)
    b = (0.4, -0.3, 0.1)
    pol = env.make_policy(_zero_body(env.obs_dim, b))
    out = env.rollout(pol, H, seed=2024)
    torch.cuda.synchronize()
    counts = torch.bincount(out["actions"].flatten().long(), minlength=3).cpu().numpy()
    p = torch.softmax(torch.tensor(b, dtype=torch.float64), -1).numpy()
    pv = R.chi_square_sf(counts, p)
    assert pv > 1e-4, (counts.tolist(), (p * H * N).tolist(), pv)
    # and a distribution that is off by 0.02 in one probability is rejected by the same test
    q = p + np.array([0.02, -0.02, 0.0])
    assert R.chi_square_sf(counts, q) < 1e-4
    env.close()


def test_continuous_noise_is_exact_with_zero_body():
    N, H = 4096, 4
    env = _factory(N, 20, continuous=True)()
    env.reset(torch.as_tensor(start_offsets(N, T_BARS, 200, 300)))
    pol = env.make_policy(_zero_body(env.obs_dim, (0.0, 0.0), continuous=True))   # mu = 0, log sigma = 0
    c = np.float32(0.5 * math.log(2 * math.pi))
    noise = _noise(H, N, True, seed=31)
    out = env.rollout(pol, H, noise=noise)
    torch.cuda.synchronize()
    assert torch.equal(out["actions"], noise), "a = mu + sigma * eps with mu = 0, sigma = 1 must be eps itself"
    assert torch.equal(out["logp"], ((-0.5 * noise) * noise - 0.0) - c)
    # in-kernel Box-Muller against the replica's uniforms
    seed = 77
    out = env.rollout(pol, H, buffers=out, seed=seed)
    torch.cuda.synchronize()
    act = out["actions"].cpu().numpy().astype(np.float64)
    t, e = np.arange(H)[:, None], np.arange(N)[None, :]
    u0, u1 = R.hash_uniform_np(seed, t, e, 0), R.hash_uniform_np(seed, t, e, 1)
    z = R.box_muller_np(u0, u1)
    r = np.sqrt(-2.0 * np.log(u0.astype(np.float64)))
    tol = 8 * 2.0 ** -24 * np.maximum(r, 2.0 ** -24)   # a few float32 ulps of the radius
    assert np.all(np.abs(act - z) <= tol), float(np.max(np.abs(act - z) / tol))
    eps = out["actions"]
    assert torch.equal(out["logp"], ((-0.5 * eps) * eps - 0.0) - c)
    env.close()


# ----------------------------------------------------------------------------------------- f. short obs ring
def test_two_slot_obs_ring_gives_the_same_rollout():
    N, H = 300, 8
    env = _factory(N, 20)()
    env.reset(torch.as_tensor(start_offsets(N, T_BARS, 200, 300)))
    _warm((env,), N, 5, False)
    pol = env.make_policy(_weights(env.obs_dim, False, seed=8))
    snap = env.get_state()
    full = {k: v.clone() for k, v in env.rollout(pol, H, seed=3).items()}
    env.set_state(snap)
    short = env.rollout(pol, H, seed=3, buffers={"obs": torch.empty((2, N, env.obs_dim), device="cuda")})
    torch.cuda.synchronize()
    for k in ("actions", "logp", "value", "reward", "done"):
        assert torch.equal(full[k], short[k]), k
    assert torch.equal(short["obs"][H % 2], full["obs"][H])
    env.close()


def test_report_h1_tightness():
    """prints the h1 statistics gathered by the tests above (largest error in bf16 ulps, fraction equal to the rounded
    fp64 reference)"""
    if not H1_STATS:
        pytest.skip("no h1 comparison ran in this session")
    worst = max(s[1] for s in H1_STATS)
    worst_big = max(s[2] for s in H1_STATS)
    least = min(s[3] for s in H1_STATS)
    print(f"\n[h1] {len(H1_STATS)} comparisons: max error {worst:.3g} bf16 ulp ({worst_big:.3g} where |h1| >= 1/16), "
          f"min fraction equal to the rounded reference {least:.5f}")
    for tag, mu, mb, fe in H1_STATS:
        print(f"[h1] {tag}: max {mu:.3g} ulp, {mb:.3g} where |h1| >= 1/16, equal {fe:.5f}")
