"""GPU (-m gpu): the fused policy kernel at hidden widths 64, 128 and 512, and at 256 through fxenv_policy_create_ex.

The patterns of test_gpu_policy_edges.py, per width:
  1. observation widths of 1, 3, 5 and 29 layer-1 k-blocks, discrete and continuous: the env side against a twin handle
     stepped with the sampled actions, h1 within check_h1 (with the same tightness floors), padded rows = the zero-row
     evaluation, value / logits / mean / log-prob against forward_ref, every comparison with its negative controls;
  2. env counts with ragged tiles, env groups 1-4 x tile hand-over off / on, rollout buffers at the front of
     sentinel-filled allocations; every group / hand-over setting bit-identical;
  3. the sampling epilogue with a zero body (logits = b_pi exactly): caller noise, greedy ties, value = b_v, the in-kernel
     Gumbel and Box-Muller draws against the replica of the counter-based generator (the head loops differ per width);
  4. the default is unchanged: create_ex(256) and fxenv_policy_create give bit-identical rollouts and h1;
  5. width 64 with action repeat, auto-reset, short episodes and start ranges;
  6. the learner: ActorCritic(hidden=h) -> make_policy infers h, and after a PPO update set_weights tracks the new net;
  7. argument errors."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn as nn

import policy_ref as R
import policy_width_ref as RW
from gym_fx_b200.synth import start_offsets
from test_gpu_policy_edges import (T_BARS, _bits16, _check_env_side, _factory, _noise, _rollout, _sentinel_buffers,
                                   _warm)

pytestmark = pytest.mark.gpu

WIDTHS = [64, 128, 512]


class _Net(nn.Module):
    def __init__(self, D, hidden, n_pi):
        super().__init__()
        self.body = nn.Sequential(nn.Linear(D, hidden), nn.Tanh(), nn.Linear(hidden, hidden), nn.Tanh())
        self.pi = nn.Linear(hidden, n_pi)
        self.v = nn.Linear(hidden, 1)


def _weights(D, hidden, continuous, seed, log_std=-0.5):
    torch.manual_seed(seed)
    w = R.weights_of(R.scaled_init(_Net(D, hidden, 1 if continuous else 3)))
    if continuous:
        w["log_std"] = torch.tensor([log_std])
    return {k: v.cuda() for k, v in w.items()}


def _zero_body(D, hidden, b_pi, b_v=0.375, continuous=False):
    """W1 = W2 = b1 = b2 = 0: tanh.approx(0) = 0, so h2 = 0 and the logits / mean are b_pi exactly."""
    n = 1 if continuous else 3
    g = torch.Generator().manual_seed(17)
    w = {"w1": torch.zeros(hidden, D), "b1": torch.zeros(hidden), "w2": torch.zeros(hidden, hidden),
         "b2": torch.zeros(hidden), "w_pi": torch.randn((n, hidden), generator=g),
         "b_pi": torch.tensor(b_pi[:n], dtype=torch.float32), "w_v": torch.randn(hidden, generator=g),
         "b_v": torch.tensor([b_v])}
    if continuous:
        w["log_std"] = torch.tensor([b_pi[1]], dtype=torch.float32)
    return {k: v.cuda() for k, v in w.items()}


def _check_h1_and_controls(pol, w, obs, N, agent, tag):
    hidden = pol.hidden
    h1 = pol.peek("h1")
    NP = (N + 127) // 128 * 128
    assert h1.shape == (NP, hidden), tag
    ref = R.forward_ref(w, obs)
    rep = R.check_h1(h1[:N], ref, obs, w)
    assert rep["bad"] == 0, (tag, rep)
    # the tightness floors of test_gpu_policy_edges.py
    assert rep["max_ulps_big"] <= 1.0 and rep["frac_equal"] >= 0.998, (tag, rep)
    ctl = RW.control_refs(w, obs, agent=agent)
    for name in R.H1_CONTROLS:
        if name in ctl and not (name == "rows_shifted" and N == 1):
            assert R.check_h1(h1[:N], ctl[name], obs, w)["bad"] > 0, f"{tag}: h1 check does not reject control {name}"
    if NP > N:   # rows past the env count: TMA fills the missing observation rows with 0 -> bf16(tanh.approx(b1))
        pad = h1[N:]
        assert torch.equal(_bits16(pad), _bits16(pad[:1].expand_as(pad))), f"{tag}: padded h1 rows differ"
        z = torch.zeros((1, obs.shape[1]), device=obs.device)
        assert R.check_h1(pad[:1], R.forward_ref(w, z), z, w)["bad"] == 0, f"{tag}: padded h1 rows"


def _check_heads(out, w, noise, H, N, continuous, tag):
    """value / logits or mean / log-prob of every step against forward_ref, with the negative controls at step 0 (as in
    test_gpu_policy_edges.py, with the controls built for the policy's width)"""
    obs, act, logp, val = out["obs"], out["actions"], out["logp"], out["value"]
    controls = [c for c in R.HEAD_CONTROLS if not (c == "rows_shifted" and N == 1)]   # one row: a shift is no change
    n_flip = 0
    for t in range(H + 1):
        ref = R.forward_ref(w, obs[t])
        assert R.head_close(val[t], ref["value"]), (tag, t, R.head_err(val[t], ref["value"]))
        if t == 0:
            ctl = RW.control_refs(w, obs[t], agent=False)
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


# ------------------------------------------------------------------------------------------------- 1. shapes
# (name, env settings, obs_dim, layer-1 k-blocks, agent scalars at the end of the row)
SHAPES = [
    ("default_w13", dict(W=13, preproc="default"), 30, 1, True),
    ("ohlcv_w20", dict(W=20), 144, 3, True),
    ("ohlcv_w41", dict(W=41), 291, 5, True),
    ("ohlcv_w256", dict(W=256), 1796, 29, True),
]


@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
@pytest.mark.parametrize("name,kw,D,kb,agent", SHAPES, ids=[s[0] for s in SHAPES])
@pytest.mark.parametrize("hidden", WIDTHS + [256])
def test_width_shape_matrix(hidden, name, kw, D, kb, agent, continuous):
    N, H = 300, 3
    kw = dict(kw)
    make = _factory(N, kw.pop("W"), continuous=continuous, **kw)
    env, twin = make(), make()
    assert env.obs_dim == D and (D + 63) // 64 == kb, "the config lowering moved this shape"
    starts = torch.as_tensor(start_offsets(N, T_BARS, 200, 300))
    env.reset(starts); twin.reset(starts)
    _warm((env, twin), N, 12, continuous)
    w = _weights(D, hidden, continuous, seed=hidden + kb)
    pol = env.make_policy(w, hidden=hidden)
    assert pol.hidden == hidden
    noise = _noise(H, N, continuous, seed=kb)
    out = _rollout(env, pol, H, noise, continuous)
    torch.cuda.synchronize()
    _check_env_side(env, twin, out, H)
    tag = f"h{hidden}/{name}/{'cont' if continuous else 'disc'}"
    _check_h1_and_controls(pol, w, out["obs"][H], N, agent, tag)   # h1 of the bootstrap evaluation
    _check_heads(out, w, noise, H, N, continuous, tag)
    env.close(); twin.close()


# -------------------------------------------------------------------------------------- 2. env counts and groups
@pytest.mark.parametrize("N", [1, 127, 129, 300, 4096 + 64])
@pytest.mark.parametrize("hidden", WIDTHS)
def test_env_counts_and_group_splits(hidden, N, monkeypatch):
    """groups 1-4 x tile hand-over 0/1 from one state and one noise tensor: identical outputs and h1, nothing written
    outside [0, N) of any buffer; the first setting is checked against the twin and the reference."""
    H, D = 3, 144
    make = _factory(N, 20)
    env, twin = make(), make()
    starts = torch.as_tensor(start_offsets(N, T_BARS, 200, 300))
    env.reset(starts); twin.reset(starts)
    _warm((env, twin), N, 8, False)
    w = _weights(D, hidden, False, seed=N + hidden)
    noise = _noise(H, N, False, seed=N)
    snap = env.get_state()
    first = None
    for groups in (1, 2, 3, 4):
        for ts in (0, 1):
            monkeypatch.setenv("FXENV_ROLLOUT_GROUPS", str(groups))
            monkeypatch.setenv("FXENV_TILE_SYNC", str(ts))
            env.set_state(snap)
            pol = env.make_policy(w)   # the rollout graph reads these settings at capture: one policy per setting
            bufs, backing, tails = _sentinel_buffers(H, N, D, torch.int32)
            out = env.rollout(pol, H, buffers=bufs, gumbel=noise)
            torch.cuda.synchronize()
            assert pol.sync_timeouts() == 0
            tag = f"h{hidden}/N{N}/g{groups}/ts{ts}"
            for k, raw in backing.items():
                assert torch.equal(raw[-tails[k].numel():], tails[k]), f"{tag}: the rollout wrote past the end of `{k}`"
            got = {k: v.clone() for k, v in out.items()}
            got["h1"] = _bits16(pol.peek("h1"))
            if first is None:
                first = got
                _check_env_side(env, twin, out, H)
                _check_h1_and_controls(pol, w, out["obs"][H], N, True, tag)
                _check_heads(out, w, noise, H, N, False, tag)
            else:
                for k in first:
                    assert torch.equal(first[k], got[k]), f"{tag}: {k} differs from groups=1, tile hand-over off"
            pol.close()
    env.close(); twin.close()


# ------------------------------------------------------------------------------------------- 3. exact epilogue
def _disc_env(N, W=20, continuous=False):
    env = _factory(N, W, continuous=continuous)()
    env.reset(torch.as_tensor(start_offsets(N, T_BARS, 200, 300)))
    return env


@pytest.mark.parametrize("hidden", WIDTHS)
def test_caller_gumbel_and_greedy_ties_with_zero_body(hidden):
    N, H = 2000, 4
    env = _disc_env(N)
    b = (0.3125, -0.1, 0.2)
    w = _zero_body(env.obs_dim, hidden, b)
    pol = env.make_policy(w)
    gum = _noise(H, N, False, seed=21 + hidden)
    out = env.rollout(pol, H, gumbel=gum)
    torch.cuda.synchronize()
    bpi = w["b_pi"]
    assert torch.equal(out["actions"], (bpi + gum).argmax(-1).to(torch.int32))   # first maximum of the float32 sums
    assert torch.equal(out["value"], torch.full_like(out["value"], 0.375))
    lp = torch.log_softmax(bpi.double(), -1)[out["actions"].long()]
    assert float((out["logp"].double() - lp).abs().max()) < 1e-6
    assert not bool(_bits16(pol.peek("h1")).any())
    for b_pi, want in (((0.25, 0.25, -0.5), 0), ((-0.5, 0.25, 0.25), 1), ((0.25, -0.5, 0.25), 0)):
        pol.set_weights(_zero_body(env.obs_dim, hidden, b_pi))
        g = env.rollout(pol, 2, deterministic=True)
        torch.cuda.synchronize()
        assert bool((g["actions"] == want).all()), (b_pi, torch.bincount(g["actions"].flatten().long(), minlength=3).tolist())
    env.close()


@pytest.mark.parametrize("hidden", WIDTHS)
def test_in_kernel_gumbel_matches_the_replica(hidden):
    N, H, seed = 4096, 4, 1234 + hidden
    env = _disc_env(N)
    b = np.array([0.1, 0.0, -0.1], dtype=np.float32)
    pol = env.make_policy(_zero_body(env.obs_dim, hidden, tuple(b.tolist())))
    out = env.rollout(pol, H, seed=seed)
    torch.cuda.synchronize()
    act = out["actions"].cpu().numpy()
    t, e, a = np.arange(H)[:, None, None], np.arange(N)[None, :, None], np.arange(3)[None, None, :]
    u = R.uniform_of_bits(R.hash_bits_np(seed, t, e, a))
    s = b.astype(np.float64)[None, None, :] + R.gumbel_of_uniform(u)
    a_ref = np.argmax(s, -1)
    # equal unless the top-two margin is inside the __logf error of the two draws + fp32 rounding
    order = np.argsort(-s, -1, kind="stable")
    pick = lambda x, j: np.take_along_axis(x, order[..., j:j + 1], -1)[..., 0]
    s1, s2 = pick(s, 0), pick(s, 1)
    err = R.fast_gumbel_err(u)
    slack = pick(err, 0) + pick(err, 1) + np.spacing(np.abs(s1).astype(np.float32)) + np.spacing(np.abs(s2).astype(np.float32))
    differ = act != a_ref
    assert not np.any(differ & ~(s1 - s2 <= slack)), "in-kernel Gumbel-max differs from the replica beyond the error bound"
    assert int(differ.sum()) <= 4
    assert torch.equal(out["value"], torch.full_like(out["value"], 0.375))
    env.close()


@pytest.mark.parametrize("hidden", WIDTHS)
def test_continuous_noise_is_exact_with_zero_body(hidden):
    N, H = 4096, 4
    env = _disc_env(N, continuous=True)
    pol = env.make_policy(_zero_body(env.obs_dim, hidden, (0.0, 0.0), continuous=True))   # mu = 0, log sigma = 0
    c = np.float32(0.5 * math.log(2 * math.pi))
    noise = _noise(H, N, True, seed=31 + hidden)
    out = env.rollout(pol, H, noise=noise)
    torch.cuda.synchronize()
    assert torch.equal(out["actions"], noise), "a = mu + sigma * eps with mu = 0, sigma = 1 must be eps itself"
    assert torch.equal(out["logp"], ((-0.5 * noise) * noise - 0.0) - c)
    assert torch.equal(out["value"], torch.full_like(out["value"], 0.375))
    seed = 77 + hidden   # in-kernel Box-Muller against the replica's uniforms
    out = env.rollout(pol, H, buffers=out, seed=seed)
    torch.cuda.synchronize()
    act = out["actions"].cpu().numpy().astype(np.float64)
    t, e = np.arange(H)[:, None], np.arange(N)[None, :]
    u0, u1 = R.hash_uniform_np(seed, t, e, 0), R.hash_uniform_np(seed, t, e, 1)
    z = R.box_muller_np(u0, u1)
    r = np.sqrt(-2.0 * np.log(u0.astype(np.float64)))
    tol = 8 * 2.0 ** -24 * np.maximum(r, 2.0 ** -24)
    assert np.all(np.abs(act - z) <= tol), float(np.max(np.abs(act - z) / tol))
    env.close()


# ------------------------------------------------------------------------------------ 4. the default is unchanged
@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_create_ex_256_equals_the_default_create(continuous):
    N, H = 300, 6
    env = _disc_env(N, continuous=continuous)
    _warm((env,), N, 5, continuous)
    w = _weights(env.obs_dim, 256, continuous, seed=5)
    ex = env.make_policy(w, hidden=256)
    legacy = env.make_policy()   # then re-created through the original entry point
    env.L.fxenv_policy_destroy(legacy._p)
    legacy._p = C.c_void_p()
    assert env.L.fxenv_policy_create(env._h, C.byref(legacy._p)) == 0
    legacy.set_weights(w)
    snap = env.get_state()
    results = []
    for pol in (ex, legacy):
        env.set_state(snap)
        out = {k: v.clone() for k, v in env.rollout(pol, H, seed=11).items()}
        out["h1"] = _bits16(pol.peek("h1"))
        torch.cuda.synchronize()
        results.append(out)
    for k in ("actions", "logp", "value", "obs", "reward", "done", "h1"):
        assert torch.equal(results[0][k], results[1][k]), k
    env.close()


# ----------------------------------------------------------------------------------------------- 5. composition
def test_width_64_with_action_repeat_and_auto_reset():
    N, H, k = 256, 24, 4
    make = _factory(N, 20, auto_reset=True, episode_bars=37)
    env, twin = make(), make()
    lo = np.asarray([(29 * i) % (T_BARS // 2) for i in range(N)], np.int64)
    hi = lo + np.asarray([[0, 1, 90, 300][i % 4] for i in range(N)], np.int64)
    for e in (env, twin):
        e.set_episode_starts(lo, hi, seed=8)
        e.set_action_repeat(k)
        e.reset()
    w = _weights(env.obs_dim, 64, False, seed=64)
    pol = env.make_policy(w)
    assert pol.hidden == 64
    noise = _noise(H, N, False, seed=4)
    out = env.rollout(pol, H, gumbel=noise)
    torch.cuda.synchronize()
    assert pol.sync_timeouts() == 0
    _check_env_side(env, twin, out, H)
    assert int(out["done"].sum()) > 0, "no episode ended"
    assert env.get_state() == twin.get_state()
    blob = env.get_state()
    g1 = {k_: v.clone() for k_, v in env.rollout(pol, 8, deterministic=True).items()}
    env.set_state(blob)
    g2 = env.rollout(pol, 8, deterministic=True)
    torch.cuda.synchronize()
    for k_ in ("obs", "actions", "reward", "done", "value", "logp"):
        assert torch.equal(g1[k_], g2[k_]), k_
    env.close(); twin.close()


# ---------------------------------------------------------------------------------------------------- 6. learner
@pytest.mark.parametrize("hidden", [64, 512])
def test_learner_update_at_width(hidden):
    from gym_fx_b200.learner import ActorCritic, ppo_update
    N, H = 512, 8
    env = _disc_env(N)
    torch.manual_seed(hidden)
    net = ActorCritic(env.obs_dim, hidden=hidden).cuda()
    pol = env.make_policy(net)
    assert pol.hidden == hidden
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    buf = env.rollout(pol, H, seed=1)
    before = {k: v.clone() for k, v in R.weights_of(net).items()}
    stats = ppo_update(net, opt, buf, torch.zeros(N, dtype=torch.uint8, device="cuda"), None, epochs=1, minibatches=2)
    assert all(math.isfinite(v) for v in stats.values() if isinstance(v, float)), stats
    assert not torch.equal(before["w1"], R.weights_of(net)["w1"]), "the update changed nothing"
    pol.set_weights(net)
    out = env.rollout(pol, H, buffers=buf, seed=2)
    torch.cuda.synchronize()
    for t in range(H + 1):
        ref = R.forward_ref(net, out["obs"][t])
        assert R.head_close(out["value"][t], ref["value"]), (hidden, t, R.head_err(out["value"][t], ref["value"]))
    env.close()


# ----------------------------------------------------------------------------------------------------- 7. errors
def test_width_errors():
    N = 130
    env = _disc_env(N)
    D = env.obs_dim
    with pytest.raises(ValueError):
        env.make_policy(hidden=96)
    w128 = _weights(D, 128, False, seed=1)
    pol = env.make_policy(hidden=64)
    with pytest.raises(ValueError, match="64-wide"):
        pol.set_weights(w128)
    with pytest.raises(ValueError):
        env.make_policy(w128, hidden=64)
    assert env.make_policy(w128).hidden == 128
    assert env.make_policy().hidden == 256
    for bad in (0, 96, 1024):
        p = C.c_void_p()
        assert env.L.fxenv_policy_create_ex(env._h, bad, C.byref(p)) == -1   # FXENV_E_INVALID
        assert not p.value
        assert b"64, 128, 256 or 512" in env.L.fxenv_last_error(env._h)
    env.close()
