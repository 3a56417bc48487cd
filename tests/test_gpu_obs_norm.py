"""GPU (-m gpu): the observation normalizer of the fused closed loop (include/fxenv.h fxenv_policy_set_obs_norm,
fxenv_obs_moments; learner.ObsNormalizer, ActorCritic(obs_norm=True)).

  * Bit-exact rows: after rollouts, every bf16 element the observe kernel (slot 0 of a one-step rollout) and the step
    kernels wrote equals bf16_rn(clamp((obs32 - mean) * rstd, -clip, clip)) with the statistics of the env's member and
    pair, pads 0 -- over LEAN / FAST5, the general emitter, padded early windows, action repeat 3, a time limit,
    per-env parameters, 1, 2 and 4 pairs and a population of 2, with random statistics and clip 3 (clipping is hit).
    Negative control: two pairs' statistics swapped.
  * An identity normalizer (mean 0, rstd 1, clip inf) gives rollouts bit-identical to none; the env side is untouched
    (step_many replays the rollout's actions from a snapshot to the same obs, reward and done).
  * Policy outputs against the float64 reference on the normalized rows, discrete and continuous, shared and separate,
    widths 64 and 512; a population member equals a single policy with its weights and normalizer, bit for bit.
  * Graph: a value update between two replays is seen, on -> off -> on works, errors leave the handle usable.
  * fxenv_obs_moments against numpy float64 (odd obs_dim, ragged row counts, one row, member slices), bit-identical
    across calls."""
import json
import math

import numpy as np
import pytest
import torch

import policy_ref as R
import scenarios as S
from gym_fx_b200 import _native
from gym_fx_b200.config import lower_config
from gym_fx_b200.learner import ActorCritic
from gym_fx_b200.synth import start_offsets, synth_candles, synth_minutes
from gym_fx_b200.vec_env import VecFxEnv

pytestmark = pytest.mark.gpu

KEYS = ("obs", "actions", "logp", "value", "reward", "done")
T_BARS = 1500


def _env(N, pairs=1, W=20, features=tuple(S.OHLCV), commission=0.0, continuous=False, episode_bars=37):
    """W % 4 == 0, OHLCV features, no costs: the LEAN kernels; commission or continuous: FAST5 general kernels; other
    features: the general emitter.  Short episodes with auto-reset: padded early windows all along the rollout."""
    cfgd = {**S.DEFAULTS, "window_size": W, "commission": commission, "feature_columns": list(features),
            "sl_pips": 3.0, "tp_pips": 4.0}
    if continuous:
        cfgd["action_space_mode"] = "continuous"
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, "strategy": "direct_fixed_sltp",
                                       "preprocessor": "feature_window_preprocessor"})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"], preprocessor_plugin=pl["preprocessor"],
                       reward_plugin=pl["reward"], columns=S.OHLCV, num_envs=N, num_pairs=pairs, order_capacity=64,
                       episode_bars=episode_bars)
    cfg.auto_reset = 1
    # the pairs on very different price levels, as EURUSD and a JPY pair
    tabs = []
    for p in range(pairs):
        t = synth_candles(T_BARS, p).copy()
        t[:, :4] *= (1.0, 120.0, 0.7, 1.3)[p % 4]
        tabs.append(t)
    env = VecFxEnv(cfg, tabs, [synth_minutes(T_BARS)] * pairs)
    env.reset(torch.as_tensor(start_offsets(N, T_BARS, 200, 300)))
    return env


def _stats(env, M, seed):
    """random per-member, per-pair statistics around the scale of the env's columns: mean [M][P][D], var [M][P][D]"""
    P, D = env.cfg.num_pairs, env.obs_dim
    obs = env.obs.double().cpu()
    g = torch.Generator().manual_seed(seed)
    mean = torch.empty(M, P, D, dtype=torch.float64)
    var = torch.empty(M, P, D, dtype=torch.float64)
    for p in range(P):
        x = obs[p::P]
        mu, sd = x.mean(0), x.std(0, unbiased=False) + 1e-3
        for m in range(M):
            mean[m, p] = mu + sd * torch.randn(D, generator=g, dtype=torch.float64) * 0.5
            var[m, p] = (sd * (0.3 + torch.rand(D, generator=g, dtype=torch.float64))) ** 2
    return mean, var


def _net(env, hidden=64, continuous=False, separate=False, mean=None, var=None, clip=3.0, seed=0):
    torch.manual_seed(seed)
    net = ActorCritic(env.obs_dim, hidden=hidden, continuous=continuous, separate=separate,
                      obs_norm=mean is not None, num_pairs=env.cfg.num_pairs)
    if continuous:
        with torch.no_grad():
            net.log_std.fill_(-0.5)
    if mean is not None:
        net.obs_norm.mean.copy_(mean)
        net.obs_norm.var.copy_(var)
        net.obs_norm.clip = clip
    return net.cuda()


def _normalized(obs, nets, P):
    """float32 [N, D] rows -> the normalized float32 rows (torch eager on the device, the formula of the kernels), each
    env with its member's (nets[m], contiguous slices) normalizer and its pair"""
    N = obs.shape[0]
    n = N // len(nets)
    out = torch.empty_like(obs)
    for m, net in enumerate(nets):
        env_ids = torch.arange(m * n, (m + 1) * n, device=obs.device)
        out[m * n:(m + 1) * n] = net.obs_norm(obs[m * n:(m + 1) * n], env_ids % P)
    return out


def _bits(t):
    return t.contiguous().view(torch.int16)


def _check_obs16(pol, want32, slot, tag):
    o16 = pol.peek("obs16", slot)
    D = want32.shape[1]
    got, want = _bits(o16[:, :D]), _bits(want32.to(torch.bfloat16))
    if not torch.equal(got, want):
        bad = (got != want).nonzero()[:5].tolist()
        raise AssertionError(f"{tag}: normalized bf16 copy of slot {slot} differs at (env, column) {bad}")
    assert not bool(_bits(o16[:, D:]).any()), f"{tag}: pad columns are not 0"


def _check_rows(env, pol, nets, tag, H=4):
    """a 1-step rollout (slot 0: the observe kernel, slot 1: the step kernel), then H steps (both slots: step kernel)"""
    P = env.cfg.num_pairs
    out = env.rollout(pol, 1, seed=3)
    torch.cuda.synchronize()
    _check_obs16(pol, _normalized(out["obs"][0], nets, P), 0, tag + "/observe")
    _check_obs16(pol, _normalized(out["obs"][1], nets, P), 1, tag + "/step")
    out = env.rollout(pol, H, seed=4)
    torch.cuda.synchronize()
    _check_obs16(pol, _normalized(out["obs"][H], nets, P), H & 1, tag + "/step H")
    _check_obs16(pol, _normalized(out["obs"][H - 1], nets, P), (H - 1) & 1, tag + "/step H-1")
    return out


# (name, env arguments, setter) -- every emit path of the bf16 copy
CASES = [
    ("lean_1pair", dict(), None),
    ("lean_2pairs", dict(pairs=2), None),
    ("fast5_general_4pairs", dict(pairs=4, commission=1e-5), None),
    ("general_emitter_f3", dict(features=("OPEN", "HIGH", "CLOSE"), W=21, pairs=2), None),
    ("continuous_fast5", dict(continuous=True, pairs=2), None),
    ("repeat3", dict(pairs=2), lambda e: e.set_action_repeat(3)),
    ("time_limit", dict(pairs=2), lambda e: e.set_time_limit(5)),
    ("env_params", dict(pairs=2), lambda e: e.set_env_params(sl_pips=np.linspace(2.0, 6.0, e.num_envs))),
]


@pytest.mark.parametrize("name,kw,setter", CASES, ids=[c[0] for c in CASES])
def test_normalized_rows_are_exact(name, kw, setter):
    N = 512
    env = _env(N, **kw)
    if setter:
        setter(env)
    cont = kw.get("continuous", False)
    mean, var = _stats(env, 1, seed=len(name))
    net = _net(env, continuous=cont, mean=mean[0], var=var[0])
    pol = env.make_policy(net)
    out = _check_rows(env, pol, [net], name)
    clipped = (_normalized(out["obs"][-1], [net], env.cfg.num_pairs).abs() == 3.0).float().mean().item()
    assert clipped > 0.001, f"{name}: clip 3 is never reached ({clipped})"
    if name.startswith("lean"):
        assert env.L.fxenv_debug_lean(env._h) == 1, f"{name}: not the LEAN kernels"
    env.close()


def test_population_rows_and_member_equivalence():
    N, M, H = 512, 2, 3
    env = _env(N, pairs=2)
    mean, var = _stats(env, M, seed=11)
    nets = [_net(env, hidden=128, mean=mean[m], var=var[m], seed=m) for m in range(M)]
    pop = env.make_policy(nets)
    _check_rows(env, pop, nets, "population")
    snap = env.get_state()
    g = torch.Generator(device="cuda").manual_seed(5)
    gumbel = -torch.log(-torch.log(torch.rand((H, N, 3), device="cuda", generator=g).clamp(1e-9, 1 - 1e-9)))
    env.set_state(snap)
    out = {k: v.clone() for k, v in env.rollout(pop, H, gumbel=gumbel).items()}
    single = env.make_policy(nets[0])
    for m in range(M):
        single.set_weights(nets[m])
        env.set_state(snap)
        ref = env.rollout(single, H, gumbel=gumbel)
        torch.cuda.synchronize()
        sl = pop.member_envs(m)
        for k in KEYS:
            assert torch.equal(out[k][:, sl], ref[k][:, sl]), f"member {m}: {k} differs from the single policy"
    env.close()


def test_negative_control_swapped_pairs():
    env = _env(256, pairs=2)
    mean, var = _stats(env, 1, seed=2)
    net = _net(env, mean=mean[0], var=var[0])
    pol = env.make_policy(net)
    snap = env.get_state()
    out = env.rollout(pol, 2, seed=1)
    torch.cuda.synchronize()
    good = pol.peek("obs16", 0).clone()
    _check_obs16(pol, _normalized(out["obs"][2], [net], 2), 0, "control")
    sw = _net(env, mean=mean[0][[1, 0]], var=var[0][[1, 0]])
    pol.set_weights(sw)
    env.set_state(snap)
    env.rollout(pol, 2, seed=1)
    torch.cuda.synchronize()
    assert not torch.equal(_bits(pol.peek("obs16", 0)), _bits(good)), "swapped pair statistics give the same rows"
    with pytest.raises(AssertionError):
        _check_obs16(pol, _normalized(out["obs"][2], [net], 2), 0, "swapped")
    env.close()


@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_identity_normalizer_is_bit_identical_and_env_untouched(continuous):
    N, H = 512, 6
    env = _env(N, pairs=2, continuous=continuous)
    net = _net(env, continuous=continuous, seed=3)
    plain = env.make_policy(net)
    P, D = 2, env.obs_dim
    ident = {**R.weights_of(net, continuous), "obs_mean": torch.zeros(P, D), "obs_rstd": torch.ones(P, D),
             "obs_clip": math.inf}
    normed = env.make_policy({k: (v.cuda() if torch.is_tensor(v) else v) for k, v in ident.items()})
    snap = env.get_state()
    outs = []
    for pol in (plain, normed):
        env.set_state(snap)
        outs.append({k: v.clone() for k, v in env.rollout(pol, H, seed=8).items()})
        torch.cuda.synchronize()
    for k in KEYS:
        assert torch.equal(outs[0][k], outs[1][k]), f"identity normalizer changes {k}"
    # the env side of a normalized rollout: step_many from the snapshot replays it exactly
    mean, var = _stats(env, 1, seed=4)
    pol = env.make_policy(_net(env, continuous=continuous, mean=mean[0], var=var[0]))
    env.set_state(snap)
    out = {k: v.clone() for k, v in env.rollout(pol, H, seed=9).items()}
    env.set_state(snap)
    ring = torch.empty((H, N, D), dtype=torch.float32, device="cuda")
    rew = torch.empty((H, N), dtype=torch.float32, device="cuda")
    term = torch.empty((H, N), dtype=torch.uint8, device="cuda")
    env.step_many(out["actions"], ring, rew, term)
    torch.cuda.synchronize()
    assert torch.equal(ring, out["obs"][1:]) and torch.equal(rew, out["reward"]) and torch.equal(term, out["done"])
    env.close()


@pytest.mark.parametrize("separate", [False, True], ids=["shared", "separate"])
@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
@pytest.mark.parametrize("hidden", [64, 512])
def test_policy_outputs_match_the_reference_on_normalized_rows(hidden, continuous, separate):
    N, H = 256, 3
    env = _env(N, pairs=2, continuous=continuous)
    mean, var = _stats(env, 1, seed=hidden)
    net = _net(env, hidden=hidden, continuous=continuous, separate=separate, mean=mean[0], var=var[0], seed=hidden)
    R.scaled_init(net)
    pol = env.make_policy(net)
    g = torch.Generator(device="cuda").manual_seed(6)
    noise = torch.randn((H, N), device="cuda", generator=g) if continuous else \
        -torch.log(-torch.log(torch.rand((H, N, 3), device="cuda", generator=g).clamp(1e-9, 1 - 1e-9)))
    out = env.rollout(pol, H, **({"noise": noise} if continuous else {"gumbel": noise}))
    torch.cuda.synchronize()
    actor = R.weights_of(net, continuous)
    critic = actor if not separate else {**actor, "w1": net.critic_body[0].weight, "b1": net.critic_body[0].bias,
                                         "w2": net.critic_body[2].weight, "b2": net.critic_body[2].bias}
    for t in range(H + 1):
        x = _normalized(out["obs"][t], [net], 2)
        ref_v = R.forward_ref(critic, x)["value"]
        assert R.head_close(out["value"][t], ref_v), (t, R.head_err(out["value"][t], ref_v))
        raw_v = R.forward_ref(critic, out["obs"][t])["value"]
        assert not R.head_close(out["value"][t], raw_v), f"step {t}: the value also matches the raw observation"
        if t == H:
            break
        head = R.forward_ref(actor, x)["head"]
        if continuous:
            want = head[:, 0] + math.exp(float(net.log_std.detach())) * noise[t].double()
            assert R.head_close(out["actions"][t], want), (t, R.head_err(out["actions"][t], want))
        else:
            lp = torch.log_softmax(head, -1).gather(1, out["actions"][t].long()[:, None]).squeeze(1)
            assert R.head_close(out["logp"][t], lp, 3e-3), (t, R.head_err(out["logp"][t], lp))
    env.close()


def test_graph_sees_value_updates_and_on_off_on():
    N = 256
    env = _env(N, pairs=2)
    mean, var = _stats(env, 2, seed=7)
    a = _net(env, mean=mean[0], var=var[0], seed=1)
    b = _net(env, mean=mean[1], var=var[1], seed=1)
    plain = _net(env, seed=1)
    pol = env.make_policy(a)
    bufs = {}
    for tag, net in (("a", a), ("b: value update", b), ("off", plain), ("on again", a)):
        pol.set_weights(net)
        out = env.rollout(pol, 2, buffers=bufs, seed=2)
        torch.cuda.synchronize()
        want = out["obs"][2] if net is plain else _normalized(out["obs"][2], [net], 2)
        _check_obs16(pol, want, 0, tag)
    # errors leave the handle and the policy usable
    L, s = env.L, env._stream()
    m32, r32 = a.obs_norm.mean32().contiguous(), a.obs_norm.rstd32().contiguous()
    assert L.fxenv_policy_set_obs_norm(pol._p, 0, m32.data_ptr(), r32.data_ptr(), 0.0, s) == -1
    assert L.fxenv_policy_set_obs_norm(pol._p, 0, m32.data_ptr(), r32.data_ptr(), float("nan"), s) == -1
    assert L.fxenv_policy_set_obs_norm(pol._p, 1, m32.data_ptr(), r32.data_ptr(), 3.0, s) == -1
    assert L.fxenv_policy_set_obs_norm(pol._p, 0, m32.data_ptr(), None, 3.0, s) == -1
    assert b"NULL" in L.fxenv_last_error(env._h)
    with pytest.raises(ValueError):
        env.obs_moments(bufs["obs"], m32, slice(5, 5))
    out = env.rollout(pol, 2, buffers=bufs, seed=2)
    torch.cuda.synchronize()
    _check_obs16(pol, _normalized(out["obs"][2], [a], 2), 0, "after errors")
    # a population with one member on and one off cannot roll out; turning the other on fixes it
    pop = env.make_policy([plain, plain])
    assert L.fxenv_policy_set_obs_norm(pop._p, 0, m32.data_ptr(), r32.data_ptr(), 3.0, s) == 0
    with pytest.raises(_native.FxEnvError, match="normalizer"):
        env.rollout(pop, 2, seed=2)
    with pytest.raises(ValueError, match="normalizer"):
        pop.set_weights([a, plain])
    with pytest.raises(ValueError, match="shape"):   # a normalizer of 1 pair for an env of 2
        pop.set_weights([ActorCritic(env.obs_dim, hidden=64, obs_norm=True, num_pairs=1).cuda()] * 2)
    pop.set_weights([a, a])
    env.rollout(pop, 2, seed=2)
    torch.cuda.synchronize()
    env.close()


def _moments_ref(x, P, e0, e1, shift):
    """numpy float64 [P, 2, D] of rows x [slots, N, D] of envs [e0, e1)"""
    x = x.astype(np.float64)
    out = np.zeros((P, 2, x.shape[2]))
    for p in range(P):
        envs = [e for e in range(e0, e1) if e % P == p]
        if envs:
            d = x[:, envs].reshape(-1, x.shape[2]) - shift[p].astype(np.float64)
            out[p, 0], out[p, 1] = d.sum(0), (d * d).sum(0)
    return out


def test_obs_moments_against_numpy():
    N, P = 300, 3
    env = _env(N, pairs=P, W=21)   # obs_dim 5 W + 2 W + 4 = 151: odd
    D = env.obs_dim
    assert D % 2 == 1
    g = torch.Generator(device="cuda").manual_seed(8)
    x = (torch.randn((5, N, D), device="cuda", generator=g) * 0.3 + torch.linspace(-4, 150, D, device="cuda")).float()
    shift = (torch.linspace(-4, 150, D, device="cuda") + 0.7).repeat(P, 1).contiguous()
    xs, sh = x.cpu().numpy(), shift.cpu().numpy()
    for slots, (e0, e1) in [(5, (0, N)), (3, (37, 211)), (1, (5, 6)), (5, (128, 256)), (2, (299, 300))]:
        xv = x[:slots].contiguous()
        got = env.obs_moments(xv, shift, slice(e0, e1))
        again = env.obs_moments(xv, shift, slice(e0, e1))
        torch.cuda.synchronize()
        assert torch.equal(got, again), "two calls differ"
        ref = _moments_ref(xs[:slots], P, e0, e1, sh)
        absd = _moments_ref(np.abs(xs[:slots] - 0), P, e0, e1, np.zeros_like(sh))  # scale of the terms
        np.testing.assert_allclose(got.cpu().numpy(), ref, rtol=1e-12, atol=1e-13 * absd.max(),
                                   err_msg=f"slots {slots}, envs [{e0}, {e1})")
    for bad in (slice(0, N, 2), slice(7, 7)):   # not contiguous, empty
        with pytest.raises(ValueError):
            env.obs_moments(x, shift, bad)
    env.close()


def test_obs_normalizer_update_on_the_device_equals_numpy():
    N, P, H = 256, 2, 4
    env = _env(N, pairs=P)
    net = _net(env, mean=torch.zeros(P, env.obs_dim, dtype=torch.float64), var=torch.ones(P, env.obs_dim, dtype=torch.float64))
    pol = env.make_policy(net)
    seen = [[] for _ in range(P)]
    for k in range(3):
        out = env.rollout(pol, H, seed=k)
        net.obs_norm.update(env, out["obs"][:H], envs=slice(64, 192))
        pol.set_weights(net)
        o = out["obs"][:H, 64:192].double().cpu().numpy()
        for p in range(P):
            seen[p].append(o[:, [i for i in range(128) if (64 + i) % P == p]].reshape(-1, env.obs_dim))
    for p in range(P):
        xx = np.concatenate(seen[p])
        assert net.obs_norm.count[p].item() == len(xx)
        np.testing.assert_allclose(net.obs_norm.mean[p].cpu().numpy(), xx.mean(0), rtol=1e-9, atol=1e-12)
        np.testing.assert_allclose(net.obs_norm.var[p].cpu().numpy(), xx.var(0), rtol=1e-7, atol=1e-15)
    env.close()


@pytest.mark.parametrize("population", [1, 2])
def test_ppo_example_with_obs_norm(population, tmp_path):
    import subprocess
    import sys
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, os.path.join(root, "examples", "ppo_rollout.py"), "--obs-norm", "--envs", "256", "--horizon", "8",
           "--updates", "3", "--population", str(population)]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["obs_norm"] and "obs-norm" in line["workload"] and line["obs_norm_update_s"] > 0, line
    assert line["obs_norm_finite"], line
    for k in ("mean_reward",) if population == 1 else ():
        assert math.isfinite(line[k]), line
