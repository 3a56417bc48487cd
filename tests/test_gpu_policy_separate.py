"""GPU (-m gpu): separate actor and critic networks in the fused closed loop (FXENV_POLICY_SEPARATE,
fx_policy_kernel<HID, CONT, true>: one CTA pair per network and tile).

The reference is the shared-body kernel, so most checks are bit for bit.  From one env snapshot:
  actor side   a shared rollout with the actor's trunk and heads and the same noise (caller, in-kernel, greedy) gives
               the separate rollout's actions, log-probs, observations, rewards and dones;
  critic side  a shared rollout with the critic's trunk and value head, its noise forcing the separate run's actions,
               gives its values;
  h1           the two column halves of the separate h1 are the two shared runs' h1;
then the fp64 host reference of each trunk (policy_ref.py) within the width tests' tolerances, negative controls each
check must reject, env counts / groups / tile hand-over / observation rings, set_weights under a cached graph, errors,
and a PPO update of ActorCritic(separate=True)."""
import ctypes as C
import math

import pytest
import torch

import policy_ref as R
from gym_fx_b200.synth import start_offsets
from test_gpu_policy_edges import T_BARS, _bits16, _check_env_side, _factory, _noise, _sentinel_buffers, _warm
from test_gpu_policy_widths import _weights

pytestmark = pytest.mark.gpu

WIDTHS = [64, 128, 256, 512]
TRUNK = ("w1", "b1", "w2", "b2")
KEYS = ("obs", "actions", "logp", "value", "reward", "done")


def _separate(actor, critic):
    """weight dict of a separate policy: the actor's trunk and heads, the critic's trunk (w1_v ...) and value head"""
    w = {k: v for k, v in actor.items() if k not in ("w_v", "b_v")}
    w.update({k + "_v": critic[k] for k in TRUNK})
    w["w_v"], w["b_v"] = critic["w_v"], critic["b_v"]
    return w


def _critic_shared(critic, actor, continuous):
    """shared-body weights whose trunk and value head are the critic's; continuous: the mean is exactly 0 and sigma 1,
    so that action = fmaf(1, eps, 0) = eps"""
    w = dict(critic)
    if continuous:
        w["w_pi"], w["b_pi"], w["log_std"] = torch.zeros_like(actor["w_pi"]), torch.zeros_like(actor["b_pi"]), torch.zeros_like(actor["log_std"])
    else:
        w["w_pi"], w["b_pi"] = actor["w_pi"], actor["b_pi"]
    return w


def _forcing_noise(actions, continuous):
    """noise that makes the critic-side shared run take the recorded actions"""
    if continuous:
        return actions.clone()
    g = torch.zeros(actions.shape + (3,), device=actions.device)
    g.scatter_(-1, actions.long()[..., None], 1e6)
    return g


def _run(env, pol, H, snap, noise=None, continuous=False, **kw):
    env.set_state(snap)
    if noise is not None:
        kw["noise" if continuous else "gumbel"] = noise
    out = {k: v.clone() for k, v in env.rollout(pol, H, **kw).items()}
    out["h1"] = _bits16(pol.peek("h1"))
    torch.cuda.synchronize()
    return out


def _pair(D, hidden, continuous, seed):
    a = _weights(D, hidden, continuous, seed=seed)
    c = _weights(D, hidden, continuous, seed=seed + 1000)
    return a, c


def _check_against_shared(env, sep, a, c, H, N, noise, continuous, tag, controls=False):
    """the separate policy `sep` against shared-body runs from the current state: actor side, critic side and h1 bit
    for bit; returns the separate run"""
    hidden = sep.hidden
    snap = env.get_state()
    out = _run(env, sep, H, snap, noise, continuous)
    actor_pol = env.make_policy(a)
    ref_a = _run(env, actor_pol, H, snap, noise, continuous)
    for k in ("obs", "actions", "logp", "reward", "done"):
        assert torch.equal(out[k], ref_a[k]), f"{tag}: {k} differs from the shared run with the actor's weights"
    critic_pol = env.make_policy(_critic_shared(c, a, continuous))
    ref_c = _run(env, critic_pol, H, snap, _forcing_noise(out["actions"], continuous), continuous)
    assert torch.equal(ref_c["actions"], out["actions"]), f"{tag}: the forcing noise did not reproduce the actions"
    assert torch.equal(out["value"], ref_c["value"]), f"{tag}: value differs from the shared run with the critic's weights"
    h1 = out["h1"]
    assert h1.shape[1] == 2 * hidden, tag
    assert torch.equal(h1[:N, :hidden], ref_a["h1"][:N]), f"{tag}: h1 actor columns"
    assert torch.equal(h1[:N, hidden:], ref_c["h1"][:N]), f"{tag}: h1 critic columns"
    if controls:   # each of the checks above rejects a wrong reference
        assert not torch.equal(out["value"], ref_a["value"]), f"{tag}: value check accepts the actor trunk's value"
        assert not torch.equal(torch.cat([h1[:N, hidden:], h1[:N, :hidden]], 1), torch.cat([ref_a["h1"][:N], ref_c["h1"][:N]], 1)), \
            f"{tag}: h1 check accepts swapped halves"
        # actor and critic trunks swapped (the heads stay)
        swapped = env.make_policy(_separate({**a, **{k: c[k] for k in TRUNK}}, {**c, **{k: a[k] for k in TRUNK}}))
        ref_s = _run(env, swapped, H, snap, noise, continuous)
        assert not torch.equal(ref_s["logp"], out["logp"]) or not torch.equal(ref_s["actions"], out["actions"]), \
            f"{tag}: actor check accepts swapped networks"
        assert not torch.equal(ref_s["value"], out["value"]), f"{tag}: critic check accepts swapped networks"
        bad = _critic_shared(c, a, continuous)
        bad["w2"] = a["w2"]
        ref_w2 = _run(env, env.make_policy(bad), H, snap, _forcing_noise(out["actions"], continuous), continuous)
        assert not torch.equal(ref_w2["value"], out["value"]), f"{tag}: critic check accepts the actor's W2"
        swapped.close()
    actor_pol.close(); critic_pol.close()
    env.set_state(snap)
    return out


def _check_reference(out, a, c, H, N, noise, continuous, tag):
    """the fp64 host reference of each trunk, with the tolerances of test_gpu_policy_widths.py"""
    hidden = a["w1"].shape[0]
    h1 = out["h1"].view(torch.bfloat16)
    obs = out["obs"]
    ra, rc = R.forward_ref(a, obs[H]), R.forward_ref(c, obs[H])
    assert R.check_h1(h1[:N, :hidden], ra, obs[H], a)["bad"] == 0, f"{tag}: actor h1"
    assert R.check_h1(h1[:N, hidden:], rc, obs[H], c)["bad"] == 0, f"{tag}: critic h1"
    assert R.check_h1(h1[:N, hidden:], ra, obs[H], a)["bad"] > 0, f"{tag}: h1 check accepts the other trunk"
    for t in range(H + 1):
        rc_t = R.forward_ref(c, obs[t])
        assert R.head_close(out["value"][t], rc_t["value"]), (tag, t, R.head_err(out["value"][t], rc_t["value"]))
        if t == 0:
            assert not R.head_close(out["value"][t], R.forward_ref(a, obs[t])["value"]), f"{tag}: value tolerance accepts the actor trunk"
        if t == H:
            break
        ra_t = R.forward_ref(a, obs[t])
        if continuous:
            want = ra_t["head"][:, 0] + math.exp(float(a["log_std"])) * noise[t].double()
            assert R.head_close(out["actions"][t], want), (tag, t, R.head_err(out["actions"][t], want))
        else:
            lp = torch.log_softmax(ra_t["head"], -1).gather(1, out["actions"][t].long()[:, None]).squeeze(1)
            assert R.head_close(out["logp"][t], lp, 3e-3), (tag, t, R.head_err(out["logp"][t], lp))


# ---------------------------------------------------------------------------------------- 1.-5. widths x modes
@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
@pytest.mark.parametrize("hidden", WIDTHS)
def test_separate_equals_two_shared_runs(hidden, continuous):
    N, H = 300, 3
    make = _factory(N, 20, continuous=continuous)
    env, twin = make(), make()
    starts = torch.as_tensor(start_offsets(N, T_BARS, 200, 300))
    env.reset(starts); twin.reset(starts)
    _warm((env, twin), N, 8, continuous)
    D = env.obs_dim
    a, c = _pair(D, hidden, continuous, seed=hidden + continuous)
    sep = env.make_policy(_separate(a, c))
    assert sep.separate and sep.hidden == hidden
    tag = f"h{hidden}/{'cont' if continuous else 'disc'}"
    noise = _noise(H, N, continuous, seed=hidden)
    out = _check_against_shared(env, sep, a, c, H, N, noise, continuous, tag, controls=True)
    _check_reference(out, a, c, H, N, noise, continuous, tag)
    # the env side against a twin stepped with the sampled actions
    out2 = env.rollout(sep, H, **({"noise": noise} if continuous else {"gumbel": noise}))
    torch.cuda.synchronize()
    _check_env_side(env, twin, out2, H)
    # in-kernel noise (same seed) and greedy rollouts: the actor side against the shared actor run
    snap = env.get_state()
    actor_pol = env.make_policy(a)
    for kw in ({"seed": 99}, {"deterministic": True}):
        s = _run(env, sep, H, snap, **kw)
        r = _run(env, actor_pol, H, snap, **kw)
        for k in ("obs", "actions", "logp", "reward", "done"):
            assert torch.equal(s[k], r[k]), f"{tag} {kw}: {k}"
    env.close(); twin.close()


# ------------------------------------------------------------------------------- 6. env counts, groups, rings
@pytest.mark.parametrize("N", [1, 127, 129, 4096 + 64])
@pytest.mark.parametrize("hidden", [128, 512])
def test_env_counts_groups_and_tile_sync(hidden, N, monkeypatch):
    """groups 1-4 x FXENV_TILE_SYNC 0 / 1 from one state: identical outputs and h1, nothing written past row N; the
    first setting against the shared runs"""
    H, continuous = 3, N % 2 == 1
    make = _factory(N, 20, continuous=continuous)
    env = make()
    env.reset(torch.as_tensor(start_offsets(N, T_BARS, 200, 300)))
    _warm((env,), N, 6, continuous)
    D = env.obs_dim
    a, c = _pair(D, hidden, continuous, seed=N + hidden)
    w = _separate(a, c)
    noise = _noise(H, N, continuous, seed=N)
    snap = env.get_state()
    first = None
    for groups in (1, 2, 3, 4):
        for ts in (0, 1):
            monkeypatch.setenv("FXENV_ROLLOUT_GROUPS", str(groups))
            monkeypatch.setenv("FXENV_TILE_SYNC", str(ts))
            env.set_state(snap)
            pol = env.make_policy(w)   # the rollout graph reads these settings at capture: one policy per setting
            tag = f"h{hidden}/N{N}/g{groups}/ts{ts}"
            if first is None:
                first = _check_against_shared(env, pol, a, c, H, N, noise, continuous, tag)
                pol.close()
                continue
            bufs, backing, tails = _sentinel_buffers(H, N, D, torch.float32 if continuous else torch.int32)
            out = env.rollout(pol, H, buffers=bufs, **({"noise": noise} if continuous else {"gumbel": noise}))
            torch.cuda.synchronize()
            assert pol.sync_timeouts() == 0
            for k, raw in backing.items():
                assert torch.equal(raw[-tails[k].numel():], tails[k]), f"{tag}: the rollout wrote past the end of `{k}`"
            for k in KEYS:
                assert torch.equal(first[k], out[k]), f"{tag}: {k} differs from groups=1, tile hand-over off"
            assert torch.equal(first["h1"], _bits16(pol.peek("h1"))), f"{tag}: h1"
            pol.close()
    env.close()


@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_two_slot_obs_ring(continuous):
    N, H = 300, 6
    env = _factory(N, 20, continuous=continuous)()
    env.reset(torch.as_tensor(start_offsets(N, T_BARS, 200, 300)))
    a, c = _pair(env.obs_dim, 256, continuous, seed=7)
    pol = env.make_policy(_separate(a, c))
    snap = env.get_state()
    full = _run(env, pol, H, snap, seed=5)
    env.set_state(snap)
    ring = {"obs": torch.empty((2, N, env.obs_dim), device="cuda")}
    out = env.rollout(pol, H, buffers=ring, seed=5)
    torch.cuda.synchronize()
    for k in ("actions", "logp", "value", "reward", "done"):
        assert torch.equal(full[k], out[k]), k
    assert torch.equal(out["obs"][H % 2], full["obs"][H]) and torch.equal(out["obs"][(H - 1) % 2], full["obs"][H - 1])
    env.close()


def test_set_weights_between_graph_replays():
    N, H = 260, 4
    env = _factory(N, 20)()
    env.reset(torch.as_tensor(start_offsets(N, T_BARS, 200, 300)))
    D = env.obs_dim
    w1, w2 = _separate(*_pair(D, 128, False, seed=1)), _separate(*_pair(D, 128, False, seed=2))
    snap = env.get_state()
    pol = env.make_policy(w1)
    bufs = env.rollout(pol, H, seed=3)   # captures the graph
    env.set_state(snap)
    pol.set_weights(w2)
    got = {k: v.clone() for k, v in env.rollout(pol, H, buffers=bufs, seed=3).items()}
    got["h1"] = _bits16(pol.peek("h1"))
    fresh = _run(env, env.make_policy(w2), H, snap, seed=3)
    for k in KEYS + ("h1",):
        assert torch.equal(got[k], fresh[k]), k
    env.close()


# ----------------------------------------------------------------------------------------------------- 7. errors
def test_errors():
    N = 130
    env = _factory(N, 20)()
    env.reset(torch.as_tensor(start_offsets(N, T_BARS, 200, 300)))
    D = env.obs_dim
    a, c = _pair(D, 64, False, seed=3)
    w = _separate(a, c)
    for flags in (2, 4, 0x80000000):
        p = C.c_void_p()
        assert env.L.fxenv_policy_create_ex2(env._h, 64, flags, C.byref(p)) == -1   # FXENV_E_INVALID
        assert not p.value
        assert b"unknown policy flags" in env.L.fxenv_last_error(env._h)
    bad = dict(w)
    bad["w2_v"] = torch.zeros(64, 32, device="cuda")
    with pytest.raises(ValueError, match="w2_v"):
        env.make_policy(bad)
    with pytest.raises(ValueError, match="separate"):
        env.make_policy(w, separate=False)
    with pytest.raises(ValueError, match="separate"):
        env.make_policy(a, separate=True)
    from gym_fx_b200.learner import ActorCritic
    shared_net, sep_net = ActorCritic(D, hidden=64).cuda(), ActorCritic(D, hidden=64, separate=True).cuda()
    assert env.make_policy(sep_net).separate and not env.make_policy(shared_net).separate
    assert env.make_policy(hidden=64, separate=True).separate and not env.make_policy().separate
    sep_pol, shared_pol = env.make_policy(hidden=64, separate=True), env.make_policy(hidden=64)
    for pol, wrong in ((sep_pol, shared_net), (shared_pol, sep_net), (sep_pol, a), (shared_pol, w)):
        with pytest.raises(ValueError):
            pol.set_weights(wrong)
    assert sep_pol.peek("h1").shape == (256, 128) and shared_pol.peek("h1").shape == (256, 64)
    env.close()


# ---------------------------------------------------------------------------------------------------- 8. learner
@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_learner_update(continuous):
    from gym_fx_b200.learner import ActorCritic, ppo_update
    N, H = 512, 8
    env = _factory(N, 20, continuous=continuous)()
    env.reset(torch.as_tensor(start_offsets(N, T_BARS, 200, 300)))
    torch.manual_seed(3)
    net = ActorCritic(env.obs_dim, hidden=128, continuous=continuous, separate=True).cuda()
    pol = env.make_policy(net)
    assert pol.separate and pol.hidden == 128
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    buf = env.rollout(pol, H, seed=1)
    before = {k: v.detach().clone() for k, v in net.state_dict().items()}
    stats = ppo_update(net, opt, buf, torch.zeros(N, dtype=torch.uint8, device="cuda"), None, epochs=1, minibatches=2)
    assert all(math.isfinite(v) for v in stats.values()), stats
    for k in ("body.0.weight", "body.2.weight", "critic_body.0.weight", "critic_body.2.weight"):
        assert not torch.equal(before[k], net.state_dict()[k]), f"the update did not move {k}"
    pol.set_weights(net)
    out = env.rollout(pol, H, buffers=buf, seed=2)
    torch.cuda.synchronize()
    actor = R.weights_of(net)
    cb = net.critic_body
    critic = {**actor, "w1": cb[0].weight, "b1": cb[0].bias, "w2": cb[2].weight, "b2": cb[2].bias}
    for t in range(H + 1):
        ref = R.forward_ref(critic, out["obs"][t])
        assert R.head_close(out["value"][t], ref["value"]), (t, R.head_err(out["value"][t], ref["value"]))
        if t < H and not continuous:
            lp = torch.log_softmax(R.forward_ref(actor, out["obs"][t])["head"], -1).gather(1, out["actions"][t].long()[:, None]).squeeze(1)
            assert R.head_close(out["logp"][t], lp, 3e-3), (t, R.head_err(out["logp"][t], lp))
    env.close()
