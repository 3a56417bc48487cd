"""GPU (-m gpu): a policy population in the fused closed loop (fxenv_policy_create_ex3, VecFxEnv.make_policy(members=M)):
M actor-critic networks of one width and layout, member m acting for the envs [m N / M, (m + 1) N / M).

The reference is the single-policy kernel, so every check is bit for bit.  From one env snapshot, a population rollout
and, for each member m, a single-policy rollout with member m's weights must agree on member m's slice of obs,
actions, log-probs, values, rewards and dones -- with caller noise, the in-kernel generator and in greedy mode, at every
width, in both action modes and both network layouts, for M = 2, 4 and N / 128 (one tile per member).  Then: a negative
control (members' weights permuted), members whose tiles straddle an env-group boundary with 1-4 groups and the tile
hand-over on and off, one member's weights replaced under a cached rollout graph, the argument errors, and a
population PPO update."""
import ctypes as C

import pytest
import torch

import policy_ref as R
from gym_fx_b200 import _native
from gym_fx_b200.synth import start_offsets
from test_gpu_policy_edges import T_BARS, _factory, _noise, _warm
from test_gpu_policy_separate import _pair, _separate
from test_gpu_policy_widths import _weights

pytestmark = pytest.mark.gpu

WIDTHS = [64, 128, 256, 512]
KEYS = ("obs", "actions", "logp", "value", "reward", "done")


def _member_weights(D, hidden, continuous, separate, M, seed):
    """M different weight dicts (separate: actor and critic trunks each)"""
    if separate:
        return [_separate(*_pair(D, hidden, continuous, seed + 10 * m)) for m in range(M)]
    return [_weights(D, hidden, continuous, seed=seed + 10 * m) for m in range(M)]


def _env(N, continuous=False):
    env = _factory(N, 20, continuous=continuous)()
    env.reset(torch.as_tensor(start_offsets(N, T_BARS, 200, 300)))
    _warm((env,), N, 6, continuous)
    return env


def _run(env, pol, H, snap, bufs, kw):
    """a rollout from `snap` into `bufs` (the same dict for every call of one policy: its rollout graph is reused)"""
    env.set_state(snap)
    out = env.rollout(pol, H, buffers=bufs, **kw)
    torch.cuda.synchronize()
    return {k: v.clone() for k, v in out.items()}


def _noise_modes(H, N, continuous, seed):
    return [{"noise" if continuous else "gumbel": _noise(H, N, continuous, seed)}, {"seed": 99}, {"deterministic": True}]


def _check_members(env, pop, ws, single, H, snap, kw, tag, out=None):
    """each member's slice of a population rollout (`out`, or one run here) against a single policy with its weights;
    returns the population run"""
    if out is None:
        out = _run(env, pop, H, snap, {}, kw)
    sbufs = {}
    for m in range(pop.members):
        single.set_weights(ws[m])
        ref = _run(env, single, H, snap, sbufs, kw)
        sl = pop.member_envs(m)
        for k in KEYS:
            assert torch.equal(out[k][:, sl], ref[k][:, sl]), f"{tag}: member {m}, {k} differs from the single policy"
    return out


# ------------------------------------------------------------------------------------- 1. member equivalence
@pytest.mark.parametrize("separate", [False, True], ids=["shared", "separate"])
@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
@pytest.mark.parametrize("hidden", WIDTHS)
def test_members_equal_single_policies(hidden, continuous, separate):
    N, H = 1024, 3   # 8 tiles: M = 2, 4 and 8 (one tile per member)
    env = _env(N, continuous)
    D = env.obs_dim
    snap = env.get_state()
    single = env.make_policy(hidden=hidden, separate=separate)
    for M in (2, 4, N // 128):
        ws = _member_weights(D, hidden, continuous, separate, M, seed=hidden + 7 * M + continuous)
        pop = env.make_policy(ws)
        assert (pop.members, pop.hidden, pop.separate) == (M, hidden, separate)
        assert [pop.member_envs(m) for m in range(M)] == [slice(m * N // M, (m + 1) * N // M) for m in range(M)]
        pbufs = {}
        for kw in _noise_modes(H, N, continuous, seed=M):
            tag = f"h{hidden}/{'cont' if continuous else 'disc'}/{'sep' if separate else 'shared'}/M{M}/{sorted(kw)[0]}"
            _check_members(env, pop, ws, single, H, snap, kw, tag, out=_run(env, pop, H, snap, pbufs, kw))
        pop.close()
    env.close()


def test_negative_control_permuted_members():
    """the comparison above rejects a population whose members' weights are rotated by one"""
    N, H, M = 512, 3, 4
    env = _env(N)
    D = env.obs_dim
    snap = env.get_state()
    ws = _member_weights(D, 128, False, False, M, seed=5)
    single = env.make_policy(hidden=128)
    kw = {"gumbel": _noise(H, N, False, seed=5)}
    good = _check_members(env, env.make_policy(ws), ws, single, H, snap, kw, "control")
    bad = _run(env, env.make_policy(ws[1:] + ws[:1]), H, snap, {}, kw)
    for m in range(M):
        sl = slice(m * N // M, (m + 1) * N // M)
        assert not torch.equal(bad["value"][:, sl], good["value"][:, sl]), f"member {m}: permuted values pass"
        assert not torch.equal(bad["logp"][:, sl], good["logp"][:, sl]), f"member {m}: permuted log-probs pass"
    with pytest.raises(AssertionError):
        _check_members(env, env.make_policy(ws[1:] + ws[:1]), ws, single, H, snap, kw, "permuted")
    env.close()


# ----------------------------------------------------------------------------------- 2. env-group boundaries
@pytest.mark.parametrize("separate", [False, True], ids=["shared", "separate"])
def test_members_across_group_boundaries(separate, monkeypatch):
    """M = 3 members of 2 tiles on 768 envs: 2 env groups of 384 envs split member 1.  Groups 1-4 x tile hand-over
    0 / 1 give identical outputs; the first setting is checked member by member against single policies."""
    N, H, M, hidden = 768, 3, 3, 128
    continuous = separate   # both action modes, across the two cases
    env = _env(N, continuous)
    D = env.obs_dim
    snap = env.get_state()
    ws = _member_weights(D, hidden, continuous, separate, M, seed=11)
    kw = {"noise" if continuous else "gumbel": _noise(H, N, continuous, seed=11)}
    first = None
    for groups in (1, 2, 3, 4):
        for ts in (0, 1):
            monkeypatch.setenv("FXENV_ROLLOUT_GROUPS", str(groups))
            monkeypatch.setenv("FXENV_TILE_SYNC", str(ts))
            pol = env.make_policy(ws)   # the rollout graph reads these settings at capture: one policy per setting
            out = _run(env, pol, H, snap, {}, kw)
            assert pol.sync_timeouts() == 0
            tag = f"{'sep' if separate else 'shared'}/g{groups}/ts{ts}"
            if first is None:
                single = env.make_policy(hidden=hidden, separate=separate)
                first = _check_members(env, pol, ws, single, H, snap, kw, tag, out=out)
                single.close()
            else:
                for k in KEYS:
                    assert torch.equal(first[k], out[k]), f"{tag}: {k} differs from groups=1, tile hand-over off"
            pol.close()
    env.close()


# ------------------------------------------------------------------------------- 3. one member's weights updated
@pytest.mark.parametrize("separate", [False, True], ids=["shared", "separate"])
def test_set_member_weights_between_graph_replays(separate):
    N, H, M, hidden, changed = 1024, 4, 4, 256, 2
    env = _env(N)
    D = env.obs_dim
    snap = env.get_state()
    ws = _member_weights(D, hidden, False, separate, M, seed=21)
    new = _member_weights(D, hidden, False, separate, 1, seed=99)[0]
    pop = env.make_policy(ws)
    bufs, kw = {}, {"seed": 3}
    before = _run(env, pop, H, snap, bufs, kw)   # captures the rollout graph
    again = _run(env, pop, H, snap, bufs, kw)    # replays it
    for k in KEYS:
        assert torch.equal(before[k], again[k]), k
    pop.set_member_weights(changed, new)
    after = _run(env, pop, H, snap, bufs, kw)    # the same buffers, seed and flags: the cached graph
    for m in range(M):
        sl = pop.member_envs(m)
        if m == changed:
            assert not torch.equal(after["value"][:, sl], before["value"][:, sl]), "the new weights were not used"
        else:
            for k in KEYS:
                assert torch.equal(after[k][:, sl], before[k][:, sl]), f"member {m}: {k} changed with member {changed}"
    fresh = _run(env, env.make_policy(ws[:changed] + [new] + ws[changed + 1:]), H, snap, {}, kw)
    for k in KEYS:
        assert torch.equal(after[k], fresh[k]), f"{k}: the updated population differs from a fresh one"
    env.close()


# --------------------------------------------------------------------------------------------------- 4. errors
def test_errors_leave_the_handle_usable():
    N = 256   # two tiles: 1 or 2 members
    env = _env(N)
    D = env.obs_dim
    L = env.L
    w, w2, w128 = (_weights(D, h, False, seed=s) for h, s in ((64, 1), (64, 2), (128, 3)))
    for members, msg in ((3, b"multiple of 128"), (4, b"multiple of 128"), (0, b"members must be >= 1"),
                         (-2, b"members must be >= 1")):
        p = C.c_void_p()
        assert L.fxenv_policy_create_ex3(env._h, 64, 0, members, C.byref(p)) == -1   # FXENV_E_INVALID
        assert not p.value and msg in L.fxenv_last_error(env._h), members
    with pytest.raises(ValueError, match="multiple of 128"):
        env.make_policy(hidden=64, members=3)
    with pytest.raises(ValueError, match="members"):
        env.make_policy(hidden=64, members=0)
    with pytest.raises(ValueError, match="weight sets"):
        env.make_policy([w, w2], members=4)
    with pytest.raises(ValueError, match="width"):
        env.make_policy([w, w128])
    pop = env.make_policy(hidden=64, members=2)
    assert pop.members == 2
    for m in (2, -1, True):
        with pytest.raises(ValueError, match="member"):
            pop.set_member_weights(m, w)
    ts = pop._tensors(w)
    pw = _native.FxPolicyWeights(*[ts[k].data_ptr() for k in ("w1", "b1", "w2", "b2", "w_pi", "b_pi", "w_v", "b_v")])
    for m in (2, -1):
        assert L.fxenv_policy_set_member_weights(pop._p, m, C.byref(pw), env._stream()) == -1
        assert b"out of range" in L.fxenv_last_error(env._h)
    with pytest.raises(ValueError, match="shape"):
        pop.set_member_weights(1, w128)
    pop.set_member_weights(0, w)
    with pytest.raises(_native.FxEnvError, match=r"\(-3\).*member 1"):   # FXENV_E_STATE
        env.rollout(pop, 2, seed=1)
    with pytest.raises(ValueError, match="weight sets"):
        pop.set_weights([w])
    with pytest.raises(ValueError, match="weight sets"):
        pop.set_weights(w)
    pop.set_member_weights(1, w2)
    snap = env.get_state()
    out = _run(env, pop, 2, snap, {}, {"seed": 1})
    assert bool(torch.isfinite(out["value"]).all())
    single = env.make_policy(hidden=64)
    _check_members(env, pop, [w, w2], single, 2, snap, {"seed": 1}, "after the errors", out=out)
    env.close()


# ---------------------------------------------------------------------------------------------------- 5. learner
@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_population_ppo_update(continuous):
    from gym_fx_b200.learner import ActorCritic, ppo_update_population
    N, H, M = 512, 8, 2
    env = _env(N, continuous)
    D = env.obs_dim
    nets = []
    for m in range(M):
        torch.manual_seed(30 + m)
        nets.append(ActorCritic(D, hidden=128, continuous=continuous).cuda())
    opts = [torch.optim.Adam(n.parameters(), lr=1e-3) for n in nets]
    pop = env.make_policy(nets)
    assert pop.members == M and pop.hidden == 128
    buf = env.rollout(pop, H, seed=1)
    before = [{k: v.detach().clone() for k, v in n.state_dict().items()} for n in nets]
    stats = ppo_update_population(nets, opts, buf, torch.zeros(N, dtype=torch.uint8, device="cuda"), None, epochs=1,
                                  minibatches=2)
    assert len(stats) == M
    for m in range(M):
        assert all(v == v for v in stats[m].values()), stats[m]
        for k in ("body.0.weight", "body.2.weight", "pi.weight", "v.weight"):
            assert not torch.equal(before[m][k], nets[m].state_dict()[k]), f"member {m}: the update did not move {k}"
    pop.set_weights(nets)
    out = env.rollout(pop, H, buffers=buf, seed=2)
    torch.cuda.synchronize()
    for m in range(M):   # each slice's values come from its own, updated member (fp64 reference, bf16 tolerance)
        sl = pop.member_envs(m)
        for t in (0, H):
            ref = R.forward_ref(R.weights_of(nets[m]), out["obs"][t][sl])
            assert R.head_close(out["value"][t][sl], ref["value"]), (m, t, R.head_err(out["value"][t][sl], ref["value"]))
            other = R.forward_ref(R.weights_of(nets[1 - m]), out["obs"][t][sl])
            assert not R.head_close(out["value"][t][sl], other["value"]), f"member {m}: the other member's values pass"
    env.close()
