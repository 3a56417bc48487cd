"""CPU (-m "not gpu"): ppo_update_population (gym_fx_b200/learner.py) -- one PPO update per member of a policy
population, each on its own contiguous slice of the envs -- against per-member ppo_update calls on hand-made slices,
a check that a member reads nothing outside its slice, and the population checks of FusedPolicy that run before any
library call."""
import math

import pytest
import torch

from gym_fx_b200.learner import ActorCritic, ppo_update, ppo_update_population


def _buffer(H, N, D, continuous, seed):
    g = torch.Generator().manual_seed(seed)
    return {"obs": torch.randn(H + 1, N, D, generator=g),
            "actions": torch.randn(H, N, generator=g) if continuous else torch.randint(0, 3, (H, N), generator=g, dtype=torch.int32),
            "logp": -torch.rand(H, N, generator=g) - 0.5, "value": torch.randn(H + 1, N, generator=g),
            "reward": torch.randn(H, N, generator=g), "done": (torch.rand(H, N, generator=g) < 0.1).to(torch.uint8)}


def _members(M, D, continuous, separate=False):
    nets, opts = [], []
    for m in range(M):
        torch.manual_seed(100 + m)
        nets.append(ActorCritic(D, hidden=8, continuous=continuous, separate=separate))
        opts.append(torch.optim.Adam(nets[-1].parameters(), lr=1e-2))
    return nets, opts


@pytest.mark.parametrize("separate", [False, True], ids=["shared", "separate"])
@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_equals_per_member_updates_on_slices(continuous, separate):
    H, M, n, D = 6, 3, 8, 10
    N = M * n
    buf = _buffer(H, N, D, continuous, seed=4)
    prev_done = (torch.arange(N) % 5 == 0).to(torch.uint8)
    nets, opts = _members(M, D, continuous, separate)
    ref_nets, ref_opts = _members(M, D, continuous, separate)
    torch.manual_seed(9)
    stats = ppo_update_population(nets, opts, buf, prev_done, None, epochs=2, minibatches=2)
    torch.manual_seed(9)
    ref_stats = []
    for m in range(M):   # the slices made by hand, as contiguous copies
        sub = {k: v[:, m * n:(m + 1) * n].clone() for k, v in buf.items()}
        ref_stats.append(ppo_update(ref_nets[m], ref_opts[m], sub, prev_done[m * n:(m + 1) * n].clone(), None, epochs=2,
                                    minibatches=2))
    assert len(stats) == M
    for m in range(M):
        assert stats[m] == ref_stats[m], m
        for (k, p), q in zip(nets[m].state_dict().items(), ref_nets[m].state_dict().values()):
            assert torch.equal(p, q), f"member {m}: {k}"
    # every member moved, and differently from the others
    fresh, _ = _members(M, D, continuous, separate)
    for m in range(M):
        assert not torch.equal(nets[m].body[0].weight, fresh[m].body[0].weight), m


def test_a_member_reads_only_its_own_envs():
    H, M, n, D = 6, 4, 8, 10
    buf = _buffer(H, M * n, D, False, seed=5)
    prev_done = torch.zeros(M * n, dtype=torch.uint8)
    keep = 2
    for k, v in buf.items():   # every other member's slice is poison
        if v.is_floating_point():
            v[:, :keep * n] = float("nan")
            v[:, (keep + 1) * n:] = float("nan")
    nets, opts = _members(M, D, False)
    before = {k: v.clone() for k, v in nets[keep].state_dict().items()}
    stats = ppo_update_population(nets, opts, buf, prev_done, None, epochs=1, minibatches=2)
    assert all(math.isfinite(v) for v in stats[keep].values()), stats[keep]
    for k, v in nets[keep].state_dict().items():
        assert bool(torch.isfinite(v).all()), k
    assert any(not torch.equal(before[k], v) for k, v in nets[keep].state_dict().items())
    assert not bool(torch.isfinite(nets[0].body[0].weight).all()), "negative control: a poisoned member goes NaN"


def test_argument_errors():
    nets, opts = _members(2, 6, False)
    buf = _buffer(2, 6, 6, False, seed=1)
    with pytest.raises(ValueError, match="optimiser"):
        ppo_update_population(nets, opts[:1], buf, torch.zeros(6, dtype=torch.uint8))
    with pytest.raises(ValueError, match="optimiser"):
        ppo_update_population([], [], buf, torch.zeros(6, dtype=torch.uint8))
    nets, opts = _members(4, 6, False)
    with pytest.raises(ValueError, match="equal member slices"):
        ppo_update_population(nets, opts, buf, torch.zeros(6, dtype=torch.uint8))


class _FakeEnv:
    """what FusedPolicy reads of a VecFxEnv before it calls the library"""
    num_envs = 512


def test_fused_policy_population_checks_before_the_library():
    from gym_fx_b200.vec_env import FusedPolicy

    w64 = ActorCritic(10, hidden=64)
    w128 = ActorCritic(10, hidden=128)
    sep = ActorCritic(10, hidden=64, separate=True)
    env = _FakeEnv()
    for kw, msg in (({"members": 0}, "members"), ({"members": -1}, "members"), ({"members": 1.5}, "members"),
                    ({"members": 3}, "multiple of 128"), ({"weights": [w64, w128]}, "width"),
                    ({"weights": [w64, sep]}, "layout"), ({"weights": [w64, w64], "members": 4}, "2 weight sets"),
                    ({"weights": w64, "members": 2}, "list"), ({"weights": [w64, w64], "hidden": 128}, "disagrees"),
                    ({"weights": [w64, w64], "separate": True}, "disagrees")):
        with pytest.raises(ValueError, match=msg):
            FusedPolicy(env, **kw)
    assert FusedPolicy._common([w64, w64], FusedPolicy._width_of, "width") == 64
