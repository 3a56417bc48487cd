"""CPU (-m "not gpu"): ActorCritic(separate=True) -- separate actor and critic networks in the learner
(gym_fx_b200/learner.py): forward shapes, which trunk each loss reaches, a PPO update on a synthetic rollout, and the
weight checks of FusedPolicy that run before any library call."""
import math

import pytest
import torch

from gym_fx_b200.learner import ActorCritic, ppo_update


@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_forward_shapes_and_trunks(continuous):
    net = ActorCritic(20, hidden=16, continuous=continuous, separate=True)
    assert net.separate and tuple(net.critic_body[0].weight.shape) == (16, 20)
    assert tuple(net.critic_body[2].weight.shape) == (16, 16)
    head, v = net(torch.randn(5, 20))
    assert head.shape == (5, 1 if continuous else 3) and v.shape == (5,)
    x = torch.randn(4, 20)
    with torch.no_grad():
        h_pi, h_v = net.body(x), net.critic_body(x)
        want_head, want_v = net.pi(h_pi), net.v(h_v).squeeze(-1)
        got_head, got_v = net(x)
    assert torch.equal(got_head, want_head) and torch.equal(got_v, want_v)
    assert not hasattr(ActorCritic(20, hidden=16), "critic_body")


def test_each_loss_reaches_only_its_own_trunk():
    torch.manual_seed(0)
    net = ActorCritic(12, hidden=8, separate=True)
    x = torch.randn(32, 12)
    logits, v = net(x)
    v.square().mean().backward(retain_graph=True)   # critic loss
    assert all(p.grad is None or not bool(p.grad.any()) for p in list(net.body.parameters()) + list(net.pi.parameters()))
    assert all(p.grad is not None and bool(p.grad.any()) for p in net.critic_body.parameters())
    net.zero_grad(set_to_none=True)
    torch.log_softmax(logits, -1)[:, 1].mean().backward()   # policy loss
    assert all(p.grad is None or not bool(p.grad.any()) for p in list(net.critic_body.parameters()) + list(net.v.parameters()))
    assert all(p.grad is not None and bool(p.grad.any()) for p in net.body.parameters())


@pytest.mark.parametrize("continuous", [False, True], ids=["discrete", "continuous"])
def test_ppo_update_moves_both_trunks(continuous):
    torch.manual_seed(1)
    H, N, D = 8, 16, 12
    net = ActorCritic(D, hidden=8, continuous=continuous, separate=True)
    opt = torch.optim.Adam(net.parameters(), lr=1e-2)
    g = torch.Generator().manual_seed(2)
    buf = {"obs": torch.randn(H + 1, N, D, generator=g),
           "actions": torch.randn(H, N, generator=g) if continuous else torch.randint(0, 3, (H, N), generator=g, dtype=torch.int32),
           "logp": torch.full((H, N), -1.1), "value": torch.randn(H + 1, N, generator=g), "reward": torch.randn(H, N, generator=g),
           "done": (torch.rand(H, N, generator=g) < 0.1).to(torch.uint8)}
    before = {k: v.detach().clone() for k, v in net.state_dict().items()}
    stats = ppo_update(net, opt, buf, torch.zeros(N, dtype=torch.uint8), None, epochs=1, minibatches=2)
    assert all(math.isfinite(v) for v in stats.values()), stats
    after = net.state_dict()
    for k in ("body.0.weight", "body.2.weight", "critic_body.0.weight", "critic_body.2.weight", "pi.weight", "v.weight"):
        assert not torch.equal(before[k], after[k]), f"{k} did not move"


def test_fused_policy_separate_inference():
    """FusedPolicy infers the layout from the weights before it creates anything in the library"""
    from gym_fx_b200.vec_env import FusedPolicy

    assert FusedPolicy._separate_of(ActorCritic(10, hidden=8, separate=True))
    assert not FusedPolicy._separate_of(ActorCritic(10, hidden=8))
    w = {"w1": torch.zeros(8, 10)}
    assert not FusedPolicy._separate_of(w)
    assert FusedPolicy._separate_of({**w, "w1_v": torch.zeros(8, 10), "b1_v": torch.zeros(8), "w2_v": torch.zeros(8, 8),
                                     "b2_v": torch.zeros(8)})
