"""CPU (-m "not gpu"): continuous action mode of the learner (gym_fx_b200/learner.py) -- the Gaussian log-prob and
entropy, a sharded continuous PPO update over gloo with world_size 2 (replicas must stay bit-identical) -- and the
greedy-rollout entry point of the C-ABI."""
import math
import os
import re
import socket
import sys

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_gaussian_log_prob_and_entropy_match_torch_distributions():
    from gym_fx_b200.learner import gaussian_entropy, gaussian_log_prob

    g = torch.Generator().manual_seed(0)
    mean = torch.randn(64, generator=g, dtype=torch.float64)
    x = torch.randn(64, generator=g, dtype=torch.float64) * 2
    for ls in (-2.0, -0.5, 0.0, 0.7):
        log_std = torch.tensor([ls], dtype=torch.float64)
        ref = torch.distributions.Normal(mean, log_std.exp())
        assert torch.allclose(gaussian_log_prob(mean, log_std, x), ref.log_prob(x), atol=1e-12, rtol=0)
        assert torch.allclose(gaussian_entropy(log_std), ref.entropy()[:1], atol=1e-12, rtol=0)


def test_continuous_actor_critic_layout():
    from gym_fx_b200.learner import ActorCritic

    net = ActorCritic(20, hidden=16, continuous=True, init_log_std=-0.5)
    assert net.pi.weight.shape == (1, 16) and net.pi.bias.shape == (1,)
    assert net.log_std.shape == (1,) and float(net.log_std.detach()) == -0.5 and net.log_std.requires_grad
    mean, v = net(torch.zeros(3, 20))
    assert mean.shape == (3, 1) and v.shape == (3,)
    torch.manual_seed(0)
    a = torch.cat([p.detach().reshape(-1) for p in ActorCritic(20, hidden=16).parameters()])
    torch.manual_seed(0)
    b = torch.cat([p.detach().reshape(-1) for p in ActorCritic(20, hidden=16, continuous=False).parameters()])
    assert torch.equal(a, b), "the discrete network must not change"


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    from gym_fx_b200.learner import ActorCritic, ppo_update

    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.manual_seed(0)                      # identical replicas
    H, N, D = 6, 8, 20
    net = ActorCritic(D, hidden=16, continuous=True, init_log_std=-0.5)
    opt = torch.optim.Adam(net.parameters(), lr=1e-2)
    g = torch.Generator().manual_seed(100 + rank)   # every rank has its own shard of the rollout
    act = torch.randn(H, N, generator=g)
    buf = {"obs": torch.randn(H + 1, N, D, generator=g), "actions": act,
           "logp": -0.5 * act * act - 0.5 * math.log(2 * math.pi) + 0.5, "value": torch.randn(H + 1, N, generator=g),
           "reward": torch.randn(H, N, generator=g), "done": (torch.rand(H, N, generator=g) < 0.15).to(torch.uint8)}
    stats = ppo_update(net, opt, buf, torch.zeros(N, dtype=torch.uint8), dist, epochs=2, minibatches=3)
    flat = torch.cat([p.detach().reshape(-1) for p in net.parameters()])
    q.put((rank, flat.numpy(), float(net.log_std), stats))
    dist.barrier()
    dist.destroy_process_group()


def test_sharded_continuous_ppo_update_over_gloo_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=120) for _ in procs], key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert np.array_equal(res[0][1], res[1][1]), "replicas diverged: the gradient all-reduce did not average"
    torch.manual_seed(0)
    sys.path.insert(0, ROOT)
    from gym_fx_b200.learner import ActorCritic
    init = torch.cat([p.detach().reshape(-1) for p in ActorCritic(20, hidden=16, continuous=True, init_log_std=-0.5).parameters()])
    assert not np.allclose(res[0][1], init.numpy()), "the update did not move the parameters"
    assert res[0][2] != -0.5, "the update did not move log sigma"
    st = res[0][3]
    assert all(math.isfinite(st[k]) for k in ("loss", "entropy", "value_loss"))


def test_library_exports_greedy_rollout():
    from gym_fx_b200 import _native

    _native.build()
    L = _native.load()
    assert hasattr(L, "fxenv_rollout_ex") and "fxenv_rollout_ex" in _native.EXPORTS
    hdr = open(os.path.join(ROOT, "include", "fxenv.h")).read()
    m = re.search(r"#define\s+FXENV_ROLLOUT_GREEDY\s+(\d+)u", hdr)
    assert m and int(m.group(1)) == _native.ROLLOUT_GREEDY
    # a missing env is rejected before anything touches a device
    assert L.fxenv_rollout_ex(None, None, None, 0, None) < 0
