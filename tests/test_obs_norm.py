"""CPU (-m "not gpu"): the learner side of the observation normalizer (gym_fx_b200/learner.py ObsNormalizer,
ActorCritic(obs_norm=True), ppo_update's pairs) -- batch merges against numpy float64 statistics of the concatenation,
forward() against a numpy float32 evaluation of the kernel's formula, state_dict, a gloo world of 2 against one rank over
all rows, and ppo_update with and without a normalizer."""
import copy
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from gym_fx_b200.learner import ActorCritic, ObsNormalizer, ppo_update, ppo_update_population

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _batches(P, D, sizes, seed):
    """per-pair rows on very different scales (a price-like column near 150, return-like columns near 3e-4, a constant
    column), as [P] lists of float32 arrays per batch"""
    rng = np.random.default_rng(seed)
    loc = rng.uniform(-2.0, 2.0, (P, D)); loc[:, 0] = 150.0 * (1 + np.arange(P))
    scale = rng.uniform(0.1, 3.0, (P, D)); scale[:, 1] = 3e-4; scale[:, 2] = 0.0
    return [[(loc[p] + scale[p] * rng.standard_normal((n, D))).astype(np.float32) for p in range(P)] for n in sizes]


def _moments(norm, rows):
    """what VecFxEnv.obs_moments returns for these rows: float64 shifted sums, shift = the float32 mean"""
    shift = norm.mean32().double().numpy()
    S = np.zeros((norm.num_pairs, 2, norm.obs_dim))
    for p, x in enumerate(rows):
        d = x.astype(np.float64) - shift[p]
        S[p, 0], S[p, 1] = d.sum(0), (d * d).sum(0)
    return torch.from_numpy(S), [len(x) for x in rows]


def test_merged_batches_equal_statistics_of_the_concatenation():
    P, D = 3, 7
    batches = _batches(P, D, [5, 40, 1, 300], seed=1)
    norm = ObsNormalizer(D, P)
    for rows in batches:
        norm.update_from_moments(*_moments(norm, rows))
    for p in range(P):
        x = np.concatenate([b[p] for b in batches]).astype(np.float64)
        assert norm.count[p].item() == len(x)
        np.testing.assert_allclose(norm.mean[p].numpy(), x.mean(0), rtol=1e-12, atol=1e-12 * np.abs(x).max())
        np.testing.assert_allclose(norm.var[p].numpy(), x.var(0), rtol=1e-12, atol=1e-24)
    assert (norm.var[:, 2] == 0).all()


def test_pair_without_rows_keeps_its_statistics():
    norm = ObsNormalizer(4, 2)
    rows = _batches(2, 4, [10], seed=2)[0]
    norm.update_from_moments(*_moments(norm, rows))
    before = norm.mean[1].clone(), norm.var[1].clone()
    S, n = _moments(norm, [rows[0], rows[1][:0]])
    norm.update_from_moments(S, n)
    assert torch.equal(norm.mean[1], before[0]) and torch.equal(norm.var[1], before[1]) and norm.count[1].item() == 10


@pytest.mark.parametrize("clip", [3.0, float("inf")])
def test_forward_is_the_kernel_formula_in_float32(clip):
    P, D, B = 4, 9, 64
    norm = ObsNormalizer(D, P, clip=clip)
    g = torch.Generator().manual_seed(3)
    norm.mean.copy_(torch.randn(P, D, generator=g, dtype=torch.float64) * 5)
    norm.var.copy_(torch.rand(P, D, generator=g, dtype=torch.float64) * 4)
    norm.var[:, 0] = 0.0                                       # a zero-variance column: (x - mean) = 0 -> 0
    x = (torch.randn(B, D, generator=g) * 20).float()
    pair = torch.arange(B) % P
    x[:, 0] = norm.mean32()[pair, 0]
    y = norm(x, pair).numpy()
    m32 = norm.mean.numpy().astype(np.float32)
    r32 = (1.0 / np.sqrt(norm.var.numpy() + 1e-8)).astype(np.float32)
    c = np.float32(clip)
    for p in range(P):
        rows = pair.numpy() == p
        t = (x.numpy()[rows] - m32[p]) * r32[p]               # float32 throughout, one rounding per operation
        ref = np.where(t < -c, -c, np.where(t > c, c, t))
        assert np.array_equal(y[rows].view(np.uint32), ref.view(np.uint32)), f"pair {p}"
    assert (y[:, 0] == 0).all()
    if np.isfinite(clip):
        assert np.abs(y).max() == clip                        # the clip is reached


def test_state_dict_round_trip():
    norm = ObsNormalizer(5, 2, clip=4.0)
    norm.update_from_moments(*_moments(norm, _batches(2, 5, [12], seed=4)[0]))
    net = ActorCritic(5, hidden=8, obs_norm=True, num_pairs=2)
    net.obs_norm.load_state_dict(norm.state_dict())
    sd = net.state_dict()
    assert {"obs_norm.mean", "obs_norm.var", "obs_norm.count"} <= set(sd)
    assert sd["obs_norm.mean"].dtype == torch.float64
    net2 = ActorCritic(5, hidden=8, obs_norm=True, num_pairs=2)
    net2.load_state_dict(sd)
    for k in ("mean", "var", "count"):
        assert torch.equal(getattr(net2.obs_norm, k), getattr(norm, k))
    assert torch.equal(net2.obs_norm.rstd32(), norm.rstd32())


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    from gym_fx_b200.learner import ObsNormalizer as ON

    dist.init_process_group("gloo", rank=rank, world_size=world)
    P, D = 2, 6
    norm = ON(D, P)
    for b in range(3):   # every rank has its own rows of each batch
        rows = _batches(P, D, [7 + rank * 3], seed=100 * b + rank)[0]
        norm.update_from_moments(*_moments(norm, rows), dist=dist)
    q.put((rank, norm.mean.numpy(), norm.var.numpy(), norm.count.numpy()))
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_over_gloo_equal_one_rank_over_all_rows():
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
    P, D = 2, 6
    one = ObsNormalizer(D, P)
    for b in range(3):   # one rank, each batch the union of both ranks' rows
        r0, r1 = (_batches(P, D, [7 + r * 3], seed=100 * b + r)[0] for r in range(2))
        one.update_from_moments(*_moments(one, [np.concatenate([r0[p], r1[p]]) for p in range(P)]))
    for rank, mean, var, count in res:
        np.testing.assert_array_equal(count, one.count.numpy())
        np.testing.assert_allclose(mean, one.mean.numpy(), rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(var, one.var.numpy(), rtol=1e-12, atol=1e-24)
    assert np.array_equal(res[0][1], res[1][1]) and np.array_equal(res[0][2], res[1][2]), "ranks disagree"


def _buffer(H, N, D, seed):
    g = torch.Generator().manual_seed(seed)
    return {"obs": torch.randn(H + 1, N, D, generator=g) * 3 + 1, "actions": torch.randint(0, 3, (H, N), generator=g, dtype=torch.int32),
            "logp": -torch.rand(H, N, generator=g) - 0.5, "value": torch.randn(H + 1, N, generator=g),
            "reward": torch.randn(H, N, generator=g), "done": (torch.rand(H, N, generator=g) < 0.1).to(torch.uint8)}


def _flat(net):
    return torch.cat([p.detach().reshape(-1) for p in net.parameters()])


def test_ppo_update_without_normalizer_ignores_env_offset():
    H, N, D = 5, 12, 8
    buf = _buffer(H, N, D, seed=5)
    torch.manual_seed(0)
    a = ActorCritic(D, hidden=16)
    b = copy.deepcopy(a)
    oa, ob = torch.optim.Adam(a.parameters(), lr=1e-2), torch.optim.Adam(b.parameters(), lr=1e-2)
    torch.manual_seed(1)
    sa = ppo_update(a, oa, buf, torch.zeros(N, dtype=torch.uint8), epochs=2, minibatches=3)
    torch.manual_seed(1)
    sb = ppo_update(b, ob, buf, torch.zeros(N, dtype=torch.uint8), epochs=2, minibatches=3, env_offset=7)
    assert torch.equal(_flat(a), _flat(b)) and sa == sb


def _normalized(buf, norm, offset):
    """the buffer with obs normalized by hand, row (t, env) with pair (offset + env) % P"""
    H1, N, D = buf["obs"].shape
    pair = ((offset + torch.arange(N)) % norm.num_pairs).repeat(H1)
    return {**buf, "obs": norm(buf["obs"].reshape(-1, D), pair).reshape(H1, N, D)}


def _normalizing_net(D, P, seed):
    torch.manual_seed(seed)
    net = ActorCritic(D, hidden=16, obs_norm=True, num_pairs=P)
    g = torch.Generator().manual_seed(seed + 1)
    net.obs_norm.mean.copy_(torch.randn(P, D, generator=g, dtype=torch.float64))
    net.obs_norm.var.copy_(torch.rand(P, D, generator=g, dtype=torch.float64) + 0.2)
    net.obs_norm.clip = 2.0
    return net


@pytest.mark.parametrize("offset", [0, 5])
def test_ppo_update_normalizes_each_row_with_its_pair(offset):
    H, N, D, P = 4, 12, 8, 3
    buf = _buffer(H, N, D, seed=6)
    net = _normalizing_net(D, P, seed=2)
    plain = ActorCritic(D, hidden=16)
    plain.load_state_dict({k: v for k, v in net.state_dict().items() if not k.startswith("obs_norm.")})
    on, op = torch.optim.Adam(net.parameters(), lr=1e-2), torch.optim.Adam(plain.parameters(), lr=1e-2)
    ref_buf = _normalized(buf, net.obs_norm, offset)
    torch.manual_seed(3)
    s1 = ppo_update(net, on, buf, torch.zeros(N, dtype=torch.uint8), epochs=2, minibatches=2, env_offset=offset)
    torch.manual_seed(3)
    s2 = ppo_update(plain, op, ref_buf, torch.zeros(N, dtype=torch.uint8), epochs=2, minibatches=2)
    assert torch.equal(_flat(net), _flat(plain)) and s1 == s2
    assert not any(p is net.obs_norm.mean for p in net.parameters())   # the statistics are buffers, not trained


def test_population_update_offsets_each_member_slice():
    H, M, n, D, P = 3, 2, 6, 5, 4
    N = M * n
    buf = _buffer(H, N, D, seed=7)
    nets = [_normalizing_net(D, P, seed=10 + m) for m in range(M)]
    refs = []
    for m in range(M):
        r = ActorCritic(D, hidden=16)
        r.load_state_dict({k: v for k, v in nets[m].state_dict().items() if not k.startswith("obs_norm.")})
        refs.append(r)
    opts = [torch.optim.Adam(x.parameters(), lr=1e-2) for x in nets]
    ropts = [torch.optim.Adam(x.parameters(), lr=1e-2) for x in refs]
    torch.manual_seed(4)
    ppo_update_population(nets, opts, buf, torch.zeros(N, dtype=torch.uint8), epochs=1, minibatches=2)
    torch.manual_seed(4)
    for m in range(M):
        sl = {k: v[:, m * n:(m + 1) * n] for k, v in buf.items()}
        ppo_update(refs[m], ropts[m], _normalized(sl, nets[m].obs_norm, m * n), torch.zeros(n, dtype=torch.uint8),
                   epochs=1, minibatches=2)
    for m in range(M):
        assert torch.equal(_flat(nets[m]), _flat(refs[m])), f"member {m}"


def test_normalizing_actor_critic_needs_the_pair():
    net = ActorCritic(4, hidden=8, obs_norm=True, num_pairs=2)
    with pytest.raises(ValueError, match="pair"):
        net(torch.zeros(3, 4))
    with pytest.raises(ValueError, match="clip"):
        ObsNormalizer(4, 1, clip=0.0)
