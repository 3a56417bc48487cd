"""CPU (-m "not gpu"): the reward normalizer (gym_fx_b200/learner.py RewardNormalizer, ppo_update(reward_norm=...))
and the numpy reference of its device scan (tests/reward_norm_ref.py) -- hand-made scans, merges against numpy
float64 statistics of the concatenated returns, state_dict, normalize() against numpy float32, a gloo world of 2 against
one rank over both ranks' returns, and ppo_update / ppo_update_population with normalizers against pre-scaled buffers."""
import copy
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from gym_fx_b200.learner import ActorCritic, RewardNormalizer, ppo_update, ppo_update_population
from reward_norm_ref import return_scan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = 0.9


def _scan1(rew, done, prev=0, ret=0.0, seen=-1, begun=1, gamma=G):
    """one env: the reference scan of columns `rew` / `done`"""
    r = np.asarray(rew, np.float32)[:, None]
    d = np.asarray(done, np.uint8)[:, None]
    R, s, out = return_scan(r, d, np.array([prev], np.uint8), np.array([ret]), np.array([seen]), np.array([begun]),
                            gamma, 0.0)
    return float(R[0]), int(s[0]), out


def test_scan_discounts_and_cuts_at_both_done_codes():
    R, seen, out = _scan1([1.0, 2.0, 3.0], [0, 0, 0], begun=4)
    r1 = 1.0; r2 = r1 * G + 2.0; r3 = r2 * G + 3.0
    assert R == r3 and seen == 4
    np.testing.assert_allclose(out, [r1 + r2 + r3, r1 * r1 + r2 * r2 + r3 * r3, 3])
    for code in (1, 2):   # termination and truncation both end the return; the step after is a reset step
        R, _, out = _scan1([1.0, 2.0, 5.0, 3.0], [0, code, 0, 0], begun=2)
        r2 = 1.0 * G + 2.0
        assert R == 3.0, code                           # reset step 2 skipped, step 3 starts from 0
        np.testing.assert_allclose(out, [1.0 + r2 + 3.0, 1.0 + r2 * r2 + 9.0, 3])


def test_scan_skips_the_first_step_after_prev_done():
    R, _, out = _scan1([7.0, 2.0], [0, 0], prev=1, begun=3)
    assert R == 2.0 and out[2] == 1


def test_scan_carries_across_two_buffers_and_clears_on_an_outside_reset():
    R0, _, out = _scan1([1.0, 2.0, 0.5], [0, 1, 0], begun=2)   # step 2 is a reset step
    assert R0 == 0.0 and out[2] == 2                            # the reset step adds nothing
    R1, s1, _ = _scan1([1.0, 2.0, 4.0], [0, 0, 0], begun=1)
    assert s1 == 1
    R2, s2, out = _scan1([1.0], [0], ret=R1, seen=s1, begun=1)      # no reset in between: carried
    assert R2 == R1 * G + 1.0 and s2 == 1 and out[0] == R2
    R3, s3, _ = _scan1([1.0], [0], ret=R1, seen=s1, begun=2)        # an explicit reset in between: cleared
    assert R3 == 1.0 and s3 == 2
    R4, _, out = _scan1([1.0, 1.0, 1.0], [1, 0, 0], ret=R1, seen=s1, begun=2)  # the new episode began at step 1
    assert R4 == 1.0 and out[0] == (R1 * G + 1.0) + 1.0 and out[2] == 2   # carried into step 0
    R5, _, _ = _scan1([1.0], [0], prev=1, ret=R1, seen=s1, begun=2)  # ... or at its step 0: kept, but step 0 is skipped
    assert R5 == R1


def test_scan_of_several_envs_equals_one_env_at_a_time():
    rng = np.random.default_rng(0)
    H, W = 9, 13
    rew = rng.standard_normal((H, W)).astype(np.float32)
    done = (rng.random((H, W)) < 0.2).astype(np.uint8) * rng.integers(1, 3, (H, W)).astype(np.uint8)
    prev = (rng.random(W) < 0.3).astype(np.uint8)
    ret, seen, begun = rng.standard_normal(W), rng.integers(0, 5, W), rng.integers(0, 8, W)
    R, s, out = return_scan(rew, done, prev, ret, seen, begun, 0.97, 0.25)
    tot = np.zeros(3)
    for j in range(W):
        Rj, sj, oj = return_scan(rew[:, j:j + 1], done[:, j:j + 1], prev[j:j + 1], ret[j:j + 1], seen[j:j + 1],
                                 begun[j:j + 1], 0.97, 0.25)
        assert Rj[0] == R[j] and sj[0] == s[j]
        tot += oj
    np.testing.assert_allclose(out, tot, rtol=1e-13)


def _returns(sizes, seed):
    rng = np.random.default_rng(seed)
    return [3e-3 + 2e-3 * rng.standard_normal(n) for n in sizes]


def _S(rn, R):
    """the sums update_from_moments takes by default: shifted by the running mean"""
    d = R - rn.mean.numpy()[0]
    return torch.tensor([d.sum(), (d * d).sum(), float(len(R))], dtype=torch.float64)


def test_merged_batches_equal_statistics_of_the_concatenation():
    batches = _returns([5, 300, 1, 0, 40], seed=1)
    rn = RewardNormalizer(8)
    for R in batches:
        rn.update_from_moments(_S(rn, R))
    x = np.concatenate(batches)
    assert rn.count.item() == len(x)
    np.testing.assert_allclose(rn.mean.numpy()[0], x.mean(), rtol=1e-12)
    np.testing.assert_allclose(rn.var.numpy()[0], x.var(), rtol=1e-12)
    other = RewardNormalizer(8)                        # sums without a shift give the same statistics
    for R in batches:
        other.update_from_moments(torch.tensor([R.sum(), (R * R).sum(), float(len(R))]), shift=0.0)
    np.testing.assert_allclose(other.var.numpy(), rn.var.numpy(), rtol=1e-9)


def test_before_the_first_update_and_with_an_empty_batch():
    rn = RewardNormalizer(3)
    assert rn.mean.item() == 0.0 and rn.var.item() == 1.0 and rn.count.item() == 0.0
    assert torch.equal(rn.seen, torch.full((3,), -1, dtype=torch.int32)) and not rn.ret.any()
    rn.update_from_moments(torch.zeros(3, dtype=torch.float64))
    assert rn.mean.item() == 0.0 and rn.var.item() == 1.0 and rn.count.item() == 0.0


@pytest.mark.parametrize("clip", [2.0, float("inf")])
def test_normalize_is_the_float32_formula(clip):
    rn = RewardNormalizer(4, clip=clip)
    rn.var.fill_(3.7e-5)
    g = torch.Generator().manual_seed(2)
    r = (torch.randn(6, 50, generator=g) * 2e-2).float()
    got = rn.normalize(r).numpy()
    s = np.float32(1.0 / np.sqrt(3.7e-5 + 1e-8))
    assert rn.scale32().dtype == torch.float32 and rn.scale32().item() == s
    t = r.numpy() * s
    c = np.float32(clip)
    ref = np.where(t < -c, -c, np.where(t > c, c, t))
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    if np.isfinite(clip):
        assert np.abs(got).max() == clip


def test_state_dict_round_trip():
    rn = RewardNormalizer(5, gamma=0.95)
    rn.update_from_moments(_S(rn, _returns([17], seed=3)[0]))
    rn.ret.copy_(torch.arange(5, dtype=torch.float64))
    rn.seen.copy_(torch.arange(5, dtype=torch.int32) + 3)
    sd = rn.state_dict()
    assert set(sd) == {"mean", "var", "count", "ret", "seen"}
    other = RewardNormalizer(5, gamma=0.95)
    other.load_state_dict(sd)
    for k in sd:
        assert torch.equal(getattr(other, k), getattr(rn, k)), k
    assert torch.equal(other.scale32(), rn.scale32())


def test_argument_errors():
    for kw in ({"gamma": 1.5}, {"gamma": -0.1}, {"gamma": float("nan")}, {"clip": 0.0}, {"clip": float("nan")},
               {"eps": 0.0}, {"eps": -1.0}, {"eps": float("inf")}):
        with pytest.raises(ValueError):
            RewardNormalizer(4, **kw)
    for n in (0, -3, 2.5):
        with pytest.raises(ValueError):
            RewardNormalizer(n)
    with pytest.raises(ValueError):
        RewardNormalizer(4).update_from_moments(torch.zeros(2, dtype=torch.float64))

    class _Env:   # the slice checks come before any call into the env
        num_envs = 16
    rn = RewardNormalizer(8)
    for envs in (slice(0, 16), slice(4, 8), slice(0, 16, 2)):
        with pytest.raises(ValueError):
            rn.update(_Env(), {}, torch.zeros(16, dtype=torch.uint8), envs=envs)
    with pytest.raises(ValueError, match="per member"):
        ppo_update_population([ActorCritic(4, hidden=8)] * 2, [None, None], _buffer(2, 4, 4, 0),
                              torch.zeros(4, dtype=torch.uint8), reward_norms=[rn])


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    from gym_fx_b200.learner import RewardNormalizer as RN

    dist.init_process_group("gloo", rank=rank, world_size=world)
    rn = RN(4)
    for b in range(3):   # every rank has its own returns of each batch
        R = _returns([9 + 4 * rank], seed=100 * b + rank)[0]
        rn.update_from_moments(_S(rn, R), dist=dist)
    q.put((rank, rn.mean.numpy(), rn.var.numpy(), rn.count.numpy()))
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_over_gloo_equal_one_rank_over_all_returns():
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
    one = RewardNormalizer(4)
    for b in range(3):
        R = np.concatenate([_returns([9 + 4 * r], seed=100 * b + r)[0] for r in range(2)])
        one.update_from_moments(_S(one, R))
    for rank, mean, var, count in res:
        np.testing.assert_array_equal(count, one.count.numpy())
        np.testing.assert_allclose(mean, one.mean.numpy(), rtol=1e-12)
        np.testing.assert_allclose(var, one.var.numpy(), rtol=1e-12)
    assert np.array_equal(res[0][1], res[1][1]) and np.array_equal(res[0][2], res[1][2]), "ranks disagree"


def _buffer(H, N, D, seed):
    g = torch.Generator().manual_seed(seed)
    return {"obs": torch.randn(H + 1, N, D, generator=g), "actions": torch.randint(0, 3, (H, N), generator=g, dtype=torch.int32),
            "logp": -torch.rand(H, N, generator=g) - 0.5, "value": torch.randn(H + 1, N, generator=g),
            "reward": torch.randn(H, N, generator=g) * 1e-3, "done": (torch.rand(H, N, generator=g) < 0.1).to(torch.uint8)}


def _flat(net):
    return torch.cat([p.detach().reshape(-1) for p in net.parameters()])


def _normalizer(n, seed):
    rn = RewardNormalizer(n, clip=3.0)
    rn.var.fill_(1e-8 * (1 + seed))
    return rn


def test_ppo_update_with_a_reward_normalizer_equals_prescaled_rewards():
    H, N, D = 5, 12, 6
    buf = _buffer(H, N, D, seed=5)
    raw = buf["reward"].clone()
    rn = _normalizer(N, 1)
    stats = copy.deepcopy(rn.state_dict())
    torch.manual_seed(0)
    a = ActorCritic(D, hidden=16)
    b = copy.deepcopy(a)
    oa, ob = torch.optim.Adam(a.parameters(), lr=1e-2), torch.optim.Adam(b.parameters(), lr=1e-2)
    scaled = {**buf, "reward": torch.clamp(buf["reward"] * rn.scale32(), -rn.clip, rn.clip)}
    assert (scaled["reward"].abs() == rn.clip).any()          # the clip is reached
    torch.manual_seed(1)
    sa = ppo_update(a, oa, buf, torch.zeros(N, dtype=torch.uint8), epochs=2, minibatches=3, reward_norm=rn)
    torch.manual_seed(1)
    sb = ppo_update(b, ob, scaled, torch.zeros(N, dtype=torch.uint8), epochs=2, minibatches=3)
    assert torch.equal(_flat(a), _flat(b)) and sa == sb
    assert torch.equal(buf["reward"], raw), "the buffer stays raw"
    assert all(torch.equal(v, stats[k]) for k, v in rn.state_dict().items()), "the update does not change the statistics"


def test_population_update_uses_each_members_normalizer():
    H, M, n, D = 4, 2, 6, 5
    N = M * n
    buf = _buffer(H, N, D, seed=7)
    torch.manual_seed(3)
    nets = [ActorCritic(D, hidden=16) for _ in range(M)]
    refs = [copy.deepcopy(x) for x in nets]
    rns = [_normalizer(n, m) for m in range(M)]
    opts = [torch.optim.Adam(x.parameters(), lr=1e-2) for x in nets]
    ropts = [torch.optim.Adam(x.parameters(), lr=1e-2) for x in refs]
    torch.manual_seed(4)
    ppo_update_population(nets, opts, buf, torch.zeros(N, dtype=torch.uint8), epochs=1, minibatches=2, reward_norms=rns)
    torch.manual_seed(4)
    for m in range(M):
        sl = {k: v[:, m * n:(m + 1) * n] for k, v in buf.items()}
        ppo_update(refs[m], ropts[m], sl, torch.zeros(n, dtype=torch.uint8), epochs=1, minibatches=2, reward_norm=rns[m])
    for m in range(M):
        assert torch.equal(_flat(nets[m]), _flat(refs[m])), f"member {m}"
