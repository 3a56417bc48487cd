"""GPU (-m gpu): the reward normalizer's return scan (include/fxenv.h fxenv_return_moments; VecFxEnv.return_moments,
learner.RewardNormalizer).

  * Three consecutive rollouts scanned against the numpy float64 reference (tests/reward_norm_ref.py), whose `begun` is
    tracked here from the resets the test knows of: carried returns and `seen` bit for bit, the sums within 1e-12 --
    short auto-reset episodes, a time limit (codes 1 and 2), action repeat 3, 2 pairs, discrete and continuous, a
    population of 2 (each member's slice), an unaligned slice, a one-env slice, horizon 1.
  * Clearing: env.reset(mask), set_state to an earlier snapshot and step_many with episode ends between two rollouts;
    envs without a reset carry their return.
  * Two calls give the same bits; NaN rewards outside the slice change nothing; a slice without a valid step leaves the
    statistics alone; RewardNormalizer.update does not synchronise the host.
  * Invalid arguments return FXENV_E_INVALID and leave the handle usable.
  * examples/ppo_rollout.py --reward-norm end to end."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import scenarios as S
from gym_fx_b200.config import lower_config
from gym_fx_b200.learner import ActorCritic, RewardNormalizer
from gym_fx_b200.synth import start_offsets, synth_candles, synth_minutes
from gym_fx_b200.vec_env import VecFxEnv
from reward_norm_ref import return_scan

pytestmark = pytest.mark.gpu

T_BARS = 1500
GAMMA, SHIFT = 0.97, 1e-4


def _env(N, pairs=1, continuous=False, episode_bars=37):
    """short episodes with auto-reset: resets all along every rollout; every env starts with one reset (begun = 1)"""
    cfgd = {**S.DEFAULTS, "window_size": 20, "feature_columns": list(S.OHLCV), "sl_pips": 3.0, "tp_pips": 4.0}
    if continuous:
        cfgd["action_space_mode"] = "continuous"
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, "strategy": "direct_fixed_sltp",
                                       "preprocessor": "feature_window_preprocessor"})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"], preprocessor_plugin=pl["preprocessor"],
                       reward_plugin=pl["reward"], columns=S.OHLCV, num_envs=N, num_pairs=pairs, order_capacity=64,
                       episode_bars=episode_bars)
    cfg.auto_reset = 1
    env = VecFxEnv(cfg, [synth_candles(T_BARS, p) for p in range(pairs)], [synth_minutes(T_BARS)] * pairs)
    env.reset(torch.as_tensor(start_offsets(N, T_BARS, 200, 300)))
    return env


def _policy(env, members=1, continuous=False):
    nets = []
    for m in range(members):
        torch.manual_seed(m)
        nets.append(ActorCritic(env.obs_dim, hidden=64, continuous=continuous).cuda())
    return env.make_policy(nets if members > 1 else nets[0])


class Tracker:
    """the env's episodes begun (as the test knows them) and the done of its last step, plus each slice's carried state"""

    def __init__(self, env, slices):
        N = env.num_envs
        self.env, self.begun, self.prev = env, np.ones(N, np.int64), np.zeros(N, np.uint8)
        self.state = {sl: (torch.zeros(sl[1] - sl[0], dtype=torch.float64, device="cuda"),
                           torch.full((sl[1] - sl[0],), -1, dtype=torch.int32, device="cuda")) for sl in slices}

    def stagger(self, groups=8, steps=5):
        """spread the episodes' phases (they all began together): `groups` rounds of `steps` hold decisions, after round g
        an explicit reset of group g"""
        env, N = self.env, self.env.num_envs
        hold = torch.zeros((steps, N), dtype=env.action_dtype, device="cuda")
        ring = torch.empty((2, N, env.obs_dim), dtype=torch.float32, device="cuda")
        rews, terms = torch.empty((steps, N), dtype=torch.float32, device="cuda"), torch.empty((steps, N), dtype=torch.uint8, device="cuda")
        for g in range(groups):
            env.step_many(hold, ring, rews, terms)
            self.stepped(terms.cpu().numpy())
            self.explicit_reset(np.arange(N) % groups == g)

    def explicit_reset(self, mask):
        self.env.reset(mask=torch.as_tensor(mask))
        self.begun[mask] += 1
        self.prev[mask] = 0

    def stepped(self, done):
        """done uint8 [K, N] of K steps just run: their reset steps began episodes"""
        done = np.asarray(done)
        self.begun += (self.prev != 0).astype(np.int64) + (done[:-1] != 0).sum(0)
        self.prev = done[-1].copy()

    def scan(self, buf, tag):
        """every slice through fxenv_return_moments and the reference; returns {slice: keep} (the carried return kept)"""
        rew, done = buf["reward"], buf["done"]
        r_np, d_np = rew.cpu().numpy(), done.cpu().numpy()
        prev = self.prev
        self.stepped(d_np)
        prev_dev = torch.as_tensor(prev).cuda()
        keeps = {}
        for (e0, e1), (ret, seen) in self.state.items():
            ret0, seen0 = ret.cpu().numpy(), seen.cpu().numpy()
            n_reset = (prev[e0:e1] != 0).astype(np.int64) + (d_np[:-1, e0:e1] != 0).sum(0)
            keeps[(e0, e1)] = self.begun[e0:e1] - n_reset == seen0
            r_ref, s_ref, o_ref = return_scan(r_np[:, e0:e1], d_np[:, e0:e1], prev[e0:e1], ret0, seen0,
                                              self.begun[e0:e1], GAMMA, SHIFT)
            out = self.env.return_moments(rew, done, prev_dev, ret, seen, GAMMA, SHIFT, slice(e0, e1))
            got = out.cpu().numpy()
            where = f"{tag}, envs [{e0}, {e1})"
            assert np.array_equal(ret.cpu().numpy().view(np.int64), r_ref.view(np.int64)), f"{where}: carried returns"
            assert np.array_equal(seen.cpu().numpy(), s_ref), f"{where}: seen != episodes begun"
            assert got[2] == o_ref[2], f"{where}: count"
            np.testing.assert_allclose(got[1], o_ref[1], rtol=1e-12, err_msg=f"{where}: S2")
            np.testing.assert_allclose(got[0], o_ref[0], rtol=1e-12, atol=1e-12 * math.sqrt(o_ref[1] * o_ref[2]),
                                       err_msg=f"{where}: S1")
        return keeps


CASES = {
    "auto-reset": dict(),
    "time limit": dict(limit=20),
    "action repeat 3": dict(repeat=3),
    "2 pairs": dict(pairs=2),
    "continuous": dict(continuous=True),
    "population of 2": dict(members=2),
    "horizon 1": dict(H=1),
}


@pytest.mark.parametrize("case", list(CASES))
def test_three_rollouts_against_the_reference(case):
    c = CASES[case]
    N, H, M = 512, c.get("H", 8), c.get("members", 1)
    env = _env(N, pairs=c.get("pairs", 1), continuous=c.get("continuous", False))
    if "repeat" in c:
        env.set_action_repeat(c["repeat"])
    pol = _policy(env, M, c.get("continuous", False))
    slices = [(0, N), (37, 211), (5, 6)] + [(m * N // M, (m + 1) * N // M) for m in range(M)] * (M > 1)
    tr = Tracker(env, slices)
    tr.stagger()
    if "limit" in c:   # set after the stagger: episodes with fewer bars left than the limit still end by exhaustion (1)
        env.set_time_limit(c["limit"])
    codes = set()
    buf = None
    for k in range(3 if H > 1 else 12):
        buf = env.rollout(pol, H, buffers=buf, seed=k)
        tr.scan(buf, f"{case}, rollout {k}")
        codes |= set(np.unique(buf["done"].cpu().numpy()).tolist())
    assert 0 in codes and 1 in codes
    if "limit" in c:
        assert 2 in codes, "the time limit truncated nothing"
    env.close()


def test_resets_between_rollouts_clear_exactly_those_envs():
    N, H = 256, 8
    env = _env(N)
    pol = _policy(env)
    tr = Tracker(env, [(0, N), (3, 100)])
    tr.stagger()
    buf = env.rollout(pol, H, seed=0)
    tr.scan(buf, "first")
    # explicit reset of a mask
    mask = np.zeros(N, bool); mask[::5] = True
    tr.explicit_reset(mask)
    buf = env.rollout(pol, H, buffers=buf, seed=1)
    keep = tr.scan(buf, "after reset(mask)")[(0, N)]
    assert np.array_equal(keep, ~mask), "explicit reset: cleared exactly the masked envs"
    # set_state to a snapshot taken before a rollout that had resets
    snap, begun_snap, prev_snap = env.get_state(), tr.begun.copy(), tr.prev.copy()
    buf = env.rollout(pol, 24, seed=2)
    tr.scan(buf, "before restore")
    rewound = tr.begun != begun_snap
    assert rewound.any() and not rewound.all()
    env.set_state(snap)
    tr.begun, tr.prev = begun_snap.copy(), prev_snap.copy()
    buf = env.rollout(pol, H, seed=3)
    keep = tr.scan(buf, "after set_state")[(0, N)]
    assert not keep[rewound].any(), "a restore past a reset clears"
    assert keep[~rewound].all(), "envs without a reset since the snapshot carry their return"
    # step_many with episode ends
    K = 12
    acts = torch.randint(0, 3, (K, N), dtype=torch.int32, device="cuda", generator=torch.Generator("cuda").manual_seed(4))
    ring = torch.empty((2, N, env.obs_dim), dtype=torch.float32, device="cuda")
    rews, terms = torch.empty((K, N), dtype=torch.float32, device="cuda"), torch.empty((K, N), dtype=torch.uint8, device="cuda")
    env.step_many(acts, ring, rews, terms)
    before = tr.begun.copy()
    tr.stepped(terms.cpu().numpy())
    began = tr.begun != before
    assert began.any() and not began.all()
    buf = env.rollout(pol, H, seed=5)
    keep = tr.scan(buf, "after step_many")[(0, N)]
    assert not keep[began].any() and keep[~began].all()
    env.close()


def test_determinism_isolation_and_empty_slices():
    N, H = 384, 8
    env = _env(N)
    pol = _policy(env)
    buf = env.rollout(pol, H, seed=1)
    prev = torch.zeros(N, dtype=torch.uint8, device="cuda")
    e0, e1 = 64, 200
    fresh = lambda: (torch.zeros(e1 - e0, dtype=torch.float64, device="cuda"),
                     torch.full((e1 - e0,), -1, dtype=torch.int32, device="cuda"))
    (r1, s1), (r2, s2), (r3, s3) = fresh(), fresh(), fresh()
    a = env.return_moments(buf["reward"], buf["done"], prev, r1, s1, GAMMA, SHIFT, slice(e0, e1))
    b = env.return_moments(buf["reward"], buf["done"], prev, r2, s2, GAMMA, SHIFT, slice(e0, e1))
    nan = buf["reward"].clone()
    nan[:, :e0] = float("nan")
    nan[:, e1:] = float("nan")
    c = env.return_moments(nan, buf["done"], prev, r3, s3, GAMMA, SHIFT, slice(e0, e1))
    torch.cuda.synchronize()
    for o, r, s in ((b, r2, s2), (c, r3, s3)):
        assert torch.equal(o.view(torch.int64), a.view(torch.int64))
        assert torch.equal(r.view(torch.int64), r1.view(torch.int64)) and torch.equal(s, s1)
    assert a[2].item() > 0 and torch.isfinite(a).all()
    # RewardNormalizer.update: no host synchronisation; a slice with no valid step leaves the statistics alone
    rn = RewardNormalizer(e1 - e0, gamma=GAMMA).cuda()
    torch.cuda.set_sync_debug_mode("error")
    try:
        rn.update(env, buf, prev, envs=slice(e0, e1))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    stats = [t.clone() for t in (rn.mean, rn.var, rn.count)]
    assert stats[2].item() == a[2].item()
    one = {"reward": buf["reward"][:1].contiguous(), "done": buf["done"][:1].contiguous()}
    rn.update(env, one, torch.ones(N, dtype=torch.uint8, device="cuda"), envs=slice(e0, e1))   # step 0 is a reset step
    for t, before in zip((rn.mean, rn.var, rn.count), stats):
        assert torch.equal(t, before)
    env.close()


def test_invalid_arguments_leave_the_handle_usable():
    N, H = 256, 4
    env = _env(N)
    pol = _policy(env)
    tr = Tracker(env, [(0, N)])
    buf = env.rollout(pol, H, seed=1)
    tr.scan(buf, "before errors")
    prev = torch.zeros(N, dtype=torch.uint8, device="cuda")
    ret, seen = torch.zeros(N, dtype=torch.float64, device="cuda"), torch.full((N,), -1, dtype=torch.int32, device="cuda")
    out = torch.empty(3, dtype=torch.float64, device="cuda")
    L, s = env.L, env._stream()
    p = [buf["reward"].data_ptr(), buf["done"].data_ptr(), prev.data_ptr()]
    good = dict(H=H, e0=0, e1=N, g=GAMMA, sh=SHIFT)
    bad = [dict(H=0), dict(e0=5, e1=5), dict(e0=-1), dict(e1=N + 1), dict(g=1.5), dict(g=-0.1), dict(g=float("nan")),
           dict(sh=float("inf")), dict(sh=float("nan"))]
    for b in bad:
        a = {**good, **b}
        rc = L.fxenv_return_moments(env._h, *p, a["H"], a["e0"], a["e1"], a["g"], a["sh"], ret.data_ptr(), seen.data_ptr(),
                                    out.data_ptr(), s)
        assert rc == -1, b
    for k in range(3):
        q = list(p); q[k] = None
        assert L.fxenv_return_moments(env._h, *q, H, 0, N, GAMMA, SHIFT, ret.data_ptr(), seen.data_ptr(), out.data_ptr(), s) == -1
    assert L.fxenv_return_moments(env._h, *p, H, 0, N, GAMMA, SHIFT, None, seen.data_ptr(), out.data_ptr(), s) == -1
    assert b"NULL" in L.fxenv_last_error(env._h) or b"null" in L.fxenv_last_error(env._h)
    with pytest.raises(ValueError):
        env.return_moments(buf["reward"], buf["done"], prev, ret[:10], seen, GAMMA, SHIFT)
    with pytest.raises(ValueError):
        env.return_moments(buf["reward"], buf["done"], prev, ret, seen, 2.0, SHIFT)
    assert torch.equal(seen, torch.full((N,), -1, dtype=torch.int32, device="cuda")), "a rejected call wrote nothing"
    buf = env.rollout(pol, H, buffers=buf, seed=2)
    tr.scan(buf, "after errors")
    env.close()


@pytest.mark.parametrize("extra", [[], ["--population", "2", "--obs-norm", "--max-episode-steps", "20", "--truncate-window"]])
def test_ppo_example_with_reward_norm(extra):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, os.path.join(root, "examples", "ppo_rollout.py"), "--reward-norm", "--envs", "256", "--horizon", "8",
           "--updates", "3"] + extra
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert line["reward_norm"] and "reward-norm" in line["workload"] and line["reward_norm_update_s"] > 0, line
    std = line["reward_norm_std"]
    stds = std if isinstance(std, list) else [std]
    assert len(stds) == (2 if extra else 1) and all(math.isfinite(x) and x > 0 for x in stds), line
    losses = [line["loss"], line["value_loss"]] if not extra else [m[k] for m in line["members"] for k in ("loss", "value_loss")]
    assert all(math.isfinite(x) for x in losses), line
