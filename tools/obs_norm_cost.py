#!/usr/bin/env python3
"""Cost of the policy's observation normalizer (include/fxenv.h fxenv_policy_set_obs_norm, fxenv_obs_moments):

  (a) rollout   µs per decision of the closed loop (VecFxEnv.rollout, horizon 32, actor-critic MLP(256, 256), discrete)
                without and with a normalizer, at the cfg4 shape (4096 envs, W = 128, 1 pair, obs_dim 900) and the cfg5
                shape (8192 envs, W = 512, 4 pairs, obs_dim 3588).  The two policies run on one handle, alternating
                within every repetition, all graphs captured and warmed before the first timed rollout; a repetition
                enqueues back-to-back rollouts between two CUDA events.  Median over the repetitions and range.
  (b) moments   the two kernels of fxenv_obs_moments over one rollout's observations ([H][N][obs_dim] float32, the
                rows obs[:H] a statistics update reads), timed with CUDA events over many calls; GB/s from the bytes
                read (H x N x obs_dim x 4: every float once; the float64 output and partial sums are below 1 % of
                that), against the H100 SXM data sheet's 3.35 TB/s of HBM3 bandwidth.

The card's name, power limit and maximum SM clock are read at the start of the same run.

Usage: python tools/obs_norm_cost.py [repetitions=7] [rollouts per repetition=5]"""
import os
import sys

sys.path[:0] = [os.path.dirname(os.path.abspath(__file__)), os.path.dirname(os.path.dirname(os.path.abspath(__file__)))]
import numpy as np
import torch

import bench
from gym_fx_b200.synth import start_offsets
from gym_fx_b200.vec_env import VecFxEnv
from policy_width_cost import H, card

HIDDEN = 256
PEAK_GBS = 3350.0


def make_env(name, rollouts):
    cfg, candles, minutes, N, D, _, desc = bench.build_workload(name)
    env = VecFxEnv(cfg, candles, minutes)
    pre = bench.preroll_steps(cfg)
    env.reset(torch.as_tensor(start_offsets(N, bench.T_BARS, pre + rollouts * H + 128, 256)))
    gen = torch.Generator(device="cuda").manual_seed(77)
    pa = torch.randint(0, 3, (64, N), generator=gen, device="cuda", dtype=torch.int32)
    ring = torch.empty((2, N, D), dtype=torch.float32, device="cuda")
    rew, term = torch.empty((64, N), dtype=torch.float32, device="cuda"), torch.empty((64, N), dtype=torch.uint8, device="cuda")
    for _ in range(-(-pre // 64)):
        env.step_many(pa, ring, rew, term)
    return env, cfg, N, D, desc


def timed(fn, calls, per):
    stream = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(calls):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (calls * per)


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 7
    batches = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    if not torch.cuda.is_available():
        sys.exit("obs_norm_cost.py needs a CUDA device")
    from gym_fx_b200.learner import ActorCritic
    print(card())
    rows = []
    for name in ("cfg4", "cfg5"):
        env, cfg, N, D, desc = make_env(name, 2 * reps * (batches + 1) + 4)
        P = int(cfg.num_pairs)
        torch.manual_seed(0)
        plain = ActorCritic(D, hidden=HIDDEN).cuda()
        normed = ActorCritic(D, hidden=HIDDEN, obs_norm=True, num_pairs=P).cuda()
        normed.load_state_dict(plain.state_dict(), strict=False)
        normed.obs_norm.update(env, env.obs[None])       # statistics of the current observation
        pols = {"off": env.make_policy(plain), "on": env.make_policy(normed)}
        bufs = {k: env.rollout(p, H, seed=2) for k, p in pols.items()}
        for k, p in pols.items():
            env.rollout(p, H, buffers=bufs[k], seed=2)
        torch.cuda.synchronize()
        per = {"off": [], "on": []}
        for _ in range(reps):
            for k in ("off", "on"):
                per[k].append(timed(lambda: env.rollout(pols[k], H, buffers=bufs[k], seed=2), batches, H))
        obs = bufs["on"]["obs"][:H]                       # one statistics update's rows
        shift = normed.obs_norm.mean32().cuda().contiguous()
        for _ in range(3):
            env.obs_moments(obs, shift)
        torch.cuda.synchronize()
        calls = 50
        us = [timed(lambda: env.obs_moments(obs, shift), calls, 1) for _ in range(reps)]
        gb = H * N * D * 4 / 1e9
        rows.append((name, desc, N, D, P, per, us, gb))
        for p in pols.values():
            p.close()
        env.close()
    cell = lambda v: f"{np.median(v):.2f} ({min(v):.2f}–{max(v):.2f})"
    print(f"closed loop (VecFxEnv.rollout, horizon {H}, width {HIDDEN}, discrete), us per decision of all envs, median of "
          f"{reps} (range); the two policies alternate in every repetition")
    print("| shape | envs | obs_dim | pairs | without | with normalizer | with / without |")
    print("|---|---|---|---|---|---|---|")
    for name, desc, N, D, P, per, _, _ in rows:
        print(f"| {name} | {N} | {D} | {P} | {cell(per['off'])} | {cell(per['on'])} | "
              f"{np.median(per['on']) / np.median(per['off']):.3f} |")
    print(f"fxenv_obs_moments over one rollout's obs[:{H}] (both kernels), us per call, median of {reps} (range)")
    print("| shape | rows x obs_dim | bytes read | time | GB/s | share of 3.35 TB/s |")
    print("|---|---|---|---|---|---|")
    for name, desc, N, D, P, _, us, gb in rows:
        t = float(np.median(us))
        print(f"| {name} | {H * N} x {D} | {gb * 1e3:.0f} MB | {cell(us)} | {gb / (t * 1e-6):.0f} | "
              f"{gb / (t * 1e-6) / PEAK_GBS * 100:.0f} % |")


if __name__ == "__main__":
    main()
