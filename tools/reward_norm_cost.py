#!/usr/bin/env python3
"""Cost of the reward normalizer (include/fxenv.h fxenv_return_moments; learner.RewardNormalizer.update) at the cfg4
shape of bench.py (4096 envs, W = 128, width-256 discrete policy), for horizons 32 and 128, beside the rollout it
follows.

For each horizon: one env pre-rolled into steady state (as bench.py), one rollout buffer, graphs captured and warmed.
Each repetition times, between CUDA events on the current stream, `rollouts` rollouts back to back, then `calls`
RewardNormalizer.update calls back to back on the last buffer (the scan kernel, the final sum and the torch merge), then
`calls` VecFxEnv.return_moments calls alone (the two kernels and their launch).  Back-to-back calls this small are
bounded by the host's enqueue rate, so a last pass under torch.profiler (after the timed ones) gives the device time of
the two return kernels alone.  The table
shows the median over the repetitions and their range, and the bytes the scan must read (H x N x 5: reward and done;
plus N prev_done, 12 N of carried state read and written).  The card's name, power limit and maximum SM clock are read
at the start of the same run.

Usage: python tools/reward_norm_cost.py [repetitions=7] [rollouts per repetition=5] [update calls per repetition=50]"""
import os
import sys

sys.path[:0] = [os.path.dirname(os.path.abspath(__file__)), os.path.dirname(os.path.dirname(os.path.abspath(__file__)))]
import numpy as np
import torch

import bench
from gym_fx_b200.synth import start_offsets
from gym_fx_b200.vec_env import VecFxEnv
from policy_width_cost import card

HIDDEN = 256
HORIZONS = (32, 128)


def make_env(H, rollouts):
    cfg, candles, minutes, N, D, _, desc = bench.build_workload("cfg4")
    env = VecFxEnv(cfg, candles, minutes)
    pre = bench.preroll_steps(cfg)
    env.reset(torch.as_tensor(start_offsets(N, bench.T_BARS, pre + rollouts * H + 128, 256)))
    gen = torch.Generator(device="cuda").manual_seed(77)
    pa = torch.randint(0, 3, (64, N), generator=gen, device="cuda", dtype=torch.int32)
    ring = torch.empty((2, N, D), dtype=torch.float32, device="cuda")
    rew, term = torch.empty((64, N), dtype=torch.float32, device="cuda"), torch.empty((64, N), dtype=torch.uint8, device="cuda")
    for _ in range(-(-pre // 64)):
        env.step_many(pa, ring, rew, term)
    return env, N, D, desc


def timed(fn, calls):
    stream = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(calls):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / calls   # us per call


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 7
    rollouts = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    calls = int(sys.argv[3]) if len(sys.argv) > 3 else 50
    if not torch.cuda.is_available():
        sys.exit("reward_norm_cost.py needs a CUDA device")
    from gym_fx_b200.learner import ActorCritic, RewardNormalizer
    print(card())
    rows = []
    for H in HORIZONS:
        env, N, D, desc = make_env(H, reps * rollouts + 4)
        torch.manual_seed(0)
        pol = env.make_policy(ActorCritic(D, hidden=HIDDEN).cuda())
        buf = env.rollout(pol, H, seed=2)
        env.rollout(pol, H, buffers=buf, seed=2)
        rn = RewardNormalizer(N).cuda()
        prev = buf["done"][-1].clone()
        for _ in range(3):
            rn.update(env, buf, prev)
        torch.cuda.synchronize()
        ret, seen = rn.ret.clone(), rn.seen.clone()
        scan = lambda: env.return_moments(buf["reward"], buf["done"], prev, ret, seen, rn.gamma, 0.0)
        roll, upd, sc = [], [], []
        for _ in range(reps):
            roll.append(timed(lambda: env.rollout(pol, H, buffers=buf, seed=2), rollouts))
            upd.append(timed(lambda: rn.update(env, buf, prev), calls))
            sc.append(timed(scan, calls))
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(20):
                scan()
            torch.cuda.synchronize()
        dev_us = sum(e.device_time_total for e in prof.key_averages() if "fx_return" in e.key) / 20
        rows.append((H, N, roll, upd, sc, dev_us))
        pol.close()
        env.close()
    cell = lambda v: f"{np.median(v):.1f} ({min(v):.1f}–{max(v):.1f})"
    print(f"{desc}; width {HIDDEN}, discrete; us per call, median of {reps} (range)")
    print("| horizon | envs | bytes read by the scan | return kernels (device) | return_moments | RewardNormalizer.update "
          "| rollout | update / rollout |")
    print("|---|---|---|---|---|---|---|---|")
    for H, N, roll, upd, sc, dev_us in rows:
        mb = (H * N * 5 + N) / 1e6
        print(f"| {H} | {N} | {mb:.2f} MB | {dev_us:.1f} | {cell(sc)} | {cell(upd)} | {cell(roll)} | "
              f"{np.median(upd) / np.median(roll) * 100:.1f} % |")


if __name__ == "__main__":
    main()
