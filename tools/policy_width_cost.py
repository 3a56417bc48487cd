#!/usr/bin/env python3
"""Cost of the policy width in the closed loop: µs per decision of VecFxEnv.rollout at the cfg4 shape of bench.py
(4096 envs, W = 128, horizon 32) for an actor-critic MLP(hidden, hidden) with hidden in {64, 128, 256, 512}, discrete
and continuous actions.

Every (width, mode) runs in every repetition, in turn, in one process: one env per mode (pre-rolled into steady state
with random actions, like bench.py), one policy per width, all graphs captured and warmed before the first timed
rollout.  A repetition of a setting enqueues its rollouts back to back between two CUDA events on the rollout stream
(as bench.py does), and the table shows the median over the repetitions and their range.  The timed rollouts of a
setting replay its cached graph (same buffers and seed).  At the end the same process runs bench.py's closed-loop block (width 256,
discrete) and prints its ms_per_step beside the 256 row, as a check that the two measure the same thing.  The card's
name, power limit and maximum SM clock are read at the start of the same run.

Usage: python tools/policy_width_cost.py [repetitions=3] [rollouts per repetition=5]"""
import os
import subprocess
import sys

sys.path[:0] = [os.path.dirname(os.path.dirname(os.path.abspath(__file__)))]
import numpy as np
import torch

import bench
from gym_fx_b200.synth import start_offsets
from gym_fx_b200.vec_env import VecFxEnv

H = 32
WIDTHS = (64, 128, 256, 512)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "nvidia-smi not available"
    return f"{torch.cuda.get_device_name(0)} ({q.splitlines()[0] if q else '?'})"


def make_env(continuous, reps, batches):
    cfg, candles, minutes, N, D, _, desc = bench.build_workload("cfg4")
    if continuous:
        cfg.action_mode = 1
    env = VecFxEnv(cfg, candles, minutes)
    pre = bench.preroll_steps(cfg)
    need = pre + (reps * (batches + 1) + 2) * H * len(WIDTHS) + 128
    env.reset(torch.as_tensor(start_offsets(N, bench.T_BARS, need, 256)))
    gen = torch.Generator(device="cuda").manual_seed(77)
    pa = (torch.rand((64, N), generator=gen, device="cuda") * 2 - 1) if continuous else \
        torch.randint(0, 3, (64, N), generator=gen, device="cuda", dtype=torch.int32)
    ring = torch.empty((2, N, D), dtype=torch.float32, device="cuda")
    rew, term = torch.empty((64, N), dtype=torch.float32, device="cuda"), torch.empty((64, N), dtype=torch.uint8, device="cuda")
    for _ in range(-(-pre // 64)):                     # episodes into steady state (bench.preroll_steps)
        env.step_many(pa, ring, rew, term)
    return env, N, D, desc


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    batches = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    if not torch.cuda.is_available():
        sys.exit("policy_width_cost.py needs a CUDA device")
    from gym_fx_b200.learner import ActorCritic
    print(card())
    envs, pols, bufs = {}, {}, {}
    desc = N = D = None
    for cont in (False, True):
        envs[cont], N, D, desc = make_env(cont, reps, batches)
        for hid in WIDTHS:
            torch.manual_seed(0)
            pols[(hid, cont)] = envs[cont].make_policy(ActorCritic(D, hidden=hid, continuous=cont).cuda())
    settings = [(hid, cont) for cont in (False, True) for hid in WIDTHS]
    for s in settings:                                   # warm-up: captures each setting's graph, then one replay
        env = envs[s[1]]
        bufs[s] = env.rollout(pols[s], H, seed=2)
        env.rollout(pols[s], H, buffers=bufs[s], seed=2)
    torch.cuda.synchronize()
    per = {s: [] for s in settings}
    for _ in range(reps):
        for s in settings:
            env = envs[s[1]]
            stream = torch.cuda.current_stream()          # VecFxEnv.rollout enqueues on the current stream
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(batches):
                env.rollout(pols[s], H, buffers=bufs[s], seed=2)
            e1.record(stream)
            e1.synchronize()
            per[s].append(e0.elapsed_time(e1) * 1e3 / (batches * H))
    for env in envs.values():
        env.close()
    print(f"{desc} -- closed loop (VecFxEnv.rollout, horizon {H}, {N} envs, obs_dim {D}), us per decision, median of {reps}")
    for cont in (False, True):
        base = np.median(per[(256, cont)])
        for hid in WIDTHS:
            v = per[(hid, cont)]
            print(f"  {'continuous' if cont else 'discrete':10s} hidden {hid:3d}: {np.median(v):7.2f} us/decision "
                  f"(range {min(v):.2f}-{max(v):.2f}, {np.median(v) / base:5.3f} x width 256)")
    blk = bench.closed_loop_block(1000, 0, 1, torch.device("cuda", 0), None)
    b_us = blk["ms_per_step"] * 1e3
    t_us = float(np.median(per[(256, False)]))
    print(f"bench.py closed_loop.ms_per_step in this run: {b_us:.2f} us/step; this tool's discrete 256 row: {t_us:.2f} "
          f"({(t_us / b_us - 1) * 100:+.1f} %)")


if __name__ == "__main__":
    main()
