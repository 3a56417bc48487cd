#!/usr/bin/env python3
"""Cost of the time limit (VecFxEnv.set_time_limit): µs per decision with truncation off (the kernels without it), on
with a limit that never fires (the truncation kernels counting decisions), and on with a limit of 500 decisions (every
env is cut once and, the workloads running with auto-reset, takes its reset step), on
  * fxenv_step_many batches of the cfg2, cfg3 and cfg5 workloads of bench.py (random actions, 64 decisions per batch);
  * the closed loop on cfg4 (VecFxEnv.rollout, horizon 32, policy MLP(256, 256) in the loop); the timed rollouts of a
    setting replay its cached graph (same buffers and seed).
A setting is timed over a window of 512 decisions right after it is set (set_time_limit restarts every env's decision
count): 8 step_many batches or 16 rollouts, one CUDA event pair around the whole window, so that "limit 500" holds each
env's cut (decision 500) and reset step (decision 501) at their steady-state rate of one per 500 decisions.  Every
setting runs in every repetition, in turn, in one process after an untimed pre-roll and a warm-up of each setting; each
figure is the median over the repetitions.  The cut restarts every env's episode, whose first window_size decisions emit
padded, cheaper rows: after "limit 500" the pre-roll runs again (untimed, truncation off), so that every window sees
full observation windows.  The steps that ended an episode (codes 1 and 2) are reported.  The card's
name, power limit and maximum SM clock are read at the start of the same run.

Usage: python tools/time_limit_cost.py [parts=cfg2,cfg3,cfg5,loop] [repetitions=3]"""
import os
import sys

sys.path[:0] = [os.path.dirname(os.path.dirname(os.path.abspath(__file__)))]
import numpy as np
import torch

import bench
from gym_fx_b200.synth import start_offsets
from gym_fx_b200.vec_env import VecFxEnv
from repeat_cost import card

KD = 64         # decisions per step_many batch
H = 32          # rollout horizon
WINDOW = 512    # decisions timed per setting and repetition (> the 500-decision limit + its reset step)
SETTINGS = {"off": 0, "never fires": 2**31 - 1, "limit 500": 500}


def report(desc, per, ended):
    print(desc)
    base = np.median(per["off"])
    for s in SETTINGS:
        v = np.median(per[s])
        print(f"  {s:12s} {v:9.2f} us/decision (range {min(per[s]):.2f}-{max(per[s]):.2f})  {v / base:6.3f} x off"
              f"  steps that ended an episode: {ended[s]}")


def measure_step_many(wl, reps):
    batches = WINDOW // KD
    cfg, candles, minutes, N, D, _, desc = bench.build_workload(wl)
    env = VecFxEnv(cfg, candles, minutes)
    pre = bench.preroll_steps(cfg)
    need = pre + (reps + 1) * (WINDOW * len(SETTINGS) + pre) + 64
    env.reset(torch.as_tensor(start_offsets(N, bench.T_BARS, need, 256)))
    gen = torch.Generator(device="cuda").manual_seed(1)
    acts = torch.randint(0, 3, (KD, N), dtype=torch.int32, device="cuda", generator=gen)
    slots = max(2, -(-int(bench.l2_bytes(0) * 1.8) // (N * D * 4)))
    ring = torch.empty((slots, N, D), dtype=torch.float32, device="cuda")
    rews = torch.empty((KD, N), dtype=torch.float32, device="cuda")
    terms = torch.empty((KD, N), dtype=torch.uint8, device="cuda")
    def preroll():                                            # windows and scaling statistics full
        for k0 in range(0, pre, KD):
            n = min(KD, pre - k0)
            env.step_many(acts[:n], ring, rews[:n], terms[:n])
    preroll()
    for m in SETTINGS.values():                               # warm-up of every setting
        env.set_time_limit(m)
        env.step_many(acts, ring, rews, terms)
    torch.cuda.synchronize()
    per = {s: [] for s in SETTINGS}
    ended = {s: 0 for s in SETTINGS}
    for _ in range(reps):
        for s, m in SETTINGS.items():
            env.set_time_limit(m)
            n_end = torch.zeros((), dtype=torch.int64, device="cuda")
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(batches):
                env.step_many(acts, ring, rews, terms)
                n_end += (terms != 0).sum()   # stream-ordered, inside the window (a few µs per 64 decisions)
            e1.record()
            torch.cuda.synchronize()
            per[s].append(e0.elapsed_time(e1) * 1e3 / WINDOW)
            ended[s] += int(n_end)
            if int(n_end):
                env.set_time_limit(0)
                preroll()
    env.close()
    report(f"{desc} -- fxenv_step_many, {KD} decisions per batch", per, ended)


def measure_loop(reps):
    batches = WINDOW // H
    from gym_fx_b200.learner import ActorCritic
    cfg, candles, minutes, N, D, _, desc = bench.build_workload("cfg4")
    env = VecFxEnv(cfg, candles, minutes)
    pre = bench.preroll_steps(cfg)
    need = pre + (reps + 1) * ((WINDOW + 2 * H) * len(SETTINGS) + pre + 64) + 128
    env.reset(torch.as_tensor(start_offsets(N, bench.T_BARS, need, 256)))
    gen = torch.Generator(device="cuda").manual_seed(77)
    pa = torch.randint(0, 3, (64, N), generator=gen, device="cuda", dtype=torch.int32)
    pring = torch.empty((2, N, D), dtype=torch.float32, device="cuda")
    prew, pterm = torch.empty((64, N), dtype=torch.float32, device="cuda"), torch.empty((64, N), dtype=torch.uint8, device="cuda")
    def preroll():
        for _ in range(-(-pre // 64)):
            env.step_many(pa, pring, prew, pterm)
    preroll()
    torch.manual_seed(0)
    net = ActorCritic(D).cuda()
    pol = env.make_policy(net)
    buf = None
    for m in SETTINGS.values():                               # warm-up (captures each setting's graph once)
        env.set_time_limit(m)
        buf = env.rollout(pol, H, buffers=buf, seed=1)
    torch.cuda.synchronize()
    per = {s: [] for s in SETTINGS}
    ended = {s: 0 for s in SETTINGS}
    for _ in range(reps):
        for s, m in SETTINGS.items():
            env.set_time_limit(m)
            # captures the setting's graph (untimed; replayed below): the window then covers decisions 33..544 of the
            # count, the 500-decision cut and its reset step included
            buf = env.rollout(pol, H, buffers=buf, seed=2)
            n_end = torch.zeros((), dtype=torch.int64, device="cuda")
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(batches):
                env.rollout(pol, H, buffers=buf, seed=2)
                n_end += (buf["done"] != 0).sum()
            e1.record()
            torch.cuda.synchronize()
            per[s].append(e0.elapsed_time(e1) * 1e3 / WINDOW)
            ended[s] += int(n_end)
            if int(n_end):
                env.set_time_limit(0)
                preroll()
    env.close()
    report(f"{desc} -- closed loop (VecFxEnv.rollout, horizon {H}, policy MLP({D},256,256))", per, ended)


if __name__ == "__main__":
    parts = sys.argv[1].split(",") if len(sys.argv) > 1 else ["cfg2", "cfg3", "cfg5", "loop"]
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    if not torch.cuda.is_available():
        sys.exit("time_limit_cost.py needs a CUDA device")
    print(card())
    for p in parts:
        if p == "loop":
            measure_loop(reps)
        else:
            measure_step_many(p, reps)
