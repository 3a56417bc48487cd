#!/usr/bin/env python3
"""Cost of the action repeat (VecFxEnv.set_action_repeat): µs per decision and µs per bar for k in {1, 2, 4, 8}, in both
modes (repeat: the action on every bar; hold: on the first bar, then hold), on
  * fxenv_step_many batches of the cfg2, cfg3 and cfg5 workloads of bench.py (random actions, 64 decisions per batch);
  * the closed loop on cfg4 (VecFxEnv.rollout, horizon 32, policy MLP(256, 256) in the loop), discrete and continuous;
    the timed rollouts of a setting replay its cached graph (same buffers and seed).
Every setting runs in every repetition, k = 1 first and then the others in turn, in one process after an untimed pre-roll
and a warm-up of each setting.  Batches are timed with CUDA events.  µs per bar is µs per decision / k: a decision runs k
bars unless it ends an episode (the episodes here run to the end of a 2^19-bar table, so only a broke account can end
one); the steps that ended an episode are reported, and where there are any the bar count is an upper bound.  The card's
name, power limit and maximum SM clock are read at the start of the same run.

Usage: python tools/repeat_cost.py [parts=cfg2,cfg3,cfg5,loop] [repetitions=3] [batches per setting=3]"""
import os
import subprocess
import sys

sys.path[:0] = [os.path.dirname(os.path.dirname(os.path.abspath(__file__)))]
import numpy as np
import torch

import bench
from gym_fx_b200.synth import start_offsets
from gym_fx_b200.vec_env import VecFxEnv

KD = 64         # decisions per step_many batch
H = 32          # rollout horizon
SETTINGS = [(1, False)] + [(k, hold) for k in (2, 4, 8) for hold in (False, True)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "nvidia-smi not available"
    return f"{torch.cuda.get_device_name(0)} ({q.splitlines()[0] if q else '?'})"


def report(desc, per_decision, ended):
    print(desc)
    base = np.median(per_decision[(1, False)])
    for s in SETTINGS:
        k, hold = s
        v = np.median(per_decision[s])
        b = v / k
        tag = "k=1" if k == 1 else f"k={k} {'hold' if hold else 'repeat'}"
        print(f"  {tag:10s} {v:9.2f} us/decision (range {min(per_decision[s]):.2f}-{max(per_decision[s]):.2f})"
              f"  {b:8.2f} us/bar ({b / base:5.3f} x k=1)  env-steps that ended an episode: {ended[s]}")


def measure_step_many(wl, reps, batches):
    cfg, candles, minutes, N, D, _, desc = bench.build_workload(wl)
    env = VecFxEnv(cfg, candles, minutes)
    pre = bench.preroll_steps(cfg)
    need = pre + (reps * batches + 1) * KD * sum(k for k, _ in SETTINGS) + 64
    env.reset(torch.as_tensor(start_offsets(N, bench.T_BARS, need, 256)))
    gen = torch.Generator(device="cuda").manual_seed(1)
    acts = torch.randint(0, 3, (KD, N), dtype=torch.int32, device="cuda", generator=gen)
    slots = max(2, -(-int(bench.l2_bytes(0) * 1.8) // (N * D * 4)))
    ring = torch.empty((slots, N, D), dtype=torch.float32, device="cuda")
    rews = torch.empty((KD, N), dtype=torch.float32, device="cuda")
    terms = torch.empty((KD, N), dtype=torch.uint8, device="cuda")
    for k0 in range(0, pre, KD):                               # windows and scaling statistics full
        n = min(KD, pre - k0)
        env.step_many(acts[:n], ring, rews[:n], terms[:n])
    for k, hold in SETTINGS:                                  # warm-up of every setting
        env.set_action_repeat(k, hold)
        env.step_many(acts, ring, rews, terms)
    torch.cuda.synchronize()
    per = {s: [] for s in SETTINGS}
    ended = {s: 0 for s in SETTINGS}
    for _ in range(reps):
        for s in SETTINGS:
            env.set_action_repeat(*s)
            times = []
            for _ in range(batches):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                env.step_many(acts, ring, rews, terms)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1) * 1e3 / KD)
                ended[s] += int(terms.sum())
            per[s].append(float(np.median(times)))
    env.close()
    report(f"{desc} -- fxenv_step_many, {KD} decisions per batch", per, ended)


def measure_loop(reps, batches, continuous):
    from gym_fx_b200.learner import ActorCritic
    cfg, candles, minutes, N, D, _, desc = bench.build_workload("cfg4")
    if continuous:
        cfg.action_mode = 1
        desc += ", continuous actions"
    env = VecFxEnv(cfg, candles, minutes)
    pre = bench.preroll_steps(cfg)
    need = pre + (reps * batches + 2) * H * sum(k for k, _ in SETTINGS) + 128
    env.reset(torch.as_tensor(start_offsets(N, bench.T_BARS, need, 256)))
    gen = torch.Generator(device="cuda").manual_seed(77)
    pa = (torch.rand((64, N), generator=gen, device="cuda") * 2 - 1) if continuous else \
        torch.randint(0, 3, (64, N), generator=gen, device="cuda", dtype=torch.int32)
    pring = torch.empty((2, N, D), dtype=torch.float32, device="cuda")
    prew, pterm = torch.empty((64, N), dtype=torch.float32, device="cuda"), torch.empty((64, N), dtype=torch.uint8, device="cuda")
    for _ in range(-(-pre // 64)):
        env.step_many(pa, pring, prew, pterm)
    del pring
    torch.manual_seed(0)
    net = ActorCritic(D, continuous=continuous).cuda()
    pol = env.make_policy(net)
    buf = None
    for k, hold in SETTINGS:                                  # warm-up (captures each setting's graph once)
        env.set_action_repeat(k, hold)
        buf = env.rollout(pol, H, buffers=buf, seed=1)
    torch.cuda.synchronize()
    per = {s: [] for s in SETTINGS}
    ended = {s: 0 for s in SETTINGS}
    for _ in range(reps):
        for s in SETTINGS:
            env.set_action_repeat(*s)
            buf = env.rollout(pol, H, buffers=buf, seed=2)   # captures the setting's graph (untimed); replayed below
            times = []
            for _ in range(batches):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                env.rollout(pol, H, buffers=buf, seed=2)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1) * 1e3 / H)
                ended[s] += int(buf["done"].sum())
            per[s].append(float(np.median(times)))
    env.close()
    report(f"{desc} -- closed loop (VecFxEnv.rollout, horizon {H}, policy MLP({D},256,256))", per, ended)


if __name__ == "__main__":
    parts = sys.argv[1].split(",") if len(sys.argv) > 1 else ["cfg2", "cfg3", "cfg5", "loop"]
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    batches = int(sys.argv[3]) if len(sys.argv) > 3 else 3
    if not torch.cuda.is_available():
        sys.exit("repeat_cost.py needs a CUDA device")
    print(card())
    for p in parts:
        if p == "loop":
            measure_loop(reps, batches, continuous=False)
            measure_loop(reps, batches, continuous=True)
        else:
            measure_step_many(p, reps, batches)
