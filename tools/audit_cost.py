#!/usr/bin/env python3
"""Cost of the bracket audit (VecFxEnv.set_bracket_audit) on the ATR workloads of bench.py: the cfg3 and cfg5 shapes run
500-step fxenv_step_many batches with the log off and on (capacity 64, drained with bracket_audit() after every batch),
alternating between the two modes in one process after an untimed pre-roll.  Each batch is timed with CUDA events from
its launch to the end of its drain (log on) or of the batch (log off).  Prints µs/step per mode (median and range over
the repetitions), the share of the drain, and the difference.

Usage: python tools/audit_cost.py [workloads=cfg3,cfg5] [repetitions=5] [batches per repetition=4]"""
import os
import sys

sys.path[:0] = [os.path.dirname(os.path.dirname(os.path.abspath(__file__)))]
import numpy as np
import torch

import bench
from gym_fx_b200.synth import start_offsets
from gym_fx_b200.vec_env import VecFxEnv

K, CAPACITY = 500, 64


def measure(wl, reps, batches):
    cfg, candles, minutes, N, D, _, desc = bench.build_workload(wl)
    env = VecFxEnv(cfg, candles, minutes)
    pre = bench.preroll_steps(cfg)
    env.reset(torch.as_tensor(start_offsets(N, bench.T_BARS, pre + (reps * batches * 2 + 2) * K, 256)))
    gen = torch.Generator(device="cuda").manual_seed(1)
    acts = torch.randint(0, 3, (K, N), dtype=torch.int32, device="cuda", generator=gen)
    slots = max(2, -(-int(bench.l2_bytes(0) * 1.8) // (N * D * 4)))
    ring = torch.empty((slots, N, D), dtype=torch.float32, device="cuda")
    rews = torch.empty((K, N), dtype=torch.float32, device="cuda")
    terms = torch.empty((K, N), dtype=torch.uint8, device="cuda")
    for k0 in range(0, pre, K):                                # windows and scaling statistics full
        n = min(K, pre - k0)
        env.step_many(acts[:n], ring, rews[:n], terms[:n])
    env.step_many(acts, ring, rews, terms)                     # warm-up
    torch.cuda.synchronize()
    per_step = {"off": [], "on": []}
    drain = {"off": [], "on": []}   # the part of a batch's time after its step_many: the drain, spread over its steps
    records = 0
    for _ in range(reps):
        for mode in ("off", "on"):
            env.set_bracket_audit(CAPACITY if mode == "on" else 0)
            times, drains = [], []
            for _ in range(batches):
                e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                e0.record()
                env.step_many(acts, ring, rews, terms)
                e1.record()
                if mode == "on":
                    records += int(env.bracket_audit()["kind"].numel())
                e2.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e2) * 1e3 / K)
                drains.append(e1.elapsed_time(e2) * 1e3 / K)
            per_step[mode].append(float(np.median(times)))
            drain[mode].append(float(np.median(drains)))
    env.close()
    print(desc)
    for mode in ("off", "on"):
        v = per_step[mode]
        print(f"  log {mode:3s}: {np.median(v):8.2f} us/step (range {min(v):.2f}-{max(v):.2f} over {reps} repetitions)")
    print(f"  of which the drain: {np.median(drain['on']):.2f} us/step")
    d = np.median(per_step["on"]) - np.median(per_step["off"])
    print(f"  on - off: {d:+.2f} us/step ({100 * d / np.median(per_step['off']):+.1f} %), "
          f"{records / (reps * batches * K * N):.3f} records per env-step")


if __name__ == "__main__":
    wls = sys.argv[1].split(",") if len(sys.argv) > 1 else ["cfg3", "cfg5"]
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    batches = int(sys.argv[3]) if len(sys.argv) > 3 else 4
    print(torch.cuda.get_device_name(0))
    for wl in wls:
        measure(wl, reps, batches)
