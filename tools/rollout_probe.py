#!/usr/bin/env python3
"""Closed-loop timing probe: H-step fxenv_rollout (fused policy kernel <-> env step) on the cfg4 shape; CUDA-event time
per step, with and without the cached graph.  Under `ncu --metrics gpu__time_duration.sum` it gives the per-kernel split.

    python tools/rollout_probe.py [H] [reps] [workload] [envs] [discrete|continuous]"""
import os, sys
sys.path[:0] = [os.path.dirname(os.path.dirname(os.path.abspath(__file__)))]
import torch
import bench
from gym_fx_b200.learner import ActorCritic
from gym_fx_b200.synth import start_offsets
from gym_fx_b200.vec_env import VecFxEnv

H = int(sys.argv[1]) if len(sys.argv) > 1 else 32
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
wl = sys.argv[3] if len(sys.argv) > 3 else "cfg4"
envs = int(sys.argv[4]) if len(sys.argv) > 4 and sys.argv[4] != "-" else None
continuous = len(sys.argv) > 5 and sys.argv[5] == "continuous"
cfg, candles, minutes, N, D, _, desc = bench.build_workload(wl, envs)
if continuous:
    cfg.action_mode = 1   # FX_ACTION_CONTINUOUS: Gaussian actor head, general (non-LEAN) step kernel
    desc += ", continuous actions"
env = VecFxEnv(cfg, candles, minutes)
env.reset(torch.as_tensor(start_offsets(N, bench.T_BARS, 4000, 256)))
torch.manual_seed(0)
net = ActorCritic(D, continuous=continuous).cuda()
pol = env.make_policy(net)
buf = env.rollout(pol, H, seed=0)
for _ in range(10):                      # past the early-episode regime
    env.rollout(pol, H, buffers=buf, seed=1)
torch.cuda.synchronize()
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
ev0.record()
for r in range(reps):
    env.rollout(pol, H, buffers=buf, seed=2 + r)
ev1.record(); torch.cuda.synchronize()
ms = ev0.elapsed_time(ev1) / reps
print(f"{desc}\nrollout H={H}: {ms * 1e3 / H:.2f} us/step ({N * H / (ms * 1e-3) / 1e6:.1f} M env-steps/s), launches {env.launch_count()}")
