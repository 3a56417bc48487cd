#!/usr/bin/env python3
"""Cost of a policy population in the closed loop, at the cfg4 shape of bench.py (4096 envs, W = 128, horizon 32) with
an actor-critic MLP(256, 256), discrete actions, for M in {1, 2, 8, 32} members:

  (a) population   one handle of 4096 envs and one policy of M members (VecFxEnv.make_policy(members=M)), member m
                   acting for envs [m 4096 / M, (m + 1) 4096 / M); M = 1 is the single policy.  µs per decision.
  (b) handles      the same M networks as M single-policy handles of 4096 / M envs each, rolled out one after the
                   other: what running M policies takes without populations.  µs per decision of all 4096 envs, i.e.
                   the time of the M rollouts divided by the horizon.

Measured like tools/policy_width_cost.py: every setting runs in every repetition, in turn, in one process, all graphs
captured and warmed before the first timed rollout; a repetition enqueues back-to-back rollouts between two CUDA events
on the current stream, and the table shows the median over the repetitions and their range.  At the end the same
process runs bench.py's closed-loop block (the same shape, a single 256-wide policy) and prints its ms_per_step beside
the M = 1 row.  The card's name, power limit and maximum SM clock are read at the start of the same run.

bf16 weight bytes per member at this shape: W1 256 x 960 (obs_dim 900 padded to a multiple of 64) + W2 256 x 256, 0.62 MB;
M members stream M times that through L2 per step.

Usage: python tools/population_cost.py [repetitions=5] [rollouts per repetition=5]"""
import os
import sys

sys.path[:0] = [os.path.dirname(os.path.abspath(__file__)), os.path.dirname(os.path.dirname(os.path.abspath(__file__)))]
import numpy as np
import torch

import bench
from gym_fx_b200.synth import start_offsets
from gym_fx_b200.vec_env import VecFxEnv
from policy_width_cost import H, card

MEMBERS = (1, 2, 8, 32)
HIDDEN = 256


_WORKLOADS = {}


def make_env(n_envs, rollouts):
    """a cfg4 handle of n_envs envs, pre-rolled into steady state with random actions like bench.py, with table room
    for `rollouts` more rollouts of horizon H"""
    if n_envs not in _WORKLOADS:                         # (the synthetic tables are built once per env count)
        _WORKLOADS[n_envs] = bench.build_workload("cfg4", n_envs)
    cfg, candles, minutes, N, D, _, desc = _WORKLOADS[n_envs]
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


def timed(fn, batches):
    stream = torch.cuda.current_stream()                  # VecFxEnv.rollout enqueues on the current stream
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(batches):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (batches * H)


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    batches = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    if not torch.cuda.is_available():
        sys.exit("population_cost.py needs a CUDA device")
    from gym_fx_b200.learner import ActorCritic
    print(card())
    per_env_rollouts = reps * (batches + 1) + 2
    env, N, D, desc = make_env(4096, per_env_rollouts * len(MEMBERS))   # (a): one handle for every M in turn
    nets = []
    for m in range(max(MEMBERS)):
        torch.manual_seed(m)
        nets.append(ActorCritic(D, hidden=HIDDEN).cuda())
    pops, bufs = {}, {}
    for M in MEMBERS:
        pops[M] = env.make_policy(nets[0] if M == 1 else nets[:M])
    handles = {}                                          # (b): M handles of N / M envs, one single policy each
    for M in MEMBERS[1:]:
        handles[M] = []
        for m in range(M):
            h, _, _, _ = make_env(N // M, per_env_rollouts)
            handles[M].append((h, h.make_policy(nets[m]), {}))
    for M in MEMBERS:                                     # warm-up: captures each graph, then one replay
        bufs[M] = env.rollout(pops[M], H, seed=2)
        env.rollout(pops[M], H, buffers=bufs[M], seed=2)
        for h, pol, b in handles.get(M, []):
            h.rollout(pol, H, buffers=b, seed=2)
            h.rollout(pol, H, buffers=b, seed=2)
    torch.cuda.synchronize()

    def pop_run(M):
        return lambda: env.rollout(pops[M], H, buffers=bufs[M], seed=2)

    def handles_run(M):
        return lambda: [h.rollout(pol, H, buffers=b, seed=2) for h, pol, b in handles[M]]

    per = {(k, M): [] for M in MEMBERS for k in ("pop", "handles") if k == "pop" or M > 1}
    for _ in range(reps):
        for M in MEMBERS:
            per[("pop", M)].append(timed(pop_run(M), batches))
            if M > 1:
                per[("handles", M)].append(timed(handles_run(M), batches))
    for M in MEMBERS:
        for h, pol, _ in handles.get(M, []):
            pol.close()
            h.close()
    env.close()
    cell = lambda k, M: f"{np.median(per[(k, M)]):.2f} ({min(per[(k, M)]):.2f}–{max(per[(k, M)]):.2f})"
    base = float(np.median(per[("pop", 1)]))
    print(f"{desc} -- closed loop (VecFxEnv.rollout, horizon {H}, {N} envs, obs_dim {D}, width {HIDDEN}, discrete), "
          f"us per decision of all {N} envs, median of {reps} (range)")
    print("| M | envs per member | member weights (bf16) | (a) population | (a) / M = 1 | (b) M handles in turn | (b) / (a) |")
    print("|---|---|---|---|---|---|---|")
    kp = (D + 63) // 64 * 64
    for M in MEMBERS:
        a = float(np.median(per[("pop", M)]))
        mb = M * (HIDDEN * kp + HIDDEN * HIDDEN) * 2 / 1e6
        b = f"{cell('handles', M)} | {float(np.median(per[('handles', M)])) / a:.2f}" if M > 1 else "(same as (a)) | –"
        print(f"| {M} | {N // M} | {mb:.1f} MB | {cell('pop', M)} | {a / base:.3f} | {b} |")
    blk = bench.closed_loop_block(1000, 0, 1, torch.device("cuda", 0), None)
    b_us = blk["ms_per_step"] * 1e3
    print(f"bench.py closed_loop.ms_per_step in this run: {b_us:.2f} us/step; this tool's M = 1 row: {base:.2f} "
          f"({(base / b_us - 1) * 100:+.1f} %)")


if __name__ == "__main__":
    main()
