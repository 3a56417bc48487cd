#!/usr/bin/env python3
"""Cost of per-env parameters (VecFxEnv.set_env_params): µs per step with the table off (the kernels without
FX_V_PARAMS), on with a uniform table equal to the config (the FX_V_PARAMS kernels reading every env's row), and on with a
heterogeneous table, on
  * cfg2 with only sl_pips / tp_pips varied per env (the LEAN kernels stay in use: fxenv_debug_lean is printed);
  * cfg3 with commission and slippage varied per env (general kernels);
  * the closed loop on cfg4 (VecFxEnv.rollout, horizon 32, policy MLP(256, 256) in the loop), with sl / tp varied and,
    separately, with commission and slippage varied (the cost-randomisation case of examples/ppo_rollout.py); the
    timed rollouts of a setting replay its cached graph (same buffers and seed).
step_many runs batches of 64 random decisions.  A setting is timed over a window of 512 steps right after it is set,
one CUDA event pair around the whole window.  Every setting runs in every repetition, in turn, in one process after an
untimed pre-roll and a warm-up of each setting; each figure is the median over the repetitions.  The card's name, power
limit and maximum SM clock are read at the start of the same run.

Usage: python tools/env_params_cost.py [parts=cfg2,cfg3,loop] [repetitions=5]"""
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
WINDOW = 512    # steps timed per setting and repetition


def settings(cfg, N, vary):
    """name -> keyword arguments of set_env_params (None: the table off)."""
    rng = np.random.default_rng(5)
    uniform = dict(commission=cfg.commission, leverage=cfg.leverage, slippage=cfg.slippage_perc, sl_pips=cfg.sl_pips,
                   tp_pips=cfg.tp_pips, k_sl=cfg.k_sl, k_tp=cfg.k_tp)
    if vary == "sltp":
        het = dict(sl_pips=rng.choice(np.linspace(5, 80, 16), N), tp_pips=rng.choice(np.linspace(5, 80, 16), N))
    else:
        het = dict(commission=rng.uniform(0.0, 1e-4, N), slippage=rng.uniform(0.0, 3e-4, N))
    return {"off": None, "uniform": uniform, f"varied {vary}": het}


def apply(env, kw):
    if kw is None:
        env.set_env_params(None)
    else:
        env.set_env_params(**kw)
    return int(env.L.fxenv_debug_lean(env._h))


def report(desc, per, lean):
    print(desc)
    base = np.median(per["off"])
    for s in per:
        v = np.median(per[s])
        print(f"  {s:16s} {v:9.2f} us/step (range {min(per[s]):.2f}-{max(per[s]):.2f})  {v / base:6.3f} x off  lean={lean[s]}")


def measure_step_many(wl, vary, reps):
    batches = WINDOW // KD
    cfg, candles, minutes, N, D, _, desc = bench.build_workload(wl)
    env = VecFxEnv(cfg, candles, minutes)
    S = settings(cfg, N, vary)
    pre = bench.preroll_steps(cfg)
    need = pre + (reps + 1) * WINDOW * len(S) + 64
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
    lean = {}
    for s, kw in S.items():                                    # warm-up of every setting
        lean[s] = apply(env, kw)
        env.step_many(acts, ring, rews, terms)
    torch.cuda.synchronize()
    per = {s: [] for s in S}
    for _ in range(reps):
        for s, kw in S.items():
            apply(env, kw)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(batches):
                env.step_many(acts, ring, rews, terms)
            e1.record()
            torch.cuda.synchronize()
            per[s].append(e0.elapsed_time(e1) * 1e3 / WINDOW)
    env.close()
    report(f"{desc} -- fxenv_step_many, {KD} decisions per batch", per, lean)


def measure_loop(vary, reps):
    batches = WINDOW // H
    from gym_fx_b200.learner import ActorCritic
    cfg, candles, minutes, N, D, _, desc = bench.build_workload("cfg4")
    env = VecFxEnv(cfg, candles, minutes)
    S = settings(cfg, N, vary)
    pre = bench.preroll_steps(cfg)
    need = pre + (reps + 1) * (WINDOW + H) * len(S) + 128
    env.reset(torch.as_tensor(start_offsets(N, bench.T_BARS, need, 256)))
    gen = torch.Generator(device="cuda").manual_seed(77)
    pa = torch.randint(0, 3, (64, N), generator=gen, device="cuda", dtype=torch.int32)
    pring = torch.empty((2, N, D), dtype=torch.float32, device="cuda")
    prew, pterm = torch.empty((64, N), dtype=torch.float32, device="cuda"), torch.empty((64, N), dtype=torch.uint8, device="cuda")
    for _ in range(-(-pre // 64)):
        env.step_many(pa, pring, prew, pterm)
    torch.manual_seed(0)
    pol = env.make_policy(ActorCritic(D).cuda())
    buf = None
    lean = {}
    for s, kw in S.items():                                    # warm-up (captures each setting's graph once)
        lean[s] = apply(env, kw)
        buf = env.rollout(pol, H, buffers=buf, seed=1)
    torch.cuda.synchronize()
    per = {s: [] for s in S}
    for _ in range(reps):
        for s, kw in S.items():
            apply(env, kw)
            buf = env.rollout(pol, H, buffers=buf, seed=2)     # (re)captures the setting's graph, untimed
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(batches):
                env.rollout(pol, H, buffers=buf, seed=2)
            e1.record()
            torch.cuda.synchronize()
            per[s].append(e0.elapsed_time(e1) * 1e3 / WINDOW)
    env.close()
    report(f"{desc} -- closed loop (VecFxEnv.rollout, horizon {H}, policy MLP({D},256,256))", per, lean)


if __name__ == "__main__":
    parts = sys.argv[1].split(",") if len(sys.argv) > 1 else ["cfg2", "cfg3", "loop"]
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    if not torch.cuda.is_available():
        sys.exit("env_params_cost.py needs a CUDA device")
    print(card())
    for p in parts:
        if p == "loop":
            measure_loop("sltp", reps)
            measure_loop("costs", reps)
        else:
            measure_step_many(p, "sltp" if p == "cfg2" else "costs", reps)
