#!/usr/bin/env python3
"""
examples/ppo_rollout.py -- PPO on the device-resident env (SURVEY section 8(f) rank 1; BASELINE configs[3] shape).

One process per GPU.  Each rank owns a shard of envs (gym_fx_b200.VecFxEnv, no collective in the step path) and a
replica of an actor-critic MLP(hidden, hidden) (--hidden 64, 128, 256 or 512; default 256).  A rollout of H steps runs entirely on the device: the fused wgmma policy
kernel and the env step kernel alternate (VecFxEnv.rollout -> fxenv_rollout, a cached CUDA graph of 2H + 2 kernels), the
observations never leave the GPU.  The PPO update is plain torch; gradients are averaged by ONE flat NCCL all-reduce per
minibatch and advantages are normalised with global statistics (gym_fx_b200.learner / gym_fx_b200.sharding).

    python examples/ppo_rollout.py --envs 4096 --horizon 32 --updates 5
    python examples/ppo_rollout.py --envs 4096 --action-space continuous --updates 5 --eval-rollouts 2
    python examples/ppo_rollout.py --envs 4096 --episode-bars 500 --holdout-frac 0.2 --eval-rollouts 2
    python examples/ppo_rollout.py --envs 4096 --action-repeat 5 --repeat-mode hold
    python examples/ppo_rollout.py --hidden 64
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 examples/ppo_rollout.py --envs 4096

--action-space continuous trains a Gaussian actor on the Box(-1, 1) action (thresholded to hold / long / short by the
env); --eval-rollouts K runs K greedy rollouts (argmax / mean action) after training and reports their mean reward.
--episode-bars B cuts the table into episodes of B bars (auto-reset starts the next one).  --holdout-frac F keeps the
last F of every table out of training: training episodes start at bars drawn from the first 1 - F (every auto-reset
draws a new one, VecFxEnv.set_episode_starts), and the greedy evaluation resets every env into the held-out tail.  The
episode records (VecFxEnv.episode_stats) then give, for training and for evaluation, the episodes finished and the mean
total return and maximum drawdown of each env's last finished episode (the reset into the tail, and one after the
evaluation, record the episodes they cut short).
--action-repeat K lets the policy decide once per K bars (VecFxEnv.set_action_repeat): a rollout step is a decision,
GAE runs per decision.  --repeat-mode repeat applies the action on every bar of the step, hold on its first bar only.
Prints one JSON line: env-steps/s (decisions) of the rollout phase (policy in the loop) and of the whole train loop, and
bars/s of the rollout phase as an upper bound (decisions x K: a step that ends an episode runs fewer bars).
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096, help="envs per GPU")
    ap.add_argument("--horizon", type=int, default=32, help="steps per rollout")
    ap.add_argument("--updates", type=int, default=5)
    ap.add_argument("--epochs", type=int, default=2)
    ap.add_argument("--minibatches", type=int, default=4)
    ap.add_argument("--workload", default="cfg4", help="bench.py workload shape (cfg4 = W=128, fixed SL/TP, sharpe)")
    ap.add_argument("--lr", type=float, default=3e-4)
    ap.add_argument("--action-space", choices=("discrete", "continuous"), default="discrete")
    ap.add_argument("--eval-rollouts", type=int, default=0, help="greedy rollouts after training")
    ap.add_argument("--episode-bars", type=int, default=0, help="bars per episode (0: an episode runs to the end of the table)")
    ap.add_argument("--holdout-frac", type=float, default=0.0,
                    help="fraction of every table held out of training for the greedy evaluation (needs --episode-bars)")
    ap.add_argument("--action-repeat", type=int, default=1, help="bars per decision (1..256)")
    ap.add_argument("--repeat-mode", choices=("repeat", "hold"), default="repeat",
                    help="repeat: the action on every bar of a step; hold: on its first bar, then hold")
    ap.add_argument("--hidden", type=int, choices=(64, 128, 256, 512), default=256,
                    help="width of both hidden layers of the actor-critic")
    args = ap.parse_args()
    continuous = args.action_space == "continuous"
    if not 0.0 <= args.holdout_frac < 1.0:
        ap.error("--holdout-frac must be in [0, 1)")
    if args.holdout_frac > 0.0 and args.episode_bars <= 0:
        ap.error("--holdout-frac needs --episode-bars (an episode must fit inside its part of the table)")
    if not 1 <= args.action_repeat <= 256:
        ap.error("--action-repeat must be in 1..256")

    import bench
    from gym_fx_b200.learner import ActorCritic, ppo_update
    from gym_fx_b200.sharding import check_pair_alignment, shard_starts
    from gym_fx_b200.vec_env import VecFxEnv

    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist = None
    if world > 1:
        import torch.distributed as dist_
        dist = dist_
        dist.init_process_group("nccl", device_id=dev)

    cfg, candles, minutes, N, D, _, desc = bench.build_workload(args.workload, args.envs)
    if continuous:
        cfg.action_mode = 1   # FX_ACTION_CONTINUOUS (action_space_mode "continuous")
        desc += ", continuous actions"
    if args.episode_bars > 0:
        cfg.episode_bars = args.episode_bars
        desc += f", episodes of {args.episode_bars} bars"
    env = VecFxEnv(cfg, candles, minutes, device=dev)
    check_pair_alignment(N, cfg.num_pairs)
    H, K = args.horizon, args.action_repeat
    if K > 1:
        env.set_action_repeat(K, hold=args.repeat_mode == "hold")
        desc += f", one decision per {K} bars ({args.repeat_mode})"
    T, L = bench.T_BARS, args.episode_bars
    split = int(T * (1.0 - args.holdout_frac))       # training bars [0, split), held-out bars [split, T)
    if args.holdout_frac > 0.0:
        if split - L < 0 or T - L < split:
            ap.error("--episode-bars is too long for the training part or the held-out part of the table")
        desc += f", last {args.holdout_frac:g} of the table held out"
        env.set_episode_starts(0, split - L, seed=0x5EED0000 + rank)   # a window [start, start + L) inside training
        env.reset()
    else:
        env.reset(torch.as_tensor(shard_starts(N, rank, world, T, (args.updates + args.eval_rollouts + 2) * H * K + 64, 256)))

    torch.backends.cuda.matmul.allow_tf32 = True
    torch.manual_seed(0)  # identical replicas on every rank
    net = ActorCritic(D, hidden=args.hidden, continuous=continuous).to(dev)
    opt = torch.optim.Adam(net.parameters(), lr=args.lr, eps=1e-5)
    policy = env.make_policy(net)
    buf = None
    prev_done = torch.zeros(N, dtype=torch.uint8, device=dev)

    t_roll = t_upd = 0.0
    stats = {}
    for it in range(args.updates):
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        buf = env.rollout(policy, H, buffers=buf, seed=1000 * rank + it)
        torch.cuda.synchronize(dev)
        t1 = time.perf_counter()
        stats = ppo_update(net, opt, buf, prev_done, dist, epochs=args.epochs, minibatches=args.minibatches)
        prev_done = buf["done"][-1].clone()
        policy.set_weights(net)                           # bf16 repack of the two hidden layers for the next rollout
        torch.cuda.synchronize(dev)
        t2 = time.perf_counter()
        if it > 0:                                        # the first iteration pays one-off set-up costs
            t_roll += t1 - t0
            t_upd += t2 - t1
        stats.update(mean_reward=float(buf["reward"].mean()), terminated_frac=float(buf["done"].float().mean()))

    def episode_report(prefix, done_before):
        """Episodes finished since `done_before` and the mean total return / max drawdown of each env's last finished one
        (envs without one are left out), summed / averaged over the ranks."""
        ep = env.episode_stats()
        new = (ep["episodes_done"] - done_before).double()
        has = (new > 0).double()
        v = torch.stack([new.sum(), has.sum(), (ep["total_return"] * has).sum(), (ep["max_drawdown_pct"] * has).sum()])
        if dist:
            dist.all_reduce(v, op=dist.ReduceOp.SUM)
        n = max(float(v[1]), 1.0)
        return {f"{prefix}_episodes": int(v[0]), f"{prefix}_mean_total_return": float(v[2]) / n if v[1] > 0 else None,
                f"{prefix}_mean_max_drawdown_pct": float(v[3]) / n if v[1] > 0 else None}

    holdout = args.holdout_frac > 0.0
    if holdout:   # every env into a fresh episode in the held-out tail; the reset records the training episodes it ends
        env.set_episode_starts(split, T - L, seed=0xE7A10000 + rank)
        env.reset()
        stats.update(episode_report("train", torch.zeros_like(env.episode_stats()["episodes_done"])))
        done0 = env.episode_stats()["episodes_done"].clone()
    if args.eval_rollouts > 0:   # greedy evaluation of the trained policy (held out: from the fresh episodes)
        rew_sum = torch.zeros((), dtype=torch.float64, device=dev)
        for _ in range(args.eval_rollouts):
            buf = env.rollout(policy, H, buffers=buf, deterministic=True)
            rew_sum += buf["reward"].double().mean()
        ev = torch.stack([rew_sum / args.eval_rollouts])
        if dist:
            dist.all_reduce(ev, op=dist.ReduceOp.SUM)
            ev /= world
        stats["eval_mean_reward"] = float(ev[0])
        if holdout:
            env.reset()          # records the evaluation episodes still running
            stats.update(episode_report("eval", done0))

    n_it = max(1, args.updates - 1)
    tt = torch.tensor([t_roll, t_upd], dtype=torch.float64, device=dev)
    if dist:
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    t_roll, t_upd = float(tt[0]), float(tt[1])
    if rank == 0:
        steps = N * world * H * n_it
        print(json.dumps({
            "example": "ppo_rollout", "workload": desc, "n_gpus": world, "envs_per_gpu": N, "horizon": H,
            "policy": f"MLP({D},{args.hidden},{args.hidden}) actor-critic ({args.action_space} actions), fused wgmma kernel in the rollout, "
                      "torch (tf32) in the update",
            "hidden": args.hidden, "rollout_env_steps_per_s": steps / max(t_roll, 1e-9), "rollout_us_per_step": t_roll / (H * n_it) * 1e6,
            "action_repeat": K, "repeat_mode": args.repeat_mode,
            "rollout_bars_per_s_upper_bound": steps * K / max(t_roll, 1e-9),
            "train_env_steps_per_s": steps / max(t_roll + t_upd, 1e-9), "update_s": t_upd / n_it, **stats}), flush=True)
    env.close()
    if dist:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
