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
    python examples/ppo_rollout.py --separate-critic --updates 5
    python examples/ppo_rollout.py --randomize-costs 1e-4,3e-4
    python examples/ppo_rollout.py --population 4 --eval-rollouts 2
    python examples/ppo_rollout.py --obs-norm --updates 5
    python examples/ppo_rollout.py --reward-norm --updates 5
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
--max-episode-steps M cuts every episode after M decisions and --truncate-window reports the end of an episode window
(--episode-bars, or the table's end) as a cut instead of an end (VecFxEnv.set_time_limit): the rollout's done codes then
tell truncations (2) from terminations (1), and GAE bootstraps through a truncation from the value of the cut episode's
last observation instead of treating the cut as the end of the market.  Before training, the envs' episodes are
staggered: in 8 groups, each reset after a different number of hold decisions, so that their cuts spread over the run
instead of falling on the same step.  terminated_frac / truncated_frac: the share of the last rollout's steps with each
code.
--randomize-costs COMM_MAX,SLIP_MAX draws each env's commission and slippage uniformly from [0, COMM_MAX] and [0, SLIP_MAX]
before every rollout (VecFxEnv.set_env_params: the values change in place, the rollout graph stays), so that the policy
does not fit one cost model.
--population M trains M policies side by side on one handle (VecFxEnv.make_policy(members=M)): member m, initialised
from seed + m (--seed) with its own optimiser, acts for the m-th contiguous slice of the envs (policy.member_envs(m)),
and one population rollout and one ppo_update_population per update train them all.  The JSON line then also holds
`members`: per member, the last update's stats and the mean total return of its envs' last finished episodes (and,
with --eval-rollouts, its greedy evaluation reward).  --envs must be a multiple of 128 x M.
--obs-norm normalizes the policy's observation with running per-pair statistics (ActorCritic(obs_norm=True),
learner.ObsNormalizer): seeded from the observation reset() returns, updated from every rollout's observations after
the PPO update (each member from its own envs), uploaded with the weights; the fused kernels apply them to the bf16
copy the policy reads.  obs_norm_update_s: the time of one statistics update.
--reward-norm scales the rewards GAE reads by the running standard deviation of the discounted return and clips them
to +-(--reward-clip) (learner.RewardNormalizer, gamma = PPO's): each member's normalizer scans its own envs' returns on
the device after every rollout, and that update's scale applies to the same rollout.  reward_norm_std: sqrt(var) of the
normalizer (a list, one per member, for a population); reward_norm_update_s: the time of one statistics update.  The
reported and evaluation rewards stay raw.
Prints one JSON line: env-steps/s (decisions) of the rollout phase (policy in the loop) and of the whole train loop, and
bars/s of the rollout phase as an upper bound (decisions x K: a step that ends an episode runs fewer bars).
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time

import numpy as np
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
    ap.add_argument("--separate-critic", action="store_true",
                    help="separate actor and critic networks of width --hidden instead of one shared body")
    ap.add_argument("--max-episode-steps", type=int, default=0,
                    help="time limit: an episode is truncated after this many decisions (0: none)")
    ap.add_argument("--truncate-window", action="store_true",
                    help="the end of an episode window is a truncation (bootstrapped), not a termination")
    ap.add_argument("--randomize-costs", default=None, metavar="COMM_MAX,SLIP_MAX",
                    help="draw each env's commission and slippage uniformly from [0, max] before every rollout")
    ap.add_argument("--population", type=int, default=1,
                    help="policies trained side by side, each on its own slice of the envs (1: one policy)")
    ap.add_argument("--seed", type=int, default=0, help="parameter seed (member m of a population: seed + m)")
    ap.add_argument("--obs-norm", action="store_true",
                    help="normalize the policy's observations with running per-pair mean / variance statistics")
    ap.add_argument("--reward-norm", action="store_true",
                    help="scale rewards by the running standard deviation of the discounted return before GAE")
    ap.add_argument("--reward-clip", type=float, default=10.0, help="clip of the scaled rewards (with --reward-norm)")
    args = ap.parse_args()
    continuous = args.action_space == "continuous"
    cost_max = None
    if args.randomize_costs is not None:
        try:
            cost_max = tuple(float(x) for x in args.randomize_costs.split(","))
        except ValueError:
            cost_max = ()
        if len(cost_max) != 2 or not (cost_max[0] >= 0.0 and 0.0 <= cost_max[1] < 1.0):
            ap.error("--randomize-costs takes COMM_MAX,SLIP_MAX with COMM_MAX >= 0 and 0 <= SLIP_MAX < 1")
    if not 0.0 <= args.holdout_frac < 1.0:
        ap.error("--holdout-frac must be in [0, 1)")
    if args.holdout_frac > 0.0 and args.episode_bars <= 0:
        ap.error("--holdout-frac needs --episode-bars (an episode must fit inside its part of the table)")
    if not 1 <= args.action_repeat <= 256:
        ap.error("--action-repeat must be in 1..256")
    if args.max_episode_steps < 0:
        ap.error("--max-episode-steps must be >= 0")
    M = args.population
    if M < 1 or args.envs % (128 * M):
        ap.error("--population must be >= 1, and --envs a multiple of 128 x --population")
    if not args.reward_clip > 0.0:
        ap.error("--reward-clip must be > 0")

    import bench
    from gym_fx_b200.learner import ActorCritic, RewardNormalizer, ppo_update, ppo_update_population
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
    if args.max_episode_steps > 0 or args.truncate_window:
        env.set_time_limit(args.max_episode_steps, truncate_window=args.truncate_window)
        if args.max_episode_steps > 0:
            desc += f", episodes truncated after {args.max_episode_steps} decisions"
        if args.truncate_window:
            desc += ", window ends truncate"
    T, L = bench.T_BARS, args.episode_bars
    truncating = args.max_episode_steps > 0 or args.truncate_window
    stagger = (args.max_episode_steps if args.max_episode_steps > 0 else L) if truncating else 0   # decisions
    split = int(T * (1.0 - args.holdout_frac))       # training bars [0, split), held-out bars [split, T)
    if args.holdout_frac > 0.0:
        if split - L < 0 or T - L < split:
            ap.error("--episode-bars is too long for the training part or the held-out part of the table")
        desc += f", last {args.holdout_frac:g} of the table held out"
        env.set_episode_starts(0, split - L, seed=0x5EED0000 + rank)   # a window [start, start + L) inside training
        env.reset()
    else:
        env.reset(torch.as_tensor(shard_starts(N, rank, world, T, (args.updates + args.eval_rollouts + 2) * H * K + 64 + stagger * K,
                                               256)))
    if stagger > 0:   # group g restarts its episode after (g + 1) / 8 of the stagger: phases 0, 1/8, ... 7/8 of it
        G, n = 8, max(1, stagger // 8)
        hold = torch.zeros((n, N), dtype=env.action_dtype, device=dev)
        ring = torch.empty((2, N, D), dtype=torch.float32, device=dev)
        rews, codes = torch.empty((n, N), dtype=torch.float32, device=dev), torch.empty((n, N), dtype=torch.uint8, device=dev)
        group = torch.arange(N, device=dev) % G
        for g in range(G):
            env.step_many(hold, ring, rews, codes)
            env.reset(mask=group == g)
        del ring, rews, codes
    done_start = env.episode_stats()["episodes_done"].clone()   # the episodes the stagger cut short are not training's

    torch.backends.cuda.matmul.allow_tf32 = True
    nets = []
    for m in range(M):
        torch.manual_seed(args.seed + m)  # identical replicas on every rank
        nets.append(ActorCritic(D, hidden=args.hidden, continuous=continuous, separate=args.separate_critic,
                                obs_norm=args.obs_norm, num_pairs=cfg.num_pairs).to(dev))
    opts = [torch.optim.Adam(n.parameters(), lr=args.lr, eps=1e-5) for n in nets]
    net, opt = nets[0], opts[0]
    member_envs = [slice(m * N // M, (m + 1) * N // M) for m in range(M)]
    if args.obs_norm:   # statistics seeded from the current observation (what reset() returned), each member's own envs
        desc += ", obs-norm (running per-pair statistics)"
        for m in range(M):
            nets[m].obs_norm.update(env, env.obs[None], envs=member_envs[m], dist=dist)
    rnorms = None
    if args.reward_norm:   # gamma: ppo_update's default, the discount of the returns GAE forms
        desc += f", reward-norm (clip {args.reward_clip:g})"
        rnorms = [RewardNormalizer(N // M, clip=args.reward_clip).to(dev) for _ in range(M)]
    policy = env.make_policy(nets if M > 1 else net)
    buf = None
    prev_done = torch.zeros(N, dtype=torch.uint8, device=dev)

    t_roll = t_upd = t_norm = t_rnorm = 0.0
    stats = {}
    member_stats = [{} for _ in range(M)]   # a population: the last update's stats of each member
    cost_rng = np.random.default_rng(0xC057 + rank) if cost_max else None
    if cost_max:
        desc += f", commission ~ U[0, {cost_max[0]:g}] and slippage ~ U[0, {cost_max[1]:g}] per env and rollout"
    for it in range(args.updates):
        if cost_max:   # per-iteration cost randomisation: the table changes in place (outside the timed rollout)
            env.set_env_params(commission=cost_rng.uniform(0.0, cost_max[0], N),
                               slippage=cost_rng.uniform(0.0, cost_max[1], N))
        torch.cuda.synchronize(dev)
        t0 = time.perf_counter()
        buf = env.rollout(policy, H, buffers=buf, seed=1000 * rank + it)
        torch.cuda.synchronize(dev)
        t1 = time.perf_counter()
        if rnorms:   # this rollout's returns first, so that the update scales with statistics that include them
            for m in range(M):
                rnorms[m].update(env, buf, prev_done, envs=member_envs[m], dist=dist)
            torch.cuda.synchronize(dev)
            if it > 0:
                t_rnorm += time.perf_counter() - t1
        if M > 1:
            member_stats = ppo_update_population(nets, opts, buf, prev_done, dist, epochs=args.epochs,
                                                 minibatches=args.minibatches, reward_norms=rnorms)
            stats = {}
        else:
            stats = ppo_update(net, opt, buf, prev_done, dist, epochs=args.epochs, minibatches=args.minibatches,
                               reward_norm=rnorms[0] if rnorms else None)
        prev_done = buf["done"][-1].clone()
        if args.obs_norm:   # after the update, which normalized with the statistics the rollout used
            torch.cuda.synchronize(dev)
            tn = time.perf_counter()
            for m in range(M):
                nets[m].obs_norm.update(env, buf["obs"][:H], envs=member_envs[m], dist=dist)
            torch.cuda.synchronize(dev)
            if it > 0:
                t_norm += time.perf_counter() - tn
        policy.set_weights(nets if M > 1 else net)        # bf16 repack of the two hidden layers (and the statistics)
        torch.cuda.synchronize(dev)
        t2 = time.perf_counter()
        if it > 0:                                        # the first iteration pays one-off set-up costs
            t_roll += t1 - t0
            t_upd += t2 - t1
        d = buf["done"]   # 0 / 1, or the codes 1 = terminated, 2 = truncated with a time limit
        stats.update(mean_reward=float(buf["reward"].mean()), terminated_frac=float((d == 1).float().mean()),
                     truncated_frac=float((d == 2).float().mean()))
        if M > 1:
            for m in range(M):
                member_stats[m]["mean_reward"] = float(buf["reward"][:, policy.member_envs(m)].mean())

    def episode_report(prefix, done_before, envs=slice(None)):
        """Episodes finished since `done_before` and the mean total return / max drawdown of each env's last finished one
        (envs without one are left out), summed / averaged over the ranks; `envs`: only these envs (a member's slice)."""
        ep = {k: v[envs] for k, v in env.episode_stats().items() if k in ("episodes_done", "total_return", "max_drawdown_pct")}
        new = (ep["episodes_done"] - done_before[envs]).double()
        has = (new > 0).double()
        v = torch.stack([new.sum(), has.sum(), (ep["total_return"] * has).sum(), (ep["max_drawdown_pct"] * has).sum()])
        if dist:
            dist.all_reduce(v, op=dist.ReduceOp.SUM)
        n = max(float(v[1]), 1.0)
        return {f"{prefix}_episodes": int(v[0]), f"{prefix}_mean_total_return": float(v[2]) / n if v[1] > 0 else None,
                f"{prefix}_mean_max_drawdown_pct": float(v[3]) / n if v[1] > 0 else None}

    holdout = args.holdout_frac > 0.0
    per_member = range(M) if M > 1 else range(0)   # a population reports each member on its own envs
    members = [dict(s) for s in member_stats]
    if holdout:   # every env into a fresh episode in the held-out tail; the reset records the training episodes it ends
        env.set_episode_starts(split, T - L, seed=0xE7A10000 + rank)
        env.reset()
        stats.update(episode_report("train", done_start))
        done0 = env.episode_stats()["episodes_done"].clone()
    for m in per_member:
        members[m].update(episode_report("train", done_start, policy.member_envs(m)))
    if args.eval_rollouts > 0:   # greedy evaluation of the trained policy (held out: from the fresh episodes)
        rew_sum = torch.zeros(1 + len(per_member), dtype=torch.float64, device=dev)   # all envs, then each member
        for _ in range(args.eval_rollouts):
            buf = env.rollout(policy, H, buffers=buf, deterministic=True)
            r = buf["reward"].double()
            rew_sum[0] += r.mean()
            for m in per_member:
                rew_sum[1 + m] += r[:, policy.member_envs(m)].mean()
        ev = rew_sum / args.eval_rollouts
        if dist:
            dist.all_reduce(ev, op=dist.ReduceOp.SUM)
            ev /= world
        stats["eval_mean_reward"] = float(ev[0])
        for m in per_member:
            members[m]["eval_mean_reward"] = float(ev[1 + m])
        if holdout:
            env.reset()          # records the evaluation episodes still running
            stats.update(episode_report("eval", done0))
            for m in per_member:
                members[m].update(episode_report("eval", done0, policy.member_envs(m)))

    n_it = max(1, args.updates - 1)
    tt = torch.tensor([t_roll, t_upd], dtype=torch.float64, device=dev)
    if dist:
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    t_roll, t_upd = float(tt[0]), float(tt[1])
    if rank == 0:
        steps = N * world * H * n_it
        print(json.dumps({
            "example": "ppo_rollout", "workload": desc, "n_gpus": world, "envs_per_gpu": N, "horizon": H,
            "policy": f"MLP({D},{args.hidden},{args.hidden}) actor-critic, {'separate actor and critic' if args.separate_critic else 'shared body'} "
                      f"({args.action_space} actions), fused wgmma kernel in the rollout, "
                      "torch (tf32) in the update",
            "hidden": args.hidden, "separate_critic": args.separate_critic, "population": M, "rollout_env_steps_per_s": steps / max(t_roll, 1e-9), "rollout_us_per_step": t_roll / (H * n_it) * 1e6,
            "action_repeat": K, "repeat_mode": args.repeat_mode, "randomize_costs": list(cost_max) if cost_max else None,
            "rollout_bars_per_s_upper_bound": steps * K / max(t_roll, 1e-9),
            "train_env_steps_per_s": steps / max(t_roll + t_upd, 1e-9), "update_s": t_upd / n_it,
            "obs_norm": args.obs_norm, "obs_norm_update_s": t_norm / n_it if args.obs_norm else None,
            "obs_norm_finite": all(bool(torch.isfinite(n.obs_norm.mean).all() and torch.isfinite(n.obs_norm.var).all())
                                   for n in nets) if args.obs_norm else None,
            "reward_norm": args.reward_norm, "reward_norm_update_s": t_rnorm / n_it if rnorms else None,
            "reward_norm_std": (None if not rnorms else [math.sqrt(float(r.var)) for r in rnorms] if M > 1
                                else math.sqrt(float(rnorms[0].var))), **stats,
            **({"members": members} if M > 1 else {})}), flush=True)
    env.close()
    if dist:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
