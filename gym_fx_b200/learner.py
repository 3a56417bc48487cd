"""
PPO learner glue for the closed loop (BASELINE configs[3]: PPO actor-critic on sharpe_reward envs, NCCL gradient
all-reduce; the MLP is 256 x 256 by default, and the fused loop also runs widths 64, 128 and 512: ActorCritic(hidden=...)).  This is CALLER code of the hot path -- the counterpart of the loop in app/main.py:57-65 for a
learned policy -- written in plain torch (autograd for the backward pass):

    rollout   VecFxEnv.rollout: fused wgmma policy kernel <-> env step kernel, H steps, nothing leaves the device
    update    GAE(lambda) -> global advantage statistics (ONE 3-float all-reduce) -> clipped PPO loss on minibatches,
              gradients averaged across ranks by ONE flat-bucket all-reduce per minibatch (gym_fx_b200.sharding)

Auto-reset semantics (include/fxenv.h, FxConfig.auto_reset): the step AFTER a termination is a reset step -- its action
is ignored, its reward is 0 and its observation jumps to the new episode.  Those transitions carry no learning signal
and are masked out of the advantage statistics and of the loss; `done[t]` cuts the GAE recursion at t.
With a time limit (VecFxEnv.set_time_limit) `done` holds codes: 1 = terminated, 2 = truncated.  A truncation also cuts
the recursion and masks the reset step after it, but its TD target keeps gamma * V(final observation) -- value[t + 1],
the value of the cut episode's last observation -- because the episode did not end in the MDP (Pardo et al., "Time
Limits in Reinforcement Learning", 2018).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .sharding import allreduce_mean_grads


class ActorCritic(nn.Module):
    """Shared-body actor-critic in the layout FusedPolicy.set_weights reads (body[0], body[2], pi, v).
    continuous=True (action_space_mode "continuous"): a Gaussian actor, `pi` = Linear(hidden, 1) gives the mean and the
    parameter `log_std` [1] the state-independent log sigma; forward() then returns (mean [B, 1], value).
    separate=True: separate actor and critic networks -- `body` feeds only `pi`, and `critic_body`, built like `body`,
    feeds `v`, so the value loss does not shape the policy's features (the layout of Stable-Baselines3's and CleanRL's
    PPO).  The fused loop runs it as two networks (VecFxEnv.make_policy infers `separate` from the module)."""

    def __init__(self, obs_dim: int, hidden: int = 256, n_actions: int = 3, continuous: bool = False,
                 init_log_std: float = 0.0, separate: bool = False):
        super().__init__()
        self.body = nn.Sequential(nn.Linear(obs_dim, hidden), nn.Tanh(), nn.Linear(hidden, hidden), nn.Tanh())
        self.pi = nn.Linear(hidden, 1 if continuous else n_actions)
        self.v = nn.Linear(hidden, 1)
        self.continuous = continuous
        self.separate = separate
        if continuous:
            self.log_std = nn.Parameter(torch.full((1,), float(init_log_std)))
        if separate:
            self.critic_body = nn.Sequential(nn.Linear(obs_dim, hidden), nn.Tanh(), nn.Linear(hidden, hidden), nn.Tanh())

    def forward(self, obs):
        h = self.body(obs)
        if self.separate:
            return self.pi(h), self.v(self.critic_body(obs)).squeeze(-1)
        return self.pi(h), self.v(h).squeeze(-1)


HALF_LOG_2PI = 0.5 * math.log(2.0 * math.pi)


def gaussian_log_prob(mean, log_std, x):
    """log N(x; mean, exp(log_std)^2), elementwise."""
    return -0.5 * ((x - mean) * torch.exp(-log_std)) ** 2 - log_std - HALF_LOG_2PI


def gaussian_entropy(log_std):
    """Entropy of N(., exp(log_std)^2): log sigma + (1 + log 2 pi) / 2."""
    return log_std + 0.5 + HALF_LOG_2PI


def gae(reward, value, done, prev_done, gamma: float = 0.99, lam: float = 0.95):
    """-> (advantage [H, N], return [H, N], valid [H, N]).  value is [H + 1, N]; done [H, N] the 0 / 1 flags or the codes
    0 / 1 = terminated / 2 = truncated; prev_done [N] = done flag or code of the step before this rollout (non-zero where
    step 0 is a reset step).  Any non-zero done[t] cuts the recursion at t and masks step t + 1; only a termination
    drops gamma * value[t + 1] from delta_t, a truncation bootstraps from it."""
    H = reward.shape[0]
    adv = torch.zeros_like(reward)
    last = torch.zeros_like(reward[0])
    cut = (done != 0).to(reward.dtype)
    boot = (done != 1).to(reward.dtype)   # 1 - terminated (FXENV_DONE_TERMINATED == 1)
    for t in reversed(range(H)):
        nd = 1.0 - cut[t]
        delta = reward[t] + gamma * value[t + 1] * boot[t] - value[t]
        last = delta + gamma * lam * nd * last
        adv[t] = last
    valid = torch.ones_like(reward)
    valid[0] = 1.0 - (prev_done != 0).to(reward.dtype)
    valid[1:] = 1.0 - cut[:-1]
    return adv, adv + value[:H], valid


def masked_global_mean_std(x, mask, dist=None, eps: float = 1e-8):
    """Mean / std of x over the valid elements of ALL ranks: one all-reduce of [sum, sum of squares, count]."""
    x64, m64 = x.reshape(-1).double(), mask.reshape(-1).double()
    s = torch.stack([(x64 * m64).sum(), (x64 * x64 * m64).sum(), m64.sum()])
    if dist is not None and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(s, op=dist.ReduceOp.SUM)
    n = s[2].clamp(min=1.0)
    mean = s[0] / n
    var = torch.clamp(s[1] / n - mean * mean, min=0.0)
    return mean.to(x.dtype), torch.sqrt(var).to(x.dtype) + eps


def ppo_update(net: ActorCritic, opt, buf: Dict[str, torch.Tensor], prev_done: torch.Tensor, dist=None, *, epochs: int = 1,
               minibatches: int = 4, clip: float = 0.2, vf_coef: float = 0.5, ent_coef: float = 0.01, max_grad_norm: float = 0.5,
               gamma: float = 0.99, lam: float = 0.95, timers: Optional[dict] = None) -> Dict[str, float]:
    """One PPO update from a rollout buffer (VecFxEnv.rollout).  `timers`, if given, receives CUDA-event pairs around the
    collectives under "allreduce" so that the caller can report their share of the update.  Floating-point actions
    (continuous action mode) are scored by the Gaussian actor of ActorCritic(continuous=True)."""
    obs, act, logp_old, val, rew, done = (buf[k] for k in ("obs", "actions", "logp", "value", "reward", "done"))
    H, N = rew.shape
    D = obs.shape[-1]
    continuous = act.is_floating_point()

    def timed(fn):
        if timers is None:
            return fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        timers.setdefault("allreduce", []).append((e0, e1))
        return out

    with torch.no_grad():
        adv, ret, valid = gae(rew, val, done, prev_done, gamma, lam)
        m, s = timed(lambda: masked_global_mean_std(adv, valid, dist))
        adv = (adv - m) / s
    b_obs = obs[:H].reshape(H * N, D)
    b_act, b_logp = (act.reshape(-1) if continuous else act.reshape(-1).long()), logp_old.reshape(-1)
    b_adv, b_ret, b_valid = adv.reshape(-1), ret.reshape(-1), valid.reshape(-1)
    params = [p for p in net.parameters()]
    mb = (H * N) // minibatches
    stats = {}
    for _ in range(epochs):
        perm = torch.randperm(H * N, device=obs.device)
        for k in range(minibatches):
            idx = perm[k * mb:(k + 1) * mb]
            w = b_valid[idx]
            wn = w.sum().clamp(min=1.0)
            logits, v = net(b_obs[idx])
            if continuous:  # logits = the Gaussian mean [mb, 1]
                new_logp = gaussian_log_prob(logits.squeeze(-1), net.log_std, b_act[idx])
            else:
                lp = torch.log_softmax(logits, -1)
                new_logp = lp.gather(1, b_act[idx, None]).squeeze(1)
            ratio = torch.exp(new_logp - b_logp[idx])
            a = b_adv[idx]
            pg = -(torch.min(ratio * a, torch.clamp(ratio, 1 - clip, 1 + clip) * a) * w).sum() / wn
            vloss = (F.mse_loss(v, b_ret[idx], reduction="none") * w).sum() / wn
            if continuous:
                ent = (gaussian_entropy(net.log_std) * w).sum() / wn
            else:
                ent = (-(lp.exp() * lp).sum(-1) * w).sum() / wn
            loss = pg + vf_coef * vloss - ent_coef * ent
            opt.zero_grad(set_to_none=True)
            loss.backward()
            timed(lambda: allreduce_mean_grads(params, dist))   # ONE flat NCCL all-reduce per minibatch
            nn.utils.clip_grad_norm_(params, max_grad_norm)
            opt.step()
            stats = {"loss": loss.detach(), "entropy": ent.detach(), "value_loss": vloss.detach()}
    return {k: float(v) for k, v in stats.items()} | {"valid_frac": float(valid.mean())}


def ppo_update_population(nets, opts, buf: Dict[str, torch.Tensor], prev_done: torch.Tensor, dist=None,
                          **kw) -> List[Dict[str, float]]:
    """One PPO update of every member of a policy population (VecFxEnv.make_policy(members=M)) from one rollout buffer:
    ppo_update(nets[m], opts[m], ...) on member m's envs, the contiguous slice [m N / M, (m + 1) N / M) of every
    buffer's env axis and of prev_done, members in order.  Each member's advantages are normalised over its own envs
    on all ranks.  kw: ppo_update's keyword arguments.  Returns one stats dict per member."""
    M = len(nets)
    if M < 1 or len(opts) != M:
        raise ValueError(f"{M} networks and {len(opts)} optimisers: one optimiser per member")
    N = int(buf["reward"].shape[1])
    if N % M:
        raise ValueError(f"{N} envs do not split into {M} equal member slices")
    n = N // M
    return [ppo_update(nets[m], opts[m], {k: v[:, m * n:(m + 1) * n] for k, v in buf.items()},
                       prev_done[m * n:(m + 1) * n], dist, **kw) for m in range(M)]
