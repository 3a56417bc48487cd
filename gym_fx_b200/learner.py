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

Observation normalization (ActorCritic(obs_norm=True), an ObsNormalizer with running per-pair statistics, the
counterpart of SB3's VecNormalize / CleanRL's NormalizeObservation).  The fused kernels normalize the bf16 copy the
policy reads, where the float32 value still exists; the rollout's float32 obs stay raw.  One iteration, statistics k:
    rollout with stats k (set_weights uploaded them)  ->  ppo_update (normalizes the raw obs with stats k, so the
    probability ratio compares like with like)  ->  net.obs_norm.update(env, obs[:H])  ->  set_weights (weights and
    stats k + 1)
A population member updates its own normalizer from its env slice (envs=policy.member_envs(m)).

Reward normalization (RewardNormalizer, the counterpart of SB3's VecNormalize(norm_reward=True) / gymnasium's
NormalizeReward): rewards divided by the running standard deviation of the discounted return and clipped, so that the
critic's targets sit near O(1) whatever the reward plugin, reward_scale, costs or leverage.  The returns are scanned on
the device (VecFxEnv.return_moments), carried per env across rollouts.  One iteration, as in SB3:
    rollout  ->  reward_norm.update(env, buf, prev_done) with this rollout's returns  ->  ppo_update(...,
    reward_norm=reward_norm) (GAE reads the rewards scaled with the updated statistics; the buffer stays raw)
A population member has its own normalizer on its own env slice.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .sharding import allreduce_mean_grads


class ObsNormalizer(nn.Module):
    """Running mean / variance of the observation columns, per currency pair (env i trades pair i % num_pairs), applied
    as y = clamp((x - mean) * rstd, -clip, clip) in float32, rstd = 1 / sqrt(var + eps) -- the formula and the float32
    statistics the fused kernels apply to the policy's bf16 observation (include/fxenv.h fxenv_policy_set_obs_norm), so
    forward() and the kernel agree bit for bit before the bf16 rounding.  A zero-variance column (the first return) maps
    to 0.  Buffers mean / var float64 [P, D] and count float64 [P] go with state_dict; before the first update the
    statistics are mean 0, var 1.  Batches merge by Chan et al.'s parallel algorithm from shifted sums (shift = the
    float32 mean), which add up across ranks with one all-reduce."""

    def __init__(self, obs_dim: int, num_pairs: int = 1, clip: float = 10.0, eps: float = 1e-8):
        super().__init__()
        if not clip > 0.0:
            raise ValueError(f"clip must be > 0 (inf allowed), got {clip}")
        self.obs_dim, self.num_pairs, self.clip, self.eps = int(obs_dim), int(num_pairs), float(clip), float(eps)
        self.register_buffer("mean", torch.zeros(num_pairs, obs_dim, dtype=torch.float64))
        self.register_buffer("var", torch.ones(num_pairs, obs_dim, dtype=torch.float64))
        self.register_buffer("count", torch.zeros(num_pairs, dtype=torch.float64))

    def mean32(self) -> torch.Tensor:
        """float32 [P, D] mean: the shift of the moments and what forward() subtracts"""
        return self.mean.float()

    def rstd32(self) -> torch.Tensor:
        """float32 [P, D] 1 / sqrt(var + eps), formed in float64"""
        return (1.0 / torch.sqrt(self.var + self.eps)).float()

    def forward(self, x: torch.Tensor, pair: torch.Tensor) -> torch.Tensor:
        """x float32 [B, D], pair [B] (each row's pair index) -> the normalized rows, float32"""
        return torch.clamp((x - self.mean32()[pair]) * self.rstd32()[pair], -self.clip, self.clip)

    @torch.no_grad()
    def update_from_moments(self, S: torch.Tensor, counts, dist=None):
        """Merge a batch given by its shifted sums S float64 [P, 2, D] (S[p, 0] = sum (x - mean32[p]), S[p, 1] = sum of
        the squares; VecFxEnv.obs_moments with shift=mean32()) over counts [P] rows per pair.  With torch.distributed
        initialised, S and counts are summed over the ranks first (one all-reduce), so every rank ends with the same
        statistics -- those of all ranks' rows."""
        P, D = self.num_pairs, self.obs_dim
        S = S.to(device=self.mean.device, dtype=torch.float64)
        if tuple(S.shape) != (P, 2, D):
            raise ValueError(f"S must have shape {(P, 2, D)}, got {tuple(S.shape)}")
        n = torch.as_tensor(counts, dtype=torch.float64, device=self.mean.device).reshape(P)
        if dist is not None and dist.is_initialized() and dist.get_world_size() > 1:
            flat = torch.cat([S.reshape(-1), n])
            dist.all_reduce(flat, op=dist.ReduceOp.SUM)
            S, n = flat[:-P].view(P, 2, D), flat[-P:]
        shift = self.mean32().double()
        nb = n.clamp(min=1.0)[:, None]
        mean_b = shift + S[:, 0] / nb
        m2_b = torch.clamp(S[:, 1] - S[:, 0] * S[:, 0] / nb, min=0.0)
        tot = self.count[:, None] + n[:, None]
        delta = mean_b - self.mean
        w = n[:, None] / tot.clamp(min=1.0)
        mean = self.mean + delta * w
        m2 = self.var * self.count[:, None] + m2_b + delta * delta * self.count[:, None] * w
        var = m2 / tot.clamp(min=1.0)
        has = (n > 0)[:, None]
        self.mean.copy_(torch.where(has, mean, self.mean))
        self.var.copy_(torch.where(has, var, self.var))
        self.count.add_(n)

    @torch.no_grad()
    def update(self, env, obs: torch.Tensor, envs: slice = slice(None), dist=None):
        """Merge rollout observations obs float32 [slots, N, D] (e.g. buf["obs"][:H]) of the envs `envs` (a contiguous
        slice: a population member's policy.member_envs(m)) into the statistics, per pair, on the device
        (VecFxEnv.obs_moments)."""
        if env.cfg.num_pairs != self.num_pairs:
            raise ValueError(f"the env has {env.cfg.num_pairs} pairs, the normalizer {self.num_pairs}")
        obs = obs.contiguous()
        e0, e1, _ = envs.indices(env.num_envs)
        S = env.obs_moments(obs, self.mean32().to(env.device).contiguous(), slice(e0, e1))
        P = self.num_pairs
        per_pair = [len(range(e0 + (p - e0) % P, e1, P)) for p in range(P)]
        self.update_from_moments(S, [c * int(obs.shape[0]) for c in per_pair], dist)


class RewardNormalizer(nn.Module):
    """Reward scaling by the running standard deviation of the discounted return, per env slice (one per population
    member): the counterpart of SB3's VecNormalize(norm_reward=True) / gymnasium's NormalizeReward, with CleanRL's
    reward clip.  normalize(r) = clamp(r * float32(1 / sqrt(var + eps)), -clip, clip); the mean is not subtracted.
    Buffers, all in state_dict: mean / var / count float64 [1] (0, 1, 0 before the first update) -- the statistics of
    the returns R_t = gamma R_{t-1} + r_t of every scanned step -- and ret float64 [num_envs] / seen int32 [num_envs]
    (zeros / -1), each env's return carried from one rollout to the next (VecFxEnv.return_moments: cut at every done,
    cleared when the env began an episode outside the scanned rollouts).  Batches merge by Chan et al.'s parallel
    algorithm from shifted sums, which add up across ranks with one all-reduce."""

    def __init__(self, num_envs: int, gamma: float = 0.99, clip: float = 10.0, eps: float = 1e-8):
        super().__init__()
        if isinstance(num_envs, bool) or int(num_envs) != num_envs or num_envs < 1:
            raise ValueError(f"num_envs must be a positive integer, got {num_envs!r}")
        if not 0.0 <= gamma <= 1.0:
            raise ValueError(f"gamma must be in [0, 1], got {gamma}")
        if not clip > 0.0:
            raise ValueError(f"clip must be > 0 (inf allowed), got {clip}")
        if not 0.0 < eps < math.inf:
            raise ValueError(f"eps must be finite and > 0, got {eps}")
        self.num_envs, self.gamma, self.clip, self.eps = int(num_envs), float(gamma), float(clip), float(eps)
        self.register_buffer("mean", torch.zeros(1, dtype=torch.float64))
        self.register_buffer("var", torch.ones(1, dtype=torch.float64))
        self.register_buffer("count", torch.zeros(1, dtype=torch.float64))
        self.register_buffer("ret", torch.zeros(self.num_envs, dtype=torch.float64))
        self.register_buffer("seen", torch.full((self.num_envs,), -1, dtype=torch.int32))

    def scale32(self) -> torch.Tensor:
        """float32 [1] 1 / sqrt(var + eps), formed in float64"""
        return (1.0 / torch.sqrt(self.var + self.eps)).float()

    def normalize(self, reward: torch.Tensor) -> torch.Tensor:
        """the scaled, clipped float32 rewards (any shape)"""
        return torch.clamp(reward * self.scale32(), -self.clip, self.clip)

    @torch.no_grad()
    def update_from_moments(self, S: torch.Tensor, dist=None, shift=None):
        """Merge a batch of returns given by its sums S float64 [3] = (sum (R - shift), sum (R - shift)^2, count);
        shift None means the running mean.  With torch.distributed initialised, S is summed over the ranks first (one
        all-reduce), so every rank ends with the same statistics -- those of all ranks' returns."""
        S = S.to(device=self.mean.device, dtype=torch.float64).reshape(-1)
        if S.numel() != 3:
            raise ValueError(f"S must have 3 elements, got {S.numel()}")
        if dist is not None and dist.is_initialized() and dist.get_world_size() > 1:
            S = S.clone()
            dist.all_reduce(S, op=dist.ReduceOp.SUM)
        s1, s2, n = S[0:1], S[1:2], S[2:3]
        base = self.mean if shift is None else torch.full_like(self.mean, float(shift))
        nb = n.clamp(min=1.0)
        mean_b = base + s1 / nb
        m2_b = torch.clamp(s2 - s1 * s1 / nb, min=0.0)
        tot = self.count + n
        delta = mean_b - self.mean
        w = n / tot.clamp(min=1.0)
        mean = self.mean + delta * w
        m2 = self.var * self.count + m2_b + delta * delta * self.count * w
        var = m2 / tot.clamp(min=1.0)
        has = n > 0
        self.mean.copy_(torch.where(has, mean, self.mean))
        self.var.copy_(torch.where(has, var, self.var))
        self.count.add_(n)

    @torch.no_grad()
    def update(self, env, buf: Dict[str, torch.Tensor], prev_done: torch.Tensor, envs: slice = slice(None), dist=None):
        """Merge the returns of a rollout buffer (VecFxEnv.rollout: its reward and done) of the envs `envs` (a contiguous
        slice of num_envs envs, e.g. a population member's policy.member_envs(m)) into the statistics, on the device and
        without a host synchronisation.  prev_done uint8 [N]: the done of the step before the rollout.  The scan's shift is
        0, not the running mean, because the mean lives on the device and the host would have to wait to read it; in
        float64 the unshifted sums lose about log10(mean^2 / var) of their 16 digits, nothing at the scale of returns."""
        if not isinstance(envs, slice) or envs.step not in (None, 1):
            raise ValueError(f"envs must be a contiguous slice, got {envs!r}")
        e0, e1, _ = envs.indices(env.num_envs)
        if e1 - e0 != self.num_envs:
            raise ValueError(f"the slice has {max(e1 - e0, 0)} envs, the normalizer {self.num_envs}")
        S = env.return_moments(buf["reward"], buf["done"], prev_done, self.ret, self.seen, self.gamma, 0.0, slice(e0, e1))
        self.update_from_moments(S, dist, shift=0.0)


class ActorCritic(nn.Module):
    """Shared-body actor-critic in the layout FusedPolicy.set_weights reads (body[0], body[2], pi, v).
    continuous=True (action_space_mode "continuous"): a Gaussian actor, `pi` = Linear(hidden, 1) gives the mean and the
    parameter `log_std` [1] the state-independent log sigma; forward() then returns (mean [B, 1], value).
    separate=True: separate actor and critic networks -- `body` feeds only `pi`, and `critic_body`, built like `body`,
    feeds `v`, so the value loss does not shape the policy's features (the layout of Stable-Baselines3's and CleanRL's
    PPO).  The fused loop runs it as two networks (VecFxEnv.make_policy infers `separate` from the module).
    obs_norm=True: an ObsNormalizer(obs_dim, num_pairs) `obs_norm` normalizes the observation first (forward needs each
    row's pair then); FusedPolicy.set_weights uploads its statistics with the weights."""

    def __init__(self, obs_dim: int, hidden: int = 256, n_actions: int = 3, continuous: bool = False,
                 init_log_std: float = 0.0, separate: bool = False, obs_norm: bool = False, num_pairs: int = 1):
        super().__init__()
        self.obs_norm = ObsNormalizer(obs_dim, num_pairs) if obs_norm else None
        self.body = nn.Sequential(nn.Linear(obs_dim, hidden), nn.Tanh(), nn.Linear(hidden, hidden), nn.Tanh())
        self.pi = nn.Linear(hidden, 1 if continuous else n_actions)
        self.v = nn.Linear(hidden, 1)
        self.continuous = continuous
        self.separate = separate
        if continuous:
            self.log_std = nn.Parameter(torch.full((1,), float(init_log_std)))
        if separate:
            self.critic_body = nn.Sequential(nn.Linear(obs_dim, hidden), nn.Tanh(), nn.Linear(hidden, hidden), nn.Tanh())

    def forward(self, obs, pair=None):
        if self.obs_norm is not None:
            if pair is None:
                raise ValueError("a normalizing ActorCritic needs each row's pair: forward(obs, pair)")
            obs = self.obs_norm(obs, pair)
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
               gamma: float = 0.99, lam: float = 0.95, timers: Optional[dict] = None, env_offset: int = 0,
               reward_norm: Optional[RewardNormalizer] = None) -> Dict[str, float]:
    """One PPO update from a rollout buffer (VecFxEnv.rollout).  `timers`, if given, receives CUDA-event pairs around the
    collectives under "allreduce" so that the caller can report their share of the update.  Floating-point actions
    (continuous action mode) are scored by the Gaussian actor of ActorCritic(continuous=True).  A net with an
    observation normalizer (net.obs_norm) gets each row's pair, (env_offset + env) % num_pairs: env_offset is the
    handle's index of the buffer's first env (a population member's first env).  reward_norm: GAE reads
    reward_norm.normalize(buf["reward"]) instead of the raw rewards (the buffer and the statistics stay as they are)."""
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
        if reward_norm is not None:
            rew = reward_norm.normalize(rew)
        adv, ret, valid = gae(rew, val, done, prev_done, gamma, lam)
        m, s = timed(lambda: masked_global_mean_std(adv, valid, dist))
        adv = (adv - m) / s
    b_obs = obs[:H].reshape(H * N, D)
    b_act, b_logp = (act.reshape(-1) if continuous else act.reshape(-1).long()), logp_old.reshape(-1)
    b_adv, b_ret, b_valid = adv.reshape(-1), ret.reshape(-1), valid.reshape(-1)
    params = [p for p in net.parameters()]
    norm = getattr(net, "obs_norm", None)
    b_pair = None if norm is None else ((env_offset + torch.arange(N, device=obs.device)) % norm.num_pairs).repeat(H)
    mb = (H * N) // minibatches
    stats = {}
    for _ in range(epochs):
        perm = torch.randperm(H * N, device=obs.device)
        for k in range(minibatches):
            idx = perm[k * mb:(k + 1) * mb]
            w = b_valid[idx]
            wn = w.sum().clamp(min=1.0)
            logits, v = net(b_obs[idx]) if b_pair is None else net(b_obs[idx], b_pair[idx])
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
                          reward_norms=None, **kw) -> List[Dict[str, float]]:
    """One PPO update of every member of a policy population (VecFxEnv.make_policy(members=M)) from one rollout buffer:
    ppo_update(nets[m], opts[m], ...) on member m's envs, the contiguous slice [m N / M, (m + 1) N / M) of every
    buffer's env axis and of prev_done, members in order.  Each member's advantages are normalised over its own envs
    on all ranks.  reward_norms: one RewardNormalizer per member (built for N / M envs), or None.  kw: ppo_update's
    keyword arguments.  Returns one stats dict per member."""
    M = len(nets)
    if M < 1 or len(opts) != M:
        raise ValueError(f"{M} networks and {len(opts)} optimisers: one optimiser per member")
    if reward_norms is not None and len(reward_norms) != M:
        raise ValueError(f"{len(reward_norms)} reward normalizers for {M} members: one per member")
    N = int(buf["reward"].shape[1])
    if N % M:
        raise ValueError(f"{N} envs do not split into {M} equal member slices")
    n = N // M
    return [ppo_update(nets[m], opts[m], {k: v[:, m * n:(m + 1) * n] for k, v in buf.items()},
                       prev_done[m * n:(m + 1) * n], dist, env_offset=m * n,
                       reward_norm=None if reward_norms is None else reward_norms[m], **kw) for m in range(M)]
