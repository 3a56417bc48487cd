"""GPU (-m gpu): the closed loop -- fused wgmma policy kernel + env step (fxenv_rollout, SURVEY 8f #1).

The policy kernel (gym_fx_b200/csrc/fx_policy.cu) is compared with a plain PyTorch fp32 reference of the same MLP:
  * against the SAME arithmetic contract evaluated in torch (bf16-rounded observation / weights / hidden activations,
    fp32 accumulation): value and log-prob to 2e-3 absolute, identical actions wherever the Gumbel-max margin exceeds the
    numerical noise;
  * against the pure fp32 MLP: rtol 1e-2-level agreement (the bf16 tolerance north_star allows for this tier);
and the env side of the rollout (observations, rewards, done flags, final account state) must be IDENTICAL to stepping a
twin env with the recorded actions through fxenv_step."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import scenarios as S
from policy_ref import forward_ref
from gym_fx_b200.config import lower_config
from gym_fx_b200.synth import start_offsets, synth_candles, synth_minutes

pytestmark = pytest.mark.gpu


class ActorCritic(nn.Module):
    def __init__(self, obs_dim, hidden=256):
        super().__init__()
        self.body = nn.Sequential(nn.Linear(obs_dim, hidden), nn.Tanh(), nn.Linear(hidden, hidden), nn.Tanh())
        self.pi = nn.Linear(hidden, 3)
        self.v = nn.Linear(hidden, 1)


def _env(N, W=128, strategy="direct_fixed_sltp", reward="pnl_reward", T=6000, **kw):
    from gym_fx_b200.vec_env import VecFxEnv
    cfgd = {**S.DEFAULTS, "window_size": W, "feature_columns": list(S.OHLCV)}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, "strategy": strategy, "reward": reward,
                                       "preprocessor": "feature_window_preprocessor"})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"], preprocessor_plugin=pl["preprocessor"],
                       reward_plugin=pl["reward"], columns=S.OHLCV, num_envs=N, order_capacity=256, **kw)
    candles, minutes = [synth_candles(T, 0)], [synth_minutes(T)]
    return cfg, candles, minutes, (lambda: VecFxEnv(cfg, candles, minutes))


def _ref_forward(net, obs, emulate_bf16):
    """-> logits [N,3], value [N] in fp32; emulate_bf16: the kernel's arithmetic contract (policy_ref.forward_ref),
    else the pure fp32 MLP."""
    if emulate_bf16:
        r = forward_ref(net, obs)
        return r["head"].float(), r["value"].float()
    w1, b1, w2, b2 = net.body[0].weight, net.body[0].bias, net.body[2].weight, net.body[2].bias
    h1 = torch.tanh(obs.double() @ w1.double().T + b1.double()).float()
    h2 = torch.tanh(h1.double() @ w2.double().T + b2.double()).float()
    logits = (h2.double() @ net.pi.weight.double().T + net.pi.bias.double()).float()
    value = (h2.double() @ net.v.weight.double().T + net.v.bias.double()).float().squeeze(-1)
    return logits, value


@pytest.mark.parametrize("N,H,tile_sync", [(512, 6, 0), (100, 4, 1), (4096, 3, 0), (4096, 5, 1)])
def test_rollout_policy_matches_torch_reference_and_env_matches_single_steps(N, H, tile_sync, monkeypatch):
    # tile_sync: the experimental per-tile hand-over between the policy and the step kernel (FXENV_TILE_SYNC, fx_kernels.cuh
    # FxTileSync) must give the same results as plain kernel order
    monkeypatch.setenv("FXENV_TILE_SYNC", str(tile_sync))
    torch.manual_seed(N)
    cfg, candles, minutes, make = _env(N)
    env, twin = make(), make()
    starts = torch.as_tensor(start_offsets(N, 6000, 400, 300))
    env.reset(starts); twin.reset(starts)
    # a few steps first so that positions / orders / non-trivial agent scalars exist
    warm = torch.randint(0, 3, (30, N), dtype=torch.int32, generator=torch.Generator().manual_seed(1)).cuda()
    for k in range(30):
        env.step(warm[k]); twin.step(warm[k])
    net = ActorCritic(env.obs_dim).cuda()
    with torch.no_grad():   # larger-than-default weights: logits that actually discriminate
        for p in net.parameters():
            p.mul_(2.0)
    pol = env.make_policy(net)
    gum = -torch.log(-torch.log(torch.rand((H, N, 3), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2)).clamp(1e-9, 1 - 1e-9)))
    out = env.rollout(pol, H, gumbel=gum)
    torch.cuda.synchronize()
    assert pol.sync_timeouts() == 0, "a tile hand-over between the policy and the step kernel was never answered"
    obs, act, logp, val, rew, done = (out[k] for k in ("obs", "actions", "logp", "value", "reward", "done"))
    assert obs.shape == (H + 1, N, env.obs_dim) and act.dtype == torch.int32
    # ---- env side: identical to single steps with the same actions
    o0 = torch.empty_like(obs[0]); twin.L.fxenv_observe(twin._h, o0.data_ptr(), twin._stream()); torch.cuda.synchronize()
    assert torch.equal(obs[0], o0), "rollout must start from the env's current observation"
    for t in range(H):
        o, r, term, _, _ = twin.step(act[t])
        assert torch.equal(o, obs[t + 1]), f"obs after step {t}"
        assert torch.equal(r, rew[t]) and torch.equal(term.to(torch.uint8), done[t]), f"reward / done at step {t}"
    for k in ("equity", "cash", "trades", "position", "n_orders"):
        assert torch.equal(env.info()[k], twin.info()[k]), k
    # ---- policy side
    with torch.no_grad():
        n_flip = 0
        for t in range(H + 1):
            lg_e, v_e = _ref_forward(net, obs[t], True)
            lg_f, v_f = _ref_forward(net, obs[t], False)
            assert torch.allclose(val[t], v_e, atol=2e-3, rtol=2e-3), (t, float((val[t] - v_e).abs().max()))
            assert torch.allclose(val[t], v_f, atol=3e-2, rtol=1e-2), (t, float((val[t] - v_f).abs().max()))
            if t == H:
                break
            lp_e = torch.log_softmax(lg_e, -1)
            sc = lg_e + gum[t]
            a_ref = sc.argmax(-1).to(torch.int32)
            top2 = sc.topk(2, -1).values
            margin = top2[:, 0] - top2[:, 1]
            same = act[t] == a_ref
            assert bool((same | (margin < 5e-3)).all()), f"step {t}: action differs where the margin is {float(margin[~same].max()):.4f}"
            n_flip += int((~same).sum())
            got_lp = lp_e.gather(1, act[t].long()[:, None]).squeeze(1)
            assert torch.allclose(logp[t], got_lp, atol=3e-3, rtol=0), (t, float((logp[t] - got_lp).abs().max()))
            lp_f = torch.log_softmax(lg_f, -1).gather(1, act[t].long()[:, None]).squeeze(1)
            assert torch.allclose(logp[t], lp_f, atol=3e-2, rtol=1e-2), (t, float((logp[t] - lp_f).abs().max()))
            assert int(act[t].min()) >= 0 and int(act[t].max()) <= 2
        assert n_flip <= max(2, H * N // 500), f"{n_flip} sampled actions differ from the reference"
        # all three actions occur and the policy is not degenerate
        assert len(torch.unique(act)) == 3
    # ---- replay of the cached graph, new weights, in-kernel sampling
    with torch.no_grad():
        for p in net.parameters():
            p.add_(0.01)
    pol.set_weights(net)
    out2 = env.rollout(pol, H, buffers=out, seed=1234)
    torch.cuda.synchronize()
    with torch.no_grad():
        lg_e, v_e = _ref_forward(net, out2["obs"][0], True)
        assert torch.allclose(out2["value"][0], v_e, atol=2e-3, rtol=2e-3)
    frac = torch.bincount(out2["actions"].flatten().long(), minlength=3).float() / out2["actions"].numel()
    assert float(frac.min()) > 0.02, f"in-kernel Gumbel sampling looks degenerate: {frac.tolist()}"
    # sampling frequencies follow softmax(logits) (first step, aggregated over envs)
    with torch.no_grad():
        p_mean = torch.softmax(lg_e, -1).mean(0)
        f0 = torch.bincount(out2["actions"][0].long(), minlength=3).float() / N
        assert float((p_mean - f0).abs().max()) < 0.12 + 2.0 / np.sqrt(N), (p_mean.tolist(), f0.tolist())
    env.close(); twin.close()


def test_rollout_other_shapes_and_errors():
    """W=256 (obs_dim 1796 -> K padded to 1856 = 29 k-blocks), ATR strategy + drawdown reward, auto-reset with short episodes."""
    from gym_fx_b200 import _native
    N, H = 300, 5
    cfg, candles, minutes, make = _env(N, W=256, strategy="direct_atr_sltp", reward="dd_penalized_reward", auto_reset=True,
                                       episode_bars=300)
    env, twin = make(), make()
    starts = torch.as_tensor(start_offsets(N, 6000, 400, 300))
    env.reset(starts); twin.reset(starts)
    net = ActorCritic(env.obs_dim).cuda()
    pol = env.make_policy()
    with pytest.raises(_native.FxEnvError, match="set_weights"):
        env.rollout(pol, H)
    pol.set_weights(net)
    out = env.rollout(pol, H, seed=7)
    torch.cuda.synchronize()
    with torch.no_grad():
        for t in range(H + 1):
            _, v_e = _ref_forward(net, out["obs"][t], True)
            assert torch.allclose(out["value"][t], v_e, atol=2e-3, rtol=2e-3), t
    for t in range(H):
        o, r, term, _, _ = twin.step(out["actions"][t])
        assert torch.equal(o, out["obs"][t + 1]) and torch.equal(r, out["reward"][t])
    with pytest.raises(ValueError):
        env.rollout(pol, H, buffers={"obs": torch.empty((1, N, env.obs_dim), device="cuda")})
    env.close(); twin.close()
