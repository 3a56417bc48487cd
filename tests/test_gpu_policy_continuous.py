"""GPU (-m gpu): the closed loop in continuous action mode (the Gaussian actor head of the fused policy kernel,
gym_fx_b200/csrc/fx_policy.cu) and greedy evaluation rollouts in both action modes (fxenv_rollout_ex,
FXENV_ROLLOUT_GREEDY).

As in test_gpu_policy.py, the kernel is compared with a torch evaluation of the same MLP under the kernel's arithmetic
contract (bf16-rounded observation / weights / hidden activations, fp32 heads), and the env side of a rollout must be
IDENTICAL to stepping a twin env with the recorded (float32) actions through fxenv_step."""
import math

import pytest
import torch

import scenarios as S
from gym_fx_b200.config import lower_config
from gym_fx_b200.learner import ActorCritic
from gym_fx_b200.synth import start_offsets, synth_candles, synth_minutes

pytestmark = pytest.mark.gpu

HALF_LOG_2PI = 0.5 * math.log(2.0 * math.pi)


def _env(N, W=128, strategy="direct_fixed_sltp", reward="pnl_reward", T=6000, continuous=True, **kw):
    from gym_fx_b200.vec_env import VecFxEnv
    cfgd = {**S.DEFAULTS, "window_size": W, "feature_columns": list(S.OHLCV)}
    if continuous:
        cfgd["action_space_mode"] = "continuous"
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, "strategy": strategy, "reward": reward,
                                       "preprocessor": "feature_window_preprocessor"})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"], preprocessor_plugin=pl["preprocessor"],
                       reward_plugin=pl["reward"], columns=S.OHLCV, num_envs=N, order_capacity=256, **kw)
    candles, minutes = [synth_candles(T, 0)], [synth_minutes(T)]
    return lambda: VecFxEnv(cfg, candles, minutes)


def _ref_forward(net, obs):
    """-> actor head output [N, n] (logits, or the Gaussian mean with n = 1), value [N]: the kernel's bf16 contract."""
    w1, b1, w2, b2 = net.body[0].weight, net.body[0].bias, net.body[2].weight, net.body[2].bias
    r = lambda t: t.to(torch.bfloat16).to(torch.float32)
    h1 = torch.tanh(r(obs).double() @ r(w1).double().T + b1.double()).float()
    h2 = torch.tanh(r(h1).double() @ r(w2).double().T + b2.double()).float()
    head = (h2.double() @ net.pi.weight.double().T + net.pi.bias.double()).float()
    value = (h2.double() @ net.v.weight.double().T + net.v.bias.double()).float().squeeze(-1)
    return head, value


def _gaussian_net(D, log_std):
    net = ActorCritic(D, continuous=True, init_log_std=log_std).cuda()
    with torch.no_grad():   # a body that makes the hidden units actually vary with the observation
        for p in net.body.parameters():
            p.mul_(2.0)
    return net


def _warm(envs, N, steps=30, continuous=True):
    g = torch.Generator().manual_seed(1)
    for _ in range(steps):
        a = (torch.rand(N, generator=g) * 2 - 1) if continuous else torch.randint(0, 3, (N,), generator=g, dtype=torch.int32)
        for e in envs:
            e.step(a.cuda())


def _check_env_side(env, twin, out, H):
    obs, act, rew, done = (out[k] for k in ("obs", "actions", "reward", "done"))
    o0 = torch.empty_like(obs[0]); twin.L.fxenv_observe(twin._h, o0.data_ptr(), twin._stream()); torch.cuda.synchronize()
    assert torch.equal(obs[0], o0), "rollout must start from the env's current observation"
    for t in range(H):
        o, r, term, _, _ = twin.step(act[t])
        assert torch.equal(o, obs[t + 1]), f"obs after step {t}"
        assert torch.equal(r, rew[t]) and torch.equal(term.to(torch.uint8), done[t]), f"reward / done at step {t}"
    for k in ("equity", "cash", "trades", "position", "n_orders", "bar_index"):
        assert torch.equal(env.info()[k], twin.info()[k]), k


@pytest.mark.parametrize("N,H", [(512, 6), (100, 4), (4096, 3)])
@pytest.mark.parametrize("tile_sync", [0, 1])
def test_continuous_rollout_matches_torch_reference_and_env_matches_single_steps(N, H, tile_sync, monkeypatch):
    monkeypatch.setenv("FXENV_TILE_SYNC", str(tile_sync))
    torch.manual_seed(N)
    make = _env(N)
    env, twin = make(), make()
    starts = torch.as_tensor(start_offsets(N, 6000, 400, 300))
    env.reset(starts); twin.reset(starts)
    _warm((env, twin), N)
    sigma = math.exp(-0.5)
    net = _gaussian_net(env.obs_dim, -0.5)
    pol = env.make_policy(net)
    noise = torch.randn((H, N), device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    out = env.rollout(pol, H, noise=noise)
    torch.cuda.synchronize()
    assert pol.sync_timeouts() == 0, "a tile hand-over between the policy and the step kernel was never answered"
    act, logp, val = out["actions"], out["logp"], out["value"]
    assert act.dtype == torch.float32 and act.shape == (H, N)
    _check_env_side(env, twin, out, H)
    with torch.no_grad():
        for t in range(H + 1):
            mu, v = _ref_forward(net, out["obs"][t])
            assert torch.allclose(val[t], v, atol=2e-3, rtol=2e-3), (t, float((val[t] - v).abs().max()))
            if t == H:
                break
            want = mu[:, 0] + sigma * noise[t]
            assert torch.allclose(act[t], want, atol=2e-3 * max(1.0, sigma), rtol=0), (t, float((act[t] - want).abs().max()))
            lp = torch.distributions.Normal(mu[:, 0], sigma).log_prob(act[t])
            assert torch.allclose(logp[t], lp, atol=3e-3, rtol=0), (t, float((logp[t] - lp).abs().max()))
    # the thresholded action reaches all three of hold / long / short
    thr = 0.33
    assert bool((act > thr).any()) and bool((act < -thr).any()) and bool((act.abs() < thr).any())
    env.close(); twin.close()


def test_continuous_rollout_other_shape_auto_reset_atr():
    """W=256 (obs_dim 1796 -> K padded to 1856), ATR strategy + drawdown reward, auto-reset with short episodes."""
    N, H = 300, 5
    make = _env(N, W=256, strategy="direct_atr_sltp", reward="dd_penalized_reward", auto_reset=True, episode_bars=300)
    env, twin = make(), make()
    starts = torch.as_tensor(start_offsets(N, 6000, 400, 300))
    env.reset(starts); twin.reset(starts)
    torch.manual_seed(3)
    sigma = math.exp(-0.3)
    net = _gaussian_net(env.obs_dim, -0.3)
    pol = env.make_policy(net)
    noise = torch.randn((H, N), device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    out = env.rollout(pol, H, noise=noise)
    torch.cuda.synchronize()
    _check_env_side(env, twin, out, H)
    with torch.no_grad():
        for t in range(H + 1):
            mu, v = _ref_forward(net, out["obs"][t])
            assert torch.allclose(out["value"][t], v, atol=2e-3, rtol=2e-3), t
            if t < H:
                assert torch.allclose(out["actions"][t], mu[:, 0] + sigma * noise[t], atol=2e-3, rtol=0), t
    env.close(); twin.close()


def test_in_kernel_normal_noise_reproducible_and_standard():
    N, H = 4096, 8
    make = _env(N)
    env = make()
    env.reset(torch.as_tensor(start_offsets(N, 6000, 400, 300)))
    _warm((env,), N)
    torch.manual_seed(5)
    net = _gaussian_net(env.obs_dim, 0.0)   # sigma = 1
    pol = env.make_policy(net)
    snap = env.get_state()
    out = env.rollout(pol, H, seed=11)
    torch.cuda.synchronize()
    first = {k: v.clone() for k, v in out.items()}
    env.set_state(snap)
    out = env.rollout(pol, H, buffers=out, seed=11)
    torch.cuda.synchronize()
    for k in first:
        assert torch.equal(first[k], out[k]), f"same seed, same state: {k} differs"
    env.set_state(snap)
    out = env.rollout(pol, H, buffers=out, seed=12)
    torch.cuda.synchronize()
    assert float((out["actions"][0] != first["actions"][0]).float().mean()) > 0.99, "another seed must draw other noise"
    # (a - mu) / sigma over the H * N draws of the first rollout: standard normal.  With n = 32768 draws the standard error
    # of the mean is 1 / sqrt(n) and that of the std about 1 / sqrt(2 n) = 0.0039: bounds of 5 standard errors.
    with torch.no_grad():
        z = torch.cat([first["actions"][t] - _ref_forward(net, first["obs"][t])[0][:, 0] for t in range(H)]).double()
    n = z.numel()
    assert abs(float(z.mean())) < 5.0 / math.sqrt(n), float(z.mean())
    assert abs(float(z.std()) - 1.0) < 0.02, float(z.std())
    assert float(z.abs().max()) < 6.5   # Box-Muller over 24-bit uniforms is bounded by sqrt(2 ln 2^25) = 5.9
    # the log-prob is that of the kernel's own draw: -z^2 / 2 - log sigma - log(2 pi) / 2
    lp = -0.5 * z * z - HALF_LOG_2PI
    assert torch.allclose(first["logp"][:H].reshape(-1).double(), lp, atol=2e-2, rtol=0)
    env.close()


def test_greedy_rollout_discrete():
    N, H = 512, 5
    make = _env(N, continuous=False)
    env, twin = make(), make()
    starts = torch.as_tensor(start_offsets(N, 6000, 400, 300))
    env.reset(starts); twin.reset(starts)
    _warm((env, twin), N, continuous=False)
    torch.manual_seed(6)
    net = ActorCritic(env.obs_dim).cuda()
    with torch.no_grad():
        for p in net.parameters():
            p.mul_(2.0)
    pol = env.make_policy(net)
    snap = env.get_state()
    out = env.rollout(pol, H, deterministic=True)
    torch.cuda.synchronize()
    first = {k: v.clone() for k, v in out.items()}
    _check_env_side(env, twin, out, H)
    with torch.no_grad():
        for t in range(H):
            lg, _ = _ref_forward(net, out["obs"][t])
            a_ref = lg.argmax(-1).to(torch.int32)
            top2 = lg.topk(2, -1).values
            margin = top2[:, 0] - top2[:, 1]
            same = out["actions"][t] == a_ref
            assert bool((same | (margin < 5e-3)).all()), t
            lp = torch.log_softmax(lg, -1).gather(1, out["actions"][t].long()[:, None]).squeeze(1)
            assert torch.allclose(out["logp"][t], lp, atol=3e-3, rtol=0), t
    assert len(torch.unique(out["actions"])) >= 2
    env.set_state(snap)
    out = env.rollout(pol, H, buffers=out, deterministic=True, seed=99)   # the seed plays no part in greedy mode
    torch.cuda.synchronize()
    for k in first:
        assert torch.equal(first[k], out[k]), f"greedy rollouts from one snapshot differ in {k}"
    # sampling again after greedy rollouts on the same buffers (the cached graph is keyed on the flags)
    env.set_state(snap)
    out = env.rollout(pol, H, buffers=out, seed=99)
    torch.cuda.synchronize()
    assert not torch.equal(first["actions"], out["actions"])
    env.close(); twin.close()


def test_greedy_rollout_continuous():
    N, H = 512, 4
    make = _env(N)
    env = make()
    env.reset(torch.as_tensor(start_offsets(N, 6000, 400, 300)))
    _warm((env,), N)
    torch.manual_seed(7)
    log_std = -0.8
    net = _gaussian_net(env.obs_dim, log_std)
    pol = env.make_policy(net)
    noise = torch.randn((H, N), device="cuda")
    out = env.rollout(pol, H, noise=noise, deterministic=True)   # noise is not read in greedy mode
    torch.cuda.synchronize()
    with torch.no_grad():
        for t in range(H):
            mu, _ = _ref_forward(net, out["obs"][t])
            assert torch.allclose(out["actions"][t], mu[:, 0], atol=2e-3, rtol=0), (t, float((out["actions"][t] - mu[:, 0]).abs().max()))
    lp = torch.full_like(out["logp"], -log_std - HALF_LOG_2PI)
    assert torch.allclose(out["logp"], lp, atol=1e-6, rtol=0)
    env.close()


def test_continuous_argument_errors():
    N, H = 128, 2
    env = _env(N)()
    env.reset()
    D = env.obs_dim
    net = _gaussian_net(D, 0.0)
    pol = env.make_policy(net)
    with pytest.raises(ValueError, match="actions"):
        env.rollout(pol, H, buffers={"actions": torch.zeros((H, N), dtype=torch.int32, device="cuda")})
    with pytest.raises(ValueError, match="gumbel"):
        env.rollout(pol, H, gumbel=torch.zeros((H, N, 3), device="cuda"))
    with pytest.raises(ValueError, match="noise"):
        env.rollout(pol, H, noise=torch.zeros((H, N, 3), device="cuda"))
    with pytest.raises(ValueError, match="noise"):
        env.rollout(pol, H, noise=torch.zeros((H, N), dtype=torch.float64, device="cuda"))
    with pytest.raises(ValueError, match="log_std"):
        pol.set_weights(ActorCritic(D).cuda())                       # a discrete net: 3 logits, no log_std
    w = {"w1": net.body[0].weight, "b1": net.body[0].bias, "w2": net.body[2].weight, "b2": net.body[2].bias,
         "w_pi": net.pi.weight, "b_pi": net.pi.bias, "w_v": net.v.weight, "b_v": net.v.bias}
    with pytest.raises(ValueError, match="log_std"):
        pol.set_weights(w)
    with pytest.raises(ValueError, match="w_pi"):
        pol.set_weights({**w, "w_pi": torch.zeros((3, 256), device="cuda"), "log_std": net.log_std})
    with pytest.raises(ValueError, match="log_std"):
        pol.set_weights({**w, "log_std": torch.zeros(2, device="cuda")})
    pol.set_weights({**w, "log_std": net.log_std})
    env.close()
    denv = _env(N, continuous=False)()
    denv.reset()
    dpol = denv.make_policy(ActorCritic(D).cuda())
    with pytest.raises(ValueError, match="noise"):
        denv.rollout(dpol, H, noise=torch.zeros((H, N), device="cuda"))
    with pytest.raises(ValueError, match="w_pi"):
        dpol.set_weights(net)                                        # a Gaussian net: one mean row
    denv.close()
