"""CPU: the host reference of the fused policy kernel (tests/policy_ref.py) and its tolerances.

The GPU tests compare kernel output with forward_ref under check_h1 / head_close, and pair every comparison with
deliberately wrong references (negative controls) that must fail it.  Here a float32 emulation of the kernel's
arithmetic (bf16 operands, fp32 accumulation, tanh perturbed by the documented tanh.approx.f32 error, bf16 h1) stands in
for the device, so the discrimination of the tolerances is shown without a GPU.  The counter-based generator replica is
checked against an independent plain-integer implementation."""
import math

import numpy as np
import pytest
import torch
import torch.nn as nn

import policy_ref as R


class _Net(nn.Module):
    def __init__(self, D, n_pi=3):
        super().__init__()
        self.body = nn.Sequential(nn.Linear(D, 256), nn.Tanh(), nn.Linear(256, 256), nn.Tanh())
        self.pi = nn.Linear(256, n_pi)
        self.v = nn.Linear(256, 1)


def _obs(N, D, seed, agent=True):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((N, D), generator=g).clamp(-4, 4)
    if agent:   # position, equity_norm, unrealized_pnl_norm, steps_remaining_norm
        x[:, D - 4] = torch.randint(-1, 2, (N,), generator=g).float()
        x[:, D - 3] = 1.0 + 0.05 * torch.randn(N, generator=g)
        x[:, D - 2] = 0.01 * torch.randn(N, generator=g)
        x[:, D - 1] = torch.rand(N, generator=g)
    return x


def _emulate_kernel(w, obs, seed):
    """float32 stand-in for the kernel: bf16 operands, fp32 accumulation over 16-wide k-steps (one wgmma k16 each),
    fp32 bias add, tanh off by up to the tanh.approx.f32 bound, bf16 h1; layer 2 likewise, fp32 heads."""
    g = torch.Generator().manual_seed(seed)
    r16 = lambda t: t.to(torch.bfloat16).to(torch.float32)
    x, w1, w2 = r16(obs), r16(w["w1"]), r16(w["w2"])

    def mm(a, b):
        acc = torch.zeros((a.shape[0], b.shape[0]), dtype=torch.float32)
        for k0 in range(0, a.shape[1], 16):
            acc = acc + a[:, k0:k0 + 16] @ b[:, k0:k0 + 16].T
        return acc

    def approx_tanh(z):
        t = torch.tanh(z)
        return t * (1.0 + (2 * torch.rand(t.shape, generator=g) - 1) * R.TANH_APPROX_REL_ERR)

    h1 = r16(approx_tanh(mm(x, w1) + w["b1"]))
    h2 = approx_tanh(mm(h1, w2) + w["b2"])
    head = h2 @ w["w_pi"].T + w["b_pi"]
    value = h2 @ w["w_v"].reshape(-1) + w["b_v"]
    return h1, head, value


@pytest.mark.parametrize("D", [30, 64, 128, 144, 256, 291, 900])
def test_tolerances_accept_the_kernel_contract_and_reject_every_negative_control(D):
    torch.manual_seed(D)
    net = R.scaled_init(_Net(D))
    w = R.weights_of(net)
    obs = _obs(257, D, D)
    h1, head, value = _emulate_kernel(w, obs, D)
    ref = R.forward_ref(w, obs)
    rep = R.check_h1(h1, ref, obs, w)
    assert rep["bad"] == 0, rep
    # the emulation puts the full tanh.approx bound on every unit of both layers, which the hardware does not reach (the
    # GPU tests hold the kernel to HEAD_TOL); the controls must still be far outside what even that allows
    e_emul = max(R.head_err(value, ref["value"]), R.head_err(head, ref["head"]))
    assert e_emul < 2 * R.HEAD_TOL, e_emul
    ctl = R.control_refs(w, obs, agent=True)
    assert set(R.H1_CONTROLS) <= set(ctl) and set(R.HEAD_CONTROLS) <= set(ctl)
    for name in R.H1_CONTROLS:
        assert R.check_h1(h1, ctl[name], obs, w)["bad"] > 0, f"h1 check does not reject control {name}"
    for name in R.HEAD_CONTROLS:
        assert R.head_err(value, ctl[name]["value"]) > 5 * R.HEAD_TOL, f"value check does not reject control {name}"
        assert R.head_err(head, ctl[name]["head"]) > 5 * R.HEAD_TOL, f"head check does not reject control {name}"


def test_h1_check_rejects_one_wrong_element_and_a_biased_rounding():
    D = 291
    torch.manual_seed(1)
    w = R.weights_of(R.scaled_init(_Net(D)))
    obs = _obs(128, D, 2)
    h1, _, _ = _emulate_kernel(w, obs, 3)
    ref = R.forward_ref(w, obs)
    # a single element two bf16 ulps off
    bad = h1.clone()
    bad[17, 200] = float(ref["h1"][17, 200] + 2 * R.bf16_ulp(ref["h1"][17, 200]))
    assert R.check_h1(bad, ref, obs, w)["bad"] >= 1
    # truncation instead of round-to-nearest-even of the observation copy: off by up to one ulp of x on every element
    x_trunc = (obs.view(torch.int32) & ~0xFFFF).view(torch.float32)
    h1_t, _, _ = _emulate_kernel(w, x_trunc, 3)
    assert R.check_h1(h1_t, ref, obs, w)["bad"] > 0


def test_bf16_helpers():
    t = torch.tensor([1.0, 0.75, -3.0, 1.0 + 2 ** -9, 0.0], dtype=torch.float64)
    assert R.bf16_ulp(t)[:3].tolist() == [2 ** -7, 2 ** -8, 2 ** -6]
    assert float(R.bf16(t)[3]) == 1.0   # tie -> even
    assert float(R.bf16_ulp(t)[4]) > 0


def test_hash_uniform_replica_matches_plain_integer_implementation():
    rng = np.random.default_rng(0)
    seeds = [0, 1, 7, 1234, 2 ** 63 + 5, 2 ** 64 - 1] + [int(s) for s in rng.integers(0, 2 ** 63, 10)]
    for seed in seeds:
        steps = rng.integers(0, 2 ** 32, 4)
        envs = rng.integers(0, 9000, 4)
        for st in list(steps) + [0, 1]:
            for e in list(envs) + [0, 8391]:
                got = R.hash_uniform_np(seed, int(st), int(e), np.arange(3))
                want = [R.hash_uniform_py(seed, int(st), int(e), a) for a in range(3)]
                assert got.dtype == np.float32 and got.tolist() == want
    u = R.hash_uniform_np(99, 3, np.arange(100000)[:, None], np.arange(3)[None, :])
    assert float(u.min()) > 0.0 and float(u.max()) <= 1.0 and abs(float(u.mean()) - 0.5) < 0.005


def test_uniform_grid_rounding_at_the_top():
    top = np.arange(2 ** 24 - 8, 2 ** 24)
    u = R.uniform_of_bits(top)
    # above 2^23 the float32 "+ 0.5" is a tie: rounds to even, so the top integer maps to exactly 1.0
    assert u[-1] == np.float32(1.0)
    assert u[-2] == u[-3] == np.float32(1.0 - 2.0 ** -23)
    assert R.uniform_of_bits(np.array([0]))[0] == np.float32(2.0 ** -25)
    g = R.gumbel_of_uniform(u)
    assert np.isinf(g[-1]) and g[-1] > 0 and np.all(np.isfinite(g[:-1]))
    # the __logf error bound admits no conclusion this close to 1, and a tight one in the bulk
    e = R.fast_gumbel_err(np.array([1.0, 1.0 - 2.0 ** -23, 0.5, 0.1, 1e-7]))
    assert np.isinf(e[0]) and np.isinf(e[1]) and np.all(e[2:] < 1e-5)


def test_box_muller_and_chi_square_helpers():
    z = R.box_muller_np(R.hash_uniform_np(5, 0, np.arange(50000), 0), R.hash_uniform_np(5, 0, np.arange(50000), 1))
    assert abs(z.mean()) < 0.03 and abs(z.std() - 1.0) < 0.02
    p = np.array([0.2, 0.3, 0.5])
    assert R.chi_square_sf(np.array([200, 300, 500]), p) > 0.99
    assert R.chi_square_sf(np.array([260, 300, 440]), p) < 1e-4
    assert math.isclose(R.chi_square_sf(np.array([10, 10]), np.array([0.5, 0.5])), 1.0)
