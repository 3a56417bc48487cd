"""CPU: the host reference of the fused policy kernel at the hidden widths other than 256 (64, 128, 512).

As in test_policy_reference.py, a float32 emulation of the kernel's arithmetic (bf16 operands, fp32 accumulation over
16-wide k-steps, tanh off by the documented tanh.approx.f32 bound, bf16 h1) stands in for the device: the tolerances
accept it at every width, and every negative control is rejected -- including the swap of the two halves of h1 (one
half per CTA of the pair, so this is what catches a CTA computing the wrong units) and the dropped last W2 k-block (at
width 64 the only one).  policy_width_ref.control_refs takes the width from the weights; on 256-wide weights it must
build exactly what policy_ref.control_refs builds for the default policy."""
import pytest
import torch
import torch.nn as nn

import policy_ref as R
import policy_width_ref as RW
from test_policy_reference import _emulate_kernel, _obs


class _Net(nn.Module):
    def __init__(self, D, hidden, n_pi=3):
        super().__init__()
        self.body = nn.Sequential(nn.Linear(D, hidden), nn.Tanh(), nn.Linear(hidden, hidden), nn.Tanh())
        self.pi = nn.Linear(hidden, n_pi)
        self.v = nn.Linear(hidden, 1)


@pytest.mark.parametrize("D", [30, 144, 291, 1796])
@pytest.mark.parametrize("hidden", [64, 128, 512])
def test_tolerances_accept_the_kernel_contract_and_reject_every_negative_control(hidden, D):
    torch.manual_seed(1000 * hidden + D)
    net = R.scaled_init(_Net(D, hidden))
    w = R.weights_of(net)
    obs = _obs(257, D, D)
    h1, head, value = _emulate_kernel(w, obs, D)
    assert h1.shape == (257, hidden)
    ref = R.forward_ref(w, obs)
    assert ref["h1"].shape == (257, hidden)
    rep = R.check_h1(h1, ref, obs, w)
    assert rep["bad"] == 0, rep
    e_emul = max(R.head_err(value, ref["value"]), R.head_err(head, ref["head"]))
    assert e_emul < 2 * R.HEAD_TOL, e_emul
    ctl = RW.control_refs(w, obs, agent=True)
    assert set(R.H1_CONTROLS) <= set(ctl) and set(R.HEAD_CONTROLS) <= set(ctl)
    for name in R.H1_CONTROLS:
        assert R.check_h1(h1, ctl[name], obs, w)["bad"] > 0, f"h1 check does not reject control {name} at width {hidden}"
    for name in R.HEAD_CONTROLS:
        assert R.head_err(value, ctl[name]["value"]) > 5 * R.HEAD_TOL, f"value check does not reject {name} at {hidden}"
        assert R.head_err(head, ctl[name]["head"]) > 5 * R.HEAD_TOL, f"head check does not reject {name} at {hidden}"


@pytest.mark.parametrize("hidden", [64, 128, 512])
def test_controls_follow_the_width_of_the_weights(hidden):
    D = 144
    torch.manual_seed(hidden)
    w = R.weights_of(R.scaled_init(_Net(D, hidden)))
    obs = _obs(64, D, 5)
    ctl = RW.control_refs(w, obs)
    good = R.forward_ref(w, obs)
    half = hidden // 2
    sw = ctl["swap_h1_halves"]["h1"]
    assert torch.equal(sw[:, :half], good["h1"][:, half:]) and torch.equal(sw[:, half:], good["h1"][:, :half])
    w2 = dict(w)
    w2["w2"] = w["w2"].clone()
    w2["w2"][:, hidden - R.BLOCK_K:] = 0   # at 64: all of W2
    assert torch.equal(ctl["drop_w2_last_kblock"]["value"], R.forward_ref(w2, obs)["value"])


@pytest.mark.parametrize("agent", [True, False])
def test_controls_on_256_wide_weights_equal_the_default_helper(agent):
    """on the default width the width-aware controls are policy_ref.control_refs, tensor for tensor"""
    D = 291
    torch.manual_seed(7)
    w = R.weights_of(R.scaled_init(_Net(D, 256)))
    obs = _obs(200, D, 9)
    got, want = RW.control_refs(w, obs, agent=agent), R.control_refs(w, obs, agent=agent)
    assert set(got) == set(want)
    for name in want:
        for k in want[name]:
            assert torch.equal(got[name][k], want[name][k]), (name, k)
