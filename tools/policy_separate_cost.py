#!/usr/bin/env python3
"""Cost of separate actor and critic networks in the closed loop: µs per decision of VecFxEnv.rollout at the cfg4 shape
of bench.py (4096 envs, W = 128, horizon 32), discrete and continuous actions, for hidden H in {64, 128, 256}:

  shared H     one MLP(H, H) body under both heads (the default policy);
  separate H   an actor MLP(H, H) and a critic MLP(H, H) (FXENV_POLICY_SEPARATE: two CTA pairs per tile);
  packed 2H    the same two networks packed into one shared body of width 2H (W1 stacked, W2 block-diagonal, each head
               zero on the other network's units): the only way to run separate networks in the fused loop before.

Measured like tools/policy_width_cost.py (its make_env and card): every setting runs in every repetition, in turn, in
one process, all graphs captured and warmed before the first timed rollout; a repetition enqueues back-to-back
rollouts between two CUDA events, and the table shows the median over the repetitions and their range.  The packed
form is also checked to give the separate policy's value (it is the same function, up to bf16 / fp32 rounding).

Usage: python tools/policy_separate_cost.py [repetitions=3] [rollouts per repetition=5]"""
import os
import sys

sys.path[:0] = [os.path.dirname(os.path.abspath(__file__)), os.path.dirname(os.path.dirname(os.path.abspath(__file__)))]
import numpy as np
import torch

from policy_width_cost import H, card, make_env

WIDTHS = (64, 128, 256)
FORMS = ("shared", "separate", "packed")


def packed(net):
    """weights of one shared body of width 2H that computes the separate net `net` exactly"""
    a, c = net.body, net.critic_body
    hid = a[0].out_features
    w2 = torch.zeros(2 * hid, 2 * hid, device=a[0].weight.device)
    w2[:hid, :hid], w2[hid:, hid:] = a[2].weight, c[2].weight
    zero = lambda t: torch.zeros_like(t)
    w = {"w1": torch.cat([a[0].weight, c[0].weight]), "b1": torch.cat([a[0].bias, c[0].bias]), "w2": w2,
         "b2": torch.cat([a[2].bias, c[2].bias]), "w_pi": torch.cat([net.pi.weight, zero(net.pi.weight)], 1),
         "b_pi": net.pi.bias, "w_v": torch.cat([zero(net.v.weight), net.v.weight], 1), "b_v": net.v.bias}
    if net.continuous:
        w["log_std"] = net.log_std
    return {k: v.detach() for k, v in w.items()}


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 3
    batches = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    if not torch.cuda.is_available():
        sys.exit("policy_separate_cost.py needs a CUDA device")
    from gym_fx_b200.learner import ActorCritic
    print(card())
    envs, pols, bufs = {}, {}, {}
    desc = N = D = None
    for cont in (False, True):
        # make_env sizes the episodes for the four settings per repetition of policy_width_cost.py; nine run here
        envs[cont], N, D, desc = make_env(cont, 3 * reps, batches)
        for hid in WIDTHS:
            torch.manual_seed(hid)
            net = ActorCritic(D, hidden=hid, continuous=cont, separate=True).cuda()
            torch.manual_seed(hid)
            pols[(hid, cont, "shared")] = envs[cont].make_policy(ActorCritic(D, hidden=hid, continuous=cont).cuda())
            pols[(hid, cont, "separate")] = envs[cont].make_policy(net)
            pols[(hid, cont, "packed")] = envs[cont].make_policy(packed(net))
    for cont in (False, True):                            # same function: packed value = separate value
        # (before the warm-up: a policy caches one rollout graph, and this 1-step rollout replaces it)
        for hid in WIDTHS:
            snap = envs[cont].get_state()
            v = []
            for f in ("separate", "packed"):
                envs[cont].set_state(snap)
                v.append(envs[cont].rollout(pols[(hid, cont, f)], 1, seed=3)["value"][0].clone())
            envs[cont].set_state(snap)
            err = float(((v[0] - v[1]).abs() / (1 + v[1].abs())).max())
            assert err < 2e-3, (hid, cont, err)
    settings = [(hid, cont, f) for cont in (False, True) for hid in WIDTHS for f in FORMS]
    for s in settings:                                    # warm-up: captures each setting's graph, then one replay
        env = envs[s[1]]
        bufs[s] = env.rollout(pols[s], H, seed=2)
        env.rollout(pols[s], H, buffers=bufs[s], seed=2)
    torch.cuda.synchronize()
    per = {s: [] for s in settings}
    for _ in range(reps):
        for s in settings:
            env = envs[s[1]]
            stream = torch.cuda.current_stream()          # VecFxEnv.rollout enqueues on the current stream
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(batches):
                env.rollout(pols[s], H, buffers=bufs[s], seed=2)
            e1.record(stream)
            e1.synchronize()
            per[s].append(e0.elapsed_time(e1) * 1e3 / (batches * H))
    for env in envs.values():
        env.close()
    print(f"{desc} -- closed loop (VecFxEnv.rollout, horizon {H}, {N} envs, obs_dim {D}), us per decision, median of {reps} "
          f"(range)")
    print("| mode | H | shared H | separate H | packed 2H | separate / shared | separate / packed |")
    print("|---|---|---|---|---|---|---|")
    for cont in (False, True):
        for hid in WIDTHS:
            m = {f: float(np.median(per[(hid, cont, f)])) for f in FORMS}
            cell = lambda f: f"{m[f]:.2f} ({min(per[(hid, cont, f)]):.2f}–{max(per[(hid, cont, f)]):.2f})"
            print(f"| {'continuous' if cont else 'discrete'} | {hid} | {cell('shared')} | {cell('separate')} | "
                  f"{cell('packed')} | {m['separate'] / m['shared']:.3f} | {m['separate'] / m['packed']:.3f} |")


if __name__ == "__main__":
    main()
