"""Negative controls of the fused policy kernel at any hidden width (64, 128, 256, 512), for the width tests.

policy_ref.control_refs builds the deliberately wrong references for the default 256-wide policy: two of them depend on
the width -- the swap of the two halves of h1 (one half per CTA of the pair) and the dropped last W2 k-block.
`control_refs` here takes the width from the rows of w1 and rebuilds those two; the others do not depend on it.  On
256-wide weights it gives exactly policy_ref.control_refs."""
from __future__ import annotations

import torch

import policy_ref as R


def control_refs(weights, obs: torch.Tensor, agent: bool = True) -> dict:
    """policy_ref.control_refs with the width-dependent controls built for the width of `weights` (the rows of w1)."""
    w = R.weights_of(weights)
    hid = w["w1"].shape[0]
    out = R.control_refs(w, obs, agent=agent)
    good = R.forward_ref(w, obs)
    out["swap_h1_halves"] = {**good, "h1": torch.cat([good["h1"][:, hid // 2:], good["h1"][:, :hid // 2]], 1)}
    w2 = dict(w)
    w2["w2"] = w["w2"].clone()
    w2["w2"][:, hid - R.BLOCK_K:] = 0   # at width 64: all of W2
    out["drop_w2_last_kblock"] = R.forward_ref(w2, obs)
    return out
