"""Host reference of the fused policy kernel (gym_fx_b200/csrc/fx_policy.cu), shared by the policy tests.

The kernel's arithmetic contract: the observation, W1 and W2 are bf16; layer 1 and layer 2 accumulate in fp32 on the
tensor cores; h1 = bf16(tanh(obs . W1^T + b1)) is stored and re-read as bf16; h2 stays fp32; biases, heads, sampling and
log-prob are fp32.  `forward_ref` evaluates that contract in fp64, `check_h1` bounds the kernel's h1 element by element,
`hash_uniform_np` replicates the in-kernel counter-based generator bit for bit, and `control_refs` builds the
deliberately wrong references every comparison must reject (negative controls)."""
from __future__ import annotations

import math

import numpy as np
import torch

HIDDEN = 256
BLOCK_K = 64      # k-block of the layer-1 / layer-2 pipelines (one 128-byte swizzled TMA box)
# PTX ISA, "tanh" (floating point): "tanh.approx.f32 implements an approximation to FP32 hyperbolic-tangent.
# Max relative error: 2^-10.987."  (The error of a bf16 rounding is up to 2^-8 relative: this is ~1/8 of a bf16 ulp.)
TANH_APPROX_REL_ERR = 2.0 ** -10.987
# CUDA Math API, intrinsic __logf(x): "For x in [0.5, 2], the maximum absolute error is 2^-21.41, otherwise, the maximum
# ulp error is 3."
LOGF_FAST_ABS_ERR = 2.0 ** -21.41
LOGF_FAST_ULP = 3.0


def bf16(t: torch.Tensor) -> torch.Tensor:
    """Round to bfloat16 (round to nearest even, via float32 like the kernel) and return as float64."""
    return t.to(torch.float32).to(torch.bfloat16).to(torch.float64)


def bf16_ulp(t: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 values (8 significant bits) at |t|, float64; bf16 has the float32 exponent range."""
    t = t.to(torch.float64).abs()
    _, e = torch.frexp(t)                       # t = m * 2^e, m in [0.5, 1)
    ulp = torch.ldexp(torch.ones_like(t), e - 8)
    return torch.where(t > 0, ulp, torch.full_like(t, 2.0 ** -133))


def weights_of(net_or_dict, continuous: bool = False) -> dict:
    """float32 parameter dict (w1, b1, w2, b2, w_pi, b_pi, w_v, b_v[, log_std]) from an ActorCritic-like module or a dict."""
    if isinstance(net_or_dict, dict):
        w = dict(net_or_dict)
    else:
        m = net_or_dict
        w = {"w1": m.body[0].weight, "b1": m.body[0].bias, "w2": m.body[2].weight, "b2": m.body[2].bias,
             "w_pi": m.pi.weight, "b_pi": m.pi.bias, "w_v": m.v.weight, "b_v": m.v.bias}
        if getattr(m, "log_std", None) is not None:
            w["log_std"] = m.log_std
    return {k: v.detach().to(torch.float32) for k, v in w.items()}


def forward_ref(weights, obs: torch.Tensor) -> dict:
    """fp64 evaluation of the kernel's contract for float32 observation rows obs [N, D].
    -> {"h1": bf16-rounded h1 [N, 256], "z1": its pre-activation, "h2": [N, 256], "head": logits [N, 3] or the Gaussian
    mean [N, 1], "value": [N]}, all float64 on obs.device."""
    w = weights_of(weights)
    dev = obs.device
    g = {k: v.to(dev) for k, v in w.items()}
    x = bf16(obs)
    z1 = x @ bf16(g["w1"]).T + g["b1"].double()
    h1 = bf16(torch.tanh(z1))
    h2 = torch.tanh(h1 @ bf16(g["w2"]).T + g["b2"].double())
    head = h2 @ g["w_pi"].double().T + g["b_pi"].double()
    value = h2 @ g["w_v"].double().reshape(-1) + g["b_v"].double().reshape(())
    return {"h1": h1, "z1": z1, "h2": h2, "head": head, "value": value}


def h1_bound(ref_h1: torch.Tensor, z1: torch.Tensor, obs: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor) -> torch.Tensor:
    """Per-element bound of |kernel h1 - ref h1|: one bf16 ulp of the reference, plus the tanh.approx.f32 error, plus an
    fp32-accumulation term (KP + 1) * 2^-24 * (sum_i |x_i w_i| + |b|) for the K-padded contraction and the bias add
    (tanh' <= 1 carries an input error to the output unchanged at most)."""
    x = bf16(obs).abs()
    kp = (obs.shape[1] + BLOCK_K - 1) // BLOCK_K * BLOCK_K
    s = x @ bf16(w1.to(obs.device)).abs().T + b1.to(obs.device).double().abs()
    return bf16_ulp(ref_h1) + TANH_APPROX_REL_ERR * torch.tanh(z1).abs() + (kp + 1) * 2.0 ** -24 * s


def check_h1(kernel_h1: torch.Tensor, ref: dict, obs: torch.Tensor, weights) -> dict:
    """Compare the kernel's h1 rows [N, 256] (bf16) with forward_ref(weights, obs).  -> {"bad": elements over the bound,
    "max_ulps": largest error in bf16 ulps of the reference, "max_ulps_big": the same over |ref| >= 1/16 (near 0 a
    bf16 ulp is far below the fp32 accumulation error), "frac_equal": fraction equal to the rounded reference}."""
    w = weights_of(weights)
    k = kernel_h1.to(torch.float64)
    r = ref["h1"]
    err = (k - r).abs()
    bound = h1_bound(r, ref["z1"], obs, w["w1"], w["b1"])
    ulps = err / bf16_ulp(r)
    big = r.abs() >= 1.0 / 16
    return {"bad": int((err > bound).sum()), "max_ulps": float(ulps.max()),
            "max_ulps_big": float(ulps[big].max()) if bool(big.any()) else 0.0,
            "frac_equal": float((err == 0).double().mean())}


def control_refs(weights, obs: torch.Tensor, agent: bool = True) -> dict:
    """Deliberately wrong references (negative controls), name -> forward_ref-like dict.  Every comparison of kernel
    output must reject the ones aimed at it:
      h1:  k-block 0 dropped, the last (possibly partial) layer-1 k-block dropped, the two 128-unit halves of h1 swapped,
           rows shifted by one, the 4 agent-scalar columns zeroed (agent: the row ends in them);
      value / head: the last W2 k-block dropped, rows shifted by one."""
    w = weights_of(weights)
    D = obs.shape[1]
    nkb = (D + BLOCK_K - 1) // BLOCK_K
    out = {}
    for name, j in (("drop_kblock_first", 0), ("drop_kblock_last", nkb - 1)):
        x = obs.clone()
        x[:, j * BLOCK_K:(j + 1) * BLOCK_K] = 0
        out[name] = forward_ref(w, x)
    good = forward_ref(w, obs)
    out["swap_h1_halves"] = {**good, "h1": torch.cat([good["h1"][:, HIDDEN // 2:], good["h1"][:, :HIDDEN // 2]], 1)}
    out["rows_shifted"] = {k: torch.roll(v, 1, 0) for k, v in good.items()}
    if agent:
        x = obs.clone()
        x[:, D - 4:] = 0
        out["agent_zeroed"] = forward_ref(w, x)
    w2 = dict(w)
    w2["w2"] = w["w2"].clone()
    w2["w2"][:, HIDDEN - BLOCK_K:] = 0
    out["drop_w2_last_kblock"] = forward_ref(w2, obs)
    return out


H1_CONTROLS = ("drop_kblock_first", "drop_kblock_last", "swap_h1_halves", "rows_shifted", "agent_zeroed")
HEAD_CONTROLS = ("drop_w2_last_kblock", "rows_shifted")
# value, logits and the Gaussian mean against forward_ref: |a - b| <= HEAD_TOL * (1 + |b|), the tolerance the policy
# tests have always used.  What it absorbs: h1 elements that round to the neighbouring bf16 value, tanh.approx.f32 in
# both layers and fp32 accumulation.
HEAD_TOL = 2e-3


def head_err(kernel: torch.Tensor, ref: torch.Tensor) -> float:
    """max |kernel - ref| / (1 + |ref|)"""
    k, r = kernel.to(torch.float64), ref.to(torch.float64).to(kernel.device)
    return float(((k - r).abs() / (1.0 + r.abs())).max())


def head_close(kernel: torch.Tensor, ref: torch.Tensor, tol: float = HEAD_TOL) -> bool:
    return head_err(kernel, ref) <= tol


def scaled_init(module, factor: float = 2.0):
    """Multiply every parameter of an nn.Module by `factor` in place (torch's default init is weak enough that a wrong
    operand could hide inside the tolerances; x2 makes every negative control fail)."""
    with torch.no_grad():
        for p in module.parameters():
            p.mul_(factor)
    return module


# ---- the in-kernel counter-based generator (fx_policy.cu: hash_uniform) ------------------------------------------------
_M64 = (1 << 64) - 1


def hash_bits_np(seed, step, env, a) -> np.ndarray:
    """The 24-bit integer k = z >> 40 of hash_uniform(seed, step, env, a), exact uint64 arithmetic (broadcasting)."""
    with np.errstate(over="ignore"):
        seed = np.asarray(seed, dtype=np.uint64)
        step = np.asarray(step, dtype=np.uint64) & np.uint64(0xFFFFFFFF)
        env = np.asarray(env, dtype=np.uint64) & np.uint64(0xFFFFFFFF)
        a = np.asarray(a, dtype=np.uint64) & np.uint64(0xFFFFFFFF)
        z = seed + np.uint64(0x9E3779B97F4A7C15) * (step * np.uint64(0x100000001B3) + (env << np.uint64(2)) + a + np.uint64(1))
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
    return (z >> np.uint64(40)).astype(np.uint32)


def uniform_of_bits(k) -> np.ndarray:
    """float32 ((float)k + 0.5f) * 2^-24, as the kernel rounds it: above 2^23 the + 0.5 is a tie that rounds to even, so
    k = 2^24 - 1 gives exactly 1.0."""
    k = np.asarray(k, dtype=np.uint32).astype(np.float32)
    return ((k + np.float32(0.5)).astype(np.float32) * np.float32(1.0 / 16777216.0)).astype(np.float32)


def hash_uniform_np(seed, step, env, a) -> np.ndarray:
    """Bit-identical numpy replica of the kernel's hash_uniform: float32 in (0, 1]."""
    return uniform_of_bits(hash_bits_np(seed, step, env, a))


def hash_uniform_py(seed: int, step: int, env: int, a: int) -> float:
    """The same generator in plain Python integers (an independent check of the numpy replica)."""
    z = (seed + 0x9E3779B97F4A7C15 * (step * 0x100000001B3 + (env << 2) + a + 1)) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    z ^= z >> 31
    return float(uniform_of_bits(z >> 40))


def gumbel_of_uniform(u: np.ndarray) -> np.ndarray:
    """fp64 Gumbel(0, 1) of the replica's uniforms, -log(-log u) (u = 1 gives +inf)."""
    u = np.asarray(u, dtype=np.float64)
    with np.errstate(divide="ignore"):
        return -np.log(-np.log(u))


def _f32_ulp(x: np.ndarray) -> np.ndarray:
    x = np.abs(np.asarray(x, dtype=np.float32))
    return np.spacing(x).astype(np.float64)


def fast_gumbel_err(u: np.ndarray) -> np.ndarray:
    """Bound of |kernel g - fp64 g| for g = -__logf(-__logf(u)) (CUDA Math API error of __logf, first-order propagation
    of the inner error through the outer log).  +inf where the inner error can reach -log u itself."""
    u = np.asarray(u, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        l = np.log(u)
        e_in = np.where(u >= 0.5, LOGF_FAST_ABS_ERR, LOGF_FAST_ULP * _f32_ulp(l))
        y = -l
        ly = np.log(np.where(y > 0, y, 1.0))
        e_out = np.where((y >= 0.5) & (y <= 2.0), LOGF_FAST_ABS_ERR, LOGF_FAST_ULP * _f32_ulp(ly))
        e = np.where(e_in < 0.5 * y, e_in / (y - e_in) + e_out, np.inf)
    return e


def box_muller_np(u0: np.ndarray, u1: np.ndarray) -> np.ndarray:
    """fp64 Box-Muller of the replica's uniforms as the continuous kernel draws it: sqrt(-2 log u0) * cos(2 pi u1)."""
    u0 = np.asarray(u0, dtype=np.float64)
    u1 = np.asarray(u1, dtype=np.float64)
    return np.sqrt(-2.0 * np.log(u0)) * np.cos(2.0 * math.pi * u1)


def chi_square_sf(counts: np.ndarray, probs: np.ndarray) -> float:
    """Upper-tail p-value of Pearson's chi-square statistic of `counts` against `probs` (len(counts) - 1 dof)."""
    from scipy import stats

    counts = np.asarray(counts, dtype=np.float64)
    exp = np.asarray(probs, dtype=np.float64) * counts.sum()
    chi2 = float(((counts - exp) ** 2 / exp).sum())
    return float(stats.chi2.sf(chi2, len(counts) - 1))
