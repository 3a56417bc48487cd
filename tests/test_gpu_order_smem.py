"""The persistent rollout kernel with each ticket's order table resident in shared memory (FXENV_ORDER_SMEM=1) against
the one that sweeps the table in global memory (FXENV_ORDER_SMEM=0), on envs of the BASELINE cfg2 shape (W=128, F=5,
direct_fixed_sltp, pnl): rewards, done flags, the observation ring, every info column and the whole state snapshot
(order tables included, stale entries past n_orders too) bit for bit, after every batch.  Each case then advances both
envs 64 single steps in lockstep: the single-step kernel reads the order tables in global memory, so a table the
resident kernel failed to write back shows up as a divergence there.

The host-side choice of the variant (shared-memory budget at 16 warps per SM) is pure arithmetic and runs without a GPU."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import scenarios as S
from gym_fx_b200 import _native
from gym_fx_b200.config import lower_config
from gym_fx_b200.synth import start_offsets, synth_candles, synth_minutes


def _choice(window, n_cols, ring, cap, force=-1):
    f = _native.load().fxenv_debug_order_smem
    f.argtypes = [C.c_int] * 5
    f.restype = C.c_int
    return f(window, n_cols, ring, cap, force)


def test_order_smem_variant_follows_the_shared_memory_budget():
    # per warp: candle window + statistics + carry record + mbarrier (5,640 B at W=128, 5 columns) + 28 B per table entry
    # (cap + 32 slack entries); 4 warps per CTA, 4 CTAs + 1 KB each must fit the SM's 228 KB
    assert _choice(128, 5, 0, 256) == 1        # cfg2: 13,704 B per warp
    assert _choice(128, 5, 0, 32) == 1
    assert _choice(128, 5, 0, 288) == 0        # 14,600 B per warp: 16 warps no longer fit
    assert _choice(128, 5, 64, 256) == 1       # a 64-return Sharpe ring still fits ...
    assert _choice(128, 5, 80, 256) == 0       # ... an 80-return one does not
    assert _choice(256, 5, 0, 256) == 0        # cfg3
    assert _choice(512, 5, 64, 256) == 0       # cfg5
    assert _choice(256, 5, 0, 256, force=1) == 1 and _choice(128, 5, 0, 256, force=0) == 0  # FXENV_ORDER_SMEM
    assert _choice(0, 5, 0, 256) < 0 and _choice(128, 5, 0, 0) < 0


def _mk(N, T, **kw):
    cfgd = {**S.DEFAULTS, "window_size": 128, "feature_columns": list(S.OHLCV), **kw.pop("cfgd", {})}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, "strategy": "direct_fixed_sltp",
                                       "preprocessor": "feature_window_preprocessor"})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"],
                       preprocessor_plugin=pl["preprocessor"], reward_plugin=pl["reward"], columns=S.OHLCV,
                       num_envs=N, **kw)
    return cfg, [synth_candles(T, 0)], [synth_minutes(T)]


def _run(resident, chunk, cfg, candles, minutes, starts, acts, singles):
    from gym_fx_b200.vec_env import VecFxEnv
    keys = ("FXENV_ORDER_SMEM", "FXENV_ENGINE", "FXENV_CHUNK")
    os.environ.update({"FXENV_ORDER_SMEM": str(resident), "FXENV_ENGINE": "persistent", "FXENV_CHUNK": str(chunk)})
    try:
        env = VecFxEnv(cfg, candles, minutes)
        env.reset(torch.as_tensor(starts))
        B, K, N = acts.shape
        out = []
        for b in range(B):
            ring = torch.zeros((3, N, env.obs_dim), dtype=torch.float32, device="cuda")
            rews = torch.zeros((K, N), dtype=torch.float32, device="cuda")
            terms = torch.zeros((K, N), dtype=torch.uint8, device="cuda")
            env.step_many(acts[b], ring, rews, terms)
            torch.cuda.synchronize()
            inf = env.info()
            out.append({"ring": ring.cpu(), "rews": rews.cpu(), "terms": terms.cpu(), "run_stats": env.run_stats().cpu(),
                        "state": torch.frombuffer(bytearray(env.get_state()), dtype=torch.uint8),
                        **{k: inf[k].cpu() for k in _native.INFO_DTYPES}})
    finally:
        for k in keys:
            os.environ.pop(k, None)
    for k in range(singles.shape[0]):
        obs, rew, term, _, inf = env.step(singles[k])
        out.append({"obs": obs.cpu(), "rew": rew.cpu(), "rew64": env.reward64.cpu(), "term": term.cpu(),
                    "run_stats": env.run_stats().cpu(), **{c: inf[c].cpu() for c in _native.INFO_DTYPES}})
    out[-1]["state"] = torch.frombuffer(bytearray(env.get_state()), dtype=torch.uint8)
    env.close()
    return out


def _agree(tag, cfg, candles, minutes, starts, chunk, K=70, batches=2, seed=0):
    N = cfg.num_envs
    g = torch.Generator().manual_seed(seed)
    acts = torch.randint(0, 3, (batches, K, N), dtype=torch.int32, generator=g).cuda()
    singles = torch.randint(0, 3, (64, N), dtype=torch.int32, generator=g).cuda()
    a = _run(1, chunk, cfg, candles, minutes, starts, acts, singles)
    b = _run(0, chunk, cfg, candles, minutes, starts, acts, singles)
    for i, (x, y) in enumerate(zip(a, b)):
        where = f"batch {i}" if i < batches else f"single step {i - batches}"
        for k in x:
            assert torch.equal(x[k], y[k]), f"{tag}, {where}: {k} differs between the resident and the global order table"
    return b


@pytest.mark.gpu
@pytest.mark.parametrize("chunk", [1, 7, 64])
def test_resident_table_matches_global_table_chunk_lengths(chunk):
    """More envs than resident warps (tickets change warps), a batch length that no chunk divides, episodes that end
    (exhausted, no auto-reset: the terminated branch runs inside tickets)."""
    N, T = 3000, 4000
    cfg, candles, minutes = _mk(N, T, order_capacity=256, episode_bars=120)
    out = _agree(f"chunk {chunk}", cfg, candles, minutes, start_offsets(N, T, 300, 300), chunk)
    assert out[-1]["n_orders"].max() > 32                 # sweeps of more than one chunk of 32 entries
    assert int(out[1]["terms"].sum()) > 0                 # episodes ended inside the batches


@pytest.mark.gpu
def test_resident_table_broke_exhausted_auto_reset_and_cold_check_submitted():
    """A small account against large orders: the check_submitted cash bound fails, so the exact simulation (cold path)
    runs on the shared copy and rejects orders; envs go broke or exhaust 40-bar episodes and auto-reset mid-ticket."""
    N, T = 3000, 4000
    cfg, candles, minutes = _mk(N, T, cfgd=dict(position_size=1500.0, initial_cash=2000.0, min_equity=1999.0),
                                order_capacity=256, auto_reset=True, episode_bars=40)
    out = _agree("broke / cold", cfg, candles, minutes, start_offsets(N, T, 300, 300), 64, seed=1)
    terms = torch.cat([o["terms"] for o in out[:2]]).sum()
    assert int(terms) >= N                                 # every env ended (and restarted) at least once
    fl = np.asarray([o["flags"].numpy() for o in out[2:]])
    assert (fl & 8).any() and (fl & 4).any()               # broke and exhausted episodes (FX_FLAG_BROKE / _EXHAUSTED)


@pytest.mark.gpu
def test_resident_table_at_capacity_and_overflow():
    """order_capacity=32: tables run full and the overflow flag is raised; pushes land in the slack entries."""
    N, T = 3000, 4000
    cfg, candles, minutes = _mk(N, T, cfgd=dict(sl_pips=80.0, tp_pips=120.0), order_capacity=32)
    out = _agree("capacity 32", cfg, candles, minutes, start_offsets(N, T, 300, 300), 64, seed=2)
    assert (out[-1]["flags"].numpy() & 16).any()
    assert 24 <= int(out[-1]["n_orders"].max()) <= 32
