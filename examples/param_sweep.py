#!/usr/bin/env python3
"""
examples/param_sweep.py -- a backtest grid in one handle: stop-loss x take-profit x commission on direct_fixed_sltp.

Every env of one VecFxEnv gets one grid point through VecFxEnv.set_env_params (per-env sl_pips, tp_pips, commission;
include/fxenv.h fxenv_set_env_params), starts at the same bar and receives the same seeded sticky action stream, so the
parameters are the only difference between the envs.  The run goes through step_many in batches; at the end the best
rows of summary() are printed (total return, max drawdown, SQN, closed trades), and --csv writes every row.

    python examples/param_sweep.py                                  # 16 SL x 16 TP x 4 commission = 1024 envs
    python examples/param_sweep.py --sl 5,10,20 --tp 10,20,40 --commission 0,2e-5 --bars 20000 --csv sweep.csv
    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 examples/param_sweep.py

Under torchrun every rank takes its slice of the grid (gym_fx_b200.sharding.shard_range) on its own GPU and prints /
writes its own rows (--csv gets a .rank<r> suffix).  The signal is a synthetic sticky action stream (hold probability
--hold), the data a synthetic 1-minute candle table (gym_fx_b200.synth): replace both with your own.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def floats(s):
    return [float(x) for x in s.split(",") if x.strip()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sl", type=floats, default=[float(x) for x in np.linspace(5, 80, 16)], help="stop-loss pips, comma-separated")
    ap.add_argument("--tp", type=floats, default=[float(x) for x in np.linspace(5, 80, 16)], help="take-profit pips, comma-separated")
    ap.add_argument("--commission", type=floats, default=[0.0, 1e-5, 2e-5, 5e-5], help="commission per unit notional, comma-separated")
    ap.add_argument("--bars", type=int, default=10000, help="bars of the backtest")
    ap.add_argument("--window", type=int, default=32, help="observation window (feature_window preprocessor)")
    ap.add_argument("--position-size", type=float, default=1000.0)
    ap.add_argument("--hold", type=float, default=0.97, help="probability that the action stream repeats its last action")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--batch", type=int, default=500, help="steps per step_many call")
    ap.add_argument("--top", type=int, default=10, help="rows to print, best total return first")
    ap.add_argument("--csv", default=None, help="write every row to this file")
    args = ap.parse_args()
    if args.bars < 2 or args.batch < 1:
        ap.error("--bars must be >= 2 and --batch >= 1")

    from gym_fx_b200.config import lower_config
    from gym_fx_b200.plugin_loader import DEFAULT_PLUGINS, build_plugins
    from gym_fx_b200.sharding import shard_range
    from gym_fx_b200.synth import synth_candles, synth_minutes
    from gym_fx_b200.vec_env import VecFxEnv

    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))

    grid = np.array([(sl, tp, c) for c in args.commission for sl in args.sl for tp in args.tp], np.float64)
    per = (len(grid) + world - 1) // world
    mine = [i for i in shard_range(per, rank, world) if i < len(grid)]
    if not mine:
        print(json.dumps({"example": "param_sweep", "rank": rank, "rows": 0}), flush=True)
        return
    pts = grid[mine]
    N = len(pts)

    cols = ("OPEN", "HIGH", "LOW", "CLOSE", "VOLUME")
    cfgd = {"window_size": args.window, "initial_cash": 10000.0, "position_size": args.position_size,
            "feature_columns": list(cols), "sl_pips": 20.0, "tp_pips": 40.0}
    pl = build_plugins(cfgd, {**DEFAULT_PLUGINS, "strategy": "direct_fixed_sltp", "preprocessor": "feature_window_preprocessor"})
    cfg = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"], preprocessor_plugin=pl["preprocessor"],
                       reward_plugin=pl["reward"], columns=cols, num_envs=N, order_capacity=64)
    T = args.bars + args.window + 2
    env = VecFxEnv(cfg, [synth_candles(T, 0, 1234 + args.seed)], [synth_minutes(T)])
    env.set_env_params(sl_pips=pts[:, 0], tp_pips=pts[:, 1], commission=pts[:, 2])
    env.reset(torch.zeros(N, dtype=torch.int64))

    # one sticky action stream, replayed to every env
    rng = np.random.default_rng(args.seed)
    stream = np.zeros(args.bars, np.int32)
    cur = 0
    for i in range(args.bars):
        if rng.random() > args.hold:
            cur = int(rng.integers(0, 3))
        stream[i] = cur
    acts = torch.as_tensor(np.repeat(stream[:, None], N, axis=1)).cuda()
    B = min(args.batch, args.bars)
    ring = torch.empty((1, N, env.obs_dim), dtype=torch.float32, device="cuda")
    rews = torch.empty((B, N), dtype=torch.float32, device="cuda")
    terms = torch.empty((B, N), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k0 in range(0, args.bars, B):
        kb = min(B, args.bars - k0)
        env.step_many(acts[k0:k0 + kb], ring, rews[:kb], terms[:kb])
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0

    sm = env.summary()
    ret, dd, sqn, trades = (sm[k].cpu().numpy() for k in ("total_return", "max_drawdown_pct", "sqn", "trades_closed"))
    rows = [dict(sl_pips=float(p[0]), tp_pips=float(p[1]), commission=float(p[2]), total_return=float(ret[i]), max_drawdown_pct=float(dd[i]),
                 sqn=float(sqn[i]), trades=int(trades[i])) for i, p in enumerate(pts)]
    order = np.argsort(-ret, kind="stable")
    print(f"{'sl_pips':>8} {'tp_pips':>8} {'commission':>11} {'total_return':>13} {'max_dd_%':>9} {'sqn':>8} {'trades':>7}")
    for i in order[:args.top]:
        r = rows[i]
        print(f"{r['sl_pips']:8.2f} {r['tp_pips']:8.2f} {r['commission']:11.2e} {r['total_return']:13.6f} "
              f"{r['max_drawdown_pct']:9.4f} {r['sqn']:8.3f} {r['trades']:7d}")
    if args.csv:
        path = args.csv if world == 1 else f"{args.csv}.rank{rank}"
        with open(path, "w") as f:
            f.write("sl_pips,tp_pips,commission,total_return,max_drawdown_pct,sqn,trades\n")
            for r in rows:
                f.write(f"{r['sl_pips']!r},{r['tp_pips']!r},{r['commission']!r},{r['total_return']!r},"
                        f"{r['max_drawdown_pct']!r},{r['sqn']!r},{r['trades']}\n")
    print(json.dumps({"example": "param_sweep", "rank": rank, "world": world, "rows": N, "bars": args.bars,
                      "env_bars_per_s": N * args.bars / max(dt, 1e-9), "seconds": dt,
                      "order_overflow_envs": sm["order_overflow_envs"], "device": torch.cuda.get_device_name()}), flush=True)
    env.close()


if __name__ == "__main__":
    main()
