"""CPU (-m "not gpu"): per-env broker and strategy parameters (fxenv_set_env_params) in the product's scalar core, and the
table helper of VecFxEnv.set_env_params.

The core (fx_core.cuh via tests/hostsim, with the row through tests/params_hostsim.cpp) steps with a base config c0 and a parameter row whose seven values all differ
from c0's; the C oracle steps with c0 with the row applied.  A use site that still read the config instead of the row
would trade with c0's commission, leverage, slippage or brackets and drift from the oracle."""
import ctypes as C

import numpy as np
import pytest

import scenarios as S
from gym_fx_b200.config import ENV_PARAM_FIELDS, FxConfig, env_params_table, lower_config
from gym_fx_b200.synth import synth_candles, synth_minutes
from env_params_hostsim import ParamsHostEnv
from hostsim.hostsim import HostSimEnv
from oracle.c_oracle import OracleVec

# the choice sets of tests/test_core_vs_oracle_random.py, in FXENV_PARAM_* order
CHOICES = {
    "commission": [0.0, 1e-5, 7e-5],
    "leverage": [1.0, 2.0, 30.0],
    "slippage": [0.0, 5e-5, 3e-4],
    "sl_pips": [2.0, 5.0, 20.0],
    "tp_pips": [3.0, 8.0, 40.0],
    "k_sl": [0.5, 2.0],
    "k_tp": [1.0, 3.0],
}
CFG_FIELD = dict(zip(ENV_PARAM_FIELDS, ("commission", "leverage", "slippage_perc", "sl_pips", "tp_pips", "k_sl", "k_tp")))


def with_row(cfg: FxConfig, row) -> FxConfig:
    """cfg with the seven fields of a parameter row applied (what one env of a handle with that row computes)."""
    out = FxConfig.from_buffer_copy(cfg)
    for name, v in zip(ENV_PARAM_FIELDS, row):
        setattr(out, CFG_FIELD[name], float(v))
    return out


def _random_case(seed):
    rng = np.random.default_rng(7000 + seed)
    strat = ["default_strategy", "direct_fixed_sltp", "direct_atr_sltp"][seed % 3]
    reward = ["pnl_reward", "sharpe_reward", "dd_penalized_reward"][(seed // 3) % 3]
    row, base = [], {}
    for name in ENV_PARAM_FIELDS:  # the row's value, and a different one for c0
        vals = CHOICES[name]
        i = int(rng.integers(0, len(vals)))
        j = (i + 1 + int(rng.integers(0, len(vals) - 1))) % len(vals)
        row.append(vals[i])
        base[name] = vals[j]
    cfgd = dict(S.DEFAULTS)
    cfgd.update(window_size=int(rng.integers(4, 24)), commission=base["commission"], leverage=base["leverage"],
                slippage_perc=base["slippage"], sl_pips=base["sl_pips"], tp_pips=base["tp_pips"], k_sl=base["k_sl"],
                k_tp=base["k_tp"], atr_period=int(rng.integers(3, 15)),
                position_size=float(rng.choice([1.0, 250.0, 4000.0, 9000.0])))  # the large ones hit margin rejections
    if strat == "direct_atr_sltp" and rng.random() < 0.5:
        cfgd.update(rel_volume=float(rng.choice([0.05, 0.4])), max_order_volume=20000.0,
                    size_mode=str(rng.choice(["fx_units", "notional"])))
    if reward == "sharpe_reward":
        cfgd.update(window=int(rng.integers(4, 40)))
    pair = int(rng.integers(0, 4))
    T = 700
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, "strategy": strat, "reward": reward})
    c0 = lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"], preprocessor_plugin=pl["preprocessor"],
                      reward_plugin=pl["reward"], columns=S.OHLCV, num_envs=1, order_capacity=1024,
                      pair_pip_size=[0.01 if pair == 3 else 1e-4])
    for name, v in base.items():  # also the fields this strategy does not read (lower_config leaves its defaults there)
        setattr(c0, CFG_FIELD[name], v)
    candles = synth_candles(T, pair, 8000 + seed)
    acts = S.make_actions(("sticky", 1900 + seed, float(rng.choice([0.2, 0.6, 0.85]))), T - 40)
    return c0, np.array(row), candles, synth_minutes(T), acts


@pytest.mark.parametrize("seed", range(36))
def test_core_with_a_parameter_row_matches_the_oracle(seed):
    c0, row, candles, minutes, acts = _random_case(seed)
    assert all(row[j] != getattr(c0, CFG_FIELD[n]) for j, n in enumerate(ENV_PARAM_FIELDS))
    core = ParamsHostEnv(c0, candles, minutes, row)
    orc = OracleVec(with_row(c0, row), [candles], [minutes])
    core.reset(0)
    orc.reset(np.zeros(1, np.int64))
    for k, a in enumerate(acts):
        r, t = core.step(a)
        _, _, r64, term = orc.step(np.array([a], np.int32))
        assert t == term[0], (seed, k)
        np.testing.assert_allclose(r, r64[0], rtol=1e-12, atol=1e-15, err_msg=f"seed {seed} step {k}: reward")
        ci, oi = core.info(), orc.info()
        assert not (ci["flags"] & 16), f"seed {seed}: order table overflow at step {k}"
        for key in ("position", "bar_index", "trades"):
            assert ci[key] == oi[key][0], (seed, k, key, ci[key], oi[key][0])
        for key in ("equity", "cash", "position_size", "position_price", "commission_paid", "price"):
            assert ci[key] == oi[key][0], (seed, k, key, repr(ci[key]), repr(oi[key][0]))
        if t:
            break
    rs, osum = core.stats(), {k: v[0] for k, v in orc.summary().items()}
    closed = core.info()["trades"]
    assert rs[2] == osum["max_drawdown_pct"] and rs[1] == osum["max_drawdown_money"], (seed, rs[:3], osum)
    assert (rs[9], rs[10], rs[11], closed) == (osum["trades_total"], osum["trades_won"], osum["trades_lost"], osum["trades_closed"])
    if closed:
        assert rs[6] / closed == osum["avg_trade_pnl"], (seed, rs[6] / closed, osum["avg_trade_pnl"])


def test_the_row_reaches_every_use_site():
    """Control: the same cases stepped with c0 alone (no row) leave the oracle of c0 + row in most cases -- the row is
    what makes them agree."""
    differ = 0
    for seed in range(12):
        c0, row, candles, minutes, acts = _random_case(seed)
        core = ParamsHostEnv(c0, candles, minutes)   # no row: the config's values
        orc = OracleVec(with_row(c0, row), [candles], [minutes])
        core.reset(0)
        orc.reset(np.zeros(1, np.int64))
        for a in acts[:300]:
            core.step(a)
            orc.step(np.array([a], np.int32), want_obs=False)
        differ += core.info()["equity"] != orc.info()["equity"][0]
    assert differ >= 8, differ


def test_a_row_equal_to_the_config_changes_nothing():
    c0, _, candles, minutes, acts = _random_case(4)
    row = [getattr(c0, CFG_FIELD[n]) for n in ENV_PARAM_FIELDS]
    a_, b_ = HostSimEnv(c0, candles, minutes), ParamsHostEnv(c0, candles, minutes, row)
    a_.reset(0)
    b_.reset(0)
    for a in acts:
        assert a_.step(a) == b_.step(a)
        assert a_.info() == b_.info()
    assert (a_.stats() == b_.stats()).all()


# ---- the table helper (VecFxEnv.set_env_params) ------------------------------------------------------------------------
def _cfg(n=4):
    cfgd = {**S.DEFAULTS, "commission": 2e-5, "leverage": 5.0, "slippage": 1e-4}
    pl = S.build_mirror_plugins(cfgd, {**S.DEFAULT_PLUGINS, "strategy": "direct_fixed_sltp"})
    return lower_config(cfgd, broker_plugin=pl["broker"], strategy_plugin=pl["strategy"], preprocessor_plugin=pl["preprocessor"],
                        reward_plugin=pl["reward"], columns=S.OHLCV, num_envs=n)


def test_table_none_takes_the_config_value():
    c = _cfg()
    t = env_params_table(c)
    assert t.shape == (4, 7) and t.dtype == np.float64
    want = [c.commission, c.leverage, c.slippage_perc, c.sl_pips, c.tp_pips, c.k_sl, c.k_tp]
    assert (t == np.array(want)[None, :]).all()
    assert want[:3] == [2e-5, 5.0, 1e-4]


def test_table_broadcasts_scalars_and_takes_arrays():
    import torch
    c = _cfg()
    t = env_params_table(c, commission=1e-4, sl_pips=[1, 2, 3, 4], tp_pips=np.arange(4.0) + 10,
                         k_tp=torch.tensor([0.5, 1.0, 1.5, 2.0], dtype=torch.float32), leverage=np.float32(2.0))
    assert (t[:, 0] == 1e-4).all()
    assert (t[:, 1] == 2.0).all()
    assert (t[:, 2] == c.slippage_perc).all()
    assert list(t[:, 3]) == [1, 2, 3, 4] and list(t[:, 4]) == [10, 11, 12, 13]
    assert (t[:, 5] == c.k_sl).all() and list(t[:, 6]) == [0.5, 1.0, 1.5, 2.0]


@pytest.mark.parametrize("field,value", [
    ("commission", float("nan")), ("sl_pips", float("inf")), ("k_sl", -float("inf")), ("leverage", 0.0),
    ("leverage", -1.0), ("slippage", -1e-9), ("slippage", 1.0), ("tp_pips", [1.0, 2.0, float("nan"), 3.0]),
])
def test_table_rejects_bad_values(field, value):
    with pytest.raises(ValueError, match=field):
        env_params_table(_cfg(), **{field: value})


@pytest.mark.parametrize("value", [[1.0, 2.0, 3.0], np.zeros((4, 1)), np.zeros(5)])
def test_table_rejects_a_wrong_length(value):
    with pytest.raises(ValueError, match="one per env"):
        env_params_table(_cfg(), commission=value)


@pytest.mark.parametrize("value", ["0.1", ["a", "b", "c", "d"], [True, False, True, False], object()])
def test_table_rejects_non_numeric_input(value):
    with pytest.raises(TypeError, match="numeric"):
        env_params_table(_cfg(), commission=value)


def test_table_rejects_unknown_fields():
    with pytest.raises(TypeError, match="unknown"):
        env_params_table(_cfg(), spread=1.0)
