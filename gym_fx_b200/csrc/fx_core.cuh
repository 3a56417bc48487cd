// fx_core.cuh -- scalar per-env state machine of the fused gym-fx step (broker, strategies, rewards, obs math).
//
// Everything here is FX_HD (host + device): the CUDA kernels in fx_kernels.cu call it from one warp per env
// (uniform scalar fp64 code, replicated across lanes), and tests/hostsim compiles the very same functions with
// g++ to pre-flight the logic on the CPU build box (test infrastructure only; the product has no CPU path).
//
// What it implements (reference = harveybc/gym-fx @ ad8bbc41; paths relative to the reference tree):
//   * BTBridgeStrategy._apply_action default order flow                app/bt_bridge.py:158-190
//   * direct_fixed_sltp.apply_action                                   strategy_plugins/direct_fixed_sltp.py:51-77
//   * direct_atr_sltp.apply_action / _compute_size / _session_state    strategy_plugins/direct_atr_sltp.py:110-255
//   * BTBridgeStrategy._publish_obs / _is_broke / notify_*             app/bt_bridge.py:109-117,192-204
//   * pnl / dd_penalized reward                                        reward_plugins/pnl_reward.py:26-36,
//                                                                      reward_plugins/dd_penalized_reward.py:30-47
//   * sharpe reward (sequential form)                                  reward_plugins/sharpe_reward.py:34-58
//   * the 4 agent scalars of both preprocessors                        preprocessor_plugins/default_preprocessor.py:54-76,
//                                                                      preprocessor_plugins/feature_window_preprocessor.py:209-232
//   * backtrader BackBroker (external dependency, restated): check_submitted, per-bar matching of
//     Market/Limit/Stop, bracket activation / OCO, _execute cash+position arithmetic, _get_value.
//
// Order table representation (differs from backtrader's object lists on purpose): one FIFO array of ENTRIES per
// env.  A bracket = a PARENT entry (limit at the signal bar's close) immediately followed by one PAIR entry
// holding BOTH children (stop @p0, limit @p1): the children are created adjacent, stay adjacent in backtrader's
// FIFO, are only ever (de)activated or cancelled together, and the stop is always examined first -- so one entry
// is an exact representation.  Stable compaction keeps FIFO order == array order.
//
// All arithmetic is fp64, one rounding per operation (compile with -fmad=false / -ffp-contract=off) so that
// cash/equity evolve bit-identically to the Python reference.
#pragma once

#include <math.h>
#include <stdint.h>

#include "../../include/fxenv.h"

#if defined(__CUDACC__)
#define FX_HD __host__ __device__ __forceinline__
#define FX_HD_COLD static __host__ __device__ __noinline__  // rare paths: keep them out of the hot instruction stream
#else
#define FX_HD inline
#define FX_HD_COLD inline
#endif

// ---- order-table entry encoding ---------------------------------------------------------------------------------
#define FXO_KIND_MASK 3u
#define FXO_MARKET 0u
#define FXO_PARENT 1u  // bracket parent: LIMIT @p0, signed size; the next entry is its PAIR
#define FXO_PAIR 2u    // bracket children: STOP @p0 and LIMIT @p1, signed size (opposite to the parent's)
#define FXO_SUBMITTED 4u      // created during the last strategy call; goes through check_submitted next bar
#define FXO_ACTIVE 8u         // PAIR: parent has completed and the children may trigger
#define FXO_ACTIVATE_NEXT 16u // PAIR: queued in broker._toactivate (activated at the start of the next bar)
#define FXO_DEAD 32u          // executed / cancelled / rejected: dropped by the next compaction
#define FXO_SELL 64u          // the entry's signed size is negative (lets the trigger scan skip loading the size)

struct FxBar {
  double o, h, l, c;
};

// The broker and strategy values fxenv_set_env_params can set per env, under their FxConfig names: the functions below
// that read them are templates on the source `PC` of the values, either the FxConfig itself (one value for every env)
// or this record (the env's row of the table).  The FxConfig instantiations are the code the library always had.
struct FxEnvParams {
  double commission, leverage, slippage_perc, sl_pips, tp_pips, k_sl, k_tp;
};

// Per-env scalar state while a step is being computed (registers).  Loaded from / stored to the device SoA.
struct FxEnvRegs {
  double cash, psize, pprice, value;
  double equity, prev_equity, price, commission_paid;
  int32_t position, bar_index, trades;
  uint32_t flags;
};

struct FxOrderTab {
  uint32_t* meta;
  double* p0;
  double* p1;
  double* sz;
  int n;           // entries in the table (live + not-yet-compacted dead ones)
  int cap;         // logical capacity (live entries); the arrays hold cap + FXO_SLACK
  int dirty_from;  // smallest index whose stored copy is stale (n => nothing to write back)
  int ndead;       // entries marked FXO_DEAD since the last compaction
  double sub_need; // sum of fx_submit_cash_bound over the entries pushed by this strategy call (set by fx_push)
  double bound_per; // max(1, 1/leverage) + |commission|, the per-unit-notional factor of that bound
};

#define FXO_SLACK 32  // physical head-room: new orders are appended before the dead ones are compacted away

FX_HD void fx_kill(FxOrderTab& t, int k) {
  const uint32_t m = t.meta[k];
  if (!(m & FXO_DEAD)) {
    t.meta[k] = m | FXO_DEAD;
    t.ndead++;
    if (k < t.dirty_from) t.dirty_from = k;
  }
}

// ---- Position.update (backtrader position.py) ------------------------------------------------------------------
FX_HD void fx_pos_update(double& psize, double& pprice, double size, double price, double& opened, double& closed) {
  const double oldsize = psize;
  psize = oldsize + size;
  if (psize == 0.0) {
    opened = 0.0; closed = size; pprice = 0.0;
  } else if (oldsize == 0.0) {
    opened = size; closed = 0.0; pprice = price;
  } else if (oldsize > 0.0) {
    if (size > 0.0) { opened = size; closed = 0.0; pprice = (pprice * oldsize + size * price) / psize; }
    else if (psize > 0.0) { opened = 0.0; closed = size; }
    else { opened = psize; closed = -oldsize; pprice = price; }
  } else {
    if (size < 0.0) { opened = size; closed = 0.0; pprice = (pprice * oldsize + size * price) / psize; }
    else if (psize < 0.0) { opened = 0.0; closed = size; }
    else { opened = psize; closed = -oldsize; pprice = price; }
  }
}

// ---- BackBroker._execute, pseudo form (check_submitted): runs on a cash / position CLONE at created.price -------
template <class PC>
FX_HD void fx_pseudo_execute(const PC& c, double size, double price, double& cash, double& ps, double& pp) {
  double opened, closed;
  fx_pos_update(ps, pp, size, price, opened, closed);
  if (closed != 0.0) {
    const double closedvalue = (-closed) * price;  // pprice_orig == created.price in pseudo mode
    double closecash = closedvalue;
    if (closedvalue > 0.0 && c.leverage != 1.0) closecash /= c.leverage;
    cash += closecash + 0.0;                       // pnl = 0 in pseudo mode
    cash -= fabs(closed) * c.commission * price;
  }
  if (opened != 0.0) {
    const double openedvalue = opened * price;
    double opencash = openedvalue;
    if (openedvalue > 0.0 && c.leverage != 1.0) opencash /= c.leverage;
    cash -= opencash;
    cash -= fabs(opened) * c.commission * price;
  }
}

// ---- end-of-run statistics: what backtrader's DrawDown / TradeAnalyzer / SQN analyzers (attached by
// app/bt_bridge.py:230-234) hold when the run ends; GymFxEnv.summary() -> metrics_plugins/default_metrics.py:48-60 reads
// max.drawdown, max.moneydown, total.total, won.total, lost.total, pnl.net.average and sqn from them.  One record of
// FX_RS_N doubles per env (the counters are stored as doubles: exact far beyond any run length).
//
// The per-fill part sits inside the hottest loop of the step (FIFO execution of the triggered orders), so it is kept to a
// few operations: the open trade's average price is NOT tracked while it equals the position's average price (which
// Position.update maintains with the very same recurrence) -- only when backtrader's Trade.update and Position.update
// diverge (a trade opened with a size for which (size * price) / size != price, or an opening bit absorbed by rounding)
// does FX_FLAG_TRADE_PRICE_OWN get set and the price kept in the record.  SQN uses the sums of pnl and pnl^2 of the
// closed trades (no division per trade; evaluated at summary time, 1e-9 relative to backtrader's fsum-based value).
enum {
  FX_RS_DD_MAXVALUE = 0,  // DrawDown._maxvalue: running peak of the broker value
  FX_RS_DD_MAX_MONEY,     // max.moneydown
  FX_RS_DD_MAX_PCT,       // max.drawdown (percent)
  FX_RS_TR_PNL,           // open Trade: gross pnl so far
  FX_RS_TR_COMM,          // open Trade: commission so far
  FX_RS_TR_PRICE,         // open Trade: average price, valid only while FX_FLAG_TRADE_PRICE_OWN is set
  FX_RS_PNL_NET,          // TradeAnalyzer pnl.net.total = sum of pnlcomm over closed trades
  FX_RS_PNL_SQ,           // sum of pnlcomm^2 over closed trades (SQN)
  FX_RS_SPARE,
  FX_RS_OPENED,           // TradeAnalyzer total.total (trades opened)
  FX_RS_WON,              // won.total  (pnlcomm >= 0)
  FX_RS_LOST,             // lost.total
  FX_RS_N
};


// Accessor the execution code is written against: the device keeps field i in lane i of one register (a single
// coalesced load / store of the record per env-step), the host build and the reset path use a plain array.
struct FxRunStatsMem {
  double* v;
  FX_HD double get(int i) const { return v[i]; }
  FX_HD void set(int i, double x) const { v[i] = x; }
  FX_HD void add(int i, double x) const { v[i] += x; }
};

struct FxRunStatsNone {  // statistics not tracked by this caller
  FX_HD double get(int) const { return 0.0; }
  FX_HD void set(int, double) const {}
  FX_HD void add(int, double) const {}
};

template <class RS> struct FxRsOn { static const bool value = true; };
template <> struct FxRsOn<FxRunStatsNone> { static const bool value = false; };

// DrawDown analyzer, one bar: notify_fund(value) then next()  [backtrader analyzers/drawdown.py, restated]
template <class RS>
FX_HD void fx_rs_drawdown(const RS& rs, double value) {
  double maxv = rs.get(FX_RS_DD_MAXVALUE);
  if (value > maxv) { maxv = value; rs.set(FX_RS_DD_MAXVALUE, maxv); }
  const double md = maxv - value;
  if (md > rs.get(FX_RS_DD_MAX_MONEY)) rs.set(FX_RS_DD_MAX_MONEY, md);
  // max.drawdown = max(max.drawdown, 100 * md / maxvalue): the division only when it can matter
  const double mp = rs.get(FX_RS_DD_MAX_PCT);
  if (100.0 * md > mp * maxv * 0.999999) {
    const double pct = 100.0 * md / maxv;
    if (pct > mp) rs.set(FX_RS_DD_MAX_PCT, pct);
  }
}

// Strategy._addnotification -> Trade.update for the two bits of one execution (closing part first, then the opening
// part), and the analyzers' notify_trade when the trade closes / opens  [backtrader strategy.py, trade.py,
// analyzers/tradeanalyzer.py, analyzers/sqn.py, restated].  oldsize / pprice_orig: the position before the execution,
// pprice_new: its average price after; pnl = (-closed) * (price - pprice_orig) as computed by _execute.
template <class RS>
FX_HD void fx_rs_trade(const RS& rs, uint32_t& flags, double oldsize, double closed, double opened, double price,
                       double pnl, double pprice_orig, double pprice_new, double closedcomm, double openedcomm, bool has_comm) {
  const bool own = (flags & FX_FLAG_TRADE_PRICE_OWN) != 0u;
  if (closed != 0.0) {
    if (has_comm) rs.add(FX_RS_TR_COMM, closedcomm);
    // comminfo.profitandloss(-size, trade.price, price); trade.price == position price unless flagged
    rs.add(FX_RS_TR_PNL, own ? (-closed) * (price - rs.get(FX_RS_TR_PRICE)) : pnl);
    if (oldsize + closed == 0.0) {         // trade.isclosed
      const double pnlcomm = rs.get(FX_RS_TR_PNL) - (has_comm ? rs.get(FX_RS_TR_COMM) : 0.0);
      rs.add(pnlcomm >= 0.0 ? FX_RS_WON : FX_RS_LOST, 1.0);
      rs.add(FX_RS_PNL_NET, pnlcomm);
      rs.add(FX_RS_PNL_SQ, pnlcomm * pnlcomm);
      rs.set(FX_RS_TR_PNL, 0.0);           // the next opening bit starts a fresh Trade()
      if (has_comm) rs.set(FX_RS_TR_COMM, 0.0);
      flags &= ~FX_FLAG_TRADE_PRICE_OWN;
    }
  }
  if (opened != 0.0) {
    const double tsize = oldsize + closed, nsize = tsize + opened;
    if (has_comm) rs.add(FX_RS_TR_COMM, openedcomm);
    if (tsize == 0.0) {                    // trade.justopened: price = (0 * 0 + size * price) / size
      rs.add(FX_RS_OPENED, 1.0);
      if (fabs(opened) != 1.0) {           // exact for unit sizes; otherwise it can be one ulp off the fill price
        const double tp = (opened * price) / nsize;
        if (tp != price) { rs.set(FX_RS_TR_PRICE, tp); flags |= FX_FLAG_TRADE_PRICE_OWN; }
      }
    } else if (fabs(nsize) > fabs(tsize)) {  // increased: the same recurrence as Position.update while the prices agree
      if (flags & FX_FLAG_TRADE_PRICE_OWN) rs.set(FX_RS_TR_PRICE, (tsize * rs.get(FX_RS_TR_PRICE) + opened * price) / nsize);
    } else {
      // Trade.update decides by |size after| > |size before|: an opening bit too small to change the size (absorbed by
      // rounding, e.g. the close() of a 1e-12 dust position executing after the position has flipped) books a pnl and
      // leaves the trade's price alone, while Position.update re-averages: from here on the two prices differ
      const double tp = (flags & FX_FLAG_TRADE_PRICE_OWN) ? rs.get(FX_RS_TR_PRICE) : pprice_orig;
      rs.add(FX_RS_TR_PNL, (-opened) * (price - tp));
      if (!(flags & FX_FLAG_TRADE_PRICE_OWN) && pprice_new != pprice_orig) { rs.set(FX_RS_TR_PRICE, pprice_orig); flags |= FX_FLAG_TRADE_PRICE_OWN; }
    }
  }
}

// ---- BackBroker._execute, real form.  Returns true if the order ended in Margin (=> cancel its bracket group) --
// PLAIN (compile time): commission == 0 and leverage == 1 -- the arithmetic that those values turn into identities
// (x / 1.0, x - 0.0) is left out; every remaining operation and its order are unchanged.
template <bool PLAIN, class RS, class PC>
FX_HD bool fx_execute(const PC& c, FxEnvRegs& e, double size, double price, const RS& rs) {
  const double pprice_orig = e.pprice, oldsize = e.psize;
  double ps = e.psize, pp = e.pprice, opened, closed;
  fx_pos_update(ps, pp, size, price, opened, closed);  // pseudoupdate on a clone
  const double pnl = (-closed) * (price - pprice_orig) * 1.0;
  double cash = e.cash;
  double closedcomm = 0.0, openedcomm = 0.0;
  if (closed != 0.0) {
    const double closedvalue = (-closed) * pprice_orig;
    double closecash = closedvalue;
    if (!PLAIN && closedvalue > 0.0 && c.leverage != 1.0) closecash /= c.leverage;
    cash += closecash + pnl * 1.0;
    if (!PLAIN) {
      closedcomm = fabs(closed) * c.commission * price;
      cash -= closedcomm;
    }
    cash += 0.0;  // stock-like cashadjust
    e.cash = cash;
  }
  const double popened = opened;
  if (opened != 0.0) {
    const double openedvalue = opened * price;
    double opencash = openedvalue;
    if (!PLAIN && openedvalue > 0.0 && c.leverage != 1.0) opencash /= c.leverage;
    cash -= opencash;
    if (!PLAIN) {
      openedcomm = fabs(opened) * c.commission * price;
      cash -= openedcomm;
    }
    if (cash < 0.0) { opened = 0.0; openedcomm = 0.0; }
    else e.cash = cash;
  }
  const bool margin = (popened != 0.0 && opened == 0.0);
  const double execsize = closed + opened;
  if (execsize != 0.0) {
    if (execsize == size) { e.psize = ps; e.pprice = pp; }  // position.update(execsize) is then exactly the clone's update
    else { double o2, c2; fx_pos_update(e.psize, e.pprice, execsize, price, o2, c2); }
    // Trade bookkeeping (strategy._addnotification): a trade closes when the closing part of the execution
    // brings the position to exactly 0 -> BTBridgeStrategy.notify_trade (app/bt_bridge.py:115-117)
    if (closed != 0.0 && oldsize + closed == 0.0) e.trades += 1;
    if (FxRsOn<RS>::value)
      fx_rs_trade(rs, e.flags, oldsize, closed, opened, price, pnl, pprice_orig, e.pprice, closedcomm, openedcomm,
                  !PLAIN && c.commission != 0.0);
    // BTBridgeStrategy.notify_order counts commission of COMPLETED orders only (app/bt_bridge.py:109-113)
    if (!PLAIN && size - execsize == 0.0) {
      double ocomm = 0.0;
      ocomm += closedcomm + openedcomm;
      e.commission_paid += ocomm;
    }
  }
  return margin;
}

// ---- matching rules (bbroker.py _try_exec_market / _try_exec_limit / _try_exec_stop) -----------------------------
// Slippage: BackBroker._slip_up / _slip_down as configured by the reference (set_slippage_perc(perc, slip_open=True,
// slip_limit=True, slip_match=True), slip_out=False -- broker_plugins/default_broker.py:50-51): the slipped price,
// capped at the bar's extreme.  perc == 0 must bypass the cap (bars whose OPEN lies outside [LOW, HIGH] exist).
FX_HD double fx_slip_up(double s, double pmax, double price) {
  if (s == 0.0) return price;
  const double pslip = price * (1 + s);
  return pslip <= pmax ? pslip : pmax;
}
FX_HD double fx_slip_down(double s, double pmin, double price) {
  if (s == 0.0) return price;
  const double pslip = price * (1 - s);
  return pslip >= pmin ? pslip : pmin;
}

FX_HD double fx_market_price(double s, bool buy, const FxBar& b) {
  return buy ? fx_slip_up(s, b.h, b.o) : fx_slip_down(s, b.l, b.o);
}

FX_HD bool fx_match_limit(double s, bool buy, double plimit, const FxBar& b, double& px) {
  if (buy) {
    if (plimit >= b.o) { px = fx_slip_up(s, b.h < plimit ? b.h : plimit, b.o); return true; }
    if (plimit >= b.l) { px = plimit; return true; }
  } else {
    if (plimit <= b.o) { px = fx_slip_down(s, plimit, b.o); return true; }  // bbroker passes plimit, not max(low, plimit)
    if (plimit <= b.h) { px = plimit; return true; }
  }
  return false;
}

FX_HD bool fx_match_stop(double s, bool buy, double pstop, const FxBar& b, double& px) {
  if (buy) {
    if (b.o >= pstop) { px = fx_slip_up(s, b.h, b.o); return true; }
    if (b.h >= pstop) { px = fx_slip_up(s, b.h, pstop); return true; }
  } else {
    if (b.o <= pstop) { px = fx_slip_down(s, b.l, b.o); return true; }
    if (b.l <= pstop) { px = fx_slip_down(s, b.l, pstop); return true; }
  }
  return false;
}

// Would entry k trade against bar b?  Pure function of the entry and the bar (lane-parallel on the device).
// The ACTIVE / DEAD / SUBMITTED state is deliberately NOT consulted here: it can change during the FIFO walk.
FX_HD bool fx_entry_hits(uint32_t meta, double p0, double p1, const FxBar& b) {
  const uint32_t kind = meta & FXO_KIND_MASK;
  const bool buy = !(meta & FXO_SELL);
  double px;
  if (kind == FXO_MARKET) return true;
  if (kind == FXO_PARENT) return fx_match_limit(0.0, buy, p0, b, px);
  return fx_match_stop(0.0, buy, p0, b, px) || fx_match_limit(0.0, buy, p1, b, px);
}

// Same test, also returning the execution price (select form: every lane of a warp evaluates it without divergence).
// The price is a pure function of (entry, bar) as well, so the FIFO walk only has to fetch it from the owning lane.
FX_HD bool fx_entry_fill(double s, uint32_t meta, double p0, double p1, const FxBar& b, double& px) {
  const uint32_t kind = meta & FXO_KIND_MASK;
  const bool buy = !(meta & FXO_SELL);
  // stop @p0 (PAIR) -- bbroker.py _try_exec_stop
  const bool s_open = buy ? (b.o >= p0) : (b.o <= p0);
  const bool s_hit = s_open || (buy ? (b.h >= p0) : (b.l <= p0));
  // limit @p0 (PARENT) or @p1 (PAIR) -- bbroker.py _try_exec_limit
  const double pl = (kind == FXO_PARENT) ? p0 : p1;
  const bool l_open = buy ? (pl >= b.o) : (pl <= b.o);
  const bool l_hit = l_open || (buy ? (pl >= b.l) : (pl <= b.h));
  bool hit;
  double base, cap;  // un-slipped price and the bound the slipped price is capped at
  bool slips = true;
  if (kind == FXO_MARKET) { hit = true; base = b.o; cap = buy ? b.h : b.l; }
  else if (kind == FXO_PAIR && s_hit) { hit = true; base = s_open ? b.o : p0; cap = buy ? b.h : b.l; }
  else { hit = l_hit; base = l_open ? b.o : pl; slips = l_open; cap = buy ? (b.h < pl ? b.h : pl) : pl; }
  px = base;
  if (s != 0.0 && slips) px = buy ? fx_slip_up(s, cap, base) : fx_slip_down(s, cap, base);
  return hit;
}

// ---- BackBroker.next, step 0: "while self._toactivate: activate()" -- per entry, lane-parallel on the device ------
FX_HD uint32_t fx_entry_begin_bar(uint32_t meta) {
  return (meta & FXO_ACTIVATE_NEXT) ? ((meta & ~FXO_ACTIVATE_NEXT) | FXO_ACTIVE) : meta;
}

// ---- BackBroker.next, step 1: check_submitted over the entries created by the previous strategy call ------------
// (they are the tail [k_begin, n) of the table).  Running pseudo-cash over ONE position clone, in submission order;
// the running cash is NOT restored after a rejection (bbroker.py keeps the negative value for the rest of the batch).
template <class PC>
FX_HD void fx_check_submitted_t(const PC& c, const FxEnvRegs& e, FxOrderTab& t, int k_begin) {
  double cash = e.cash, ps = e.psize, pp = e.pprice;
  for (int k = k_begin; k < t.n; k++) {
    const uint32_t m = t.meta[k];
    if (!(m & FXO_SUBMITTED) || (m & FXO_DEAD)) continue;
    const uint32_t kind = m & FXO_KIND_MASK;
    const double sz = t.sz[k];
    bool margin = false;
    fx_pseudo_execute(c, sz, t.p0[k], cash, ps, pp);  // market / limit parent / stop child at created.price
    margin = !(cash >= 0.0);
    if (kind == FXO_PAIR && !margin) {                // then the limit child
      fx_pseudo_execute(c, sz, t.p1[k], cash, ps, pp);
      margin = !(cash >= 0.0);
    }
    if (!margin) {
      t.meta[k] = m & ~FXO_SUBMITTED;
      if (k < t.dirty_from) t.dirty_from = k;
      continue;
    }
    fx_kill(t, k);
    if (kind == FXO_PARENT) fx_kill(t, k + 1);  // children: _take_children -> Rejected
    if (kind == FXO_PAIR) fx_kill(t, k - 1);    // a child going Margin cancels the (already accepted) group
  }
}
FX_HD_COLD void fx_check_submitted(const FxConfig& c, const FxEnvRegs& e, FxOrderTab& t, int k_begin) {
  fx_check_submitted_t(c, e, t, k_begin);
}
FX_HD_COLD void fx_check_submitted(const FxEnvParams& c, const FxEnvRegs& e, FxOrderTab& t, int k_begin) {
  fx_check_submitted_t(c, e, t, k_begin);
}

// Upper bound of the pseudo-cash that check_submitted can take away for one submitted entry: every pseudo-execution
// lowers the running cash by at most |size| * price * (max(1, 1/leverage) + commission) (closing a short or opening a
// long; the other two cases ADD cash).  A PAIR is two pseudo-executions (stop child @p0, limit child @p1).
// If cash >= 1.001 * (sum of the bounds of all submitted entries) no order can be rejected, and the exact sequential
// simulation can be skipped without changing any outcome (the simulation only decides accept / reject).
template <class PC>
FX_HD double fx_bound_per(const PC& c) { return (c.leverage < 1.0 ? 1.0 / c.leverage : 1.0) + fabs(c.commission); }

template <class PC>
FX_HD double fx_submit_cash_bound(const PC& c, uint32_t meta, double p0, double p1, double sz) {
  const double per = fx_bound_per(c);
  double need = fabs(sz) * fabs(p0) * per;
  if ((meta & FXO_KIND_MASK) == FXO_PAIR) need += fabs(sz) * fabs(p1) * per;
  return need;
}

// ---- BackBroker.next, step 2: execute entry k (known to hit) in FIFO position ------------------------------------
// p: the broker values (the config, or the env's row of the per-env table)
template <class RS, class PC>
FX_HD void fx_exec_entry(const FxConfig& c, const PC& p, FxEnvRegs& e, FxOrderTab& t, int k, const FxBar& b, const RS& rs) {
  const uint32_t m = t.meta[k];
  if (m & (FXO_DEAD | FXO_SUBMITTED)) return;
  const uint32_t kind = m & FXO_KIND_MASK;
  const bool buy = !(m & FXO_SELL);
  const double s = p.slippage_perc;
  double px = b.o;
  bool go;
  if (kind == FXO_MARKET) { go = true; px = fx_market_price(s, buy, b); }
  else if (kind == FXO_PARENT) go = fx_match_limit(s, buy, t.p0[k], b, px);
  else go = (m & FXO_ACTIVE) && (fx_match_stop(s, buy, t.p0[k], b, px) || fx_match_limit(s, buy, t.p1[k], b, px));
  if (!go) return;
  // Completed or Margin: either way the entry leaves the table.  A child that completes cancels its sibling, a child
  // or parent that goes Margin cancels its whole group -- for a PAIR both mean "the pair is gone".
  const bool margin = fx_execute<false>(p, e, t.sz[k], px, rs);
  fx_kill(t, k);
  if (kind == FXO_PARENT) {
    if (margin) fx_kill(t, k + 1);
    else t.meta[k + 1] |= (c.children_same_bar ? FXO_ACTIVE : FXO_ACTIVATE_NEXT);
  }
}
template <class RS>
FX_HD void fx_exec_entry(const FxConfig& c, FxEnvRegs& e, FxOrderTab& t, int k, const FxBar& b, const RS& rs) {
  fx_exec_entry(c, c, e, t, k, b, rs);
}

// ---- BackBroker._get_value (shortcash valuation; the long side is un-levered) -------------------------------------
template <bool PLAIN = false, class PC>
FX_HD void fx_mark_to_market(const PC& c, FxEnvRegs& e, double pclose) {
  double unl = 0.0;
  double dvalue = e.psize * pclose;
  const double dunreal = e.psize * (pclose - e.pprice) * 1.0;
  if (dvalue > 0.0) { dvalue -= dunreal; unl += PLAIN ? dvalue : dvalue / c.leverage; unl += dunreal; }
  else unl += dvalue;
  e.value = e.cash + unl;
}

// ---- order creation (Strategy.buy/sell/close/buy_bracket/sell_bracket) -------------------------------------------
FX_HD bool fx_room(FxOrderTab& t, int need, uint32_t& flags) {
  if (t.n - t.ndead + need <= t.cap && t.n + need <= t.cap + FXO_SLACK) return true;
  flags |= FX_FLAG_ORDER_OVERFLOW;
  return false;
}

FX_HD void fx_push(FxOrderTab& t, uint32_t meta, double p0, double p1, double sz) {
  t.sub_need += fabs(sz) * fabs(p0) * t.bound_per;
  if ((meta & FXO_KIND_MASK) == FXO_PAIR) t.sub_need += fabs(sz) * fabs(p1) * t.bound_per;
  const int k = t.n++;
  t.meta[k] = meta | (sz < 0.0 ? FXO_SELL : 0u); t.p0[k] = p0; t.p1[k] = p1; t.sz[k] = sz;
  if (k < t.dirty_from) t.dirty_from = k;
}

FX_HD void fx_order_market(FxOrderTab& t, double size, double pclose) {
  if (size != 0.0) fx_push(t, FXO_MARKET | FXO_SUBMITTED, pclose, 0.0, size);
}

// OrderBase.__init__: "if not self.price" -> created.price = close of the creation bar (also for price == 0.0)
FX_HD void fx_order_bracket(FxOrderTab& t, bool buy, double size, double stopprice, double limitprice, double pclose) {
  const double s = buy ? fabs(size) : -fabs(size);
  fx_push(t, FXO_PARENT | FXO_SUBMITTED, pclose, 0.0, s);
  fx_push(t, FXO_PAIR | FXO_SUBMITTED, stopprice != 0.0 ? stopprice : pclose, limitprice != 0.0 ? limitprice : pclose, -s);
}

FX_HD int fx_close_need(double pos) { return pos != 0.0 ? 1 : 0; }

FX_HD void fx_order_close(FxOrderTab& t, double pos, double pclose) {
  if (pos > 0.0) fx_order_market(t, -fabs(pos), pclose);
  else if (pos < 0.0) fx_order_market(t, fabs(pos), pclose);
}

// direct_atr_sltp._compute_size (strategy_plugins/direct_atr_sltp.py:204-224)
FX_HD double fx_atr_size(const FxConfig& c, double cash, double pclose) {
  if (!c.use_rel_volume) return c.strat_position_size;
  double raw;
  if (c.size_mode == FX_SIZE_NOTIONAL) raw = pclose > 0.0 ? (cash * c.rel_volume * c.strat_leverage) / pclose : 0.0;
  else raw = cash * c.rel_volume * c.strat_leverage;
  const double m = raw < c.max_order_volume ? raw : c.max_order_volume;
  return c.min_order_volume > m ? c.min_order_volume : m;
}

// direct_atr_sltp: true range of one bar (:121-126)
FX_HD double fx_true_range(double high, double low, double prev_close, bool has_prev) {
  if (!has_prev) return high - low;
  double tr = high - low;
  const double b = fabs(high - prev_close), d = fabs(low - prev_close);
  if (b > tr) tr = b;
  if (d > tr) tr = d;
  return tr;
}

// CPython >= 3.12 sum(): Neumaier step. Start with s = x0, comp = 0; finish with fx_neumaier_done.
FX_HD void fx_neumaier_add(double& s, double& comp, double x) {
  const double t = s + x;
  if (fabs(s) >= fabs(x)) comp += (s - t) + x;
  else comp += (x - t) + s;
  s = t;
}

FX_HD double fx_neumaier_done(double s, double comp) {
  if (comp != 0.0 && !isinf(comp) && !isnan(comp)) s += comp;
  return s;
}

// direct_atr_sltp._session_state (:233-255): minute of the week from minutes since the Unix epoch
FX_HD void fx_session_state(const FxConfig& c, int64_t minutes, bool& in_entry, bool& in_close) {
  int64_t day = minutes / 1440, mod = minutes % 1440;
  if (mod < 0) { mod += 1440; day -= 1; }
  const int64_t wd = ((day + 3) % 7 + 7) % 7;  // 1970-01-01 was a Thursday (weekday() == 3)
  const int64_t cur = wd * 1440 + mod;
  const int64_t st = (int64_t)c.entry_dow_start * 1440 + (int64_t)c.entry_hour_start * 60;
  const int64_t en = (int64_t)c.force_close_dow * 1440 + (int64_t)c.force_close_hour * 60;
  in_entry = (st <= cur && cur < en);
  in_close = !in_entry;
}

// The decision direct_atr_sltp reports to its bracket audit (strategy_plugins/direct_atr_sltp.py:138-142, :188-191,
// :199-202): kind FXENV_AU_KIND_* (FXENV_AU_KIND_NONE: no record this call); stop / limit / size / atr as the reference
// logs them (size = the signed position before the close for a session force-close, whose stop / limit / atr are unset).
// Set whether or not the orders find room in the table: the reference's order list is unbounded.
struct FxAudit {
  int kind;
  double stop, limit, size, atr;
};

// ---- BTBridgeStrategy._apply_action at the current bar ------------------------------------------------------------
// atr / atr_ready: simple-mean ATR of the env's TR deque (only read for FX_STRATEGY_ATR_SLTP).
// au: the ATR strategy's audit record of this call (the other strategies leave it untouched).
// p: sl_pips / tp_pips / k_sl / k_tp (the config, or the env's row of the per-env table).
template <class PC>
FX_HD void fx_apply_action(const FxConfig& c, const PC& p, int strategy, FxEnvRegs& e, FxOrderTab& t, int action,
                           const FxBar& b, int pair, double atr, bool atr_ready, bool has_minutes, int64_t minutes,
                           FxAudit& au) {
  const double pos = e.psize, pclose = b.c;
  if (strategy == FX_STRATEGY_DEFAULT) {  // app/bt_bridge.py:171-190 (market orders)
    const double size = c.position_size;
    if (action == 1) {
      if (pos < 0.0) { if (fx_room(t, 2, e.flags)) { fx_order_close(t, pos, pclose); fx_order_market(t, fabs(size), pclose); } }
      else if (pos == 0.0) { if (fx_room(t, 1, e.flags)) fx_order_market(t, fabs(size), pclose); }
    } else if (action == 2) {
      if (pos > 0.0) { if (fx_room(t, 2, e.flags)) { fx_order_close(t, pos, pclose); fx_order_market(t, -fabs(size), pclose); } }
      else if (pos == 0.0) { if (fx_room(t, 1, e.flags)) fx_order_market(t, -fabs(size), pclose); }
    }
    return;
  }
  double size, sl, tp;
  if (strategy == FX_STRATEGY_FIXED_SLTP) {  // direct_fixed_sltp.py:51-77
    if (action == 0) return;
    const double pip = c.pair_pip_size[pair] != 0.0 ? c.pair_pip_size[pair] : c.pip_size;
    size = c.strat_position_size;
    sl = p.sl_pips * pip;
    tp = p.tp_pips * pip;
  } else {  // direct_atr_sltp.py:110-202
    au.kind = FXENV_AU_KIND_NONE;
    size = fx_atr_size(c, e.cash, pclose);
    bool in_entry = true, in_close = false;
    if (c.session_filter && has_minutes) fx_session_state(c, minutes, in_entry, in_close);
    if (in_close && pos != 0.0) {
      au.kind = FXENV_AU_KIND_FORCE_CLOSE; au.size = pos;
      if (fx_room(t, 1, e.flags)) fx_order_close(t, pos, pclose);
      return;
    }
    if (action == 0) return;
    if (c.session_filter && !in_entry) return;
    if (!atr_ready || atr <= 0.0 || size <= 0.0 || pclose <= 0.0) return;
    sl = p.k_sl * atr;
    tp = p.k_tp * atr;
    if (c.use_min_frac) { const double fl = c.min_sltp_frac * pclose; if (fl > sl) sl = fl; if (fl > tp) tp = fl; }
    if (c.use_max_frac) { const double ce = c.max_sltp_frac * pclose; if (ce < sl) sl = ce; if (ce < tp) tp = ce; }
    if (tp >= pclose) tp = pclose * 0.5;
    if (action == 1 ? pos <= 0.0 : pos >= 0.0) {
      const bool buy = action == 1;
      au.kind = buy ? FXENV_AU_KIND_LONG : FXENV_AU_KIND_SHORT;
      au.stop = buy ? pclose - sl : pclose + sl;
      au.limit = buy ? pclose + tp : pclose - tp;
      au.size = size; au.atr = atr;
    }
  }
  if (action == 1) {
    if (pos <= 0.0 && fx_room(t, fx_close_need(pos) + 2, e.flags)) {
      if (pos < 0.0) fx_order_close(t, pos, pclose);
      fx_order_bracket(t, true, size, pclose - sl, pclose + tp, pclose);
    }
  } else if (action == 2) {
    if (pos >= 0.0 && fx_room(t, fx_close_need(pos) + 2, e.flags)) {
      if (pos > 0.0) fx_order_close(t, pos, pclose);
      fx_order_bracket(t, false, size, pclose + sl, pclose - tp, pclose);
    }
  }
}

// The same calls with the config's values, and for callers that keep no audit.
FX_HD void fx_apply_action(const FxConfig& c, int strategy, FxEnvRegs& e, FxOrderTab& t, int action, const FxBar& b,
                           int pair, double atr, bool atr_ready, bool has_minutes, int64_t minutes, FxAudit& au) {
  fx_apply_action(c, c, strategy, e, t, action, b, pair, atr, atr_ready, has_minutes, minutes, au);
}
template <class PC>
FX_HD void fx_apply_action(const FxConfig& c, const PC& p, int strategy, FxEnvRegs& e, FxOrderTab& t, int action,
                           const FxBar& b, int pair, double atr, bool atr_ready, bool has_minutes, int64_t minutes) {
  FxAudit au;
  fx_apply_action(c, p, strategy, e, t, action, b, pair, atr, atr_ready, has_minutes, minutes, au);
}
FX_HD void fx_apply_action(const FxConfig& c, int strategy, FxEnvRegs& e, FxOrderTab& t, int action, const FxBar& b,
                           int pair, double atr, bool atr_ready, bool has_minutes, int64_t minutes) {
  fx_apply_action(c, c, strategy, e, t, action, b, pair, atr, atr_ready, has_minutes, minutes);
}

// ---- app/env.py:187-204 ---------------------------------------------------------------------------------------------
FX_HD int fx_coerce_discrete(int a) { return (a == 0 || a == 1 || a == 2) ? a : 0; }

FX_HD int fx_coerce_continuous(const FxConfig& c, float v) {
  const double val = (double)v;
  const double thr = c.continuous_action_threshold != 0.0 ? c.continuous_action_threshold : 0.33;
  if (val >= thr) return 1;
  if (val <= -thr) return 2;
  return 0;
}

// ---- BTBridgeStrategy._publish_obs (app/bt_bridge.py:192-201) ----------------------------------------------------
FX_HD void fx_publish(FxEnvRegs& e, double pclose, int32_t t_local) {
  e.prev_equity = e.equity;
  e.equity = e.value;
  e.position = e.psize > 0.0 ? 1 : (e.psize < 0.0 ? -1 : 0);
  e.price = pclose;
  e.bar_index = t_local + 1;
}

// ---- rewards ---------------------------------------------------------------------------------------------------------
FX_HD double fx_reward_pnl(const FxConfig& c, const FxEnvRegs& e) {
  return (e.equity - e.prev_equity) / c.reward_initial_cash * c.reward_scale;
}

FX_HD double fx_reward_dd(const FxConfig& c, const FxEnvRegs& e, double& peak, int32_t& last_step) {
  if (e.bar_index <= last_step) peak = 0.0;
  last_step = e.bar_index;
  double m = peak;
  if (e.equity > m) m = e.equity;
  if (e.prev_equity > m) m = e.prev_equity;
  peak = m;
  const double pnl_norm = (e.equity - e.prev_equity) / c.reward_initial_cash;
  const double dd_norm = peak > 0.0 ? (peak - e.equity) / c.reward_initial_cash : 0.0;
  return pnl_norm - c.penalty_lambda * dd_norm;
}

// sharpe: ring push (deque(maxlen=W).append) into ring[slot * stride]; returns the new length
FX_HD int fx_sharpe_push(double* ring, int64_t stride, int W, int32_t& len, int32_t& head, int32_t& last_step,
                         int32_t step, double r) {
  if (step <= last_step) { len = 0; head = 0; }
  last_step = step;
  if (len == W) { ring[head * stride] = r; head = (head + 1) % W; }
  else { ring[((head + len) % W) * stride] = r; len++; }
  return len;
}

// sharpe: sequential (Python-order) evaluation over ring[((head+i) % W) * stride], i < n
FX_HD double fx_sharpe_eval(const double* ring, int64_t stride, int W, int n, int head, double ann) {
  if (n < 2) return 0.0;
  int idx = head % W;
  double s = ring[idx * stride], comp = 0.0;
  for (int i = 1; i < n; i++) { idx = (idx + 1 == W) ? 0 : idx + 1; fx_neumaier_add(s, comp, ring[idx * stride]); }
  const double mean = fx_neumaier_done(s, comp) / (double)n;
  idx = head % W;
  double d = ring[idx * stride] - mean;
  s = d * d; comp = 0.0;
  for (int i = 1; i < n; i++) {
    idx = (idx + 1 == W) ? 0 : idx + 1;
    d = ring[idx * stride] - mean;
    fx_neumaier_add(s, comp, d * d);
  }
  const double var = fx_neumaier_done(s, comp) / (double)(n - 1);
  const double sd = sqrt(var);
  if (sd <= 0.0) return 0.0;
  return (mean / sd) * sqrt(ann);
}

// Welford update of the running (mean, M2) of one feature column with the n-th row (n >= 1 after the update);
// used while the z-score history is still growing (warm-up of the rolling window, or expanding_zscore).
FX_HD void fx_welford_add(double& mean, double& m2, double x, int n) {
  const double d = x - mean;
  mean += d / (double)n;
  m2 += d * (x - mean);
}

// ---- observation element math ---------------------------------------------------------------------------------------
// np.clip (float32) then np.nan_to_num(nan=0, posinf=clip, neginf=-clip)  (feature_window_preprocessor.py:119-123)
FX_HD float fx_clip_nan(float v, float clipf, bool do_clip) {
  if (do_clip) { if (v < -clipf) v = -clipf; if (v > clipf) v = clipf; }
  if (v != v) return 0.0f;
  if (isinf(v)) return v > 0.0f ? clipf : -clipf;
  return v;
}

// the 4 agent scalars.  ref_price: default preprocessor -> fp64 last window price; feature_window -> the
// float32-rounded last window price (it reads obs["prices"][-1] back) or the bridge price without a price window.
// `inv_ic` = 1 / initial_cash (fp64, computed once on the host): x * inv_ic differs from x / ic by <= 1 ulp of fp64,
// invisible after the float32 cast the reference applies to these values (obs tolerance 1e-5).
FX_HD void fx_agent_scalars(const FxConfig& c, const FxEnvRegs& e, int32_t total_bars, double ref_price, double inv_ic,
                            float out[4]) {
  const double ic = c.initial_cash != 0.0 ? c.initial_cash : 1.0;
  const double upnl = (double)e.position * (e.price - ref_price) * c.obs_position_size;
  int32_t rem = total_bars - e.bar_index;
  if (rem < 0) rem = 0;
  const int32_t den = total_bars > 1 ? total_bars : 1;
  out[0] = (float)(double)e.position;
  out[1] = (float)((e.equity - ic) * inv_ic);
  out[2] = (float)(upnl * inv_ic);
  out[3] = (float)((double)rem / (double)den);
}

FX_HD int64_t fx_obs_dim(const FxConfig& c) {
  const int64_t W = c.window_size;
  if (c.preproc == FX_PREPROC_DEFAULT) return 2 * W + 4;
  return W * c.n_features + (c.include_price_window ? 2 * W : 0) + (c.include_agent_state ? 4 : 0);
}
