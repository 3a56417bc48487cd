/*
 * tests/episode_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * The episode starts and records of include/fxenv.h (fxenv_set_reset_starts, FXENV_EP_*) restated on top of the C oracle:
 * oracle/fxenv_oracle.c is compiled into this library unchanged, and the functions below read a finished episode from
 * the oracle's own analyzer state.  tests/episode_oracle.py drives them (draws, counters, auto-reset steps).
 */
#include "../oracle/fxenv_oracle.c"

/* lo + high 64 bits of splitmix64(seed ^ (env << 32 | k)) * span */
int64_t fxe_draw_start(uint64_t seed, int32_t env, int32_t k, int64_t lo, uint64_t span) {
  uint64_t z = seed ^ (((uint64_t)(uint32_t)env << 32) | (uint64_t)(uint32_t)k);
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return lo + (int64_t)(uint64_t)(((unsigned __int128)z * span) >> 64);
}

int fxe_started(const FxoEnv* e) { return (e->flags & FX_FLAG_STARTED) != 0; }

/* The record of the episode the env is in (FXENV_EPISODE_STATS doubles); START and INDEX are the caller's. */
void fxe_record(const FxoEnv* e, double* r) {
  double sq = 0.0;   /* SQN's sum of squares over the closed trades, in closing order */
  for (int i = 0; i < e->sqn_n; i++) sq += e->sqn_pnl[i] * e->sqn_pnl[i];
  r[FXENV_EP_START] = 0.0;
  r[FXENV_EP_BARS] = e->bar_index;
  r[FXENV_EP_EQUITY] = e->equity;
  r[FXENV_EP_COMMISSION] = e->commission_paid;
  r[FXENV_EP_END_FLAGS] = e->flags & (FX_FLAG_TERMINATED | FX_FLAG_EXHAUSTED | FX_FLAG_BROKE);
  r[FXENV_EP_DD_MAX_PCT] = e->an_max_drawdown;
  r[FXENV_EP_DD_MAX_MONEY] = e->an_max_moneydown;
  r[FXENV_EP_PNL_NET] = e->an_pnl_net;
  r[FXENV_EP_PNL_SQ] = sq;
  r[FXENV_EP_OPENED] = e->an_opened;
  r[FXENV_EP_CLOSED] = e->an_closed;
  r[FXENV_EP_WON] = e->an_won;
  r[FXENV_EP_LOST] = e->an_lost;
  r[FXENV_EP_INDEX] = 0.0;
}
