/*
 * tests/audit_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * The bracket audit of direct_atr_sltp (include/fxenv.h, FXENV_AU_*) read off the C oracle: oracle/fxenv_oracle.c is
 * compiled into this library unchanged, and fxa_step runs one fxo_step, then derives the record from the orders that
 * step's strategy call created (they are the ones with a ref the env had not issued before the step):
 *   a bracket parent (limit order that is its own group) -> long / short bracket: stop / limit = its children's prices,
 *     size = |parent size|, atr = the simple mean of the oracle's TR deque;
 *   a lone market order -> session force-close (the ATR strategy places no other market order without a bracket),
 *     size = the position it closes.
 * tests/audit_ref.py drives it.
 */
#include "../oracle/fxenv_oracle.c"

/* One fxo_step.  Returns 1 and fills rec[FXENV_AU_FIELDS] (EPISODE left to the caller) if the step logged a record. */
int fxa_step(FxoEnv* e, double action, float* obs, double* reward, uint8_t* terminated, double* rec) {
  const int ref0 = e->next_ref;
  fxo_step(e, action, obs, reward, terminated);
  const OOrder *parent = NULL, *stop = NULL, *limit = NULL, *market = NULL;
  for (int i = 0; i < e->n_ord; i++) {
    const OOrder* o = &e->ord[i];
    if (o->ref < ref0) continue;
    if (o->type == OT_MARKET) market = o;
    else if (o->group == o->ref) parent = o;
    else if (o->type == OT_STOP) stop = o;
    else limit = o;
  }
  if (!parent && !market) return 0;
  rec[FXENV_AU_BAR] = (double)(e->start + e->t);
  rec[FXENV_AU_EPISODE] = 0.0;
  rec[FXENV_AU_ENTRY] = row(e, e->t)[3];
  if (parent) {
    rec[FXENV_AU_KIND] = parent->size > 0 ? FXENV_AU_KIND_LONG : FXENV_AU_KIND_SHORT;
    rec[FXENV_AU_STOP] = stop->price;
    rec[FXENV_AU_LIMIT] = limit->price;
    rec[FXENV_AU_SIZE] = fabs(parent->size);
    rec[FXENV_AU_ATR] = py_sum(e->tr_buf, e->tr_len) / (double)e->tr_len;
  } else {
    rec[FXENV_AU_KIND] = FXENV_AU_KIND_FORCE_CLOSE;
    rec[FXENV_AU_STOP] = rec[FXENV_AU_LIMIT] = rec[FXENV_AU_ATR] = NAN;
    rec[FXENV_AU_SIZE] = -market->size;
  }
  return 1;
}
