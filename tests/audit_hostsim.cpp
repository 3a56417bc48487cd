// tests/audit_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// tests/hostsim (the g++ build of the product's fx_core.cuh) with the bracket audit: fx_hostsim.cpp is compiled into this
// library unchanged, except that its one fx_apply_action call is routed through fx_apply_action_audited, which makes the
// same call with the product's FxAudit out-parameter and keeps the records of each env (fields FXENV_AU_*; EPISODE 0:
// the host build has no episode counter).  tests/audit_ref.py drives it.
#include <array>
#include <map>
#include <vector>

#include "../gym_fx_b200/csrc/fx_core.cuh"

static void fx_apply_action_audited(void* h, int32_t t, const FxConfig& c, int strategy, FxEnvRegs& e, FxOrderTab& tab,
                                    int action, const FxBar& b, int pair, double atr, bool atr_ready, bool has_minutes,
                                    int64_t minutes);
#define fx_apply_action(...) fx_apply_action_audited(h, t, __VA_ARGS__)
#include "hostsim/fx_hostsim.cpp"
#undef fx_apply_action

static std::map<void*, std::vector<std::array<double, FXENV_AU_FIELDS>>> g_records;

static void fx_apply_action_audited(void* hv, int32_t t, const FxConfig& c, int strategy, FxEnvRegs& e, FxOrderTab& tab,
                                    int action, const FxBar& b, int pair, double atr, bool atr_ready, bool has_minutes,
                                    int64_t minutes) {
  FxAudit au;
  au.kind = FXENV_AU_KIND_NONE;
  fx_apply_action(c, strategy, e, tab, action, b, pair, atr, atr_ready, has_minutes, minutes, au);
  if (au.kind == FXENV_AU_KIND_NONE) return;
  const HsEnv* h = static_cast<const HsEnv*>(hv);
  const bool fc = au.kind == FXENV_AU_KIND_FORCE_CLOSE;
  std::array<double, FXENV_AU_FIELDS> r;
  r[FXENV_AU_KIND] = au.kind;
  r[FXENV_AU_BAR] = (double)(h->start + t);
  r[FXENV_AU_EPISODE] = 0.0;
  r[FXENV_AU_ENTRY] = b.c;
  r[FXENV_AU_STOP] = fc ? NAN : au.stop;
  r[FXENV_AU_LIMIT] = fc ? NAN : au.limit;
  r[FXENV_AU_SIZE] = au.size;
  r[FXENV_AU_ATR] = fc ? NAN : au.atr;
  g_records[hv].push_back(r);
}

extern "C" {

// Copies up to `cap` records of env h (oldest first) into out[cap][FXENV_AU_FIELDS]; returns how many it holds.
int hsa_records(void* h, double* out, int cap) {
  const auto& v = g_records[h];
  for (int i = 0; i < (int)v.size() && i < cap; i++)
    for (int j = 0; j < FXENV_AU_FIELDS; j++) out[i * FXENV_AU_FIELDS + j] = v[i][j];
  return (int)v.size();
}

void hsa_forget(void* h) { g_records.erase(h); }

}  // extern "C"
