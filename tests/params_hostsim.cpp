// tests/params_hostsim.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// tests/hostsim (the g++ build of the product's fx_core.cuh) stepping the core with a per-env parameter row (FxEnvParams,
// include/fxenv.h fxenv_set_env_params).  fx_hostsim.cpp is compiled into this library unchanged, except that its calls
// of the core functions that read the seven values (commission, leverage, slippage_perc, sl_pips, tp_pips, k_sl, k_tp)
// are routed to the overloads that take them from the env's row, as the step kernels built with FX_V_PARAMS do: the
// config keeps feeding every other field.  tests/env_params_hostsim.py drives it.
#include <map>

#include "../gym_fx_b200/csrc/fx_core.cuh"

struct HsEnv;
static const FxEnvParams& hsp_row(const HsEnv* h);
#define fx_bound_per(c) fx_bound_per(hsp_row(h))
#define fx_check_submitted(c, ...) fx_check_submitted(hsp_row(h), __VA_ARGS__)
#define fx_exec_entry(c, ...) fx_exec_entry(c, hsp_row(h), __VA_ARGS__)
#define fx_mark_to_market(c, ...) fx_mark_to_market(hsp_row(h), __VA_ARGS__)
#define fx_apply_action(c, ...) fx_apply_action(c, hsp_row(h), __VA_ARGS__)
#include "hostsim/fx_hostsim.cpp"
#undef fx_bound_per
#undef fx_check_submitted
#undef fx_exec_entry
#undef fx_mark_to_market
#undef fx_apply_action

static std::map<const HsEnv*, FxEnvParams> g_rows;

// the env's row, or (none set) the config's own values
static const FxEnvParams& hsp_row(const HsEnv* h) {
  const auto it = g_rows.find(h);
  if (it != g_rows.end()) return it->second;
  static thread_local FxEnvParams cfg_row;
  const FxConfig& c = h->c;
  cfg_row = FxEnvParams{c.commission, c.leverage, c.slippage_perc, c.sl_pips, c.tp_pips, c.k_sl, c.k_tp};
  return cfg_row;
}

extern "C" {

// row: FXENV_ENV_PARAMS values in FXENV_PARAM_* order, or NULL (the config's values)
void hsp_set_params(HsEnv* h, const double* row) {
  if (!row) { g_rows.erase(h); return; }
  g_rows[h] = FxEnvParams{row[FXENV_PARAM_COMMISSION], row[FXENV_PARAM_LEVERAGE], row[FXENV_PARAM_SLIPPAGE],
                          row[FXENV_PARAM_SL_PIPS], row[FXENV_PARAM_TP_PIPS], row[FXENV_PARAM_K_SL], row[FXENV_PARAM_K_TP]};
}

}  // extern "C"
