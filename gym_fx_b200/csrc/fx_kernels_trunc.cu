// fx_kernels_trunc.cu -- the step / rollout kernels of fx_env_step.cuh with truncation (FX_V_TRUNC, fxenv_set_time_limit).
// A translation unit of its own so that both halves of the kernels compile in parallel.
#include "fx_env_step.cuh"

FxEnvKernels fx_trunc_kernels(int strategy, int reward, unsigned key) {
  return fx_variant_lookup<FX_V_TRUNC>(strategy, reward, key);
}
