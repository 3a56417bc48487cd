// fx_kernels_params_trunc.cu -- the step / rollout kernels of fx_env_step.cuh with per-env parameters (FX_V_PARAMS) and
// truncation (FX_V_TRUNC).  A translation unit of its own so that the kernel halves compile in parallel.
#include "fx_env_step.cuh"

FxEnvKernels fx_params_trunc_kernels(int strategy, int reward, unsigned key) {
  return fx_variant_lookup<FX_V_PARAMS | FX_V_TRUNC>(strategy, reward, key);
}
