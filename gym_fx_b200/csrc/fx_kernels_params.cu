// fx_kernels_params.cu -- the step / rollout kernels of fx_env_step.cuh with per-env parameters (FX_V_PARAMS,
// fxenv_set_env_params) and without truncation.  A translation unit of its own so that the kernel halves compile in
// parallel, and so that a handle that never sets a table never loads these kernels.
#include "fx_env_step.cuh"

FxEnvKernels fx_params_kernels(int strategy, int reward, unsigned key) {
  return fx_variant_lookup<FX_V_PARAMS>(strategy, reward, key);
}
