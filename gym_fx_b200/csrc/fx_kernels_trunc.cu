// fx_kernels_trunc.cu -- the truncation instantiations of the step / rollout kernels (include/fxenv.h,
// fxenv_set_time_limit): fx_kernels.cu with FX_KERNELS_TRUNC, its kernels inside namespace fx_trunc.  A translation unit
// of its own, so that the kernels that run with truncation off are not touched and both halves compile in parallel.
#define FX_KERNELS_TRUNC 1
#include "fx_kernels.cu"
