// fe_kernels_ik.cu -- the step kernel of control_type="ik" (fe_ik.h), compiled to its own sm_90a cubin: the stock kernels of
// fe_kernels.cu stay the binary they were profiled as.  Same launch shape as fe_env_step_kernel: one warp = one env, envs packed into
// blocks by fe_order_kernel.
#include <stdint.h>

#include "../../include/furniture_b200.h"
#include "fe_ik.h"

extern "C" __global__ void __launch_bounds__(32 * FE_MAX_WPB) fe_env_ik_step_kernel(FeState st, FeEnvState es, FeIkArgs ik, const fe_model* __restrict__ m,
                                                            const fe_scene* __restrict__ sc, fe_config cfg, FeOpt opt, const float* __restrict__ actions,
                                                            float* reward, uint8_t* done, int32_t* info, int slice_words, const int* __restrict__ slots) {
  const int wib = threadIdx.x >> 5, slot = blockIdx.x * (blockDim.x >> 5) + wib;
  const int env = slots[slot];
  if (env < 0) return; // unused slot
  FeEnv e;
  fe_env_bind(&e, fe_smem + (size_t)wib * (slice_words + FE_ENV_EXTRA_WORDS), m, sc, &cfg, opt, st, es, env, slice_words);
  fe_load(e.w, st, env);
  fe_env_load_groups(&e);
  fe_env_ik_step_one(&e, ik, actions, reward, done, info);
  fe_env_store_groups(&e);
  fe_store(e.w, st, env);
}
