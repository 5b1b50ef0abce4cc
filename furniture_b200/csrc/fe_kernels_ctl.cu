// fe_kernels_ctl.cu -- the step kernel of the torque controllers (fe_ctl.h) and the test hook of their arithmetic, compiled to their own
// sm_90a cubin (like fe_kernels_ik.cu: the stock kernels stay the profiled binary).  Same launch shape as fe_env_step_kernel.
#include <stdint.h>

#include "../../include/furniture_b200.h"
#include "fe_ik.h"
#include "fe_ctl.h"

extern "C" __global__ void __launch_bounds__(32 * FE_MAX_WPB) fe_env_ctl_step_kernel(FeState st, FeEnvState es, FeCtlArgs ctl, const fe_model* __restrict__ m,
                                                             const fe_scene* __restrict__ sc, fe_config cfg, FeOpt opt, const float* __restrict__ actions,
                                                             float* reward, uint8_t* done, int32_t* info, int slice_words, const int* __restrict__ slots) {
  const int wib = threadIdx.x >> 5, slot = blockIdx.x * (blockDim.x >> 5) + wib;
  const int env = slots[slot];
  if (env < 0) return; // unused slot
  FeEnv e;
  fe_env_bind(&e, fe_smem + (size_t)wib * (slice_words + FE_ENV_EXTRA_WORDS), m, sc, &cfg, opt, st, es, env, slice_words);
  fe_load(e.w, st, env);
  fe_env_load_groups(&e);
  fe_env_ctl_step_one(&e, ctl, actions, reward, done, info);
  fe_env_store_groups(&e);
  fe_store(e.w, st, env);
}

extern "C" __global__ void fe_ctl_eval_kernel(const fe_ctl_config* c, int n_episodes, const int32_t* first, const int32_t* count, const uint8_t* reset,
                                   const uint8_t* policy_step, const double* action, const FeCtlIn* in, double* tau) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_episodes) return;
  fe_ctl_eval_episode(c, first[e], count[e], reset, policy_step, action, in, tau);
}
