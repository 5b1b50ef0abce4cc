// fe_kernels.cu -- the sm_90a kernels, compiled to a cubin (nvcc -cubin) that the host library embeds and loads through
// the driver API: one module instance per (device, slice layout).  The slice layout table `fe_c_lay` is a __constant__
// object of the module, so every instance carries its own copy and handles of different models (a mixed-furniture batch)
// run concurrently on their own streams without re-uploading it.
// One warp = one environment; the warp's working set lives in dynamic shared memory for the whole call (all nsub mj_steps of an
// env step run without touching HBM except for the model tables, which stay in L1/L2).
#include <stdint.h>

#include "../../include/furniture_b200.h"
#include "fe_ik.h"
#include "fe_ctl.h"

// ---------------------------------------------------------------- kernels

extern "C" __global__ void __launch_bounds__(32 * FE_MAX_WPB) fe_sim_kernel(FeState s, const fe_model* __restrict__ m, FeOpt opt, int nsub, int mode, FeDebug dbg, int slice_words) {
  const int wib = threadIdx.x >> 5, slot = blockIdx.x * (blockDim.x >> 5) + wib;
  if (slot >= s.N) return;
  const int env = slot;
  fe_run_env(s, m, opt, env, nsub, mode, fe_smem + (size_t)wib * slice_words, dbg);
}

// the step kernels, one per control type: same launch shape, envs packed into blocks by fe_order_kernel
extern "C" __global__ void __launch_bounds__(32 * FE_MAX_WPB) fe_env_step_kernel(FeState st, FeEnvState es, const fe_model* __restrict__ m, const fe_scene* __restrict__ sc,
                                                         fe_config cfg, FeOpt opt, const float* __restrict__ actions, float* reward, uint8_t* done,
                                                         int32_t* info, int slice_words, const int* __restrict__ slots) {
  const int wib = threadIdx.x >> 5, slot = blockIdx.x * (blockDim.x >> 5) + wib;
  const int env = slots[slot];
  if (env < 0) return; // unused slot (blocks of heavy envs are deliberately left partly empty)
  fe_env_run(fe_smem + (size_t)wib * (slice_words + FE_ENV_EXTRA_WORDS), m, sc, &cfg, opt, st, es, env, slice_words, [&](FeEnv* e) { fe_env_step_one(e, actions, reward, done, info); });
}

extern "C" __global__ void __launch_bounds__(32 * FE_MAX_WPB) fe_env_ik_step_kernel(FeState st, FeEnvState es, FeIkArgs ik, const fe_model* __restrict__ m,
                                                            const fe_scene* __restrict__ sc, fe_config cfg, FeOpt opt, const float* __restrict__ actions,
                                                            float* reward, uint8_t* done, int32_t* info, int slice_words, const int* __restrict__ slots) {
  const int wib = threadIdx.x >> 5, slot = blockIdx.x * (blockDim.x >> 5) + wib;
  const int env = slots[slot];
  if (env < 0) return; // unused slot (blocks of heavy envs are deliberately left partly empty)
  fe_env_run(fe_smem + (size_t)wib * (slice_words + FE_ENV_EXTRA_WORDS), m, sc, &cfg, opt, st, es, env, slice_words, [&](FeEnv* e) { fe_env_ik_step_one(e, ik, actions, reward, done, info); });
}

extern "C" __global__ void __launch_bounds__(32 * FE_MAX_WPB) fe_env_ctl_step_kernel(FeState st, FeEnvState es, FeCtlArgs ctl, const fe_model* __restrict__ m,
                                                             const fe_scene* __restrict__ sc, fe_config cfg, FeOpt opt, const float* __restrict__ actions,
                                                             float* reward, uint8_t* done, int32_t* info, int slice_words, const int* __restrict__ slots) {
  const int wib = threadIdx.x >> 5, slot = blockIdx.x * (blockDim.x >> 5) + wib;
  const int env = slots[slot];
  if (env < 0) return; // unused slot (blocks of heavy envs are deliberately left partly empty)
  fe_env_run(fe_smem + (size_t)wib * (slice_words + FE_ENV_EXTRA_WORDS), m, sc, &cfg, opt, st, es, env, slice_words, [&](FeEnv* e) { fe_env_ctl_step_one(e, ctl, actions, reward, done, info); });
}

extern "C" __global__ void __launch_bounds__(32 * FE_MAX_WPB) fe_env_reset_kernel(FeState st, FeEnvState es, const fe_model* __restrict__ m, const fe_scene* __restrict__ sc,
                                                          fe_config cfg, FeOpt opt, const uint8_t* __restrict__ mask, int slice_words) {
  const int wib = threadIdx.x >> 5, env = blockIdx.x * (blockDim.x >> 5) + wib;
  if (env >= st.N) return;
  if (mask && !mask[env]) return;
  fe_env_run(fe_smem + (size_t)wib * (slice_words + FE_ENV_EXTRA_WORDS), m, sc, &cfg, opt, st, es, env, slice_words, [&](FeEnv* e) { fe_env_reset_one(e); });
}

// Packs the envs into blocks for the next step from the work their last step took (cycles in the five phases, barrier
// waits excluded).  Counting sort on a log-scale key (16 buckets per octave), heaviest first, into order[].  The warps of a
// block run in lockstep, so like goes with like; and the few envs far heavier than the median (robot coupled to a part:
// the big Newton solve) bound the whole step by their own latency, which is lowest when few warps share the SM: they get
// blocks with only `heavy_k` of the warp slots used, launched first, while the light envs fill the other SMs.
#define FE_ORDER_BUCKETS 256
#define FE_ORDER_HEAVY_SHIFT 18 /* heavy: 18 buckets above the median, 2^(18/16) = 2.2x the median work */
#define FE_ORDER_HEAVY_K 7      /* warp slots used in a block of heavy envs (7 of 14); half the block where it holds fewer than 8 */
#define FE_ORDER_DECAY 0.85f    /* per-step decay of an env's predicted work */
extern "C" __global__ void __launch_bounds__(1024) fe_order_kernel(int N, const int* __restrict__ stats, int* __restrict__ order, int* __restrict__ slots, int nslots,
                                                        int wpb, float* __restrict__ pred) {
  __shared__ int hist[FE_ORDER_BUCKETS], start[FE_ORDER_BUCKETS], nheavy;
  const int tid = threadIdx.x, heavy_k = wpb > FE_ORDER_HEAVY_K ? FE_ORDER_HEAVY_K : wpb / 2;
  if (tid < FE_ORDER_BUCKETS) hist[tid] = 0;
  // predicted work of the next step: the last step's, but an env that was heavy a few steps ago is still suspect
  for (int e = tid; e < N; e += 1024) {
    const int* st = stats + (size_t)e * FE_NSTAT;
    const float work = (float)st[FE_STAT_KIN] + (float)st[FE_STAT_COLLIDE] + (float)st[FE_STAT_ASSEMBLE] + (float)st[FE_STAT_SOLVE] + (float)st[FE_STAT_INTEGRATE]; // cycles / 16
    pred[e] = fmaxf(work, FE_ORDER_DECAY * pred[e]);
  }
  __syncthreads();
  auto bucket_of = [&](int e) {
    const float work = pred[e];
    int b = (int)(16.f * log2f(fmaxf(work, 1.f) * (1.f / 1024.f)));                               // bucket 0 below 16k cycles
    b = b < 0 ? 0 : (b > FE_ORDER_BUCKETS - 1 ? FE_ORDER_BUCKETS - 1 : b);
    return FE_ORDER_BUCKETS - 1 - b; // heaviest first
  };
  for (int e = tid; e < N; e += 1024) atomicAdd(&hist[bucket_of(e)], 1);
  __syncthreads();
  if (tid == 0) {
    int acc = 0, med = -1;
    for (int b = 0; b < FE_ORDER_BUCKETS; ++b) { start[b] = acc; acc += hist[b]; if (med < 0 && 2 * acc >= N) med = b; }
    // heavy: at least FE_ORDER_HEAVY_SHIFT buckets (sixteenths of an octave) above the median bucket
    const int hb = med - FE_ORDER_HEAVY_SHIFT; // last heavy bucket (buckets are in heaviest-first order)
    const int H = (heavy_k > 0 && heavy_k < wpb && hb >= 0) ? start[hb] + hist[hb] : 0;
    const int cap = heavy_k * FE_EXTRA_BLOCKS;
    nheavy = H > cap ? cap : H;
  }
  __syncthreads();
  for (int e = tid; e < N; e += 1024) order[atomicAdd(&start[bucket_of(e)], 1)] = e;
  for (int i = tid; i < nslots; i += 1024) slots[i] = -1;
  __syncthreads();
  const int H = nheavy, HB = heavy_k > 0 ? (H + heavy_k - 1) / heavy_k : 0;
  for (int r = tid; r < N; r += 1024) {
    const int slot = r < H ? (r / heavy_k) * wpb + r % heavy_k : HB * wpb + (r - H);
    slots[slot] = order[r];
  }
}

extern "C" __global__ void fe_is_aligned_kernel(int n, const double* p1, const double* m1, const double* p2, const double* m2, const double* cs, const double* sn,
                                     const int32_t* nang, const double* thr, uint8_t* aligned, double* tq) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double q[4] = {0, 0, 0, 0};
  bool set = false;
  const bool ok = fe_is_aligned_d(p1 + 3 * i, m1 + 9 * i, p2 + 3 * i, m2 + 9 * i, nang[i], cs + 4 * i, sn + 4 * i, thr + 4 * i, q, &set);
  aligned[i] = ok ? 1 : 0;
  const double nanv = __longlong_as_double(0x7ff8000000000000LL);
  for (int k = 0; k < 4; ++k) tq[4 * i + k] = set ? q[k] : nanv;
}


extern "C" __global__ void fe_dense_eval_kernel(const fe_dense_config* c, const fe_dense_recipe* rc, const double* thr, int n_goal, int n_episodes, const int32_t* first,
                                     const int32_t* count, int nsite, int npart, int act_dim, const double* spos, const double* smat, const double* ppos,
                                     const uint8_t* touch, const uint8_t* reset, const uint8_t* connected, const double* ac, double* reward, uint8_t* done, double* info) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_episodes) return;
  fe_dense_eval_episode(c, rc, thr, n_goal, first[e], count[e], nsite, npart, act_dim, spos, smat, ppos, touch, reset, connected, ac, reward, done, info);
}

// test hook of the torque controllers' arithmetic (fe_ctl_eval): one thread per episode of records
extern "C" __global__ void fe_ctl_eval_kernel(const fe_ctl_config* c, int n_episodes, const int32_t* first, const int32_t* count, const uint8_t* reset,
                                   const uint8_t* policy_step, const double* action, const FeCtlIn* in, double* tau) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_episodes) return;
  fe_ctl_eval_episode(c, first[e], count[e], reset, policy_step, action, in, tau);
}
