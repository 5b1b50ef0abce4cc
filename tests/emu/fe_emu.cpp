// fe_emu.cpp -- lane-emulated build of the engine (TEST HARNESS ONLY, never loaded by the package).
// The same kernel source as furniture_b200/csrc/fe_kernels.cu, compiled by g++ with every lane region run as a 32-trip
// loop, behind the same C-ABI, so that `-m "not gpu"` tests can exercise the kernel logic without a GPU.
#define FE_EMULATE 1
#define PLAT_IS_CUDA 0
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <vector>
struct fe_handle;
static void* plat_alloc(size_t bytes) { return malloc(bytes); }
static void plat_free(void* p) { free(p); }
static void plat_memset0(void* p, size_t n) { memset(p, 0, n); }
static void plat_upload(void* d, const void* h, size_t n) { memcpy(d, h, n); }
static void plat_download(void* h, const void* d, size_t n) { memcpy(h, d, n); }
static int plat_init(fe_handle*) { return 0; }
static void plat_fini(fe_handle*) {}
static void plat_sync(fe_handle*) {}
static int plat_enter(fe_handle*) { return -1; }
static void plat_leave(fe_handle*, int) {}
static int plat_run_sim(fe_handle* h, int nsub, int mode, void* stream);
static int plat_run_reset(fe_handle* h, const uint8_t* mask, void* stream);
static int plat_run_step(fe_handle* h, const float* actions, float* reward, uint8_t* done, int32_t* info, void* stream);
static int plat_step_host(fe_handle* h, const float* actions, float* obs, float* reward, uint8_t* done, int32_t* info);
static void plat_copy_d2d(fe_handle*, void* dst, const void* src, size_t n, void*) { if (dst != src) memcpy(dst, src, n); }
static int plat_is_aligned(fe_handle* h, int n, const double* p1, const double* m1, const double* p2, const double* m2, const double* angles,
                           const int32_t* nangles, const double* thr, uint8_t* aligned, double* tq);

static int plat_dense_eval(fe_handle* h, const struct fe_dense_config* dc, const struct fe_dense_recipe* rc, const double* thr, int n_goal, int n_episodes,
                           const int32_t* first, const int32_t* count, int n_records, int nsite, int npart, int act_dim, const double* spos, const double* smat,
                           const double* ppos, const uint8_t* touch, const uint8_t* reset, const uint8_t* connected, const double* ac, double* reward,
                           uint8_t* done, double* info);
static int plat_ctl_eval(fe_handle* h, const struct fe_ctl_config* cc, int n_episodes, const int32_t* first, const int32_t* count, int n_records, const uint8_t* reset,
                         const uint8_t* policy_step, const double* action, const struct FeCtlIn* in, double* torques);

#include "../../furniture_b200/csrc/fe_api.inl"

static int plat_run_sim(fe_handle* h, int nsub, int mode, void*) {
  fe_h_lay = h->lay;
  std::vector<float> slice(h->slice_words + FE_ENV_EXTRA_WORDS);
  for (int env = 0; env < h->N; ++env) fe_run_env(h->st, h->dm, h->opt, env, nsub, mode, slice.data(), h->dbg);
  return 0;
}
static int plat_run_reset(fe_handle* h, const uint8_t* mask, void*) {
  fe_h_lay = h->lay;
  std::vector<double> slice((h->slice_words + FE_ENV_EXTRA_WORDS) / 2 + 8);
  for (int env = 0; env < h->N; ++env)
    if (!mask || mask[env]) fe_env_run((float*)slice.data(), h->dm, h->ds, &h->cfg, h->opt, h->st, h->es, env, h->slice_words, [&](FeEnv* e) { fe_env_reset_one(e); });
  return 0;
}
static int plat_run_step(fe_handle* h, const float* actions, float* reward, uint8_t* done, int32_t* info, void*) {
  fe_h_lay = h->lay;
  std::vector<double> slice((h->slice_words + FE_ENV_EXTRA_WORDS) / 2 + 8);
  for (int env = 0; env < h->N; ++env)
    fe_env_run((float*)slice.data(), h->dm, h->ds, &h->cfg, h->opt, h->st, h->es, env, h->slice_words, [&](FeEnv* e) {
      if (h->ctl.c) fe_env_ctl_step_one(e, h->ctl, actions, reward, done, info);
      else if (h->ik.c) fe_env_ik_step_one(e, h->ik, actions, reward, done, info);
      else fe_env_step_one(e, actions, reward, done, info);
    });
  return 0;
}
static int plat_step_host(fe_handle* h, const float* actions, float* obs, float* reward, uint8_t* done, int32_t* info) {
  int rc = plat_run_step(h, actions, reward ? reward : (float*)h->dev_rew, done ? done : (uint8_t*)h->dev_done, info ? info : (int32_t*)h->dev_info, nullptr);
  if (obs) memcpy(obs, h->es.obs, sizeof(float) * (size_t)h->N * h->hs.obs_dim);
  return rc;
}
static int plat_is_aligned(fe_handle*, int n, const double* p1, const double* m1, const double* p2, const double* m2, const double* angles,
                           const int32_t* nangles, const double* thr, uint8_t* aligned, double* tq) {
  for (int i = 0; i < n; ++i) {
    double cs[4], sn[4], q[4] = {0, 0, 0, 0};
    for (int k = 0; k < 4; ++k) { double a = angles[4 * i + k] / 180 * 3.141592653589793; cs[k] = cos(a); sn[k] = sin(a); }
    bool set = false;
    aligned[i] = fe_is_aligned_d(p1 + 3 * i, m1 + 9 * i, p2 + 3 * i, m2 + 9 * i, nangles[i], cs, sn, thr + 4 * i, q, &set) ? 1 : 0;
    for (int k = 0; k < 4; ++k) tq[4 * i + k] = set ? q[k] : NAN;
  }
  return 0;
}
static int plat_dense_eval(fe_handle*, const fe_dense_config* dc, const fe_dense_recipe* rc, const double* thr, int n_goal, int n_episodes, const int32_t* first,
                           const int32_t* count, int, int nsite, int npart, int act_dim, const double* spos, const double* smat, const double* ppos,
                           const uint8_t* touch, const uint8_t* reset, const uint8_t* connected, const double* ac, double* reward, uint8_t* done, double* info) {
  for (int e = 0; e < n_episodes; ++e)
    fe_dense_eval_episode(dc, rc, thr, n_goal, first[e], count[e], nsite, npart, act_dim, spos, smat, ppos, touch, reset, connected, ac, reward, done, info);
  return 0;
}
static int plat_ctl_eval(fe_handle*, const fe_ctl_config* cc, int n_episodes, const int32_t* first, const int32_t* count, int, const uint8_t* reset,
                         const uint8_t* policy_step, const double* action, const FeCtlIn* in, double* torques) {
  for (int e = 0; e < n_episodes; ++e) fe_ctl_eval_episode(cc, first[e], count[e], reset, policy_step, action, in, torques);
  return 0;
}
