// fe_driver.h -- per-env state in HBM (env-major arrays: one env's record is contiguous, so a warp's lanes read
// consecutive words), the load/store between HBM and the warp slice, and the per-env entry points the kernels call.
#pragma once
#include "fe_engine.h"

#define FE_MAX_WPB 16      /* warps (= envs) per block of the sim / step / reset kernels */
#define FE_EXTRA_BLOCKS 132 /* spare blocks of the step grid, one per SM of an H100 SXM: heavy envs get partly empty blocks */

struct FeState {
  int N;
  float *qpos, *qvel, *warm, *ctrl, *qfrc_applied, *gravcomp, *eq_data; // [N][nq|nv|nv|nu|nr|npart|7 neq]
  float* mpos;                                                          // [N][3 nmov] world positions of the movable static geoms
  int *contype, *conaff, *eq_active;                                    // [N][ngeom|ngeom|neq]
  float *bias;                                                          // [N][nr]  qfrc_bias of the last forward pass
  float *lpos, *lquat, *lvel;                                           // [N][nlink][3|4|6] of the last forward pass
  int *touch;                                                           // [N][npart]
  int *flags, *ncon, *niter;                                            // [N]  flags: FE_FLAG_* bits
  int* order;                                                           // [N] rank -> env: the envs by the predicted work of their next step, heaviest first (written by fe_order_kernel)
  int* stats;                                                           // [N][FE_NSTAT] per call: the FE_STAT_* columns
  float* coop;                                                          // [N][FeLayout::coop_words] the cooperative solver's arrays (FE_COOP_*)
};

// optional dump of one forward pass (all nullable, [N][dim])
struct FeDebug {
  float *Mr, *fs, *as, *linert, *x, *fc, *c_dist, *c_pos, *c_frame, *c_aref, *c_D, *c_f, *lmat, *S;
  int *c_geom, *c_state;
  float *c_mu, *c_fric;                 // [N][maxcon] regularised and plain friction coefficient of each contact
  float *w_aref, *w_D, *w_f;            // [N][6 neq] weld rows (3 translational, 3 rotational); rows of inactive welds are stale
  float *l_sign, *l_aref, *l_D, *l_f;   // [N][nr] joint-limit rows: side (+1 lower, -1 upper, 0 none), aref, D, force
};

FE_FN void fe_load(FeWarp* w, const FeState& s, int env) {
  const fe_model* m = w->m;
#define LD(field, n) for (int i = lane; i < (n); i += 32) w->field()[i] = s.field[(size_t)env * (n) + i];
  LANES_BEGIN
    LD(qpos, m->nq) LD(qvel, m->nv) LD(warm, m->nv) LD(ctrl, m->nu) LD(qfrc_applied, m->nr) LD(gravcomp, m->npart) LD(eq_data, 7 * m->neq) LD(mpos, 3 * m->nmov)
    LD(contype, m->ngeom) LD(conaff, m->ngeom) LD(eq_active, m->neq) LD(bias, m->nr)
    w->u()[lane] = 0; // FE_U_STAT + FE_NSTAT <= 32
    if (lane == 0) w->coop = s.coop + (size_t)env * FE_LAY.coop_words;
  LANES_END
#undef LD
}
FE_FN void fe_store(FeWarp* w, const FeState& s, int env) {
  const fe_model* m = w->m;
#define ST(field, n) for (int i = lane; i < (n); i += 32) s.field[(size_t)env * (n) + i] = w->field()[i];
  LANES_BEGIN
    ST(qpos, m->nq) ST(qvel, m->nv) ST(warm, m->nv) ST(ctrl, m->nu) ST(qfrc_applied, m->nr) ST(gravcomp, m->npart) ST(eq_data, 7 * m->neq) ST(mpos, 3 * m->nmov)
    ST(contype, m->ngeom) ST(conaff, m->ngeom) ST(eq_active, m->neq)
    ST(bias, m->nr) ST(lpos, 3 * m->nlink) ST(lquat, 4 * m->nlink) ST(lvel, 6 * m->nlink) ST(touch, m->npart)
    if (lane == 0) { s.flags[env] |= w->u()[FE_U_FLAGS]; s.ncon[env] = w->u()[FE_U_NCON]; s.niter[env] = w->u()[FE_U_NITER]; }
    if (lane < FE_NSTAT) s.stats[(size_t)env * FE_NSTAT + lane] = w->u()[FE_U_STAT + lane];
  LANES_END
#undef ST
}
FE_FN void fe_dump(FeWarp* w, const FeDebug& d, int env) {
  const fe_model* m = w->m;
  const int mc = w->opt.maxcon;
#define DP(field, n) if (d.field) for (int i = lane; i < (n); i += 32) d.field[(size_t)env * (n) + i] = w->field()[i];
  LANES_BEGIN
    DP(Mr, m->nr * m->nr) DP(fs, m->nv) DP(as, m->nv) DP(linert, 10 * m->nlink) DP(x, m->nv) DP(fc, m->nv) DP(lmat, 9 * m->nlink) DP(S, 6 * m->nr)
    DP(c_dist, mc) DP(c_pos, 3 * mc) DP(c_aref, 3 * mc) DP(c_D, 2 * mc) DP(c_f, 3 * mc) DP(c_geom, mc) DP(c_state, mc)
    DP(c_mu, mc) DP(c_fric, mc) DP(w_aref, 6 * m->neq) DP(w_D, 6 * m->neq) DP(w_f, 6 * m->neq)
    DP(l_sign, m->nr) DP(l_aref, m->nr) DP(l_D, m->nr) DP(l_f, m->nr)
    if (d.c_frame) for (int c = lane; c < mc; c += 32) { float F[9]; fe_frame_load(w, c, F); for (int k = 0; k < 9; ++k) d.c_frame[(size_t)env * 9 * mc + 9 * c + k] = F[k]; }
  LANES_END
#undef DP
}

// nsub mj_steps of one env. mode 0: step; mode 1: forward only (mj_forward, no integration), with optional dump.
FE_FN void fe_run_env(const FeState& s, const fe_model* m, const FeOpt& opt, int env, int nsub, int mode, float* slice, const FeDebug& dbg) {
  FeWarp* w = fe_warp_bind(slice, m, opt);
  fe_load(w, s, env);
  if (mode == 1) { fe_forward(w); fe_dump(w, dbg, env); }
  else for (int i = 0; i < nsub; ++i) fe_substep_lockstep(w);
  fe_store(w, s, env);
}
