// fe_dense.h -- the phase-based dense reward of FurnitureSawyerDenseRewardEnv, evaluated by lane 0 of the warp that owns the env
// right after the physics of the step (furniture/env/furniture_sawyer_dense.py):
//   fe_dense_begin_episode <- _reset_reward_variables :128-139
//   fe_dense_begin_subtask <- _update_reward_variables :150-219, _set_next_subtask :141-148
//   fe_dense_step          <- _collect_values :225-280, _compute_reward :282-586, the eight phase terms :588-943,
//                             _stable_grip_reward :945-985, _gripper_penalty :987-1003, _ctrl_penalty :1005-1009,
//                             _move_other_part_penalty :1011-1022, _project_connector_forward (furniture.py:1178-1199)
// All arithmetic is float64 in numpy's operation order (the np* helpers of fe_env.h); Python's min/max semantics are kept
// (pymin/pymax below: a NaN first argument stays, C's fmin/fmax would drop it).  The machine is templated on the "world" it reads, so
// that the same code runs on the env's slice (FeSliceWorld in fe_env.h) and on explicit poses (FeArrayWorld: the golden-vector
// test hook fe_dense_eval).  One deviation from the reference, stated in oracle/dense_oracle.py as well: prev[GRASP] exists in both
// reward modes (the reference raises AttributeError in _grasp_leg_reward when diff_rew is off).
#pragma once

#include "fe_dense_types.h"

FE_HD double pymin(double a, double b) { return b < a ? b : a; }
FE_HD double pymax(double a, double b) { return b > a ? b : a; }
FE_HD void dv_sub(double* r, const double* a, const double* b) { r[0] = ndsub(a[0], b[0]); r[1] = ndsub(a[1], b[1]); r[2] = ndsub(a[2], b[2]); }
FE_HD double dv_dist(const double* a, const double* b) { double d[3]; dv_sub(d, a, b); return npnorm(d); }
FE_HD double dv_dist_xy(const double* a, const double* b) { const double x = ndsub(a[0], b[0]), y = ndsub(a[1], b[1]); return ndsqrt(ndfma(y, y, ndmul(x, x))); }
FE_HD void dv_col(double* r, const double* m, int c) { r[0] = m[c]; r[1] = m[3 + c]; r[2] = m[6 + c]; }

// (pos(g_l) + pos(g_r)) / 2 and pos(g_r) - pos(g_l)
template <class W>
FE_HD void fe_dense_grasp(const W& w, const fe_dense_recipe* rc, int s, double* mid, double* vec) {
  double l[3], r[3];
  w.site_pos(rc->gl_site[s], l);
  w.site_pos(rc->gr_site[s], r);
  for (int k = 0; k < 3; ++k) { mid[k] = nddiv(ndadd(l[k], r[k]), 2.0); if (vec) vec[k] = ndsub(r[k], l[k]); }
}

template <class W>
FE_HDN void fe_dense_begin_subtask(const W& w, const fe_dense_config* c, const fe_dense_recipe* rc, FeDenseState* st) {
  const int s = st->subtask;
  st->dropped = st->table_moved = st->lifted = 0;
  st->fine_aligned = 0;
  w.site_pos(rc->table_site[s], st->table_site0);
  w.part_pos(rc->leg_part[s], st->leg0);
  st->lift_target[0] = ndadd(st->leg0[0], 0.0); st->lift_target[1] = ndadd(st->leg0[1], 0.0); st->lift_target[2] = ndadd(st->leg0[2], rc->waypoint_z[s]);
  double eef[3];
  w.site_pos(rc->griptip_site, eef);
  st->phase = c->reset_robot_after_attach ? FE_PH_ABOVE_LEG : FE_PH_INIT_EEF;
  if (rc->grip_init_len[s] > 0) {
    for (int k = 0; k < 3; ++k) st->init_eef[k] = ndadd(eef[k], rc->grip_init[s][k]);
    if (rc->grip_init_len[s] == 4) st->init_eef[2] = ndsub(rc->grip_init[s][3], 0.085);
  } else {
    st->phase = FE_PH_ABOVE_LEG;
  }
  if (st->diff_rew) {
    if (st->phase == FE_PH_ABOVE_LEG) {
      double g[3];
      fe_dense_grasp(w, rc, s, g, (double*)nullptr);
      g[0] = ndadd(g[0], 0.0); g[1] = ndadd(g[1], 0.0); g[2] = ndadd(g[2], 0.05);
      st->prev[FE_DP_ABOVE_LEG] = dv_dist(eef, g);
    } else {
      st->prev[FE_DP_INIT_EEF] = dv_dist(eef, st->init_eef);
    }
    st->prev[FE_DP_GRASP] = -1.0;
    st->prev[FE_DP_LIFT_Z] = rc->waypoint_z[s];
    st->prev[FE_DP_LIFT_XY] = 0.0;
  }
}

// `first`: the subtask the episode starts at, the number of recipe steps the reset preassembled.  Their legs' grasp-target pairs are claimed in
// recipe order (:130-138), which is the order the packed gl_site / gr_site were resolved in: subtask `first` holds the pair it would claim.
template <class W>
FE_HDN void fe_dense_begin_episode(const W& w, const fe_dense_config* c, const fe_dense_recipe* rc, int first, FeDenseState* st) {
  st->subtask = first;
  st->success = 0;
  st->diff_rew = c->diff_rew; // the shaped terms keep their prev[] slots only in diff mode: the mode holds for the whole episode
  for (int k = 0; k < FE_DP_N; ++k) st->prev[k] = 0.0;
  st->prev[FE_DP_GRASP] = -1.0;
  for (int k = 0; k < 3; ++k) st->init_eef[k] = 0.0;
  fe_dense_begin_subtask(w, c, rc, st);
}

// shaped term of a quantity x with memory: diff_rew (the episode's) -> coef * mult * (f(x) - f(prev)) (or the reverse), prev := x; else the plain term
#define FE_DENSE_SHAPED(out, slot, x, coef, mult, FEXPR, reversed, plain)            \
  do {                                                                               \
    if (st->diff_rew) {                                                              \
      double v_ = (x);            const double cur_ = (FEXPR);                       \
      v_ = st->prev[slot];        const double old_ = (FEXPR);                       \
      out = ndmul(ndmul((reversed) ? ndsub(old_, cur_) : ndsub(cur_, old_), (coef)), (mult)); \
      st->prev[slot] = (x);                                                          \
    } else {                                                                         \
      out = (plain);                                                                 \
    }                                                                                \
  } while (0)

template <class W>
FE_HDN void fe_dense_step(const W& w, const fe_dense_config* c, const fe_dense_recipe* rc, const double* thr /* alignment thresholds (4) */, int n_goal,
                          FeDenseState* st, const double* ac, int act_dim, int connected, double* reward_out, int* done_out, double* info) {
  const int s = st->subtask;
  const double P = c->phase_bonus;
  int done = 0;
  double bonus = 0.0;
  st->success = 0;
  // ---- what the world looks like (_collect_values)
  const int touched = w.touch_both(rc->leg_part[s]) ? 1 : 0;
  double eef[3], grasp[3], gvec[3], leg[3], lsp[3], lsm[9], tsp[3], tsm[9], gm[9], gp_[3];
  w.site_pos(rc->griptip_site, eef);
  fe_dense_grasp(w, rc, s, grasp, gvec);
  w.part_pos(rc->leg_part[s], leg);
  w.site_pose(rc->leg_site[s], lsp, lsm);
  w.site_pose(rc->table_site[s], tsp, tsm);
  w.site_pose(rc->grip_site, gp_, gm);
  double leg_up[3], leg_fw[3], table_up[3], table_fw[3], fw_rot[3];
  dv_col(leg_up, lsm, 2); dv_col(leg_fw, lsm, 1); dv_col(table_up, tsm, 2); dv_col(table_fw, tsm, 1);
  if (rc->n_allowed[s] > 0) { // _project_connector_forward(leg_site, table_site, angle)
    double k[3], cr[3];
    np_unit_vector_f32(k, leg_up);
    npcross(cr, k, leg_fw);
    if (rc->has_angle[s]) for (int i = 0; i < 3; ++i) fw_rot[i] = ndadd(ndmul(rc->angle_cos[s], leg_fw[i]), ndmul(rc->angle_sin[s], cr[i]));
    else np_rotate_towards(fw_rot, leg_fw, cr, table_fw);
  } else {
    for (int i = 0; i < 3; ++i) fw_rot[i] = leg_fw[i];
  }
  double above[3] = {ndadd(tsp[0], 0.0), ndadd(tsp[1], 0.0), ndadd(tsp[2], rc->z_finedist)};
  const bool safe_grasp = touched && (eef[2] < ndsub(grasp[2], 0.0));
  const double d_site = dv_dist(tsp, lsp), d_above = dv_dist(above, lsp);
  const double up_sim = np_cos_siml(leg_up, table_up), fw_sim = np_cos_siml(fw_rot, table_fw);
  double neg_up[3] = {-table_up[0], -table_up[1], -table_up[2]}, l_t[3], t_l[3];
  dv_sub(l_t, lsp, tsp); dv_sub(t_l, tsp, lsp);
  const double proj_t = np_cos_siml(neg_up, l_t), proj_l = np_cos_siml(leg_up, t_l);
  const double disp = dv_dist(tsp, st->table_site0);
  double sq = 0.0;
  for (int k = 0; k < act_dim - 2; ++k) sq = k == 0 ? ndmul(ac[0], ac[0]) : ndfma(ac[k], ac[k], sq);
  const double a_grip = ac[act_dim - 2], a_conn = ac[act_dim - 1];
  const double ctrl = ndmul(ndsqrt(sq), -c->ctrl_penalty_coef);
  const double other = ndmul(-c->move_other_part_penalty_coef, disp);
  const bool moved = disp > 0.1;
  // ---- _stable_grip_reward: evaluated for the phase at entry (its verdict feeds the shortcuts) and again for the phase after them
  double eef_up[3], eef_fw[3], neg_fw[3];
  dv_col(eef_up, gm, 2); dv_col(eef_fw, gm, 1);
  for (int i = 0; i < 3; ++i) neg_fw[i] = -eef_fw[i];
  const double down[3] = {0.0, 0.0, -1.0};
  const double up_d = np_cos_siml(eef_up, down);
  const double fw_d = pymax(np_cos_siml(eef_fw, gvec), np_cos_siml(neg_fw, gvec));
  const double up_rew = ndmul(c->eef_up_dist_coef, ndsub(up_d, 1.0)), fw_rew = ndmul(ndsub(fabs(fw_d), 1.0), c->eef_forward_dist_coef);
  bool grip_ok = true;
  if (st->phase <= FE_PH_LIFT) grip_ok = grip_ok && up_d > c->eef_rot_threshold;
  if (st->phase >= FE_PH_ABOVE_LEG && st->phase <= FE_PH_LIFT) grip_ok = grip_ok && fw_d > c->eef_rot_threshold;
  int skips = 0;
  if (!c->phase_ob) { // shortcuts a policy may take
    if (safe_grasp && grip_ok && st->phase < FE_PH_GRASP) { skips |= 1; st->phase = FE_PH_LIFT; }
    if (touched && (st->phase == FE_PH_LIFT || st->phase == FE_PH_ALIGN)) {
      if ((d_site < c->move_pos_threshold || d_above < c->move_pos_threshold) && up_sim > c->move_rot_threshold && fw_sim > c->move_rot_threshold) {
        skips |= 2;
        st->phase = FE_PH_FINE;
        st->prev[FE_DP_MOVE_POS] = d_site; st->prev[FE_DP_MOVE_UP] = up_sim; st->prev[FE_DP_MOVE_FWD] = fw_sim;
        st->prev[FE_DP_PROJ_T] = proj_t; st->prev[FE_DP_PROJ_L] = proj_l;
      }
    }
  }
  const int drop_leg = (st->phase > FE_PH_GRASP && !touched && !st->dropped && !connected) ? 1 : 0;
  const int table_moved_now = (moved && !st->table_moved) ? 1 : 0;
  double grip_rew = 0.0;
  grip_ok = true;
  if (st->phase <= FE_PH_LIFT) { grip_rew = ndadd(grip_rew, up_rew); grip_ok = grip_ok && up_d > c->eef_rot_threshold; }
  if (st->phase >= FE_PH_ABOVE_LEG && st->phase <= FE_PH_LIFT) { grip_rew = ndadd(grip_rew, fw_rew); grip_ok = grip_ok && fw_d > c->eef_rot_threshold; }
  const bool open_phase = st->phase <= FE_PH_LOWER_EEF;
  const bool hand_ok = open_phase ? a_grip < 0.0 : a_grip > 0.0;
  const double hand = ndmul(open_phase ? -a_grip : a_grip, c->gripper_penalty_coef);

#define FE_DENSE_MISHAP(flag, cost) do { st->flag = 1; done = c->early_termination ? 1 : 0; if (c->early_termination) bonus = ndsub(bonus, (cost)); } while (0)
#define FE_DENSE_ATTACHED() do { bonus = ndadd(bonus, ndmul(P, 2.0)); bonus = ndsub(bonus, ndmul((double)st->fine_aligned, c->aligned_bonus_coef)); \
    st->phase = FE_PH_INIT_EEF; st->subtask += 1; if (st->subtask == n_goal || st->subtask >= rc->nsub) { done = 1; st->success = 1; } \
    else { fe_dense_begin_subtask(w, c, rc, st); done = 0; st->success = 0; } } while (0)
#define FE_DENSE_ALIGNED() fe_is_aligned_d(lsp, lsm, tsp, tsm, rc->n_allowed[s], rc->allowed_cos[s], rc->allowed_sin[s], thr, tq_, &tq_set_)

  const int phase = st->phase;
  double term = 0.0, tq_[4];
  bool tq_set_;
  // lower_eef / grasp_leg share this term
  double lower_target[3] = {ndadd(grasp[0], 0.0), ndadd(grasp[1], 0.0), ndadd(grasp[2], -0.015)};
  if (phase != FE_PH_FINE && connected) {
    const bool correct = FE_DENSE_ALIGNED();
    if (moved) FE_DENSE_MISHAP(table_moved, P);
    else if (correct) FE_DENSE_ATTACHED();
    else { st->success = 0; done = 1; }
  } else if (phase == FE_PH_INIT_EEF) {
    const double d = dv_dist(eef, st->init_eef);
    FE_DENSE_SHAPED(term, FE_DP_INIT_EEF, d, c->init_eef_pos_dist_coef, 10.0, exp(ndmul(-10.0, pymin(v_, 0.5))), false, ndmul(-d, c->init_eef_pos_dist_coef));
    if (d < 0.03 && grip_ok && hand_ok) {
      st->phase += 1;
      bonus = ndadd(bonus, P);
      double t[3] = {ndadd(grasp[0], 0.0), ndadd(grasp[1], 0.0), ndadd(grasp[2], 0.05)};
      st->prev[FE_DP_ABOVE_LEG] = dv_dist(eef, t);
    }
  } else if (phase == FE_PH_ABOVE_LEG) {
    double t[3] = {ndadd(grasp[0], 0.0), ndadd(grasp[1], 0.0), ndadd(grasp[2], 0.05)};
    const double d = dv_dist(eef, t);
    FE_DENSE_SHAPED(term, FE_DP_ABOVE_LEG, d, c->move_eef_pos_dist_coef, 10.0, pymin(v_, 1.0), true, ndmul(-d, c->move_eef_pos_dist_coef));
    if (d < 0.03 && grip_ok && hand_ok) {
      st->phase += 1;
      bonus = ndadd(bonus, P);
      st->prev[FE_DP_EEF_LEG] = dv_dist(eef, lower_target);
    }
  } else if (phase == FE_PH_LOWER_EEF || phase == FE_PH_GRASP) {
    const double d = dv_dist(eef, lower_target);
    FE_DENSE_SHAPED(term, FE_DP_EEF_LEG, d, c->lower_eef_pos_dist_coef, 10.0, pymin(v_, 0.2), true, ndmul(-d, c->lower_eef_pos_dist_coef));
    if (phase == FE_PH_LOWER_EEF) {
      const bool ok = dv_dist_xy(eef, lower_target) < 0.02 && fabs(ndsub(eef[2], lower_target[2])) < 0.015;
      if (ok && grip_ok && hand_ok) { bonus = ndadd(bonus, P); st->phase += 1; }
    } else {
      term = ndadd(term, ndmul(ndsub(a_grip, st->prev[FE_DP_GRASP]), c->grasp_dist_coef));
      st->prev[FE_DP_GRASP] = a_grip;
      if (touched && safe_grasp && grip_ok) { st->phase += 1; bonus = ndadd(bonus, P); }
    }
  } else if (phase == FE_PH_LIFT) {
    const double xy = dv_dist_xy(st->lift_target, leg), z = fabs(ndsub(st->lift_target[2], leg[2]));
    double rz, rxy;
    FE_DENSE_SHAPED(rz, FE_DP_LIFT_Z, z, c->lift_z_dist_coef, 10.0, pymin(v_, 0.5), true, ndmul(-z, c->lift_z_dist_coef));
    FE_DENSE_SHAPED(rxy, FE_DP_LIFT_XY, xy, c->lift_xy_dist_coef, 10.0, pymin(v_, 0.8), true, ndmul(-xy, c->lift_xy_dist_coef));
    term = ndadd(rxy, rz);
    if (touched && leg[2] > ndadd(st->leg0[2], 0.01) && safe_grasp && !st->lifted) { st->lifted = 1; term = ndadd(term, nddiv(P, 2.0)); }
    if (!touched) term = pymin(term, 0.0);
    if (!touched) FE_DENSE_MISHAP(dropped, nddiv(P, 2.0));
    else if (moved) FE_DENSE_MISHAP(table_moved, nddiv(P, 2.0));
    else if (xy < c->lift_xy_pos_threshold && z < c->lift_z_pos_threshold) {
      st->phase += 1;
      bonus = ndadd(bonus, P);
      st->prev[FE_DP_MOVE_POS] = 0.0; st->prev[FE_DP_MOVE_UP] = up_sim; st->prev[FE_DP_MOVE_FWD] = fw_sim;
    }
  } else if (phase == FE_PH_ALIGN || phase == FE_PH_MOVE) {
    double rp, ru, rf;
    bool ok;
    if (phase == FE_PH_ALIGN) {
      const double d = dv_dist(st->lift_target, leg);
      FE_DENSE_SHAPED(rp, FE_DP_MOVE_POS, d, c->align_pos_dist_coef, 10.0, pymin(v_, 0.4), true, ndmul(-d, c->align_pos_dist_coef));
      FE_DENSE_SHAPED(ru, FE_DP_MOVE_UP, up_sim, c->align_rot_dist_coef, 10.0, v_, false, ndmul(ndsub(up_sim, 1.0), c->align_rot_dist_coef));
      FE_DENSE_SHAPED(rf, FE_DP_MOVE_FWD, fw_sim, c->align_rot_dist_coef, 10.0, v_, false, ndmul(ndsub(fw_sim, 1.0), c->align_rot_dist_coef));
      ok = d < c->align_pos_threshold && up_sim > c->align_rot_threshold && fw_sim > c->align_rot_threshold && touched;
    } else {
      FE_DENSE_SHAPED(rp, FE_DP_MOVE_POS, d_above, c->move_pos_dist_coef, 10.0, pymin(v_, 0.5), true, ndmul(-d_site, c->move_pos_dist_coef));
      FE_DENSE_SHAPED(ru, FE_DP_MOVE_UP, up_sim, c->move_rot_dist_coef, 10.0, pymax(v_, 0.0), false, ndmul(ndsub(up_sim, 1.0), c->move_rot_dist_coef));
      FE_DENSE_SHAPED(rf, FE_DP_MOVE_FWD, fw_sim, c->move_rot_dist_coef, 10.0, pymax(v_, 0.0), false, ndmul(ndsub(fw_sim, 1.0), c->move_rot_dist_coef));
      ok = (d_above < c->move_pos_threshold || d_site < c->move_pos_threshold) && up_sim > c->move_rot_threshold && fw_sim > c->move_rot_threshold && touched;
    }
    if (!touched) { rp = pymin(rp, 0.0); ru = pymin(ru, 0.0); rf = pymin(rf, 0.0); }
    term = ndadd(ndadd(rp, ru), rf);
    if (!touched) FE_DENSE_MISHAP(dropped, nddiv(P, 2.0));
    else if (moved) FE_DENSE_MISHAP(table_moved, nddiv(P, 2.0));
    else if (ok) {
      st->phase += 1;
      bonus = ndadd(bonus, ndmul(P, 2.0));
      if (phase == FE_PH_ALIGN) st->prev[FE_DP_MOVE_POS] = d_above;
      else { st->prev[FE_DP_MOVE_POS] = d_site; st->prev[FE_DP_PROJ_T] = proj_t; st->prev[FE_DP_PROJ_L] = proj_l; }
    }
  } else { // move_leg_fine
    const double kf = c->move_fine_rot_dist_coef, lo = ndsub(c->move_rot_threshold, 0.1);
    double rp, ru, rf, rt, rl;
    FE_DENSE_SHAPED(rp, FE_DP_MOVE_POS, d_site, c->move_fine_pos_dist_coef, 10.0, exp(ndmul(c->move_fine_pos_exp_coef, v_)), false, ndmul(-d_site, c->move_fine_pos_dist_coef));
    FE_DENSE_SHAPED(ru, FE_DP_MOVE_UP, up_sim, kf, 10.0, exp(ndmul(-2.0, ndsub(1.0, pymax(v_, lo)))), false, ndmul(ndsub(up_sim, 1.0), kf));
    FE_DENSE_SHAPED(rf, FE_DP_MOVE_FWD, fw_sim, kf, 10.0, exp(ndmul(-2.0, ndsub(1.0, pymax(v_, lo)))), false, ndmul(ndsub(fw_sim, 1.0), kf));
    FE_DENSE_SHAPED(rt, FE_DP_PROJ_T, proj_t, kf, 5.0, exp(ndmul(-3.0, ndsub(1.0, pymax(fabs(v_), 0.5)))), false, nddiv(ndmul(ndsub(proj_t, 1.0), kf), 10.0));
    FE_DENSE_SHAPED(rl, FE_DP_PROJ_L, proj_l, kf, 5.0, exp(ndmul(-3.0, ndsub(1.0, pymax(fabs(v_), 0.5)))), false, nddiv(ndmul(ndsub(proj_l, 1.0), kf), 10.0));
    const bool aligned = FE_DENSE_ALIGNED();
    const bool good = connected && aligned;
    if (!touched) { rp = pymin(rp, 0.0); ru = pymin(ru, 0.0); rf = pymin(rf, 0.0); rt = pymin(rt, 0.0); rl = pymin(rl, 0.0); }
    term = ndadd(ndadd(ndadd(ndadd(rp, ru), rf), rt), rl);
    if (aligned) { st->fine_aligned += 1; term = ndadd(term, ndmul(ndadd(a_conn, 1.0), c->aligned_bonus_coef)); }
    if (connected) term = 0.0;
    if (moved) FE_DENSE_MISHAP(table_moved, P);
    else if (good) FE_DENSE_ATTACHED();
    else if (connected) { done = 1; st->success = 0; }
    if (!touched && !good) FE_DENSE_MISHAP(dropped, P);
  }
  double reward = ndadd(0.0, ndadd(ndadd(ctrl, term), grip_rew));
  reward = ndadd(reward, ndadd(ndadd(hand, bonus), other));
  double drop_pen = 0.0;
  if (st->dropped && !c->early_termination) { reward = ndsub(reward, c->drop_penalty_coef); drop_pen = -c->drop_penalty_coef; }
  *reward_out = reward;
  *done_out = done;
  if (info) {
    info[0] = (double)st->phase; info[1] = (double)st->subtask; info[2] = bonus; info[3] = ctrl; info[4] = hand; info[5] = other; info[6] = drop_pen;
    info[7] = (double)touched; info[8] = (double)drop_leg; info[9] = (double)table_moved_now; info[10] = grip_ok ? 1.0 : 0.0; info[11] = (double)skips;
  }
#undef FE_DENSE_MISHAP
#undef FE_DENSE_ATTACHED
#undef FE_DENSE_ALIGNED
}

// explicit poses (test hook fe_dense_eval): sites and parts are indices into per-record arrays
struct FeArrayWorld {
  const double* spos;  // [nsite][3]
  const double* smat;  // [nsite][9] row-major
  const double* ppos;  // [npart][3]
  const uint8_t* touch; // [npart] both fingers on the part
  FE_MEMBER void site_pos(int s, double* p) const { p[0] = spos[3 * s]; p[1] = spos[3 * s + 1]; p[2] = spos[3 * s + 2]; }
  FE_MEMBER void site_pose(int s, double* p, double* m) const { site_pos(s, p); for (int k = 0; k < 9; ++k) m[k] = smat[9 * s + k]; }
  FE_MEMBER void part_pos(int q, double* p) const { p[0] = ppos[3 * q]; p[1] = ppos[3 * q + 1]; p[2] = ppos[3 * q + 2]; }
  FE_MEMBER bool touch_both(int q) const { return touch[q] != 0; }
};

// one thread walks the records of one episode: a record with reset != 0 starts the episode on the world it shows, at subtask reset - 1
FE_HDN void fe_dense_eval_episode(const fe_dense_config* c, const fe_dense_recipe* rc, const double* thr, int n_goal, int first, int count, int nsite, int npart,
                                  int act_dim, const double* spos, const double* smat, const double* ppos, const uint8_t* touch, const uint8_t* reset,
                                  const uint8_t* connected, const double* ac, double* reward, uint8_t* done, double* info) {
  FeDenseState st;
  for (int t = first; t < first + count; ++t) {
    FeArrayWorld w = {spos + (size_t)t * nsite * 3, smat + (size_t)t * nsite * 9, ppos + (size_t)t * npart * 3, touch + (size_t)t * npart};
    double* inf = info + (size_t)t * FE_DENSE_INFO;
    if (reset[t]) {
      fe_dense_begin_episode(w, c, rc, reset[t] - 1, &st);
      reward[t] = 0.0; done[t] = 0;
      for (int k = 0; k < FE_DENSE_INFO; ++k) inf[k] = 0.0;
      inf[0] = (double)st.phase; inf[1] = (double)st.subtask;
    } else {
      int d = 0;
      fe_dense_step(w, c, rc, thr, n_goal, &st, ac + (size_t)t * act_dim, act_dim, connected[t], reward + t, &d, inf);
      done[t] = (uint8_t)(d | (st.success ? 2 : 0));
    }
  }
}
