// fe_ctl.h -- the five torque controllers of furniture/env/controllers/arm_controller.py (NEW_CONTROLLERS, furniture.py:41-47), evaluated by
// lane 0 of the env's warp before every mj_step (FurnitureEnv._pre_action :1706-1759 inside _do_controller_step :3065-3093):
//   fe_ctl_torques <- Controller.transform_action :98-105, linear_interpolate :157-164, calculate_orientation_error :179-201,
//                     JointTorqueController.action_to_torques :275-303, JointVelocityController :345-366, JointImpedanceController :432-496,
//                     PositionOrientationController :639-739 with update_model_opspace :752-799 and set_goal_position / _orientation
//                     :801-812, PositionController :925-930 -- parameters of controllers/controller_config.hjson (host: controllers.py)
// float64 throughout; one function, five modes, because the reference's classes share one skeleton (see oracle/controller_oracle.py, which
// is pinned to the reference's own classes; this file is checked against the same golden records through fe_ctl_eval).
// Kept quirks: the ramp is ramp_steps = floor(0.2 * control_freq / timestep) = 2000 mj_steps long; the position controller fixes its
// orientation goal once per controller lifetime (ori_set survives resets).
#pragma once
#include "fe_env.h"

enum { FE_CTL_JOINT_TORQUE = 0, FE_CTL_JOINT_VELOCITY = 1, FE_CTL_JOINT_IMPEDANCE = 2, FE_CTL_POS_ORI = 3, FE_CTL_POS = 4 };

struct FeCtlState { // per env, in HBM
  int32_t step, ori_set, started, pad_;
  double last[7], start[7], delta[7];                                     // joint-space goal ramp
  double last_pos[3], pos_start[3], pos_delta[3];                         // operational-space position ramp
  double last_ori[9], ori_start[9], ori_delta[3], ori_goal[9];            // orientation ramp (row-major matrices) and goal
};
struct FeCtlIn { // what Controller.update_model reads from the simulator (:107-126, update_mass_matrix :128-137)
  double pos[3], R[9], velp[3], velr[3], q[7], qvel[7], Jx[21], Jr[21], M[49];
};

FE_HD void ctl_euler2mat(double* m, const double* e) { // transform_utils.euler2mat (:360-380), row-major
  const double ai = -e[2], aj = -e[1], ak = -e[0];
  const double si = sin(ai), sj = sin(aj), sk = sin(ak), ci = cos(ai), cj = cos(aj), ck = cos(ak);
  const double cc = ci * ck, cs = ci * sk, sc = si * ck, ss = si * sk;
  m[0] = cj * ci; m[1] = cj * si; m[2] = -sj;
  m[3] = sj * cs - sc; m[4] = sj * ss + cc; m[5] = cj * sk;
  m[6] = sj * cc + ss; m[7] = sj * sc - cs; m[8] = cj * ck;
}
FE_HD void ctl_cross(double* r, const double* a, const double* b) { r[0] = a[1] * b[2] - a[2] * b[1]; r[1] = a[2] * b[0] - a[0] * b[2]; r[2] = a[0] * b[1] - a[1] * b[0]; }
// 0.5 * sum of cross(current column, desired column)
FE_HD void ctl_ori_error(double* e, const double* desired, const double* current) {
  e[0] = e[1] = e[2] = 0.0;
  for (int c = 0; c < 3; ++c) {
    const double a[3] = {current[c], current[3 + c], current[6 + c]}, b[3] = {desired[c], desired[3 + c], desired[6 + c]};
    double x[3];
    ctl_cross(x, a, b);
    e[0] += x[0]; e[1] += x[1]; e[2] += x[2];
  }
  e[0] *= 0.5; e[1] *= 0.5; e[2] *= 0.5;
}
// r = euler2mat(-d)^T * base
FE_HD void ctl_rotate_by(double* r, const double* d, const double* base) {
  const double nd[3] = {-d[0], -d[1], -d[2]};
  double E[9];
  ctl_euler2mat(E, nd);
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r[3 * i + j] = E[i] * base[j] + E[3 + i] * base[3 + j] + E[6 + i] * base[6 + j];
}
// pseudo-inverse of a symmetric positive semi-definite 3x3 with the reference's singular-value threshold (:784-793): Jacobi eigenvalues
FE_HDN void ctl_pinv_sym3(double* P, const double* A_in, double threshold) {
  double A[9], V[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  for (int k = 0; k < 9; ++k) A[k] = A_in[k];
  for (int sweep = 0; sweep < 30; ++sweep) {
    const double off = fabs(A[1]) + fabs(A[2]) + fabs(A[5]);
    if (off < 1e-300) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        const double apq = A[3 * p + q];
        if (fabs(apq) < 1e-300) continue;
        const double theta = (A[3 * q + q] - A[3 * p + p]) / (2.0 * apq);
        const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0)), c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; ++k) { const double akp = A[3 * k + p], akq = A[3 * k + q]; A[3 * k + p] = c * akp - s * akq; A[3 * k + q] = s * akp + c * akq; }
        for (int k = 0; k < 3; ++k) { const double apk = A[3 * p + k], aqk = A[3 * q + k]; A[3 * p + k] = c * apk - s * aqk; A[3 * q + k] = s * apk + c * aqk; }
        for (int k = 0; k < 3; ++k) { const double vkp = V[3 * k + p], vkq = V[3 * k + q]; V[3 * k + p] = c * vkp - s * vkq; V[3 * k + q] = s * vkp + c * vkq; }
      }
  }
  for (int k = 0; k < 9; ++k) P[k] = 0.0;
  for (int e = 0; e < 3; ++e) {
    const double s = fabs(A[4 * e]); // singular value of a symmetric matrix
    if (s < threshold) continue;
    const double inv = (A[4 * e] < 0 ? -1.0 : 1.0) / s;
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) P[3 * i + j] += inv * V[3 * i + e] * V[3 * j + e];
  }
}
// X = M^-1 B for the symmetric positive definite 7x7 M (Cholesky), B 7 x nb column-major in X on entry
FE_HDN void ctl_spd7_solve(const double* M, double* X, int nb) {
  double L[49];
  for (int i = 0; i < 7; ++i)
    for (int j = 0; j <= i; ++j) {
      double s = M[7 * i + j];
      for (int k = 0; k < j; ++k) s -= L[7 * i + k] * L[7 * j + k];
      L[7 * i + j] = i == j ? sqrt(s) : s / L[7 * j + j];
    }
  for (int b = 0; b < nb; ++b) {
    double* x = X + 7 * b;
    for (int i = 0; i < 7; ++i) { double s = x[i]; for (int k = 0; k < i; ++k) s -= L[7 * i + k] * x[k]; x[i] = s / L[7 * i + i]; }
    for (int i = 6; i >= 0; --i) { double s = x[i]; for (int k = i + 1; k < 7; ++k) s -= L[7 * k + i] * x[k]; x[i] = s / L[7 * i + i]; }
  }
}

FE_HDN void fe_ctl_reset(const fe_ctl_config* c, FeCtlState* s) { // Controller.reset of the five classes; ori_set is not touched
  s->step = 0;
  for (int k = 0; k < 7; ++k) s->last[k] = 0.0;
  for (int k = 0; k < 3; ++k) s->last_pos[k] = 0.0;
  for (int k = 0; k < 9; ++k) s->last_ori[k] = (k % 4 == 0) ? 1.0 : 0.0;
}

FE_HDN void fe_ctl_torques(const fe_ctl_config* c, FeCtlState* s, const double* action, int policy_step, const FeCtlIn* in, double* tau) {
  const int n = c->control_dim;
  double a[7];
  for (int k = 0; k < n; ++k) { const double v = action[k] < -1.0 ? -1.0 : (action[k] > 1.0 ? 1.0 : action[k]); a[k] = v * c->control_max[k]; }
  const double steps = c->ramp_steps;
  if (c->mode <= FE_CTL_JOINT_IMPEDANCE) {
    if (policy_step) {
      s->step = 0;
      double goal[7];
      if (c->mode == FE_CTL_JOINT_IMPEDANCE) {
        bool zero = true;
        for (int k = 0; k < 7; ++k) { goal[k] = in->q[k] + a[k]; zero = zero && s->last[k] == 0.0; }
        if (zero) for (int k = 0; k < 7; ++k) s->last[k] = in->q[k];
      } else {
        for (int k = 0; k < 7; ++k) goal[k] = a[k];
      }
      for (int k = 0; k < 7; ++k) { s->start[k] = s->last[k]; s->delta[k] = (goal[k] - s->last[k]) / steps; }
    }
    for (int k = 0; k < 7; ++k) s->last[k] = s->start[k] + (double)(s->step + 1) * s->delta[k];
    if ((double)s->step < steps - 1.0) s->step += 1;
    if (c->mode == FE_CTL_JOINT_TORQUE) { for (int k = 0; k < 7; ++k) tau[k] = s->last[k]; return; }
    if (c->mode == FE_CTL_JOINT_VELOCITY) { for (int k = 0; k < 7; ++k) tau[k] = c->kv[k] * (s->last[k] - in->qvel[k]); return; }
    double v[7], nrm = 0.0, t[7];
    for (int k = 0; k < 7; ++k) { v[k] = in->qvel[k]; nrm += v[k] * v[k]; }
    nrm = sqrt(nrm);
    if (nrm > 7.0) for (int k = 0; k < 7; ++k) v[k] = v[k] / (nrm * 7.0);
    for (int k = 0; k < 7; ++k) { const double kvk = 2.0 * sqrt(c->kp[k]) * c->damping[k]; t[k] = c->kp[k] * (s->last[k] - in->q[k]) - kvk * v[k]; }
    for (int i = 0; i < 7; ++i) { double acc = 0.0; for (int k = 0; k < 7; ++k) acc += in->M[7 * i + k] * t[k]; tau[i] = acc; }
    return;
  }
  // ---- operational space
  if (policy_step) {
    s->step = 0;
    double goal_pos[3];
    for (int k = 0; k < 3; ++k) goal_pos[k] = in->pos[k] + a[k];
    if (c->mode == FE_CTL_POS_ORI) ctl_rotate_by(s->ori_goal, a + 3, in->R);
    else if (!s->ori_set) { for (int k = 0; k < 9; ++k) s->ori_goal[k] = in->R[k]; s->ori_set = 1; }
    if (s->last_pos[0] == 0.0 && s->last_pos[1] == 0.0 && s->last_pos[2] == 0.0) for (int k = 0; k < 3; ++k) s->last_pos[k] = in->pos[k];
    bool eye = true;
    for (int k = 0; k < 9; ++k) eye = eye && s->last_ori[k] == ((k % 4 == 0) ? 1.0 : 0.0);
    if (eye) for (int k = 0; k < 9; ++k) s->last_ori[k] = in->R[k];
    for (int k = 0; k < 3; ++k) { s->pos_start[k] = s->last_pos[k]; s->pos_delta[k] = (goal_pos[k] - s->last_pos[k]) / steps; }
    double e[3];
    ctl_ori_error(e, s->ori_goal, s->last_ori);
    for (int k = 0; k < 3; ++k) s->ori_delta[k] = e[k] / steps;
    for (int k = 0; k < 9; ++k) s->ori_start[k] = s->last_ori[k];
  }
  const double f = (double)(s->step + 1);
  for (int k = 0; k < 3; ++k) s->last_pos[k] = s->pos_start[k] + f * s->pos_delta[k];
  { const double d[3] = {f * s->ori_delta[0], f * s->ori_delta[1], f * s->ori_delta[2]}; ctl_rotate_by(s->last_ori, d, s->ori_start); }
  if ((double)s->step < steps - 1.0) s->step += 1;
  double force[3], torque[3], oe[3], kv[6];
  for (int k = 0; k < 6; ++k) kv[k] = 2.0 * sqrt(c->kp[k]) * c->damping[k];
  ctl_ori_error(oe, s->last_ori, in->R);
  for (int k = 0; k < 3; ++k) { force[k] = (s->last_pos[k] - in->pos[k]) * c->kp[k] - in->velp[k] * kv[k]; torque[k] = oe[k] * c->kp[3 + k] - in->velr[k] * kv[3 + k]; }
  // lambda_x = pinv(Jx M^-1 Jx^T), lambda_r = pinv(Jr M^-1 Jr^T)
  double X[42], A[9], lam[9], wrench[6];
  for (int part = 0; part < 2; ++part) {
    const double* J = part == 0 ? in->Jx : in->Jr;
    for (int b = 0; b < 3; ++b) for (int k = 0; k < 7; ++k) X[7 * b + k] = J[7 * b + k]; // columns of J^T
    ctl_spd7_solve(in->M, X, 3);
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) { double acc = 0.0; for (int k = 0; k < 7; ++k) acc += J[7 * i + k] * X[7 * j + k]; A[3 * i + j] = acc; }
    for (int i = 0; i < 3; ++i) for (int j = i + 1; j < 3; ++j) { const double m_ = 0.5 * (A[3 * i + j] + A[3 * j + i]); A[3 * i + j] = A[3 * j + i] = m_; }
    ctl_pinv_sym3(lam, A, 0.00025);
    const double* w_in = part == 0 ? force : torque;
    for (int i = 0; i < 3; ++i) wrench[3 * part + i] = lam[3 * i] * w_in[0] + lam[3 * i + 1] * w_in[1] + lam[3 * i + 2] * w_in[2];
  }
  for (int k = 0; k < 7; ++k) {
    double acc = 0.0;
    for (int i = 0; i < 3; ++i) acc += in->Jx[7 * i + k] * wrench[i] + in->Jr[7 * i + k] * wrench[3 + i];
    tau[k] = acc;
  }
}

// test hook: one thread walks the records of one episode (a record with reset != 0 starts with a fresh controller)
FE_HDN void fe_ctl_eval_episode(const fe_ctl_config* c, int first, int count, const uint8_t* reset, const uint8_t* policy_step, const double* action /* [7] per record */,
                                const FeCtlIn* in, double* tau /* [7] per record */) {
  FeCtlState s;
  s.ori_set = 0; s.started = 0;
  for (int t = first; t < first + count; ++t) {
    if (reset[t]) { s.ori_set = 0; fe_ctl_reset(c, &s); }
    fe_ctl_torques(c, &s, action + (size_t)7 * t, policy_step[t], in + t, tau + (size_t)7 * t);
  }
}

// ---------------------------------------------------------------- the env step under a torque controller
struct FeCtlArgs {
  const fe_ctl_config* c;
  FeCtlState* st;
};

// Controller.update_model (:107-126) + update_mass_matrix (:128-137): the hand body's pose and velocity, the arm's joint state, the hand
// Jacobian (mj_jacBody: rows about the body origin) and the arm block of the joint-space inertia, from the last forward pass in the slice
FE_HDN void fe_ctl_read(FeEnv* e, const fe_ctl_config* c, FeCtlIn* in) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const fe_scene* sc = e->sc;
  const int hl = sc->hand_link[0], nr = m->nr;
  const float* Rl = w->lmat() + 9 * hl;
  float t[3], hp[3], hq[4], Rh[9], vel[3];
  m3mulv(t, Rl, c->hand_pos);
  v3add(hp, w->lpos() + 3 * hl, t);
  qmul(hq, w->lquat() + 4 * hl, c->hand_quat);
  qnormalize(hq);
  q2mat(Rh, hq);
  fe_point_vel(w, w->lvel(), hl, hp, vel);
  for (int k = 0; k < 3; ++k) { in->pos[k] = (double)hp[k]; in->velp[k] = (double)vel[k]; in->velr[k] = (double)w->lvel()[6 * hl + k]; }
  for (int k = 0; k < 9; ++k) in->R[k] = (double)Rh[k];
  const float Pr[3] = {m->robot_ref[0], m->robot_ref[1], m->robot_ref[2]};
  float d[3];
  v3sub(d, hp, Pr);
  for (int k = 0; k < 7; ++k) {
    const int da = sc->arm_dof[k];
    in->q[k] = (double)w->qpos()[da];
    in->qvel[k] = (double)w->qvel()[da];
    const float* S = w->S() + 6 * da; // [axis; (anchor - Pr) x axis]: spatial velocity about robot_ref per unit joint velocity
    float cr[3] = {0.f, 0.f, 0.f}, ang[3] = {0.f, 0.f, 0.f}, lin[3] = {0.f, 0.f, 0.f};
    if ((m->link_ancmask[hl] >> da) & 1) { v3cpy(ang, S); v3cross(cr, S, d); v3add(lin, S + 3, cr); }
    for (int i = 0; i < 3; ++i) { in->Jx[7 * i + k] = (double)lin[i]; in->Jr[7 * i + k] = (double)ang[i]; }
    for (int j = 0; j < 7; ++j) in->M[7 * k + j] = (double)w->Mr()[da * nr + sc->arm_dof[j]];
  }
}

// FurnitureEnv.step with one of the NEW_CONTROLLERS for the one-arm env: _do_controller_step (furniture.py:3065-3093) with _pre_action
// (:1706-1759) before every mj_step; action = [arm command (control_dim), gripper, connect]
FE_FN void fe_env_ctl_step_one(FeEnv* e, FeCtlArgs ctl, const float* action, float* reward_out, uint8_t* done_out, int32_t* info_out) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const fe_scene* sc = e->sc;
  const fe_ctl_config* c = ctl.c;
  const int act_dim = c->control_dim + 2;
  const float* a = action + (size_t)e->env * act_dim;
  float grip = a[act_dim - 2];
  if (e->cfg->discrete_grip) grip = grip < 0.f ? -1.f : 1.f; // furniture_sawyer.py:73-74
  const float connect = a[act_dim - 1];
  FeCtlState* st = ctl.st + e->env;
  LANES_BEGIN
    if (lane == 0) {
      if (e->es.episode_len[e->env] == 0) fe_ctl_reset(c, st); // _reset: controller.reset() (furniture.py:1885-1887)
      fe_env_clear_flags(e);
    }
  LANES_END
  fe_forward(w); // sim.forward() ahead of the loop (:3080): the first _pre_action reads fresh kinematics
  for (int i = 0; i < e->cfg->nsub; ++i) {
    LANES_BEGIN
      if (lane == 0) {
        double arm[7] = {0, 0, 0, 0, 0, 0, 0}, tau[7];
        for (int k = 0; k < c->control_dim; ++k) arm[k] = (double)a[k];
        { const double x = arm[0] * c->move_speed, y = arm[1] * c->move_speed, z = arm[2] * c->move_speed; arm[0] = -y; arm[1] = x; arm[2] = z; } // :3069-3071, every controller
        FeCtlIn in;
        fe_ctl_read(e, c, &in);
        fe_ctl_torques(c, st, arm, i == 0, &in, tau);
        for (int u = 0; u < m->nu; ++u) {
          const int src = sc->act_src[u];
          if (src < sc->narm) w->ctrl()[u] = w->bias()[sc->arm_dof[src]] + (float)tau[src]; // ctrl = qfrc_bias + torques (:1756-1758)
          else { const float lo = m->act_ctrlrange[u][0], hi = m->act_ctrlrange[u][1]; w->ctrl()[u] = 0.5f * (hi + lo) + 0.5f * (hi - lo) * (sc->act_sign[u] * grip); } // apply_rescaled_action (:1722-1727)
        }
      }
    LANES_END
    fe_substep_lockstep(w);
  }
  const int fail = (w->u()[FE_U_FLAGS] & FE_FLAG_DIVERGED) ? 1 : 0;
  fe_env_finish(e, a, act_dim, connect, fail, fail, reward_out, done_out, info_out);
}
