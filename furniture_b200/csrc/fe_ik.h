// fe_ik.h -- control_type="ik" for the one-arm (Sawyer) env, executed by the warp that owns the env:
//   fe_env_ik_step_one <- FurnitureEnv._do_ik_step (furniture/env/furniture.py:2899-2996) inside FurnitureEnv.step: action scaling and axis
//                         swap, workspace clip (_bounded_d_pos :1252-1258), the accumulated orientation target with the reference's
//                         quaternion conventions (transform_utils.euler_to_quat :617-630 fed an (x,y,z,w) array), _make_input :1332-1343,
//                         SawyerIKController.get_control (controllers/sawyer_ik_controller.py:46-87): target += 0.3 dpos, inverse
//                         kinematics from the current joints, joint velocities -5 (q - q_cmd) clipped to [-1, 1]; then action_repeat x
//                         { _setup_action, _do_simulation } with the velocities recomputed in between (:2977-2995)
//   fe_ik_solve        <- replaces the pybullet solve (p.calculateInverseKinematics, :177-215, :248-281; pybullet and its URDF are not
//                         available): damped least squares on the arm's own chain, lane 0, float32 -- furniture_b200/ik.py: solve_ik is
//                         the same algorithm in float64 (oracle/ik_oracle.py)
// The part of an env step that follows the simulation (connect, reward, termination, observation) is the one of fe_env.h:
// fe_ik_controls / fe_ik_finish below restate fe_env_step_one's blocks with the policy action (8 numbers) and the low-level action
// (7 velocities + gripper) as separate arguments.  fe_env.h itself is left untouched on purpose: its step kernel is the stock build
// that is profiled and benched (profiles/); fold the two once a capture of the folded build is taken.
#pragma once
#include "fe_env.h"

struct FeIkState { // per env, in HBM; [arm]: right, left
  float s[2][4];          // _initial_<arm>_hand_quat: the accumulated orientation target, components as the reference stores them
  float target_pos[2][3]; // ik_robot_target_pos_<arm>, base frame
  float q_cmd[14];        // commanded_joint_positions (right arm, then left)
  float low[16];          // low-level action of the current repeat: the joint velocities of every arm, then one gripper action per arm
  int32_t iters[2];
};
struct FeIkArgs {
  const fe_ik_config* c;
  FeIkState* st;
};

// ---- quaternions in the reference's two conventions
FE_HD void ik_hamilton(float* r, const float* a, const float* b) { // first component scalar
  const float w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  const float y = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1], z = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
  r[0] = w; r[1] = x; r[2] = y; r[3] = z;
}
FE_HD void ik_xyzw_mul(float* r, const float* q1, const float* q0) { // transform_utils.quat_multiply(quaternion1, quaternion0)
  const float x0 = q0[0], y0 = q0[1], z0 = q0[2], w0 = q0[3], x1 = q1[0], y1 = q1[1], z1 = q1[2], w1 = q1[3];
  r[0] = x1 * w0 + y1 * z0 - z1 * y0 + w1 * x0; r[1] = -x1 * z0 + y1 * w0 + z1 * x0 + w1 * y0;
  r[2] = x1 * y0 - y1 * x0 + z1 * w0 + w1 * z0; r[3] = -x1 * x0 - y1 * y0 - z1 * z0 + w1 * w0;
}
FE_HD void ik_xyzw_to_mat(float* R, const float* q) { // transform_utils.quat2mat
  const float n = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  if (n < 8.8817842e-16f) { for (int k = 0; k < 9; ++k) R[k] = (k % 4 == 0) ? 1.f : 0.f; return; }
  const float sc = sqrtf(2.0f / n), w = q[3] * sc, x = q[0] * sc, y = q[1] * sc, z = q[2] * sc;
  R[0] = 1.f - y * y - z * z; R[1] = x * y - z * w; R[2] = x * z + y * w;
  R[3] = x * y + z * w; R[4] = 1.f - x * x - z * z; R[5] = y * z - x * w;
  R[6] = x * z - y * w; R[7] = y * z + x * w; R[8] = 1.f - x * x - y * y;
}
FE_HD void ik_mat_to_wxyz(float* q, const float* R) { // rotation matrix -> unit quaternion (w, x, y, z), largest component first
  const float tr = R[0] + R[4] + R[8];
  if (tr > 0.f) { const float s = sqrtf(tr + 1.f) * 2.f; q[0] = 0.25f * s; q[1] = (R[7] - R[5]) / s; q[2] = (R[2] - R[6]) / s; q[3] = (R[3] - R[1]) / s; }
  else if (R[0] > R[4] && R[0] > R[8]) { const float s = sqrtf(1.f + R[0] - R[4] - R[8]) * 2.f; q[0] = (R[7] - R[5]) / s; q[1] = 0.25f * s; q[2] = (R[1] + R[3]) / s; q[3] = (R[2] + R[6]) / s; }
  else if (R[4] > R[8]) { const float s = sqrtf(1.f + R[4] - R[0] - R[8]) * 2.f; q[0] = (R[2] - R[6]) / s; q[1] = (R[1] + R[3]) / s; q[2] = 0.25f * s; q[3] = (R[5] + R[7]) / s; }
  else { const float s = sqrtf(1.f + R[8] - R[0] - R[4]) * 2.f; q[0] = (R[3] - R[1]) / s; q[1] = (R[2] + R[6]) / s; q[2] = (R[5] + R[7]) / s; q[3] = 0.25f * s; }
  qnormalize(q);
}

// ---- the arm: joint k's body frame in the frame of joint k-1's body at zero angle (fe_ik_config), hinge about (jpos, jaxis)
FE_HD void fe_ik_fk(const fe_ik_arm* c, const float* q, float* hp, float* hq, float* anchors, float* axes) {
  float p[3] = {0.f, 0.f, 0.f}, quat[4] = {1.f, 0.f, 0.f, 0.f};
  for (int k = 0; k < 7; ++k) {
    float R[9], t[3], p0[3], q0[4], R0[9], ql[4], R1[9];
    q2mat(R, quat);
    m3mulv(t, R, c->link_pos[k]);
    v3add(p0, p, t);
    qmul(q0, quat, c->link_quat[k]);
    q2mat(R0, q0);
    m3mulv(t, R0, c->jpos[k]);
    v3add(anchors + 3 * k, p0, t);
    m3mulv(axes + 3 * k, R0, c->jaxis[k]);
    const float sn = sinf(0.5f * q[k]), cs = cosf(0.5f * q[k]);
    ql[0] = cs; ql[1] = c->jaxis[k][0] * sn; ql[2] = c->jaxis[k][1] * sn; ql[3] = c->jaxis[k][2] * sn;
    qmul(quat, q0, ql);
    qnormalize(quat);
    q2mat(R1, quat);
    m3mulv(t, R1, c->jpos[k]);
    v3sub(p, anchors + 3 * k, t);
  }
  float R[9], t[3];
  q2mat(R, quat);
  m3mulv(t, R, c->hand_pos);
  v3add(hp, p, t);
  qmul(hq, quat, c->hand_quat);
  qnormalize(hq);
}

// damped least squares from q (in / out) to the world target (tp, tq wxyz); returns the number of iterations used
FE_HDN int fe_ik_solve(const fe_ik_config* c, const fe_ik_arm* arm, float* q, const float* tp, const float* tq) {
  const float lam2 = c->damping * c->damping;
  int it = 0;
  for (; it < c->max_iters; ++it) {
    float hp[3], hq[4], an[21], ax[21], e[6], J[42];
    fe_ik_fk(arm, q, hp, hq, an, ax);
    v3sub(e, tp, hp);
    { // rotation vector of tq * conj(hq)
      const float cq[4] = {hq[0], -hq[1], -hq[2], -hq[3]};
      float d[4];
      qmul(d, tq, cq);
      if (d[0] < 0.f) { d[0] = -d[0]; d[1] = -d[1]; d[2] = -d[2]; d[3] = -d[3]; }
      const float n = sqrtf(d[1] * d[1] + d[2] * d[2] + d[3] * d[3]);
      const float f = n < 1e-9f ? 2.f : 2.f * atan2f(n, d[0]) / n;
      e[3] = f * d[1]; e[4] = f * d[2]; e[5] = f * d[3];
    }
    const float np_ = v3norm(e), nr_ = v3norm(e + 3);
    if (np_ < c->tol_pos && nr_ < c->tol_rot) break;
    if (np_ > c->max_step_pos) { const float f = c->max_step_pos / np_; e[0] *= f; e[1] *= f; e[2] *= f; }
    if (nr_ > c->max_step_rot) { const float f = c->max_step_rot / nr_; e[3] *= f; e[4] *= f; e[5] *= f; }
    for (int k = 0; k < 7; ++k) { // column k: [axis x (hand - anchor); axis]
      float d[3], cr[3];
      v3sub(d, hp, an + 3 * k);
      v3cross(cr, ax + 3 * k, d);
      for (int i = 0; i < 3; ++i) { J[7 * i + k] = cr[i]; J[7 * (3 + i) + k] = ax[3 * k + i]; }
    }
    float A[21], z[7], rhs[6];
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j <= i; ++j) {
        float s = i == j ? lam2 : 0.f;
        for (int k = 0; k < 7; ++k) s += J[7 * i + k] * J[7 * j + k];
        A[i * (i + 1) / 2 + j] = s;
      }
    for (int k = 0; k < 7; ++k) z[k] = c->null_gain * (arm->rest_pose[k] - q[k]);
    for (int i = 0; i < 6; ++i) { float s = e[i]; for (int k = 0; k < 7; ++k) s -= J[7 * i + k] * z[k]; rhs[i] = s; }
    fe_chol6(A);
    fe_chol6_solve(A, rhs);
    for (int k = 0; k < 7; ++k) {
      float dq = z[k];
      for (int i = 0; i < 6; ++i) dq += J[7 * i + k] * rhs[i];
      q[k] = fminf(fmaxf(q[k] + dq, arm->lower[k]), arm->upper[k]);
    }
  }
  return it;
}

// _setup_action + gravity compensation with the low-level action `a` (arm velocities, then the gripper action `grip`)
FE_HD void fe_ik_controls(FeEnv* e, const float* a, float grip) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const fe_scene* sc = e->sc;
  const fe_config* cfg = e->cfg;
  LANES_BEGIN
    for (int u = lane; u < m->nu; u += 32) { // _setup_action, furniture.py:3332-3367
      const int src = sc->act_src[u];
      float v = src == sc->grip_action_index ? grip : a[src];
      if (cfg->rescale_actions) v = fminf(fmaxf(v, -1.f), 1.f);
      v *= sc->act_sign[u];
      if (cfg->rescale_actions) {
        const float lo = m->act_ctrlrange[u][0], hi = m->act_ctrlrange[u][1];
        v = 0.5f * (hi + lo) + 0.5f * (hi - lo) * v;
      }
      w->ctrl()[u] = v;
    }
    for (int i = lane; i < sc->narm; i += 32) w->qfrc_applied()[sc->arm_dof[i]] = w->bias()[sc->arm_dof[i]]; // gravity compensation, :3372-3377
    for (int i = lane; i < sc->ngrip; i += 32) w->qfrc_applied()[sc->grip_dof[i]] = w->bias()[sc->grip_dof[i]];
    if (lane == 0) { e->ei[0] = 0; e->ei[1] = -1; e->ei[6] = 0; w->u()[2] = 0; }
  LANES_END
}

// what follows the simulation in FurnitureEnv.step, with the policy action `a` (act_dim numbers) for reward and connect
// `fail`: some _do_simulation of this step raised; `reset_now`: the last one did, so the env has not been reset for it yet
FE_HD void fe_ik_finish(FeEnv* e, const float* a, int act_dim, float connect, int fail, int reset_now, float* reward_out, uint8_t* done_out, int32_t* info_out) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const fe_scene* sc = e->sc;
  const fe_config* cfg = e->cfg;
  const int np = m->npart, env = e->env;
  FE_SYNC;
  if (reset_now) {
    fe_env_reset_one(e);
  } else {
    if (connect > 0.f) { // furniture.py:1290-1322: per arm, the first part both of its fingers touch; stop at the first connection
      for (int arm = 0; arm < sc->narms; ++arm) {
        const int both = arm == 0 ? 3 : 24;
        int part = -1;
        for (int p = 0; p < np; ++p) if ((w->touch()[p] & both) == both) { part = p; break; }
        if (part >= 0) {
          fe_try_connect_scan(e, part);
          if (e->ei[0]) { fe_connect(e); break; }
        }
      }
    }
    const int repin = e->ei[1];
    FE_SYNC; // every lane has read the flag before lane 0 clears it
    if (repin >= 0) { // furniture.py:426-436: re-pin the merged group at the recorded pose, one more step
      LANES_BEGIN
        if (lane == 0) {
          const int b1 = e->ei[1], qa = m->link_qadr[m->nrlink + b1];
          double tr[3] = {e->ed[4] - (double)w->qpos()[qa], e->ed[5] - (double)w->qpos()[qa + 1], e->ed[6] - (double)w->qpos()[qa + 2]};
          fe_move_group(e, b1, tr, e->ed + 7, 0.f);
          e->ei[1] = -1;
        }
      LANES_END
      fe_fwd_step(e);
      if (w->u()[2] & 8) { fail = 1; fe_env_reset_one(e); }
    }
  }
  // reward (furniture.py:482-541), termination (:440-445, :451-480)
  LANES_BEGIN
    if (lane == 0) {
      float touch_r = 0.f, pick_r = 0.f;
      int* touched = e->es.touched + (size_t)env * np;
      int* picked = e->es.picked + (size_t)env * np;
      if (!fail)
        for (int arm = 0; arm < sc->narms; ++arm) // furniture.py:492-523: both fingers of the same arm
          for (int p = 0; p < np; ++p) {
            const int t = w->touch()[p], both = arm == 0 ? 3 : 24;
            if ((t & both) == both) {
              if (!touched[p]) { touched[p] = 1; touch_r += cfg->touch_reward; }
              if (!(t & 4) && !picked[p]) { picked[p] = 1; pick_r += cfg->pick_reward; }
            }
          }
      const int nc = e->es.num_connected[env];
      const float success_r = cfg->success_reward * (float)(nc - e->es.prev_num_connected[env]);
      const int connected_now = nc != e->es.prev_num_connected[env]; // _connected: a connection was made during this step
      e->es.prev_num_connected[env] = nc;
      float sq = 0.f;
      for (int k = 0; k < act_dim; ++k) sq += a[k] * a[k];
      float reward = success_r + touch_r + pick_r - cfg->ctrl_penalty_coef * sq;
      int success = (nc == np - 1 && np > 1) ? 1 : 0;
      int done = success;
      if (e->es.dense) { // FurnitureSawyerEnv._step: reward, _done, info = _compute_reward(a); done = done or _done (furniture_sawyer.py:66-84)
        FeSliceWorld world = {w};
        const double thr[4] = {cfg->alignment_pos_dist, cfg->alignment_rot_dist_up, cfg->alignment_rot_dist_forward, cfg->alignment_project_dist};
        double ad[FE_MAXU + 2], dr = 0.0, di[FE_DENSE_INFO];
        for (int k = 0; k < act_dim; ++k) ad[k] = (double)a[k];
        int dd = 0;
        FeDenseState* ds = e->es.dstate + env;
        fe_dense_step(world, e->es.dense, &sc->dense, thr, np - 1, ds, ad, act_dim, connected_now, &dr, &dd, di);
        reward = (float)dr;
        success = ds->success;
        done = done || dd;
        float* dinf = e->es.dinfo + (size_t)env * FE_DENSE_INFO;
        for (int k = 0; k < FE_DENSE_INFO; ++k) dinf[k] = (float)di[k];
      }
      const int len = ++e->es.episode_len[env];
      float penalty = 0.f;
      if (len == cfg->max_episode_steps || fail) { done = 1; if (fail) penalty = -cfg->unstable_penalty_coef; }
      reward += penalty;
      reward_out[env] = reward;
      done_out[env] = (uint8_t)done;
      if (e->es.packed) { float* pk = e->es.packed + (size_t)env * (sc->obs_dim + 2) + sc->obs_dim; pk[0] = reward; pk[1] = done ? 1.f : 0.f; }
      int32_t* info = info_out + (size_t)env * FE_INFO_DIM;
      info[0] = nc; info[1] = success; info[2] = fail; info[3] = len; info[4] = w->u()[0]; info[5] = w->u()[3];
      e->es.done[env] = done;
      // An unstable episode resets twice, as the reference does: once inside _do_simulation's except branch
      // (furniture.py:2889-2897) and once more by the VecEnv worker because the step returned done (subproc_vec_env.py:16-20).
      // The second reset zeroes the episode length that _after_step just incremented and consumes its own random draws,
      // so the env's generator stays draw-for-draw on the reference's stream.
      e->ei[6] = done;
    }
  LANES_END
  if (e->ei[6]) fe_env_reset_one(e); else fe_write_obs(e);
}

// first get_control of the step (lane 0), one arm: hand pose of the last forward pass -> targets -> joint command -> first velocities.
// `a` points at this arm's (move, rotate) numbers
FE_HDN void fe_ik_command(FeEnv* e, const FeIkArgs& ik, int arm_i, const float* a) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const fe_ik_config* c = ik.c;
  const fe_ik_arm* arm = &c->arm[arm_i];
  FeIkState* st = ik.st + e->env;
  const int hl = e->sc->hand_link[arm_i];
  const float* lp = e->st.lpos + ((size_t)e->env * m->nlink + hl) * 3;  // sim.data.body_xpos / body_xmat: kinematics of the last forward pass
  const float* lq = e->st.lquat + ((size_t)e->env * m->nlink + hl) * 4;
  float Rl[9], t[3], hand_p[3], hand_q[4], Rh[9], Rb[9], hb[3], Rhb[9], cur[4], cw[4];
  const float lqv[4] = {lq[0], lq[1], lq[2], lq[3]};
  q2mat(Rl, lqv);
  m3mulv(t, Rl, arm->hand_pos);
  hand_p[0] = lp[0] + t[0]; hand_p[1] = lp[1] + t[1]; hand_p[2] = lp[2] + t[2];
  qmul(hand_q, lqv, arm->hand_quat);
  qnormalize(hand_q);
  q2mat(Rh, hand_q);
  q2mat(Rb, c->base_quat);
  v3sub(t, hand_p, c->base_pos);
  m3tmulv(hb, Rb, t);                                      // pose_in_base_from_name("<arm>_hand"), furniture.py:3381-3398
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) Rhb[3 * i + j] = Rb[i] * Rh[j] + Rb[3 + i] * Rh[3 + j] + Rb[6 + i] * Rh[6 + j];
  ik_mat_to_wxyz(cw, Rhb);
  cur[0] = cw[1]; cur[1] = cw[2]; cur[2] = cw[3]; cur[3] = cw[0]; // _<arm>_hand_quat, (x, y, z, w)
  float* s_acc = st->s[arm_i];
  float* target = st->target_pos[arm_i];
  if (e->es.episode_len[e->env] == 0) {                     // _reset's tail: _initial_<arm>_hand_quat = _<arm>_hand_quat; controller.sync_state()
    for (int k = 0; k < 4; ++k) s_acc[k] = cur[k];
    v3cpy(target, hb);
  }
  // action[:3] * move_speed, axes swapped, clipped to the workspace (world position of the hand)
  const float mv[3] = {-a[1] * c->move_speed, a[0] * c->move_speed, a[2] * c->move_speed};
  float dpos[3];
  for (int k = 0; k < 3; ++k) dpos[k] = fminf(fmaxf(mv[k], c->min_pos[k] - hand_p[k]), c->max_pos[k] - hand_p[k]);
  float rq[4], rot[9], Rw[9], tq[4], tp[3];
  if (c->quaternion_mode) { // "ik_quaternion": rotation = quat2mat(cur * convert_quat(action[3:7])), furniture.py:3013, :3027 (_make_input)
    const float aq[4] = {a[4], a[5], a[6], a[3]};
    ik_xyzw_mul(rq, cur, aq);
  } else {
    // euler_to_quat(action[3:6] * rotate_speed, s): q3 q2 q1 about z, y, x; s read as if (w, x, y, z)
    float qe[4], t4[4], s_new[4];
    {
      const float hx = 0.5f * a[3] * c->rotate_speed * 0.017453292519943295f, hy = 0.5f * a[4] * c->rotate_speed * 0.017453292519943295f,
                  hz = 0.5f * a[5] * c->rotate_speed * 0.017453292519943295f;
      const float q1[4] = {cosf(hx), sinf(hx), 0.f, 0.f}, q2[4] = {cosf(hy), 0.f, sinf(hy), 0.f}, q3[4] = {cosf(hz), 0.f, 0.f, sinf(hz)};
      ik_hamilton(t4, q3, q2);
      ik_hamilton(qe, t4, q1);
    }
    ik_hamilton(s_new, s_acc, qe);
    for (int k = 0; k < 4; ++k) s_acc[k] = s_new[k];
    // d_quat = quat_inverse(cur) * s; rotation = quat2mat(cur * d_quat)  (all (x, y, z, w))
    float inv[4], dq[4];
    { const float n = cur[0] * cur[0] + cur[1] * cur[1] + cur[2] * cur[2] + cur[3] * cur[3]; inv[0] = -cur[0] / n; inv[1] = -cur[1] / n; inv[2] = -cur[2] / n; inv[3] = cur[3] / n; }
    ik_xyzw_mul(dq, inv, s_new);
    ik_xyzw_mul(rq, cur, dq);
  }
  ik_xyzw_to_mat(rot, rq);
  for (int k = 0; k < 3; ++k) target[k] += dpos[k] * c->user_sensitivity;
  m3mulv(t, Rb, target);
  v3add(tp, c->base_pos, t);
  m3mul(Rw, Rb, rot);
  ik_mat_to_wxyz(tq, Rw);
  float q[7];
  for (int k = 0; k < 7; ++k) q[k] = w->qpos()[arm->arm_qadr[k]];
  st->iters[arm_i] = fe_ik_solve(c, arm, q, tp, tq);
  for (int k = 0; k < 7; ++k) { st->q_cmd[7 * arm_i + k] = q[k]; st->low[7 * arm_i + k] = fminf(fmaxf(-c->kp * (w->qpos()[arm->arm_qadr[k]] - q[k]), -1.f), 1.f); }
}

// FurnitureEnv.step with control_type="ik" / "ik_quaternion" for one env.  Actions: per arm (move 3, rotate 3 or a quaternion), then one
// gripper action per arm, then connect (furniture_sawyer.py:60-63, furniture_baxter.py:52-62)
FE_FN void fe_env_ik_step_one(FeEnv* e, FeIkArgs ik, const float* action, float* reward_out, uint8_t* done_out, int32_t* info_out) {
  FeWarp* w = e->w;
  const fe_ik_config* c = ik.c;
  const int na = c->narms, per = c->quaternion_mode ? 7 : 6, act_dim = na * per + na + 1;
  const float* a = action + (size_t)e->env * act_dim;
  float grip = a[act_dim - 2];
  if (e->cfg->discrete_grip) grip = grip < 0.f ? -1.f : 1.f; // FurnitureSawyerEnv._step only (furniture_sawyer.py:73-74); unused with two arms
  const float connect = a[act_dim - 1];
  FeIkState* st = ik.st + e->env;
  LANES_BEGIN
    if (lane == 0) {
      for (int arm = 0; arm < na; ++arm) {
        fe_ik_command(e, ik, arm, a + arm * per);
        st->low[7 * na + arm] = na == 1 ? grip : a[na * per + arm];
      }
    }
  LANES_END
  int fail = 0, reset_now = 0;
  for (int r = 0; r < c->action_repeat; ++r) {
    if (r > 0) { // closed loop: get_control() without arguments, furniture.py:2988-2995
      LANES_BEGIN
        if (lane < 7 * na) st->low[lane] = fminf(fmaxf(-c->kp * (w->qpos()[c->arm[lane / 7].arm_qadr[lane % 7]] - st->q_cmd[lane]), -1.f), 1.f);
      LANES_END
    }
    fe_ik_controls(e, st->low, grip);
    for (int i = 0; i < e->cfg->nsub; ++i) fe_substep_lockstep(w);
    if (w->u()[2] & 8) { // _do_simulation's except branch: reset, then the remaining repeats run on the new episode (furniture.py:2889-2897)
      fail = 1;
      FE_SYNC;
      if (r + 1 < c->action_repeat) fe_env_reset_one(e); else reset_now = 1;
    }
  }
  fe_ik_finish(e, a, act_dim, connect, fail, reset_now, reward_out, done_out, info_out);
}
