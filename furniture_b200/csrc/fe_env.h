// fe_env.h -- the FurnitureEnv logic that sits around the mj_step loop, executed by the same warp that owns the env,
// so that no host round trip breaks the batch:
//   fe_env_step_one  : FurnitureEnv.step -> FurnitureSawyerEnv._step -> _step_continuous (action mapping, gravity
//                      compensation, nsub mj_steps, finger-contact scan, _try_connect/_is_aligned/_connect), post-connect
//                      re-pin, _get_obs, _compute_reward, _after_step, VecEnv auto-reset
//                      (furniture/env/furniture.py:364-480, :1260-1330, :3332-3379; furniture_sawyer.py:66-155); its parts before and
//                      after the simulation, fe_env_controls / fe_env_finish, are also those of the IK and torque-controller steps
//   fe_env_reset_one : FurnitureEnv._reset settle protocol (furniture.py:1406-1663) with a counter-based per-env RNG
//   fe_is_aligned_d  : _is_aligned in float64 with numpy's exact arithmetic (float32 unit_vector, FMA-chain dots)
#pragma once
#include "fe_driver.h"
#include "fe_dense_types.h"

#define FE_SCENE_MAGIC 0x46455344 /* "FESD" */
#define FE_MAXCONN 48
#define FE_INFO_DIM 6
#define FE_REWARD_INFO 4  /* success_reward, touch_reward, pick_reward, ctrl_penalty of FurnitureEnv._compute_reward (furniture.py:535-540) */
#define FE_EPISODE_INFO 2 /* episode_reward, episode_unstable of FurnitureEnv._after_step (furniture.py:469-476) */

// the observation flags of config/furniture.py (robot_ob, object_ob, object_ob_all, subtask_ob; read at furniture.py:103-107) as the bits of
// fe_scene.obs_layout, each set where the flag differs from its default, so that 0 is the default row [object_ob (7 per part) | robot_ob]
#define FE_OBS_NO_ROBOT 1      /* robot_ob = False */
#define FE_OBS_NO_OBJECT 2     /* object_ob = False */
#define FE_OBS_PAIR_ONLY 4     /* object_ob_all = False: object_ob holds the two parts of the current subtask, 14 numbers */
#define FE_OBS_SUBTASK 8       /* subtask_ob = True: [part1 + 1, part2 + 1] after object_ob */

typedef struct fe_scene {
  int32_t magic, struct_bytes;
  int32_t obs_dim, act_dim, robot_ob_dim, nconn, npart, narm, ngrip; // narm / ngrip: arm / gripper joints of all arms together
  int32_t narms;                                                      // 1 (Sawyer) or 2 (Baxter: right, left -- furniture.py:89-92)
  // action -> actuator map: ctrl[u] = bias_u + weight_u * sign_u * clip(action[src_u]) (furniture.py:3332-3367)
  int32_t act_src[FE_MAXU];
  float act_sign[FE_MAXU];
  int32_t grip_action_index, connect_action_index;
  // connector sites in model site-id order (furniture.py:954-961); names "A-B,ang..,conn_siteN" interned as (a, b)
  int32_t conn_site[FE_MAXCONN], conn_part[FE_MAXCONN], conn_a[FE_MAXCONN], conn_b[FE_MAXCONN], conn_nangles[FE_MAXCONN];
  double conn_cos[FE_MAXCONN][4], conn_sin[FE_MAXCONN][4]; // cos/sin(angle/180*pi) evaluated on the host in float64
  int32_t eq_part1[FE_MAXEQ], eq_part2[FE_MAXEQ];
  int32_t part_site_start[FE_MAXPART + 1], part_sites[FE_MAXSITE]; // sites per part for _get_bounding_box
  int32_t eef_site[2], hand_link[2]; // per arm: grip site and the link that carries the "<arm>_hand" body
  float hand_quat[2][4];
  // robot dof of every arm joint (mujoco_robot.joints order: right arm, then left) and of every gripper joint (right gripper, then
  // left); the other robot dofs (Baxter's head_pan) get neither gravity compensation nor a reset pose (furniture.py:3372-3377, :1761-1779)
  int32_t arm_dof[FE_MAXRDOF], grip_dof[8];
  float robot_init_qpos[FE_MAXRDOF]; // arm joints (arm_dof order), then gripper joints (grip_dof order)
  float part_init_pos[FE_MAXPART][3], part_init_quat[FE_MAXPART][4], part_radius[FE_MAXPART];
  int32_t phase_ob;            // 1: obs ends with the 8-way one-hot of the dense reward's phase (furniture_sawyer_dense.py:100-117); counted in obs_dim
  int32_t obs_layout;          // FE_OBS_* bits of fe_set_obs_layout; 0 = the reference's default flags, the layout of a scene file
  fe_dense_recipe dense;       // assembly recipe for the dense reward (nsub = 0: the furniture has none)
} fe_scene;

struct FeEnvState {
  float* obs;                                  // [N][obs_dim]
  // the last observation row and qpos / qvel of the episode an env's step ended, written by that step before its auto-reset; the rows of
  // envs whose step did not end an episode are left as they are
  float *terminal_obs, *terminal_qpos, *terminal_qvel; // [N][obs_dim], [N][nq], [N][nv]
  float* packed;                               // optional second output of a step: rows [obs | reward | done | info | dense_info | terminal_obs]
                                               // (float) -- the send buffer of the multi-GPU all-gather, written by the step kernel itself
  int pk_stride;                               // floats per packed row: obs_dim + 2 and the optional columns fe_set_packed_layout asks for
  int pk_info, pk_dense, pk_term;              // first column of info (int32 bits), dense_info, terminal_obs in a packed row; -1 = absent
  int pk_step;                                 // first column of the step-info block [reward_info | episode_info] (fe_set_packed_step_info); -1 = absent
  int *group, *site_connected;                 // [N][npart], [N][nsite]
  int *num_connected, *prev_num_connected, *touched, *picked, *episode_len, *done;
  int *preassembled, *num_connects;            // [N] set_subtask (furniture.py:204-207): recipe steps connected by the env's next reset; connections asked for, -1 = None
  int* success_num_conn;                       // [N] _success_num_conn as the env's last reset left it (furniture.py:1477-1481)
  int* subtask_part;                           // [N][2] _subtask_part1 / _subtask_part2, -1 = none left (furniture.py:2723-2736)
  uint32_t* mt;                                // [N][624] MT19937 state of the env's numpy RandomState(seed + env)
  int* mt_pos;                                 // [N] position in the state (624 = regenerate before the next draw)
  // recorded starts, _init_qpos (furniture.py:121-130, :315-316, :1433-1434): a bank shared by the envs, and per env the entry its resets start from
  const float *init_qpos, *init_qvel;          // [n_init][nq], [n_init][nv] (fe_set_init_states)
  int n_init;
  int *init_state, *init_pick;                 // [N] bank index of the env's _init_qpos, -1 = None; leading entries its resets pick from, 0 = no load_init_states
  uint32_t* init_mt;                           // [N][624] MT19937 of the pick, numpy RandomState(seed + 2**20 + env); laid out like mt
  int* init_mt_pos;                            // [N]
  // fix_init / fix_init_parts (config/furniture.py:116-127): the placement a random-placement reset remembers (furniture.py:1519-1532),
  // the reference's init_pos / init_quat, and whether it holds one (init_pos is not None)
  int *fix_init, *fix_init_parts, *fix_have;   // [N] 0 / 1, bit mask over parts in XML order, 0 / 1
  double* fix_pose;                            // [N][npart][7] position, quaternion (w, x, y, z)
  int* reset_arm;                              // [N] reset_robot_after_attach (config/furniture.py:169-174)
  int* arm_resync;                             // [N] a connection sent the arm home: the next IK command re-seeds its position target
  int* substeps;                               // [N] mj_steps of the env's step: int(control_timestep / model_timestep) (furniture.py:2878)
  int* no_collision;                           // [N] 0 / 1: the agent's masks stay 0 (config/furniture.py no_collision, furniture.py:1962-1965)
  int* assembled;                              // [N] 0 / 1: episodes start with every weld on, the parts at qpos0 (config/furniture.py:307-312)
  // the task options of config/furniture.py per env, in fe_config's types: filled from it at creation, read instead of it by the kernels
  double* alignment;                           // [N][4] alignment_pos_dist, _rot_dist_up, _rot_dist_forward, _project_dist (:203-226), thr[] order
  int* auto_align;                             // [N] 0 / 1 (:95-100)
  float* placement_rand;                       // [N][3] furn_xyz_rand, furn_rot_rand, agent_xyz_rand (:177-194)
  float* reward_coef;                          // [N][5] success_reward, touch_reward, pick_reward, ctrl_penalty_coef, unstable_penalty_coef (:291-295)
  int* max_episode_steps;                      // [N] (:163-168)
  int *robot_contype, *robot_conaff;           // [N][ngeom] saved robot masks during reset
  float* episode_reward;                       // [N] _episode_reward: the rewards of the episode so far, before the unstable penalty (furniture.py:459-461)
  // the step's info dict (furniture.py:451-541): the sparse reward's four terms of every step (NULL on a dense handle, whose terms are dinfo),
  // and {episode_reward + penalty, episode_unstable = penalty} of the episode a step ended, written by that step; other rows are left as they are
  float* reward_info;                          // [N][FE_REWARD_INFO] success_reward, touch_reward, pick_reward, ctrl_penalty
  float* episode_info;                         // [N][FE_EPISODE_INFO]
  // dense (phase-based) reward, fe_dense.h: NULL = the sparse reward of FurnitureEnv._compute_reward
  const fe_dense_config* dense;                // [N] each env's coefficients and flags; lane 0 reads its row once per step
  FeDenseState* dstate;                        // [N]
  float* dinfo;                                // [N][FE_DENSE_INFO]
};

// the geoms no_collision switches off.  The reference zeroes the masks of every geom under the robot's worldbody, grippers included
// (furniture.py:1962-1965); among the geoms the engine keeps (those that can collide) that is every one that belongs to neither a furniture
// part nor the floor: FE_TAG_ROBOT (the robot's contact geoms, which the reset switches off) and the agent's other colliding geoms
// (the torque Sawyer's controller box and pedestal feet, Baxter's head, pedestal and left wrist)
FE_BOTH bool fe_geom_is_agent(int tag) { return !(tag & FE_TAG_FLOOR) && ((tag >> FE_TAG_PART_SHIFT) & 0x3FFFFF) == 0; }

// ---------------------------------------------------------------- float64 helpers with numpy's arithmetic
#if FE_DEVICE_BUILD
FE_HD double ndmul(double a, double b) { return __dmul_rn(a, b); }
FE_HD double ndadd(double a, double b) { return __dadd_rn(a, b); }
FE_HD double ndsub(double a, double b) { return __dsub_rn(a, b); }
FE_HD double nddiv(double a, double b) { return __ddiv_rn(a, b); }
FE_HD double ndfma(double a, double b, double c) { return __fma_rn(a, b, c); }
FE_HD double ndsqrt(double a) { return __dsqrt_rn(a); }
FE_HD float fmul32(float a, float b) { return __fmul_rn(a, b); }
FE_HD float fdiv32(float a, float b) { return __fdiv_rn(a, b); }
#else
FE_HD double ndmul(double a, double b) { return a * b; }
FE_HD double ndadd(double a, double b) { return a + b; }
FE_HD double ndsub(double a, double b) { return a - b; }
FE_HD double nddiv(double a, double b) { return a / b; }
FE_HD double ndfma(double a, double b, double c) { return fma(a, b, c); }
FE_HD double ndsqrt(double a) { return sqrt(a); }
FE_HD float fmul32(float a, float b) { return a * b; }
FE_HD float fdiv32(float a, float b) { return a / b; }
#endif
FE_HD double npdot(const double* a, const double* b) { return ndfma(a[2], b[2], ndfma(a[1], b[1], ndmul(a[0], b[0]))); } // cblas_ddot, n = 3
FE_HD double npnorm(const double* a) { return ndsqrt(npdot(a, a)); }
FE_HD void npcross(double* r, const double* a, const double* b) {
  double x = ndsub(ndmul(a[1], b[2]), ndmul(a[2], b[1])), y = ndsub(ndmul(a[2], b[0]), ndmul(a[0], b[2])), z = ndsub(ndmul(a[0], b[1]), ndmul(a[1], b[0]));
  r[0] = x; r[1] = y; r[2] = z;
}
// transform_utils.unit_vector (float32 copy, in-place divide by the float32-rounded norm), returned upcast
FE_HD void np_unit_vector_f32(double* out, const double* v) {
  float d[3] = {(float)v[0], (float)v[1], (float)v[2]};
  float dot = (float)ndadd(ndadd((double)fmul32(d[0], d[0]), (double)fmul32(d[1], d[1])), (double)fmul32(d[2], d[2]));
  float s = (float)ndsqrt((double)dot);
  out[0] = (double)fdiv32(d[0], s); out[1] = (double)fdiv32(d[1], s); out[2] = (double)fdiv32(d[2], s);
}
FE_HD double np_cos_siml(const double* a, const double* b) { return nddiv(nddiv(npdot(a, b), npnorm(a)), npnorm(b)); }
FE_HD void np_normed(double* r, const double* a) { double n = npnorm(a); r[0] = nddiv(a[0], n); r[1] = nddiv(a[1], n); r[2] = nddiv(a[2], n); }
// transform_utils.lookat_to_quat(forward, up) -> xyzw, returned here as wxyz (convert_quat(..., "wxyz"))
FE_HDN void np_lookat_wxyz(double* out, const double* forward, const double* up) {
  double v[3], v2[3], v3[3], t[3], q[4] = {0, 0, 0, 0};
  np_normed(v, forward);
  np_normed(t, up);
  npcross(v2, t, v);
  np_normed(v2, v2);
  npcross(v3, v, v2);
  const double m00 = v2[0], m01 = v2[1], m02 = v2[2], m10 = v3[0], m11 = v3[1], m12 = v3[2], m20 = v[0], m21 = v[1], m22 = v[2];
  const double num8 = ndadd(ndadd(m00, m11), m22);
  if (num8 > 0) {
    double num = ndsqrt(ndadd(num8, 1.0));
    q[3] = ndmul(num, 0.5);
    num = nddiv(0.5, num);
    q[0] = ndmul(ndsub(m12, m21), num); q[1] = ndmul(ndsub(m20, m02), num); q[2] = ndmul(ndsub(m01, m10), num);
  } else if (m00 >= m11 && m00 >= m22) {
    double num7 = ndsqrt(ndsub(ndsub(ndadd(1.0, m00), m11), m22)), num4 = nddiv(0.5, num7);
    q[0] = ndmul(0.5, num7); q[1] = ndmul(ndadd(m01, m10), num4); q[2] = ndmul(ndadd(m02, m20), num4); q[3] = ndmul(ndsub(m12, m21), num4);
  } else if (m11 > m22) {
    double num6 = ndsqrt(ndsub(ndsub(ndadd(1.0, m11), m00), m22)), num3 = nddiv(0.5, num6);
    q[0] = ndmul(ndadd(m10, m01), num3); q[1] = ndmul(0.5, num6); q[2] = ndmul(ndadd(m21, m12), num3); q[3] = ndmul(ndsub(m20, m02), num3);
  } else {
    double num5 = ndsqrt(ndsub(ndsub(ndadd(1.0, m22), m00), m11)), num2 = nddiv(0.5, num5);
    q[0] = ndmul(ndadd(m20, m02), num2); q[1] = ndmul(ndadd(m21, m12), num2); q[2] = ndmul(0.5, num5); q[3] = ndmul(ndsub(m01, m10), num2);
  }
  out[0] = q[3]; out[1] = q[0]; out[2] = q[1]; out[3] = q[2];
}
// the better of transform_utils.rotate_vector_cos_siml(f1, up1, cos_siml(f1, f2), +-1) by cos_siml with f2; cr = cross(unit_vector(up1), f1)
FE_HD void np_rotate_towards(double* fr, const double* f1, const double* cr, const double* f2) {
  const double c = np_cos_siml(f1, f2);
  const double s = ndsqrt(ndsub(1.0, ndmul(c, c)));
  double fp[3], fn[3];
  for (int i = 0; i < 3; ++i) { fp[i] = ndadd(ndmul(c, f1[i]), ndmul(ndmul(1.0, s), cr[i])); fn[i] = ndadd(ndmul(c, f1[i]), ndmul(ndmul(-1.0, s), cr[i])); }
  const bool pos = np_cos_siml(fp, f2) > np_cos_siml(fn, f2);
  for (int i = 0; i < 3; ++i) fr[i] = pos ? fp[i] : fn[i];
}
// FurnitureEnv._is_aligned (furniture.py:1057-1153). m*: row-major site rotation. cs/sn: cos/sin of the allowed angles.
// Returns the decision; *tq_set tells whether _target_connector_xquat was assigned, tq its value (wxyz).
FE_HDN bool fe_is_aligned_d(const double* p1, const double* m1, const double* p2, const double* m2, int nang, const double* cs, const double* sn,
                           const double* thr, double* tq, bool* tq_set) {
  const double up1[3] = {m1[2], m1[5], m1[8]}, up2[3] = {m2[2], m2[5], m2[8]}, f1[3] = {m1[1], m1[4], m1[7]}, f2[3] = {m2[1], m2[4], m2[7]};
  double d12[3] = {ndsub(p1[0], p2[0]), ndsub(p1[1], p2[1]), ndsub(p1[2], p2[2])}, d21[3] = {ndsub(p2[0], p1[0]), ndsub(p2[1], p1[1]), ndsub(p2[2], p1[2])};
  const double pos_dist = npnorm(d12);
  const double rot_up = np_cos_siml(up1, up2);
  double u[3];
  np_unit_vector_f32(u, d21);
  const double proj12 = npdot(up1, u);
  np_unit_vector_f32(u, d12);
  const double proj21 = npdot(up2, u);
  bool fwd_ok = false;
  *tq_set = false;
  double k[3], cr[3], fr[3];
  np_unit_vector_f32(k, up1);
  npcross(cr, k, f1);
  if (nang == 0) {
    fwd_ok = true;
    np_rotate_towards(fr, f1, cr, f2);
    np_lookat_wxyz(tq, up1, fr);
    *tq_set = true;
  } else {
    for (int a = 0; a < nang; ++a) {
      for (int i = 0; i < 3; ++i) fr[i] = ndadd(ndmul(cs[a], f1[i]), ndmul(sn[a], cr[i]));
      if (np_cos_siml(fr, f2) > thr[2]) {
        fwd_ok = true;
        np_lookat_wxyz(tq, up1, fr);
        *tq_set = true;
        break;
      }
    }
  }
  if (pos_dist < thr[0] && rot_up > thr[1] && fwd_ok && fabs(proj12) > thr[3] && fabs(proj21) > thr[3]) return true;
  if (pos_dist < nddiv(thr[0], 2.0) && rot_up > thr[1] && fwd_ok) return true;
  return false;
}
// FurnitureEnv._project_connector_quat(connector1, connector2, angle) (furniture.py:1201-1222): connector2's xquat (wxyz) when aligned with
// connector1.  m*: row-major site rotation; cs / sn: cos / sin of the recipe angle when it gives one.
FE_HDN void fe_project_connector_quat_d(const double* m1, const double* m2, int has_angle, double cs, double sn, double* tq) {
  const double up1[3] = {m1[2], m1[5], m1[8]}, f1[3] = {m1[1], m1[4], m1[7]}, f2[3] = {m2[1], m2[4], m2[7]};
  double k[3], cr[3], fr[3];
  np_unit_vector_f32(k, up1);
  npcross(cr, k, f1);
  if (has_angle) for (int i = 0; i < 3; ++i) fr[i] = ndadd(ndmul(cs, f1[i]), ndmul(sn, cr[i]));
  else np_rotate_towards(fr, f1, cr, f2);
  np_lookat_wxyz(tq, up1, fr);
}

#include "fe_dense.h"

// ---- pyquaternion semantics in float64 (w,x,y,z), used by the connect path (transform_utils.py:633-664)
FE_HD void dq_mul(double* r, const double* a, const double* b) {
  double w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], x = a[1] * b[0] + a[0] * b[1] - a[3] * b[2] + a[2] * b[3];
  double y = a[2] * b[0] + a[3] * b[1] + a[0] * b[2] - a[1] * b[3], z = a[3] * b[0] - a[2] * b[1] + a[1] * b[2] + a[0] * b[3];
  r[0] = w; r[1] = x; r[2] = y; r[3] = z;
}
FE_HD void dq_inv(double* r, const double* q) {
  double ss = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  r[0] = q[0] / ss; r[1] = -q[1] / ss; r[2] = -q[2] / ss; r[3] = -q[3] / ss;
}
FE_HD void dq_rotate(double* r, const double* q_in, const double* v) {
  double q[4] = {q_in[0], q_in[1], q_in[2], q_in[3]};
  double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  if (fabs(1.0 - n) >= 1e-14 && n > 0) { q[0] /= n; q[1] /= n; q[2] /= n; q[3] /= n; }
  double qv[4] = {0, v[0], v[1], v[2]}, t[4], c[4] = {q[0], -q[1], -q[2], -q[3]}, o[4];
  dq_mul(t, q, qv);
  dq_mul(o, t, c);
  r[0] = o[1]; r[1] = o[2]; r[2] = o[3];
}
// T.transform_to_target_quat(qpos_base, qpos, target_quat) on 7-vectors (pos, wxyz)
FE_HDN void d_transform_to_target(const double* base, const double* q, const double* target, double* new_pos, double* new_quat) {
  double inv[4], rel[4], d[3] = {q[0] - base[0], q[1] - base[1], q[2] - base[2]}, r[3];
  dq_inv(inv, base + 3);
  dq_mul(rel, target, inv);
  dq_rotate(r, rel, d);
  new_pos[0] = r[0] + base[0]; new_pos[1] = r[1] + base[1]; new_pos[2] = r[2] + base[2];
  dq_mul(new_quat, rel, q + 3);
}

// ---------------------------------------------------------------- per-env RNG: the reference's own generator.
// Every reference env draws from numpy's RandomState(config.seed) (furniture.py:72; seed + rank per VecEnv worker,
// env/base.py:77): MT19937 seeded by init_genrand, doubles as (a >> 5, b >> 6) -> (a * 2^26 + b) / 2^53, and
// uniform(low, high) = low + (high - low) * double, two roundings (numpy legacy distributions).  The state lives in HBM
// (2.5 KB per env) and only lane 0 touches it, in reset.
#define FE_MT_N 624
#define FE_MT_M 397
FE_HD void fe_mt_twist(uint32_t* mt) {
  int i = 0;
  for (; i < FE_MT_N - FE_MT_M; ++i) { const uint32_t y = (mt[i] & 0x80000000u) | (mt[i + 1] & 0x7fffffffu); mt[i] = mt[i + FE_MT_M] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u); }
  for (; i < FE_MT_N - 1; ++i) { const uint32_t y = (mt[i] & 0x80000000u) | (mt[i + 1] & 0x7fffffffu); mt[i] = mt[i + (FE_MT_M - FE_MT_N)] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u); }
  const uint32_t y = (mt[FE_MT_N - 1] & 0x80000000u) | (mt[0] & 0x7fffffffu);
  mt[FE_MT_N - 1] = mt[FE_MT_M - 1] ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
}
FE_HD uint32_t fe_mt_u32(uint32_t* mt, int* pos) {
  if (*pos >= FE_MT_N) { fe_mt_twist(mt); *pos = 0; }
  uint32_t y = mt[(*pos)++];
  y ^= y >> 11; y ^= (y << 7) & 0x9d2c5680u; y ^= (y << 15) & 0xefc60000u; y ^= y >> 18;
  return y;
}
FE_HD double fe_mt_double(uint32_t* mt, int* pos) {
  const uint32_t a = fe_mt_u32(mt, pos) >> 5, b = fe_mt_u32(mt, pos) >> 6;
  return nddiv(ndadd(ndmul((double)a, 67108864.0), (double)b), 9007199254740992.0);
}
// RandomState.uniform(low, high): low + (high - low) * random_sample()
FE_HD double fe_mt_uniform(uint32_t* mt, int* pos, double lo, double hi) { return ndadd(lo, ndmul(ndsub(hi, lo), fe_mt_double(mt, pos))); }
// RandomState.randint(0, n), which RandomState.choice(n items) draws: no draw for n = 1, else masked rejection on 32-bit draws
FE_HD int fe_mt_randint(uint32_t* mt, int* pos, int n) {
  const uint32_t rng = (uint32_t)(n - 1);
  if (rng == 0) return 0;
  uint32_t mask = rng;
  mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
  uint32_t v;
  do v = fe_mt_u32(mt, pos) & mask; while (v > rng);
  return (int)v;
}

// ---------------------------------------------------------------- env context of one warp
// Scratch of the connect path, the re-pin and the auto-reset: values lane 0 hands to the other lanes and to later parts of the step
struct FeEnvScratchD {
  double target_quat[4]; // of the aligned connector pair (fe_try_connect_scan -> fe_connect)
  double body1_pose[7];  // _connected_body1 after the connection: the re-pin moves its group back to this pose
  double spare_;
  double lift;           // lowest site z of the two connected groups (floor clearance)
};
struct FeEnvScratchI {
  int aligned;           // fe_try_connect_scan found an aligned pair and no reset has followed: _connected, a connection made during this step
  int repin;             // part to re-pin at body1_pose after the step (_connected_body1), -1 = none
  int site1, site2;      // sites of the aligned pair
  int conn1, conn2;      // their connector indices
  int done;              // the step ends the episode: auto-reset
  int dense_pair;        // the dense reward moved on to its next subtask during this step: its recipe pair replaces subtask_part after the observation
};
struct FeEnv {
  FeWarp* w;      // header of the env's slice
  const fe_scene* sc;
  const fe_config* cfg;
  int env;
  // smem-resident env scratch, ahead of the two state structs so that their size does not move it
  int* group;     // [npart] union-find parents (furniture.py:2738-2759)
  FeEnvScratchI* si;
  FeEnvScratchD* sd;
  FeState st;
  FeEnvState es;
};

FE_HD int fe_find(int* g, int i) { while (g[i] != i) i = g[i]; return i; } // path compression does not change results

// _get_next_subtask (furniture.py:2723-2736), lane 0: the first weld in model order whose two parts lie in different groups (_find_group,
// :2738-2747), -1 / -1 when there is none.  The reference calls it at the end of every _connect (:917) and of _reset (:1653).
FE_HD void fe_next_subtask(FeEnv* e) {
  const fe_scene* sc = e->sc;
  int p1 = -1, p2 = -1;
  for (int q = 0; q < e->w->m->neq; ++q)
    if (fe_find(e->group, sc->eq_part1[q]) != fe_find(e->group, sc->eq_part2[q])) { p1 = sc->eq_part1[q]; p2 = sc->eq_part2[q]; break; }
  e->es.subtask_part[2 * e->env] = p1;
  e->es.subtask_part[2 * e->env + 1] = p2;
}
// FurnitureSawyerDenseRewardEnv._update_reward_variables (furniture_sawyer_dense.py:149-162), lane 0: the pair becomes recipe step s's (leg, table).
// The table is the part that carries the step's table site.
FE_HD void fe_dense_subtask_pair(FeEnv* e, int s) {
  const fe_model* m = e->w->m;
  e->es.subtask_part[2 * e->env] = e->sc->dense.leg_part[s];
  e->es.subtask_part[2 * e->env + 1] = m->site_link[e->sc->dense.table_site[s]] - m->nrlink;
}

// site world pose (float64) from the link poses of the last forward pass held in the warp slice
FE_HDN void fe_site_pose_d(const FeWarp* w, int site, double* pos, double* mat, double* quat) {
  const fe_model* m = w->m;
  const int l = m->site_link[site];
  float R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, P[3] = {0, 0, 0}, Q[4] = {1, 0, 0, 0};
  if (l >= 0) { for (int k = 0; k < 9; ++k) R[k] = w->lmat()[9 * l + k]; v3cpy(P, w->lpos() + 3 * l); for (int k = 0; k < 4; ++k) Q[k] = w->lquat()[4 * l + k]; }
  const float* sp = m->site_pos[site];
  const float* sq = m->site_quat[site];
  for (int i = 0; i < 3; ++i) pos[i] = (double)P[i] + (double)R[3 * i] * sp[0] + (double)R[3 * i + 1] * sp[1] + (double)R[3 * i + 2] * sp[2];
  double bq[4] = {Q[0], Q[1], Q[2], Q[3]}, s4[4] = {sq[0], sq[1], sq[2], sq[3]}, q[4];
  dq_mul(q, bq, s4);
  if (quat) for (int k = 0; k < 4; ++k) quat[k] = q[k];
  if (mat) {
    float Sm[9], sqf[4] = {sq[0], sq[1], sq[2], sq[3]}, Mx[9];
    q2mat(Sm, sqf);
    m3mul(Mx, R, Sm);
    for (int k = 0; k < 9; ++k) mat[k] = (double)Mx[k];
  }
}

// _finger_contact: both fingers of arm `arm` touch the part whose touch bits are `t` (bits 0 / 1: arm 0's fingers, 3 / 4: arm 1's)
FE_HD bool fe_both_fingers(int t, int arm) { const int both = arm == 0 ? 3 : 24; return (t & both) == both; }

// the dense reward's view of the env: poses of the last forward pass, as _get_obs and the connect scan see them
struct FeSliceWorld {
  const FeWarp* w;
  FE_MEMBER void site_pos(int s, double* p) const { fe_site_pose_d(w, s, p, nullptr, nullptr); }
  FE_MEMBER void site_pose(int s, double* p, double* m) const { fe_site_pose_d(w, s, p, m, nullptr); }
  FE_MEMBER void part_pos(int q, double* p) const { const float* lp = w->lpos() + 3 * (w->m->nrlink + q); p[0] = (double)lp[0]; p[1] = (double)lp[1]; p[2] = (double)lp[2]; }
  FE_MEMBER bool touch_both(int q) const { return fe_both_fingers(w->touch()[q], 0); } // _finger_contact(leg): the (only) arm
};

// _stop_object(obj, gravity=gc): xfrc_applied -> gravity-compensation factor, qvel = 0 (furniture.py:2778-2800)
FE_HD void fe_stop_part(FeWarp* w, int p, float gc) {
  const int da = w->m->link_dadr[w->m->nrlink + p];
  w->gravcomp()[p] = gc;
  for (int k = 0; k < 6; ++k) w->qvel()[da + k] = 0.f;
}
// _move_objects_translation_quat(obj, translation, target_quat, gravity=0): rigidly move obj's whole group and stop every part of it
// (furniture.py:1163-1176).  Without `stop` it is the move of _move_rotate_object, which keeps the parts' velocities and gravity compensation.
// A null target_quat is obj's own quaternion.
FE_HDN void fe_move_group(FeEnv* e, int obj, const double* translation, const double* target_quat, bool stop) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const int qb = m->link_qadr[m->nrlink + obj];
  double base[7];
  for (int k = 0; k < 7; ++k) base[k] = (double)w->qpos()[qb + k];
  const int g = fe_find(e->group, obj);
  for (int i = 0; i < m->npart; ++i) {
    if (fe_find(e->group, i) != g) continue;
    const int qa = m->link_qadr[m->nrlink + i];
    double q[7], np_[3], nq[4];
    for (int k = 0; k < 7; ++k) q[k] = (double)w->qpos()[qa + k];
    d_transform_to_target(base, q, target_quat ? target_quat : base + 3, np_, nq);
    for (int k = 0; k < 3; ++k) w->qpos()[qa + k] = (float)(np_[k] + translation[k]);
    for (int k = 0; k < 4; ++k) w->qpos()[qa + 3 + k] = (float)nq[k];
    if (stop) fe_stop_part(w, i, 0.f);
  }
}
// min z over every site of every part in obj's group, starting from 0 (furniture.py:749-769)
FE_HDN double fe_group_min_z(FeEnv* e, int obj) {
  FeWarp* w = e->w;
  const int g = fe_find(e->group, obj);
  double mn = 0.0;
  for (int i = 0; i < w->m->npart; ++i) {
    if (fe_find(e->group, i) != g) continue;
    for (int s = e->sc->part_site_start[i]; s < e->sc->part_site_start[i + 1]; ++s) {
      double p[3];
      fe_site_pose_d(w, e->sc->part_sites[s], p, nullptr, nullptr);
      if (p[2] < mn) mn = p[2];
    }
  }
  return mn;
}

// forward + step as the reference issues them (the extra sim.forward() has no effect on the state)
FE_FN void fe_fwd_step(FeEnv* e) { fe_substep(e->w); }

// _try_connect(part1) for arm agents (part2 = None, _num_connect_steps = 0), furniture.py:926-1042.
// Runs on lane 0; leaves the aligned pair in si->site1 .. conn2 and the target quat in sd->target_quat; si->aligned = 1 if aligned.
FE_FN void fe_try_connect_scan(FeEnv* e, int part1) {
  FeWarp* w = e->w;
  const fe_scene* sc = e->sc;
  LANES_BEGIN
    if (lane == 0) {
      e->si->aligned = 0;
      const int g1 = fe_find(e->group, part1);
      const int* connected = e->es.site_connected + (size_t)e->env * w->m->nsite;
      const double* al = e->es.alignment + (size_t)e->env * 4;
      const double thr[4] = {al[0], al[1], al[2], al[3]};
      bool found = w->m->neq > 0; // some weld joins bodies of the two candidate sets (body2_ids = every part)
      for (int i = 0; i < sc->nconn && found && !e->si->aligned; ++i) {
        if (fe_find(e->group, sc->conn_part[i]) != g1) continue;
        for (int j = 0; j < sc->nconn; ++j) {
          const int s1 = sc->conn_site[i], s2 = sc->conn_site[j];
          if (connected[s1] || connected[s2]) continue;
          if (!(sc->conn_a[i] == sc->conn_b[j] && sc->conn_b[i] == sc->conn_a[j])) continue;
          double p1[3], m1[9], p2[3], m2[9], tq[4];
          bool tq_set;
          fe_site_pose_d(w, s1, p1, m1, nullptr);
          fe_site_pose_d(w, s2, p2, m2, nullptr);
          const bool ok = fe_is_aligned_d(p1, m1, p2, m2, sc->conn_nangles[i], sc->conn_cos[i], sc->conn_sin[i], thr, tq, &tq_set);
          if (tq_set) for (int k = 0; k < 4; ++k) e->sd->target_quat[k] = tq[k];
          if (ok) { e->si->aligned = 1; e->si->site1 = s1; e->si->site2 = s2; e->si->conn1 = i; e->si->conn2 = j; break; }
        }
      }
    }
  LANES_END
}

// _connect(site1, site2, auto_align) (furniture.py:847-924) for arm agents: the pair in si->site1 .. conn2, its target quat in sd->target_quat.
// `align`: FE_ALIGN_CONFIG follows the env's auto_align (a connection made by the policy); the reset's preassembly passes auto_align=_init_qpos is None
// (furniture.py:1556): FE_ALIGN_ALWAYS after random placement, FE_ALIGN_NEVER on a recorded start
enum { FE_ALIGN_CONFIG = 0, FE_ALIGN_ALWAYS = 1, FE_ALIGN_NEVER = 2 };
// _initialize_robot_pos (furniture.py:1761-1779), lane 0: fresh noise on every call, the arm joints at their start pose plus the noise, the
// gripper open; qvel untouched.  Called by the reset's robot poses and by fe_connect under reset_robot_after_attach
FE_HDN void fe_init_robot_pos(FeEnv* e) {
  FeWarp* w = e->w;
  const fe_scene* sc = e->sc;
  uint32_t* mt = e->es.mt + (size_t)e->env * FE_MT_N;
  int pos = e->es.mt_pos[e->env];
  const double r = (double)e->es.placement_rand[(size_t)e->env * 3 + 2]; // agent_xyz_rand; _init_random(shape, "agent") = rng.uniform(-r, r, size=7), furniture.py:336-349
  for (int i = 0; i < sc->narm; ++i) w->qpos()[sc->arm_dof[i]] = (float)ndadd((double)sc->robot_init_qpos[i], fe_mt_uniform(mt, &pos, -r, r));
  for (int i = 0; i < sc->ngrip; ++i) w->qpos()[sc->grip_dof[i]] = sc->robot_init_qpos[sc->narm + i];
  e->es.mt_pos[e->env] = pos;
}
FE_FN void fe_connect(FeEnv* e, int align) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const fe_scene* sc = e->sc;
  const int s1 = e->si->site1, s2 = e->si->site2, body1 = sc->conn_part[e->si->conn1], body2 = sc->conn_part[e->si->conn2];
  LANES_BEGIN
    if (lane == 0) {
      int* connected = e->es.site_connected + (size_t)e->env * m->nsite;
      connected[s1] = 1; connected[s2] = 1;
      const int g1 = fe_find(e->group, body1), g2 = fe_find(e->group, body2);
      for (int g = 0; g < m->ngeom; ++g) { // collision groups, furniture.py:869-878
        const int p = ((m->geom_tag[g] >> FE_TAG_PART_SHIFT) & 0xff) - 1;
        if (p < 0) continue;
        const int gp = fe_find(e->group, p);
        if ((gp == g1 || gp == g2) && w->contype()[g] != 0) { w->contype()[g] = (1 << 30) - 1 - (1 << (g1 + 1)); w->conaff()[g] = 1 << (g1 + 1); }
      }
      if (align == FE_ALIGN_ALWAYS || (align == FE_ALIGN_CONFIG && e->es.auto_align[e->env])) { // _align_connectors -> _move_site_to_target (furniture.py:1224-1250)
        double target[7], base[7], sp[3], sq[4];
        fe_site_pose_d(w, s1, sp, nullptr, sq);
        for (int k = 0; k < 3; ++k) target[k] = sp[k];
        for (int k = 0; k < 4; ++k) target[3 + k] = e->sd->target_quat[k];
        fe_site_pose_d(w, s2, sp, nullptr, sq);
        for (int k = 0; k < 3; ++k) base[k] = sp[k];
        for (int k = 0; k < 4; ++k) base[3 + k] = sq[k];
        const int qa = m->link_qadr[m->nrlink + body2];
        double bq[7], np_[3], nq[4], nsp[3], nsq[4];
        for (int k = 0; k < 7; ++k) bq[k] = (double)w->qpos()[qa + k];
        d_transform_to_target(base, bq, target + 3, np_, nq);
        d_transform_to_target(bq, base, nq, nsp, nsq);
        double tr[3] = {target[0] - nsp[0], target[1] - nsp[1], target[2] - nsp[2]};
        fe_move_group(e, body2, tr, nq, true);
      }
    }
  LANES_END
  fe_fwd_step(e);
  // floor clearance (furniture.py:888-896): lift both groups if any of their sites is below z = 0
  double lift = 0.0;
  LANES_BEGIN
    if (lane == 0) {
      double mn = fe_group_min_z(e, body1), mn2 = fe_group_min_z(e, body2);
      if (mn2 < mn) mn = mn2;
      e->sd->lift = mn;
    }
  LANES_END
  lift = e->sd->lift;
  if (lift < 0.0) {
    for (int which = 0; which < 2; ++which) { // _move_rotate_object(body, offset, [0,0,0]) incl. the step inside _is_inside
      LANES_BEGIN
        if (lane == 0) {
          const double tr[3] = {0, 0, -lift};
          fe_move_group(e, which == 0 ? body1 : body2, tr, nullptr, false); // _move_rotate_object does not stop the parts
        }
      LANES_END
      fe_fwd_step(e);
    }
  }
  fe_fwd_step(e);
  LANES_BEGIN
    if (lane == 0) { // _activate_weld(body1, body2), furniture.py:2761-2776
      for (int q = 0; q < m->neq; ++q) {
        const int a = sc->eq_part1[q], b = sc->eq_part2[q];
        if ((a == body1 || a == body2) && (b == body1 || b == body2)) {
          const int qa = m->link_qadr[m->nrlink + a], qb = m->link_qadr[m->nrlink + b];
          double q1[7], q2[7], inv[4], d[3], r[3], rq[4];
          for (int k = 0; k < 7; ++k) { q1[k] = (double)w->qpos()[qa + k]; q2[k] = (double)w->qpos()[qb + k]; }
          dq_inv(inv, q1 + 3);
          dq_mul(rq, inv, q2 + 3);
          d[0] = q2[0] - q1[0]; d[1] = q2[1] - q1[1]; d[2] = q2[2] - q1[2];
          dq_rotate(r, inv, d);
          for (int k = 0; k < 3; ++k) w->eq_data()[7 * q + k] = (float)r[k];
          for (int k = 0; k < 4; ++k) w->eq_data()[7 * q + 3 + k] = (float)rq[k];
          w->eq_active()[q] = 1;
          const int p1 = fe_find(e->group, body1), p2 = fe_find(e->group, body2);
          e->group[p1] = p2;
        }
      }
      e->es.num_connected[e->env] += 1;
      fe_next_subtask(e);   // :917
      e->si->repin = body1; // _connected_body1 and its pose
      const int qa = m->link_qadr[m->nrlink + body1];
      for (int k = 0; k < 7; ++k) e->sd->body1_pose[k] = (double)w->qpos()[qa + k];
      if (e->es.reset_arm[e->env]) { fe_init_robot_pos(e); e->es.arm_resync[e->env] = 1; } // :919-924, every _connect (the reset's preassembly too)
    }
  LANES_END
}

// robot_ob of every arm from rb on, by every lane: per arm qpos, qvel, gripper qpos, eef pos, quat (xyzw), velp, velr (furniture_sawyer.py:103-155,
// furniture_baxter.py:98-155)
FE_HD void fe_write_robot_ob(FeEnv* e, float* rb, int lane) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const fe_scene* sc = e->sc;
  const int nar = sc->narms > 0 ? sc->narms : 1, na = sc->narm / nar, ngr = sc->ngrip / nar, per = 2 * na + ngr + 13;
  for (int arm = 0; arm < sc->narms; ++arm) {
    float* r = rb + arm * per;
    for (int d = lane; d < na; d += 32) { const int dof = sc->arm_dof[arm * na + d]; r[d] = w->qpos()[dof]; r[na + d] = w->qvel()[dof]; }
    for (int d = lane; d < ngr; d += 32) r[2 * na + d] = w->qpos()[sc->grip_dof[arm * ngr + d]];
    if (lane == 0 && sc->eef_site[arm] >= 0) {
      float* o = r + 2 * na + ngr;
      const int s = sc->eef_site[arm], l = m->site_link[s], hl = sc->hand_link[arm];
      float t[3], sp[3], q[4];
      m3mulv(t, w->lmat() + 9 * l, m->site_pos[s]);
      v3add(sp, w->lpos() + 3 * l, t);
      v3cpy(o, sp);
      qmul(q, w->lquat() + 4 * hl, sc->hand_quat[arm]);
      o[3] = q[1]; o[4] = q[2]; o[5] = q[3]; o[6] = q[0]; // xyzw
      fe_point_vel(w, w->lvel(), l, sp, o + 7);
      v3cpy(o + 10, w->lvel() + 6 * l);
    }
  }
}

// _get_obs under the flags of fe_set_obs_layout (furniture.py:1344-1387): the row [object_ob | subtask_ob | robot_ob | phase_ob], each entry present
// as its flag asks, written to `ob` and, when `packed` is set, to that second row too.  The default flags give object_ob (7 per part, XML order)
// then robot_ob (furniture_sawyer.py:103-155).  It shows the subtask pair held in subtask_part, which the step's dense reward has not moved yet.
FE_FN void fe_write_obs(FeEnv* e, float* ob, float* packed) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const fe_scene* sc = e->sc;
  const int lay = sc->obs_layout, nrl = m->nrlink, np = m->npart;
  const int* pair = e->es.subtask_part + 2 * e->env;
  const bool all = !(lay & (FE_OBS_NO_OBJECT | FE_OBS_PAIR_ONLY)), two = (lay & (FE_OBS_NO_OBJECT | FE_OBS_PAIR_ONLY)) == FE_OBS_PAIR_ONLY;
  const int nobj = all ? 7 * np : (two ? 14 : 0), nsub = (lay & FE_OBS_SUBTASK) ? 2 : 0;
  for (int pass = 0; pass < (packed ? 2 : 1); ++pass) {
  if (pass == 1) ob = packed;
  LANES_BEGIN
    const int p1 = pair[0], p2 = pair[1];
    if (all) {
      for (int p = lane; p < np; p += 32) {
        for (int k = 0; k < 3; ++k) ob[7 * p + k] = w->lpos()[3 * (nrl + p) + k];
        for (int k = 0; k < 4; ++k) ob[7 * p + 3 + k] = w->lquat()[4 * (nrl + p) + k];
      }
    } else if (two && lane < 14) { // the loop over _object_names keeps the pair's parts in part order; none left: np.zeros(14) (:1364-1375)
      const int p = lane < 7 ? (p1 < p2 ? p1 : p2) : (p1 < p2 ? p2 : p1), k = lane % 7;
      ob[lane] = p1 < 0 ? 0.f : (k < 3 ? w->lpos()[3 * (nrl + p) + k] : w->lquat()[4 * (nrl + p) + k - 3]);
    }
    if (nsub && lane < 2) ob[nobj + lane] = (float)((lane == 0 ? p1 : p2) + 1); // [_subtask_part1 + 1, _subtask_part2 + 1] (:1379-1382)
    if (!(lay & FE_OBS_NO_ROBOT)) fe_write_robot_ob(e, ob + nobj + nsub, lane);
    if (sc->phase_ob && lane < 8) ob[sc->obs_dim - 8 + lane] = (e->es.dstate && e->es.dstate[e->env].phase == lane) ? 1.f : 0.f;
  LANES_END
  }
}
// the env's rows of the step's outputs: obs, and the obs columns of the packed row of fe_env_step_packed when it runs
FE_HD void fe_write_step_obs(FeEnv* e) {
  const int od = e->sc->obs_dim;
  fe_write_obs(e, e->es.obs + (size_t)e->env * od, e->es.packed ? e->es.packed + (size_t)e->env * e->es.pk_stride : nullptr);
}
// the episode that ends in this step, before the auto-reset overwrites the slice: its last observation row (the row fe_write_step_obs would
// have written) into terminal_obs and the packed row's terminal slot when the layout has one, its qpos / qvel into terminal_qpos / terminal_qvel
FE_FN void fe_write_terminal(FeEnv* e) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const size_t env = (size_t)e->env;
  float* pk = e->es.packed && e->es.pk_term >= 0 ? e->es.packed + env * e->es.pk_stride + e->es.pk_term : nullptr;
  fe_write_obs(e, e->es.terminal_obs + env * e->sc->obs_dim, pk);
  float* q = e->es.terminal_qpos + env * m->nq;
  float* v = e->es.terminal_qvel + env * m->nv;
  LANES_BEGIN
    for (int i = lane; i < m->nq; i += 32) q[i] = w->qpos()[i];
    for (int i = lane; i < m->nv; i += 32) v[i] = w->qvel()[i];
  LANES_END
}

// stabilise furniture: 10 x { stop(gravity=0); 10 x { forward; step; slow } }  (furniture.py:1535-1540, :1560-1566)
FE_FN void fe_env_stabilise(FeEnv* e) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const int nrl = m->nrlink, np = m->npart;
  for (int outer = 0; outer < 10; ++outer) {
    LANES_BEGIN for (int p = lane; p < np; p += 32) fe_stop_part(w, p, 0.f); LANES_END
    for (int inner = 0; inner < 10; ++inner) {
      fe_fwd_step(e);
      LANES_BEGIN
        for (int p = lane; p < np; p += 32) { // _slow_object: full gravity compensation + velocity clip (furniture.py:2821-2842)
          const int da = m->link_dadr[nrl + p];
          w->gravcomp()[p] = 1.f;
          for (int k = 0; k < 6; ++k) w->qvel()[da + k] = fminf(fmaxf(w->qvel()[da + k], -0.2f), 0.2f);
        }
      LANES_END
    }
  }
}

// the pair and the target of the preassembly's i-th connection (furniture.py:1544-1555), left where fe_try_connect_scan leaves an aligned pair.
// _connect(site2_id, site1_id): the table's connector is _connect's site1, so the leg's group is moved onto the table.
FE_FN void fe_env_preassemble_pair(FeEnv* e, int i) {
  const fe_scene* sc = e->sc;
  const fe_dense_recipe* rc = &sc->dense;
  LANES_BEGIN
    if (lane == 0) {
      const int s1 = rc->table_site[i], s2 = rc->leg_site[i];
      double p[3], m1[9], m2[9];
      fe_site_pose_d(e->w, s1, p, m1, nullptr);
      fe_site_pose_d(e->w, s2, p, m2, nullptr);
      fe_project_connector_quat_d(m1, m2, rc->has_angle[i], rc->angle_cos[i], rc->angle_sin[i], e->sd->target_quat);
      e->si->site1 = s1; e->si->site2 = s2;
      for (int c = 0; c < sc->nconn; ++c) { if (sc->conn_site[c] == s1) e->si->conn1 = c; if (sc->conn_site[c] == s2) e->si->conn2 = c; }
    }
  LANES_END
}

// gravity compensation, this lane's share: qfrc_applied = qfrc_bias of the last forward pass on the arm and gripper dofs (furniture.py:3372-3377)
FE_HD void fe_gravity_comp(FeEnv* e, int lane) {
  FeWarp* w = e->w;
  const fe_scene* sc = e->sc;
  for (int i = lane; i < sc->narm; i += 32) w->qfrc_applied()[sc->arm_dof[i]] = w->bias()[sc->arm_dof[i]];
  for (int i = lane; i < sc->ngrip; i += 32) w->qfrc_applied()[sc->grip_dof[i]] = w->bias()[sc->grip_dof[i]];
}
// the robot's collisions back on, this lane's share: the masks fe_env_reset_clear saved, or 0 under no_collision, whose saved masks are the
// agent's zeros (furniture.py:1586-1595, :1962-1965)
FE_HD void fe_restore_robot_masks(FeEnv* e, int lane) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const int ng = m->ngeom;
  const int* rct = e->es.robot_contype + (size_t)e->env * ng;
  const int* rca = e->es.robot_conaff + (size_t)e->env * ng;
  const bool off = e->es.no_collision[e->env] != 0;
  for (int g = lane; g < ng; g += 32) if (m->geom_tag[g] & FE_TAG_ROBOT) { w->contype()[g] = off ? 0 : rct[g]; w->conaff()[g] = off ? 0 : rca[g]; }
}

// FurnitureEnv._reset (furniture.py:1406-1663) in non-inlined parts called one after the other by fe_env_reset_one, so that the connect path of
// the preassembly does not stack on their frames.  This one, shared by both branches of `if self._init_qpos:`: the size-factor draw, sim.reset()
// and the episode's bookkeeping with the robot's collisions off (:1428-1503), `pre` recipe steps to preassemble
FE_FN void fe_env_reset_clear(FeEnv* e, int pre) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const fe_config* cfg = e->cfg;
  const int nr = m->nr, np = m->npart, ng = m->ngeom;
  int* rct = e->es.robot_contype + (size_t)e->env * ng;
  int* rca = e->es.robot_conaff + (size_t)e->env * ng;
  const bool off = e->es.no_collision[e->env] != 0;
  LANES_BEGIN
    // sim.reset(): data only (model arrays such as masks / eq_data persist)
    for (int i = lane; i < m->nq; i += 32) w->qpos()[i] = 0.f;
    for (int i = lane; i < m->nv; i += 32) { w->qvel()[i] = 0.f; w->warm()[i] = 0.f; }
    for (int i = lane; i < m->nu; i += 32) w->ctrl()[i] = 0.f;
    for (int i = lane; i < nr; i += 32) w->qfrc_applied()[i] = 0.f;
    for (int i = lane; i < np; i += 32) { w->gravcomp()[i] = 0.f; e->group[i] = i; e->es.touched[(size_t)e->env * np + i] = 0; e->es.picked[(size_t)e->env * np + i] = 0; }
    for (int g = lane; g < ng; g += 32) {
      const int tag = m->geom_tag[g];
      if (tag & FE_TAG_ROBOT) { rct[g] = w->contype()[g]; rca[g] = w->conaff()[g]; w->contype()[g] = 0; w->conaff()[g] = 0; } // furniture.py:1441-1453
      if (tag & (1 << 30)) { w->contype()[g] = 1; w->conaff()[g] = 1; }                                                    // :1456-1461
      if (off && fe_geom_is_agent(tag)) { w->contype()[g] = 0; w->conaff()[g] = 0; }                                     // no_collision (:1962-1965)
    }
    const int weld = e->es.assembled[e->env];
    for (int q = lane; q < m->neq; q += 32) w->eq_active()[q] = weld; // :1501-1503: 1 if assembled else 0, eq_data kept as the model holds it
    for (int s = lane; s < m->nsite; s += 32) e->es.site_connected[(size_t)e->env * m->nsite + s] = 0;
    if (lane == 0) {
      e->es.num_connected[e->env] = 0; e->es.prev_num_connected[e->env] = 0; e->es.episode_len[e->env] = 0; e->es.episode_reward[e->env] = 0.f;
      const int ask = e->es.num_connects[e->env];
      e->es.success_num_conn[e->env] = ask >= 0 ? ask + pre : np - 1; // furniture.py:1477-1481
      e->si->aligned = 0;                                             // _connected = False (:1468)
      w->u()[FE_U_FLAGS] = 0;
      if (cfg->furn_size_rand != 0.f) { // _reset draws a size factor first (furniture.py:1428-1431; it only edits the XML tree)
        int pos = e->es.mt_pos[e->env];
        (void)fe_mt_double(e->es.mt + (size_t)e->env * FE_MT_N, &pos);
        e->es.mt_pos[e->env] = pos;
      }
    }
  LANES_END
}
// _place_objects and the first settle loop (:1519-1540).  The env's remembered placement fix_pose is the reference's init_pos / init_quat:
// with fix_init and a placement held, the parts start there and nothing is drawn (:1522); otherwise the sampler runs and its placement is
// remembered (:1520-1525), the parts of fix_init_parts planted at their remembered pose and placed first (:1397-1404) once there is one.
// Under assembled the sampler still draws and init_pos is still updated, but no part is moved (:1526-1532): they stay at qpos0, in group 0
FE_FN void fe_env_reset_place(FeEnv* e) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const fe_scene* sc = e->sc;
  const int nrl = m->nrlink, np = m->npart;
  LANES_BEGIN
    if (lane == 0) { // UniformRandomSampler.sample (placement_sampler.py:137-190): xy noise, z + 0.01, +furn_rot_rand deg about x
      const int env = e->env, have = e->es.fix_have[env];
      double* fp = e->es.fix_pose + (size_t)env * np * 7;
      const unsigned fixed = e->es.fix_init[env] && have ? (1u << np) - 1u : (have ? (unsigned)e->es.fix_init_parts[env] : 0u);
      uint32_t* mt = e->es.mt + (size_t)env * FE_MT_N;
      int pos = e->es.mt_pos[env];
      const float* rnd = e->es.placement_rand + (size_t)env * 3; // furn_xyz_rand, furn_rot_rand
      const double half = 0.5 * (double)rnd[1] * 3.14159265358979323846 / 180.0;
      const double qx[4] = {cos(half), sin(half), 0.0, 0.0};
      const double r_xy = (double)rnd[0], r_rot = (double)rnd[1];
      double px[FE_MAXPART], py[FE_MAXPART]; // placed so far, in double like the sampler's Qpos list
      for (int p = 0; p < np; ++p) {
        const int qa = m->link_qadr[nrl + p];
        if ((fixed >> p) & 1u) { // placed_objects_orig: at its remembered pose, z and quaternion included, no draw (:150-158)
          px[p] = fp[7 * p]; py[p] = fp[7 * p + 1];
          for (int k = 0; k < 7; ++k) w->qpos()[qa + k] = (float)fp[7 * p + k];
        }
      }
      for (int p = 0; p < np; ++p) {
        if ((fixed >> p) & 1u) continue;
        const int qa = m->link_qadr[nrl + p];
        double x = 0, y = 0;
        for (int tries = 0; tries < 10000; ++tries) { // draw order of the reference: x, y per try; the rotation draw after a valid try
          x = ndadd((double)sc->part_init_pos[p][0], fe_mt_uniform(mt, &pos, -r_xy, r_xy));
          y = ndadd((double)sc->part_init_pos[p][1], fe_mt_uniform(mt, &pos, -r_xy, r_xy));
          bool valid = true;
          for (int o = 0; o < np; ++o) { // the fixed parts and the parts placed before p; the outcome does not depend on the order
            if (!(o < p || ((fixed >> o) & 1u)) || o == p) continue;
            const double dx = x - px[o], dy = y - py[o];
            if (ndsqrt(ndadd(ndmul(dx, dx), ndmul(dy, dy))) <= (double)sc->part_radius[o] + (double)sc->part_radius[p]) { valid = false; break; } // np.linalg.norm
          }
          if (valid) break;
        }
        (void)fe_mt_uniform(mt, &pos, r_rot, r_rot); // sample_quat: rng.uniform(high=max, low=max), a draw whose value is always max
        px[p] = x; py[p] = y;
        const float z = sc->part_init_pos[p][2] + 0.01f;
        w->qpos()[qa] = (float)x; w->qpos()[qa + 1] = (float)y; w->qpos()[qa + 2] = z;
        double q0[4] = {sc->part_init_quat[p][0], sc->part_init_quat[p][1], sc->part_init_quat[p][2], sc->part_init_quat[p][3]}, q[4];
        dq_mul(q, q0, qx);
        for (int k = 0; k < 4; ++k) w->qpos()[qa + 3 + k] = (float)q[k];
        // init_pos.update: remembered as planted, so that a later fix_init start is this one bit for bit
        fp[7 * p] = x; fp[7 * p + 1] = y; fp[7 * p + 2] = (double)z;
        for (int k = 0; k < 4; ++k) fp[7 * p + 3 + k] = q[k];
      }
      e->es.fix_have[env] = 1;
      e->es.mt_pos[env] = pos;
      if (e->es.assembled[env]) // `if self._config.assembled: self._object_group[i] = 0` instead of _set_qpos
        for (int p = 0; p < np; ++p) { // qpos0 of a part's free joint is its link frame at qpos0, which the model holds (engine_model.py)
          const int qa = m->link_qadr[nrl + p];
          for (int k = 0; k < 3; ++k) w->qpos()[qa + k] = m->link_pos[nrl + p][k];
          for (int k = 0; k < 4; ++k) w->qpos()[qa + 3 + k] = m->link_quat[nrl + p][k];
          e->group[p] = 0;
        }
    }
  LANES_END
  fe_env_stabilise(e);
}
// gravity compensation and 101 robot poses, the second one with the robot's collisions back on (:1569-1612)
FE_FN void fe_env_reset_robot(FeEnv* e) {
  // gravity compensation, robot pose, one step with robot collisions still off (furniture.py:1569-1584)
  for (int phase = 0; phase < 101; ++phase) {
    LANES_BEGIN
      if (phase <= 1) fe_gravity_comp(e, lane);
      if (phase == 1) fe_restore_robot_masks(e, lane); // :1586-1595
      if (lane == 0) fe_init_robot_pos(e);
    LANES_END
    fe_fwd_step(e);
  }
}
// shared by both branches again: the sync block (furniture.py:1621-1628), gravity compensation from that forward pass, 100 settle steps
// (:1639-1641), the episode's first observation
FE_FN void fe_env_reset_sync(FeEnv* e, int pre) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const fe_scene* sc = e->sc;
  const int nr = m->nr, np = m->npart;
  LANES_BEGIN
    for (int i = lane; i < m->nu; i += 32) w->ctrl()[i] = 0.f;
    for (int i = lane; i < nr; i += 32) w->qfrc_applied()[i] = 0.f;
    for (int i = lane; i < np; i += 32) w->gravcomp()[i] = 0.f;
    for (int i = lane; i < m->nv; i += 32) w->warm()[i] = 0.f;
  LANES_END
  fe_forward(e->w);
  LANES_BEGIN fe_gravity_comp(e, lane); LANES_END
  for (int i = 0; i < 100; ++i) fe_fwd_step(e);
  LANES_BEGIN
    if (lane == 0) {
      e->es.done[e->env] = 0;
      e->si->repin = -1; // _connected_body1 = None (:1558): the preassembly leaves no re-pin pending
      fe_next_subtask(e); // :1653, after the preassembly in both branches
      if (e->es.dense) { // FurnitureSawyerDenseRewardEnv._reset: _reset_reward_variables on the settled scene
        FeSliceWorld world = {w};
        fe_dense_begin_episode(world, e->es.dense + e->env, &sc->dense, pre, e->es.dstate + e->env); // dense_info keeps the last step's terms (the terminal step's, after an auto-reset)
        fe_dense_subtask_pair(e, pre);
      }
    }
  LANES_END
  fe_write_step_obs(e);
}
// set_env_state(_init_qpos) (furniture.py:1794-1798) from bank entry s: _stop_objects(gravity=0), qpos and qvel, ctrl = 0.  `robot`: the first call
// of the reset, which switches the robot's collisions back on (:1505-1517)
FE_FN void fe_env_set_init_state(FeEnv* e, int s, bool robot) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const float* q = e->es.init_qpos + (size_t)s * m->nq;
  const float* v = e->es.init_qvel + (size_t)s * m->nv;
  LANES_BEGIN
    for (int p = lane; p < m->npart; p += 32) w->gravcomp()[p] = 0.f;
    for (int i = lane; i < m->nq; i += 32) w->qpos()[i] = q[i];
    for (int i = lane; i < m->nv; i += 32) w->qvel()[i] = v[i];
    for (int i = lane; i < m->nu; i += 32) w->ctrl()[i] = 0.f;
    if (robot) fe_restore_robot_masks(e, lane);
  LANES_END
}
// the pick before every reset (furniture.py:1433-1434): `if np.random.rand() > 0.2: set_init_qpos(np.random.choice(states))` over the first
// init_pick bank entries, drawn from the env's init_mt; a failed draw keeps the env's start.  Returns the start, -1 = None (random placement);
// an index past the bank counts as None
FE_FN int fe_env_pick_start(FeEnv* e) {
  const int env = e->env, n_init = e->es.n_init;
  LANES_BEGIN
    if (lane == 0) {
      const int n = e->es.init_pick[env] < n_init ? e->es.init_pick[env] : n_init;
      if (n > 0) {
        uint32_t* mt = e->es.init_mt + (size_t)env * FE_MT_N;
        int pos = e->es.init_mt_pos[env];
        if (fe_mt_double(mt, &pos) > 0.2) e->es.init_state[env] = fe_mt_randint(mt, &pos, n);
        e->es.init_mt_pos[env] = pos;
      }
    }
  LANES_END
  const int s = e->es.init_state[env];
  return s < n_init ? s : -1;
}
// the warp slice is (re)initialised here, caller stores it
FE_FN void fe_env_reset_one(FeEnv* e) {
  const fe_scene* sc = e->sc;
  const int want = e->es.preassembled[e->env], cap = sc->dense.nsub - (e->es.dense && sc->dense.nsub > 0 ? 1 : 0); // a recipe prefix; the dense reward needs a subtask left
  const int pre = want < 0 ? 0 : (want > cap ? cap : want);
  const int s = fe_env_pick_start(e);
  fe_env_reset_clear(e, pre);
  if (s < 0) {
    fe_env_reset_place(e);
    for (int i = 0; i < pre; ++i) { fe_env_preassemble_pair(e, i); fe_connect(e, FE_ALIGN_ALWAYS); } // :1542-1558, robot collisions still off
    if (pre > 0) fe_env_stabilise(e);                                                                // :1560-1566
    fe_env_reset_robot(e);
  } else { // `if self._init_qpos:` (:1505-1518): no placement, no settle loop, no random draw; the parts start unwelded
    fe_env_set_init_state(e, s, true);
    fe_forward(e->w);
    for (int i = 0; i < pre; ++i) { fe_env_preassemble_pair(e, i); fe_connect(e, FE_ALIGN_NEVER); } // :1542-1558, robot collisions on
    // The settle loop after the preassembly (:1560-1566) and the forward pass of :1568 are skipped: the second set_env_state (:1617) and the
    // sync block (:1621-1627) overwrite all they produce (qpos, qvel, xfrc, qfrc, warmstart, time); the welds' eq_data is set before them.
    fe_env_set_init_state(e, s, false);
  }
  fe_env_reset_sync(e, pre);
}
// the reset of _do_simulation's except branch (furniture.py:2889-2897), which clears the env's start first: set_init_qpos(None)
FE_HD void fe_env_reset_unstable(FeEnv* e) {
  LANES_BEGIN if (lane == 0) e->es.init_state[e->env] = -1; LANES_END
  fe_env_reset_one(e);
}

// no_collision: the agent's masks stay 0 through the env's steps, whatever wrote them since (furniture.py:1962-1965)
FE_HD void fe_env_agent_masks(FeEnv* e) {
  if (!e->es.no_collision[e->env]) return;
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  LANES_BEGIN
    for (int g = lane; g < m->ngeom; g += 32) if (fe_geom_is_agent(m->geom_tag[g])) { w->contype()[g] = 0; w->conaff()[g] = 0; }
  LANES_END
}
// the per-step flags: no connection found, no re-pin pending, no auto-reset due, no simulation failure yet (lane 0)
FE_HD void fe_env_clear_flags(FeEnv* e) { e->si->aligned = 0; e->si->repin = -1; e->si->done = 0; e->w->u()[FE_U_FLAGS] = 0; }

// _setup_action + gravity compensation with the low-level action `a` (indexed by act_src) and the gripper action `grip`
FE_HD void fe_env_controls(FeEnv* e, const float* a, float grip) {
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
    fe_gravity_comp(e, lane);
    if (lane == 0) fe_env_clear_flags(e);
  LANES_END
}

// what follows the simulation in FurnitureEnv.step, with the policy action `a` (act_dim numbers) for reward and connect
// `fail`: some _do_simulation of this step raised; `reset_now`: the last one did, so the env has not been reset for it yet
FE_HD void fe_env_finish(FeEnv* e, const float* a, int act_dim, float connect, int fail, int reset_now, float* reward_out, uint8_t* done_out, int32_t* info_out) {
  FeWarp* w = e->w;
  const fe_model* m = w->m;
  const fe_scene* sc = e->sc;
  const int np = m->npart, env = e->env;
  FE_SYNC;
  if (reset_now) {
    fe_env_reset_unstable(e);
  } else {
    if (connect > 0.f) { // furniture.py:1290-1322: per arm, the first part both of its fingers touch; stop at the first connection
      for (int arm = 0; arm < sc->narms; ++arm) {
        int part = -1;
        for (int p = 0; p < np; ++p) if (fe_both_fingers(w->touch()[p], arm)) { part = p; break; }
        if (part >= 0) {
          fe_try_connect_scan(e, part);
          if (e->si->aligned) { fe_connect(e, FE_ALIGN_CONFIG); break; }
        }
      }
    }
    const int repin = e->si->repin;
    FE_SYNC; // every lane has read the flag before lane 0 clears it
    if (repin >= 0) { // furniture.py:426-436: re-pin the merged group at the recorded pose, one more step
      LANES_BEGIN
        if (lane == 0) {
          const int b1 = e->si->repin, qa = m->link_qadr[m->nrlink + b1];
          double tr[3] = {e->sd->body1_pose[0] - (double)w->qpos()[qa], e->sd->body1_pose[1] - (double)w->qpos()[qa + 1], e->sd->body1_pose[2] - (double)w->qpos()[qa + 2]};
          fe_move_group(e, b1, tr, e->sd->body1_pose + 3, true);
          e->si->repin = -1;
        }
      LANES_END
      fe_fwd_step(e);
      // the re-pin step diverged: the device's stand-in for the reference, whose re-pin step has no except branch and would raise.  The
      // episode ends as an unstable one, and the reset clears the env's start as _do_simulation's except branch does.
      if (w->u()[FE_U_FLAGS] & FE_FLAG_DIVERGED) { fail = 1; fe_env_reset_unstable(e); }
    }
  }
  // reward (furniture.py:482-541), termination (:440-445, :451-480)
  LANES_BEGIN
    if (lane == 0) {
      float* pk = e->es.packed ? e->es.packed + (size_t)env * e->es.pk_stride : nullptr; // the env's packed row of fe_env_step_packed
      const float* coef = e->es.reward_coef + (size_t)env * 5; // success, touch, pick, ctrl_penalty, unstable_penalty
      float touch_r = 0.f, pick_r = 0.f;
      int* touched = e->es.touched + (size_t)env * np;
      int* picked = e->es.picked + (size_t)env * np;
      if (!fail)
        for (int arm = 0; arm < sc->narms; ++arm) // furniture.py:492-523: both fingers of the same arm
          for (int p = 0; p < np; ++p) {
            const int t = w->touch()[p];
            if (fe_both_fingers(t, arm)) {
              if (!touched[p]) { touched[p] = 1; touch_r += coef[1]; }
              if (!(t & 4) && !picked[p]) { picked[p] = 1; pick_r += coef[2]; }
            }
          }
      const int nc = e->es.num_connected[env];
      const float success_r = coef[0] * (float)(nc - e->es.prev_num_connected[env]);
      const int connected_now = e->si->aligned; // _connected: a connection was made during this step (the legs a reset preassembles are not one)
      e->es.prev_num_connected[env] = nc;
      float sq = 0.f;
      for (int k = 0; k < act_dim; ++k) sq += a[k] * a[k];
      float reward = success_r + touch_r + pick_r - coef[3] * sq;
      // _compute_reward's info (furniture.py:535-540): the terms the reward is made of.  ctrl_penalty (_ctrl_penalty, :549) is the part of the
      // reward the control penalty makes: the reward less the other three in their order.  That is -coef[3] * sq, up to the single rounding
      // of the product the device fuses into the reward, and the four terms add up to the reward exactly.
      const float terms[FE_REWARD_INFO] = {success_r, touch_r, pick_r, reward - (success_r + touch_r + pick_r)};
      const int n_goal = e->es.success_num_conn[env];
      int success = (nc == n_goal && np > 1) ? 1 : 0;
      int done = success;
      e->si->dense_pair = 0;
      if (e->es.dense) { // FurnitureSawyerEnv._step: reward, _done, info = _compute_reward(a); done = done or _done (furniture_sawyer.py:66-84)
        FeSliceWorld world = {w};
        const double* al = e->es.alignment + (size_t)env * 4;
        const double thr[4] = {al[0], al[1], al[2], al[3]};
        double ad[FE_MAXU + 2], dr = 0.0, di[FE_DENSE_INFO];
        for (int k = 0; k < act_dim; ++k) ad[k] = (double)a[k];
        int dd = 0;
        FeDenseState* ds = e->es.dstate + env;
        const int sub0 = ds->subtask;
        fe_dense_step(world, e->es.dense + e->env, &sc->dense, thr, n_goal, ds, ad, act_dim, connected_now, &dr, &dd, di);
        e->si->dense_pair = ds->subtask != sub0 && !ds->success; // _set_next_subtask moved on without finishing (furniture_sawyer_dense.py:141-147)
        reward = (float)dr;
        success = ds->success;
        done = done || dd;
        float* dinf = e->es.dinfo + (size_t)env * FE_DENSE_INFO;
        float* pkd = pk && e->es.pk_dense >= 0 ? pk + e->es.pk_dense : nullptr;
        for (int k = 0; k < FE_DENSE_INFO; ++k) { dinf[k] = (float)di[k]; if (pkd) pkd[k] = (float)di[k]; }
      }
      const int len = ++e->es.episode_len[env];
      // _after_step (furniture.py:459-476): the episode's return before the penalty.  After an unstable step the reset inside the step has
      // zeroed it, as _do_simulation's except branch does (:2889-2897 -> _after_reset :355-356), so that episode reports this step alone.
      const float ep_r = e->es.episode_reward[env] += reward;
      float penalty = 0.f;
      if (len == e->es.max_episode_steps[env] || fail) { done = 1; if (fail) penalty = -coef[4]; }
      reward += penalty;
      reward_out[env] = reward;
      done_out[env] = (uint8_t)done;
      const int32_t iv[FE_INFO_DIM] = {nc, success, fail, len, w->u()[FE_U_NCON], w->u()[FE_U_NITER]};
      const float ep[FE_EPISODE_INFO] = {ep_r + penalty, penalty};
      if (e->es.reward_info) for (int k = 0; k < FE_REWARD_INFO; ++k) e->es.reward_info[(size_t)env * FE_REWARD_INFO + k] = terms[k];
      if (done) for (int k = 0; k < FE_EPISODE_INFO; ++k) e->es.episode_info[(size_t)env * FE_EPISODE_INFO + k] = ep[k];
      if (pk) {
        pk[sc->obs_dim] = reward; pk[sc->obs_dim + 1] = done ? 1.f : 0.f;
        // the info row as int32 bit patterns, which the float32 all-gather carries unchanged
        if (e->es.pk_info >= 0) for (int k = 0; k < FE_INFO_DIM; ++k) ((int32_t*)(pk + e->es.pk_info))[k] = iv[k];
        // the step-info block: the reward terms (NaN on a dense handle, which has none), the episode record where done as in episode_info
        if (e->es.pk_step >= 0) {
          float* ps = pk + e->es.pk_step;
          for (int k = 0; k < FE_REWARD_INFO; ++k) ps[k] = e->es.reward_info ? terms[k] : nanf("");
          if (done) for (int k = 0; k < FE_EPISODE_INFO; ++k) ps[FE_REWARD_INFO + k] = ep[k];
        }
      }
      int32_t* info = info_out + (size_t)env * FE_INFO_DIM;
      for (int k = 0; k < FE_INFO_DIM; ++k) info[k] = iv[k];
      e->es.done[env] = done;
      // An unstable episode resets twice, as the reference does: once inside _do_simulation's except branch
      // (furniture.py:2889-2897) and once more by the VecEnv worker because the step returned done (subproc_vec_env.py:16-20).
      // The second reset zeroes the episode length that _after_step just incremented and consumes its own random draws,
      // so the env's generator stays draw-for-draw on the reference's stream.
      e->si->done = done;
    }
  LANES_END
  if (e->si->done) {
    // The finished episode's last observation and state, taken between the two resets of an unstable step: after the one of _do_simulation's
    // except branch, whose freshly reset world is what the reference's step returns (furniture.py:2889-2897), and before the auto-reset
    fe_write_terminal(e);
    fe_env_reset_one(e);
  } else {
    fe_write_step_obs(e);
    // FurnitureSawyerEnv._step takes the observation before _compute_reward (furniture_sawyer.py:66-84): it shows the pair as the connect scan
    // left it, and the dense reward's new subtask pair is the env's from here on
    LANES_BEGIN if (lane == 0 && e->si->dense_pair) fe_dense_subtask_pair(e, e->es.dstate[env].subtask); LANES_END
  }
}

// FurnitureEnv.step for one env; writes reward / done / info; auto-resets when done (subproc_vec_env.py:16-20)
FE_FN void fe_env_step_one(FeEnv* e, const float* action, float* reward_out, uint8_t* done_out, int32_t* info_out) {
  FeWarp* w = e->w;
  const fe_scene* sc = e->sc;
  const fe_config* cfg = e->cfg;
  const float* a = action + (size_t)e->env * sc->act_dim;
  float grip = sc->grip_action_index >= 0 ? a[sc->grip_action_index] : 0.f;
  if (cfg->discrete_grip) grip = grip < 0.f ? -1.f : 1.f; // FurnitureSawyerEnv._step only (furniture_sawyer.py:73-74); Baxter: index -1
  const float connect = a[sc->connect_action_index];
  fe_env_controls(e, a, grip);
  fe_env_agent_masks(e);
  fe_substeps_mixed(w, e->es.substeps[e->env]); // _do_simulation, furniture.py:2877-2879
  const int fail = (w->u()[FE_U_FLAGS] & FE_FLAG_DIVERGED) ? 1 : 0; // MujocoException path, :2889-2897
  fe_env_finish(e, a, sc->act_dim, connect, fail, fail, reward_out, done_out, info_out);
}

// per-env context set-up shared by the CUDA kernels and the emulation loop
FE_FN void fe_env_bind(FeEnv* e, float* slice, const fe_model* m, const fe_scene* sc, const fe_config* cfg, const FeOpt& opt, const FeState& st,
                       const FeEnvState& es, int env, int slice_words_physics) {
  e->w = fe_warp_bind(slice, m, opt);
  e->sc = sc; e->cfg = cfg; e->st = st; e->es = es; e->env = env;
  float* extra = slice + slice_words_physics;
  e->sd = (FeEnvScratchD*)extra;     // 8-byte aligned: slices are multiples of 32 words
  e->si = (FeEnvScratchI*)(extra + 32);
  e->group = (int*)(extra + 40);     // FE_MAXPART ints
}
#define FE_ENV_EXTRA_WORDS 64
static_assert(sizeof(FeEnvScratchD) <= 4 * 32, "the double scratch ends before the int scratch at word 32");
static_assert(sizeof(FeEnvScratchI) <= 4 * (40 - 32), "the int scratch ends before group at word 40");
static_assert(40 + FE_MAXPART <= FE_ENV_EXTRA_WORDS, "group ends within the env's extra words");
FE_FN void fe_env_load_groups(FeEnv* e) {
  const int np = e->w->m->npart;
  LANES_BEGIN for (int p = lane; p < np; p += 32) e->group[p] = e->es.group[(size_t)e->env * np + p]; LANES_END
}
FE_FN void fe_env_store_groups(FeEnv* e) {
  const int np = e->w->m->npart;
  LANES_BEGIN for (int p = lane; p < np; p += 32) e->es.group[(size_t)e->env * np + p] = e->group[p]; LANES_END
}
// one env in its slice: bind, load the env's state from HBM, run `body(FeEnv*)` (a reset or a step), store the state back
template <class Body>
FE_HD void fe_env_run(float* slice, const fe_model* m, const fe_scene* sc, const fe_config* cfg, const FeOpt& opt, const FeState& st, const FeEnvState& es,
                      int env, int slice_words_physics, Body body) {
  FeEnv e;
  fe_env_bind(&e, slice, m, sc, cfg, opt, st, es, env, slice_words_physics);
  fe_load(e.w, st, env);
  fe_env_load_groups(&e);
  body(&e);
  fe_env_store_groups(&e);
  fe_store(e.w, st, env);
}
