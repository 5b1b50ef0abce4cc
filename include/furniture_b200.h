/* furniture_b200.h -- C-ABI of the H100-native (sm_90a) batched physics backend.
 *
 * The reference has no FFI seam of its own: FurnitureEnv drives the closed MuJoCo 2.0 binary through mujoco-py
 * (SURVEY.md 8b-B2).  This header is the seam a maintainer would bind instead; every entry point names the
 * reference call it replaces.  Plain pointers and sizes only; no torch types.
 *
 *   fe_create        <- load_model_from_xml + MjSim(model)          furniture/env/models/base.py:113-115, furniture.py:1837-1838
 *   fe_sim_forward   <- sim.forward()   (17 call sites, e.g.)        furniture/env/furniture.py:2877
 *   fe_sim_step      <- sim.step()      (12 call sites, e.g.)        furniture/env/furniture.py:2878-2879
 *   fe_set_field/fe_get_field <- sim.data.* / sim.model.* views     furniture.py:1622-1627, :2784-2800, :875-878, :2772-2775
 *   fe_get_state/fe_set_state <- get_env_state / set_env_state      furniture/env/furniture.py:1781-1803, :3095-3105
 *   fe_env_reset     <- FurnitureEnv.reset() -> _reset()             furniture/env/furniture.py:318-334, :1406-1663
 *   fe_env_step      <- FurnitureEnv.step() (incl. _step_continuous, _try_connect/_is_aligned/_connect, _get_obs,
 *                       _compute_reward, _after_step; VecEnv auto-reset) furniture.py:364-385, :405-449, :1260-1330,
 *                       :926-1153, :847-924, furniture_sawyer.py:66-155, util/subproc_vec_env.py:16-20
 *   fe_is_aligned    <- FurnitureEnv._is_aligned on explicit site poses (test hook)  furniture.py:1057-1153
 *   fe_enable_dense_reward <- FurnitureSawyerDenseRewardEnv (env id IKEASawyerDense-v0): _compute_reward and the phase machine
 *                       around it replace the sparse reward inside fe_env_step         furniture_sawyer_dense.py:18-1022
 *   fe_dense_eval    <- the same reward machine on explicit poses (test hook)          furniture_sawyer_dense.py:225-586
 *
 * Conventions: every function returns 0 on success or a negative code and records a message retrievable with
 * fe_last_error(); a handle is bound to one CUDA device, is not thread-safe, and all work is issued on the stream
 * passed in (NULL = default stream).  "dev" pointers are device memory, "host" pointers are host memory.  All
 * per-env arrays at the boundary are env-major and contiguous: (n_envs, dim).
 */
#ifndef FURNITURE_B200_H
#define FURNITURE_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct fe_handle fe_handle;

typedef struct fe_config {
  int32_t struct_bytes;      /* sizeof(fe_config), checked */
  int32_t maxcon;            /* contact capacity per env (MuJoCo: nconmax, base.xml:5); an env that overflows raises bit 0 of `flags` */
  int32_t newton_iters;      /* max Newton iterations per mj_step (MuJoCo default 100) */
  int32_t ls_iters;          /* max line-search evaluations per Newton iteration */
  float tolerance;           /* solver tolerance on scaled improvement / gradient (MuJoCo: 1e-8 in double) */
  int32_t nsub;              /* mj_steps per env step = int(control_timestep / model_timestep), furniture.py:2878 */
  int32_t max_episode_steps; /* config/furniture.py:164 */
  int32_t discrete_grip, rescale_actions, auto_align; /* config/furniture.py:75, :90, :96 */
  double alignment_pos_dist, alignment_rot_dist_up, alignment_rot_dist_forward, alignment_project_dist; /* :203-226 */
  float ctrl_penalty_coef, unstable_penalty_coef, success_reward, touch_reward, pick_reward;            /* :291-295 */
  float furn_xyz_rand, furn_rot_rand, agent_xyz_rand; /* :177-194 */
  float furn_size_rand;      /* :196-201; != 0: every env's generator gives one draw at creation and one per reset to the size factor
                                (furniture.py:1989-1991, :1428-1431); the geometry itself is fixed by the scene handed to fe_create */
  uint64_t seed;             /* env i draws its resets from numpy's RandomState(seed + i) stream: MT19937 state per env
                                (fields mt_state / mt_pos), the reference's draw order (furniture.py:72, env/base.py:77) */
} fe_config;

/* coefficients of the dense reward: config/furniture_sawyer_dense.py:5-71 (defaults there), ctrl_penalty_coef of config/furniture.py:291 */
typedef struct fe_dense_config {
  int32_t struct_bytes; /* sizeof(fe_dense_config), checked */
  int32_t diff_rew, early_termination, phase_ob, reset_robot_after_attach, pad_;
  double phase_bonus, ctrl_penalty_coef, eef_forward_dist_coef, eef_up_dist_coef, eef_rot_threshold, gripper_penalty_coef, move_other_part_penalty_coef,
      drop_penalty_coef, init_eef_pos_dist_coef, move_eef_pos_dist_coef, lower_eef_pos_dist_coef, grasp_dist_coef, lift_z_dist_coef, lift_xy_dist_coef,
      lift_z_pos_threshold, lift_xy_pos_threshold, align_pos_dist_coef, align_rot_dist_coef, align_pos_threshold, align_rot_threshold, move_pos_dist_coef,
      move_rot_dist_coef, move_pos_threshold, move_rot_threshold, move_fine_pos_exp_coef, move_fine_pos_dist_coef, move_fine_rot_dist_coef,
      aligned_bonus_coef;
} fe_dense_config;

/* sizes of the blobs the host packs (furniture_b200/engine_model.py, furniture_b200/scene.py) */
size_t fe_model_sizeof(void);
size_t fe_scene_sizeof(void);
size_t fe_config_sizeof(void);
size_t fe_dense_recipe_sizeof(void); /* the recipe block inside the scene blob (fe_dense_recipe, csrc/fe_dense.h) */
/* 1 if this library drives a CUDA device, 0 for the lane-emulated test build (never shipped) */
int fe_is_cuda(void);

int fe_create(const void* model_blob, size_t model_bytes, const void* scene_blob, size_t scene_bytes, const fe_config* cfg, int n_envs,
              int device, fe_handle** out);
/* Same, from a scene file: the two blobs as written by fe_scene_file_write (magic "FEB1", sizes, fe_model, fe_scene).  The
   files furniture_b200/compiled/<agent>_<furniture>.feb are produced offline by tools/compile_models.py from the composed MJCF
   (models/base.py:76-116 + load_model_from_xml), so that a binder in any language creates a handle with this one call and no
   Python at run time. */
int fe_create_from_file(const char* scene_file, const fe_config* cfg, int n_envs, int device, fe_handle** out);
int fe_scene_file_write(const char* scene_file, const void* model_blob, size_t model_bytes, const void* scene_blob, size_t scene_bytes);
void fe_destroy(fe_handle* h);
const char* fe_last_error(const fe_handle* h); /* h may be NULL: last creation error */

int fe_num_envs(const fe_handle* h);
int fe_obs_dim(const fe_handle* h);    /* robot_ob (29 for Sawyer impedance) + object_ob (7 per part) */
int fe_action_dim(const fe_handle* h); /* dof: 7 joint velocities + gripper + connect for Sawyer impedance */
int fe_info_dim(const fe_handle* h);   /* int32 per env: num_connected, success, unstable, episode_length, ncon, solver iters */
int fe_smem_bytes_per_env(const fe_handle* h); /* shared-memory working set of one env (one warp) */

/* ---- simulator surface (MjSim) */
int fe_sim_forward(fe_handle* h, void* stream);
int fe_sim_step(fe_handle* h, int nsub, void* stream);
/* named per-env arrays, host side; bytes must equal n_envs * dim * sizeof(elem). Names: qpos qvel ctrl qfrc_applied
   qacc_warmstart gravcomp eq_data eq_active geom_contype geom_conaffinity mt_state (624 x uint32) mt_pos (read/write); qfrc_bias link_xpos link_xquat
   link_xmat link_vel touch ncon niter flags + the debug fields of the last fe_sim_forward (read only) */
int fe_get_field(fe_handle* h, const char* name, void* dst_host, size_t bytes);
int fe_set_field(fe_handle* h, const char* name, const void* src_host, size_t bytes);
int fe_field_dim(fe_handle* h, const char* name, int* dim, int* elem_bytes);
int fe_get_state(fe_handle* h, float* qpos_host, float* qvel_host);
int fe_set_state(fe_handle* h, const float* qpos_host, const float* qvel_host);

/* ---- environment surface (FurnitureEnv / VecEnv) */
int fe_env_reset(fe_handle* h, const uint8_t* env_mask_dev /* NULL = all */, float* obs_dev, void* stream);
int fe_env_step(fe_handle* h, const float* actions_dev, float* obs_dev, float* reward_dev, uint8_t* done_dev, int32_t* info_dev,
                void* stream);
/* same step, results written by the kernel as rows [obs | reward | done] of (obs_dim + 2) floats: the send buffer of the
   observation all-gather over env shards (SURVEY.md 8e; the reference's counterpart is the pipe of
   util/subproc_vec_env.py:100-113 that carries (ob, reward, done, info) of every worker back to the caller) */
int fe_env_step_packed(fe_handle* h, const float* actions_dev, float* packed_dev, int32_t* info_dev, void* stream);
/* same call with host buffers: H2D of the actions and D2H of the results happen inside (pinned staging) */
int fe_env_step_host(fe_handle* h, const float* actions_host, float* obs_host, float* reward_host, uint8_t* done_host, int32_t* info_host);
/* FurnitureGym.set_max_episode_steps -> FurnitureEnv.set_max_episode_steps (furniture_gym.py:35-37, furniture.py:271-272):
   takes effect from the next step */
int fe_set_max_episode_steps(fe_handle* h, int max_episode_steps);
/* Switch the handle to the dense reward; call before the first fe_env_reset.  The scene must carry a recipe, and dc->phase_ob must agree
 * with the scene (the one-hot phase is part of obs_dim).  fe_env_step then returns the dense reward / done / success, and field
 * "dense_info" holds (n_envs, fe_dense_info_dim()) float32 per step: phase, subtask, phase_bonus, ctrl_penalty, gripper_penalty,
 * move_other_part_penalty, drop_penalty, touch, drop_leg, table_moved, stable_grip_succ, skips (bit 0 to lift_leg, bit 1 to move_leg_fine). */
int fe_enable_dense_reward(fe_handle* h, const fe_dense_config* dc);
int fe_dense_info_dim(void);
/* device pointer of the internal obs buffer after the last step/reset: (n_envs, obs_dim) float32 */
const float* fe_obs_dev(const fe_handle* h);

/* ---- test hook: the device _is_aligned on explicit site poses (float64), n independent cases */
int fe_is_aligned(fe_handle* h, int n, const double* p1, const double* m1, const double* p2, const double* m2, const double* angles /* (n,4) */,
                  const int32_t* nangles, const double* thr /* (n,4) */, uint8_t* aligned_host, double* target_quat_host /* (n,4) wxyz, NaN if unset */);

/* ---- test hook: the device reward machine on explicit poses.  Records [first[e], first[e] + count[e]) form episode e and are walked in
 * order by one thread; a record with reset != 0 starts the episode on the world it shows.  Per record: site_pos (nsite,3), site_mat
 * (nsite,9 row-major), part_pos (npart,3), touch (npart: both fingers on the part), connected, ac (act_dim).  The ids inside the recipe
 * blob index these arrays.  Outputs per record: reward, done (bit 0 done, bit 1 success), info (fe_dense_info_dim() doubles). */
int fe_dense_eval(fe_handle* h, const fe_dense_config* dc, const void* recipe_blob, size_t recipe_bytes, const double* thr4, int n_goal, int n_episodes,
                  const int32_t* first, const int32_t* count, int n_records, int nsite, int npart, int act_dim, const double* site_pos,
                  const double* site_mat, const double* part_pos, const uint8_t* touch, const uint8_t* reset, const uint8_t* connected, const double* ac,
                  double* reward_host, uint8_t* done_host, double* info_host);

/* ---- control_type="ik" for the one-arm env: FurnitureEnv._do_ik_step (furniture.py:2899-2996) + SawyerIKController
 * (controllers/sawyer_ik_controller.py) with the pybullet solve replaced by a damped-least-squares IK on the arm's own chain, run inside
 * the step kernel.  Speeds: config/furniture.py:84-89; workspace and the three repeats: furniture.py:166-172; sensitivity 0.3, gain 5,
 * joint damping 0.1, rest pose, limits: sawyer_ik_controller.py (Baxter: 1.0, 2, 0.7, baxter_ik_controller.py).  The chain (host: furniture_b200/ik.py: arm_chain) lists, per arm joint,
 * its body frame in the previous joint body's frame at zero angle and the hinge (anchor, axis) in its body frame. */
typedef struct fe_ik_arm {
  float rest_pose[7], lower[7], upper[7];
  float link_pos[7][3], link_quat[7][4], jaxis[7][3], jpos[7][3];
  float hand_pos[3], hand_quat[4]; /* "<arm>_hand" in the last joint body's frame */
  int32_t arm_qadr[7];             /* qpos index of every joint of this arm */
  int32_t pad_;
} fe_ik_arm;
typedef struct fe_ik_config {
  int32_t struct_bytes, action_repeat, max_iters;
  int32_t quaternion_mode; /* 1: control_type="ik_quaternion" (furniture.py:2998-3058): actions are move 3, quaternion (w,x,y,z) relative to the hand, gripper, connect */
  float move_speed, rotate_speed, user_sensitivity, kp, damping, null_gain, tol_pos, tol_rot, max_step_pos, max_step_rot;
  float min_pos[3], max_pos[3];
  float base_pos[3], base_quat[4]; /* the robot base in the world: targets are kept in its frame */
  int32_t narms, pad_;             /* 1 (Sawyer) or 2 (Baxter: right, then left; actions (move, rotate) per arm, then the grippers, then connect) */
  fe_ik_arm arm[2];
} fe_ik_config;
/* Switch the handle to control_type="ik": fe_env_step then takes (n_envs, 8) actions (move 3, rotate 3, gripper, connect) and
 * fe_action_dim() returns 8.  Field "ik_state" holds per env, for two arms (the second unused with one): accumulated target quaternions
 * (2 x 4), target positions in the base frame (2 x 3), commanded joints (14), last low-level action (16) as float32, then the iteration counts
 * of the last solves (2 x int32). */
int fe_enable_ik(fe_handle* h, const fe_ik_config* ikc);

/* ---- the torque controllers of controllers/arm_controller.py (NEW_CONTROLLERS): parameters of one controller (host: furniture_b200/
 * controllers.py from controllers/controller_config.hjson).  mode: 0 joint_torque, 1 joint_velocity, 2 joint_impedance, 3 position_orientation,
 * 4 position.  ramp_steps = floor(0.2 * control_freq / model timestep) as the reference computes it (arm_controller.py:111). */
typedef struct fe_ctl_config {
  int32_t struct_bytes, mode, control_dim, pad_;
  double move_speed;                              /* _do_controller_step scales and swaps action[:3] for every controller (furniture.py:3069-3071) */
  double control_max[7], kp[7], damping[7], kv[7];
  double ramp_steps;
  float hand_pos[3], hand_quat[4];                /* right_hand in the frame of the link that carries it */
} fe_ctl_config;
/* Switch the handle (one-arm env on the torque-actuated robot, robots/sawyer/robot_torque.xml) to one of these controllers: fe_env_step then
 * takes (n_envs, control_dim + 2) actions -- the controller's command, the gripper, connect -- and runs _do_controller_step
 * (furniture.py:3065-3093): sim.forward(), then before every mj_step the controller turns the hand pose / velocity, the hand Jacobian and
 * the arm block of the joint-space inertia of the last forward pass into joint torques, ctrl = qfrc_bias + torques (_pre_action :1706-1759). */
int fe_enable_controller(fe_handle* h, const fe_ctl_config* cc);
/* test hook: the device controller arithmetic on explicit simulator readings.  Records [first[e], first[e] + count[e]) form episode e; per
 * record: reset / policy_step flags, action (7 doubles, the first control_dim used) and the readings as 123 doubles: pos 3, R 9 (row-major),
 * velp 3, velr 3, q 7, qvel 7, Jx 21, Jr 21 (3 x 7 row-major), M 49.  Output: torques (7 doubles per record). */
int fe_ctl_eval(fe_handle* h, const fe_ctl_config* cc, int n_episodes, const int32_t* first, const int32_t* count, int n_records, const uint8_t* reset,
                const uint8_t* policy_step, const double* action, const double* readings, double* torques_host);

#ifdef __cplusplus
}
#endif
#endif
