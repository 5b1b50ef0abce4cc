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
 *   fe_set_init_states <- the states of --load_init_states / --load_demo / set_init_qpos   furniture.py:121-130, :315-316
 *   fe_env_step      <- FurnitureEnv.step() (incl. _step_continuous, _try_connect/_is_aligned/_connect, _get_obs,
 *                       _compute_reward, _after_step; VecEnv auto-reset) furniture.py:364-385, :405-449, :1260-1330,
 *                       :926-1153, :847-924, furniture_sawyer.py:66-155, util/subproc_vec_env.py:16-20
 *   fe_is_aligned    <- FurnitureEnv._is_aligned on explicit site poses (test hook)  furniture.py:1057-1153
 *   fe_enable_dense_reward <- FurnitureSawyerDenseRewardEnv (env id IKEASawyerDense-v0): _compute_reward and the phase machine
 *                       around it replace the sparse reward inside fe_env_step         furniture_sawyer_dense.py:18-1022
 *   fe_dense_eval    <- the same reward machine on explicit poses (test hook)          furniture_sawyer_dense.py:225-586
 *   fe_set_obs_layout <- the observation flags robot_ob / object_ob / object_ob_all / subtask_ob, with _get_next_subtask
 *                       tracked per env inside the kernels    furniture.py:103-107, :215-252, :1344-1387, :2723-2759
 *   fe_terminal_obs_dev / fe_terminal_qpos_dev / fe_terminal_qvel_dev <- the terminal `ob` of FurnitureEnv.step and the state
 *                       get_env_state gives at that point     furniture.py:364-385, :1781-1792
 *   fe_reward_info_dev / fe_episode_info_dev <- the `info` dict of FurnitureEnv.step: _compute_reward's four terms and
 *                       _after_step's episode record           furniture.py:451-541, :543-550
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
  int32_t maxcon;            /* contact capacity per env (MuJoCo: nconmax, base.xml:5); an env that overflows raises FE_FLAG_CONTACT_FULL in `flags` */
  int32_t newton_iters;      /* max Newton iterations per mj_step (MuJoCo default 100) */
  int32_t ls_iters;          /* max line-search evaluations per Newton iteration */
  float tolerance;           /* solver tolerance on scaled improvement / gradient (MuJoCo: 1e-8 in double) */
  int32_t nsub;              /* mj_steps per env step = int(control_timestep / model_timestep), furniture.py:2878: every env's substeps at fe_create */
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
int fe_obs_dim(const fe_handle* h);    /* object_ob (7 per part) + robot_ob (29 for Sawyer impedance) by default; see fe_set_obs_layout */
int fe_action_dim(const fe_handle* h); /* dof: 7 joint velocities + gripper + connect for Sawyer impedance */
int fe_info_dim(const fe_handle* h);   /* int32 per env: num_connected, success, unstable, episode_length, ncon, solver iters */
int fe_smem_bytes_per_env(const fe_handle* h); /* shared-memory working set of one env (one warp) */

/* ---- simulator surface (MjSim) */
int fe_sim_forward(fe_handle* h, void* stream);
int fe_sim_step(fe_handle* h, int nsub, void* stream);
/* named per-env arrays, host side; bytes must equal n_envs * dim * sizeof(elem). Names: qpos qvel ctrl qfrc_applied
   qacc_warmstart gravcomp eq_data eq_active geom_contype geom_conaffinity mt_state (624 x uint32) mt_pos (read/write); qfrc_bias link_xpos link_xquat
   link_xmat link_vel touch ncon niter + the debug fields of the last fe_sim_forward (read only); flags (int32, the FE_FLAG_* bits below;
   read/write); stats (int32, one per FE_STAT_* column below; read only); order (int32, one per env: the env ids by the predicted work of their
   next env step, heaviest first, the order in which the step packs envs into blocks); preassembled num_connects (int32, one per env,
   read/write: FurnitureEnv.set_subtask, furniture.py:204-207.  An env's next reset, an auto-reset included, connects the first `preassembled`
   steps of the scene's assembly recipe before it places the robot, and the episode then succeeds at num_connects + preassembled connections,
   or with every part connected when num_connects is -1); init_state init_pick init_mt_state (624 x uint32) init_mt_pos (int32, one per env,
   read/write: the env's recorded start, see fe_set_init_states); subtask_part (2 x int32 per env, read only: _subtask_part1 / _subtask_part2,
   the two parts of the env's current subtask, -1 / -1 when none is left -- see fe_set_obs_layout); fix_init fix_init_parts fix_have (int32,
   one per env, read/write: config/furniture.py:116-127.  fix_init = 1 with fix_have = 1: the env's random-placement resets plant fix_pose and
   draw nothing; otherwise they sample, planting the parts whose bit is set in fix_init_parts at fix_pose first when fix_have = 1, and store
   the placement into fix_pose with fix_have = 1 -- furniture.py:1389-1404, :1519-1532; a recorded start ignores both); fix_pose (7 x float64
   per part, XML order, read/write: position and quaternion w, x, y, z, the reference's init_pos / init_quat; fe_create leaves fix_have = 0,
   the XML poses are the caller's to seed); reset_robot_after_attach (int32, one per env, read/write: every connection, the reset's
   preassembly included, ends with _initialize_robot_pos, furniture.py:916-924, and the IK step re-seeds its position target; a dense handle
   sets it from fe_dense_config.reset_robot_after_attach); substeps (int32, one per env, read/write: the env's mj_steps per env step,
   int(control_timestep / model_timestep) of furniture.py:2878 for its control_freq; fe_create sets fe_config.nsub.  The stock step runs it,
   the IK step runs it once per closed-loop repeat, the torque-controller step evaluates the controller before each of them; envs with
   different counts share one launch); no_collision (int32, one per env, read/write: config/furniture.py's no_collision, furniture.py:1962-1965:
   while 1, contype = conaffinity = 0 on every geom of the agent -- every colliding geom that is neither a furniture part's nor the floor --
   through steps and resets.  Writing it changes the env's geom_contype / geom_conaffinity at once: 0 where it turns on, the model's compiled
   masks where it turns off); assembled (int32, one per env, read/write: config/furniture.py:307-312.  From the env's next reset on, an
   auto-reset included, every weld starts on with the eq_data the env holds, and a random-placement reset still draws and stores its
   placement but leaves the parts at the model's qpos0 (their link frames), all in one group -- furniture.py:1501-1532; a recorded start
   turns the welds on and merges no group); the task options of config/furniture.py, per env, read by the kernels in place of the same
   fe_config members and set from them by fe_create: alignment (4 x float64 per env, read/write: alignment_pos_dist, alignment_rot_dist_up,
   alignment_rot_dist_forward, alignment_project_dist, :203-226) and auto_align (int32, one per env, read/write: :95-100), from the env's next
   step; placement_rand (3 x float32 per env, read/write: furn_xyz_rand, furn_rot_rand, agent_xyz_rand, :177-194), from the env's next reset,
   agent_xyz_rand also from its next connection under reset_robot_after_attach; reward_coef (5 x float32 per env, read/write: success_reward,
   touch_reward, pick_reward, ctrl_penalty_coef, unstable_penalty_coef, :291-295), from the env's next step; max_episode_steps (int32, one
   per env, read/write: :163-168), at once, an episode ending when its length equals it (fe_set_max_episode_steps writes every env's);
   dense_config (one fe_dense_config per env, typestr "|V" + its size, read/write, a dense handle only: fe_enable_dense_reward fills every
   row with its argument): the env's coefficients, thresholds and flags of the dense reward, from its next step, but diff_rew, which an
   episode keeps from its start (the shaped terms difference against values kept in that mode only).  Writing it sets every env's
   reset_robot_after_attach from its row.  fe_set_field refuses rows whose struct_bytes is not sizeof(fe_dense_config), whose diff_rew,
   early_termination or reset_robot_after_attach is outside {0, 1}, whose phase_ob disagrees with the handle's (the obs width is the
   handle's) or that hold a non-finite coefficient or threshold.
   fe_set_field refuses flags outside {0, 1}, substeps below 1, fix_init_parts bits at or beyond the
   number of parts, non-finite fix_pose values or zero quaternions, fix_have = 1 for an env whose fix_pose was never written, non-finite
   alignment / placement_rand / reward_coef values, max_episode_steps below 1 and, in a dense handle, a reset_robot_after_attach that
   differs from the env's dense_config row or a reward_coef whose first four columns differ from the handle's fe_config (the phase machine
   replaces those terms; its ctrl_penalty_coef is fe_dense_config's) */
int fe_get_field(fe_handle* h, const char* name, void* dst_host, size_t bytes);
int fe_set_field(fe_handle* h, const char* name, const void* src_host, size_t bytes);
int fe_field_dim(fe_handle* h, const char* name, int* dim, int* elem_bytes);
/* the numpy typestr of one element of field `name`: "<i4" (int32), "<u4" (uint32), "<f4" (float32), "<f8" (float64) or "|u1" (bytes, the
   struct-valued fields ik_state, ctl_state and dense_state); NULL for an unknown name, with fe_last_error set */
const char* fe_field_dtype(fe_handle* h, const char* name);
int fe_get_state(fe_handle* h, float* qpos_host, float* qvel_host);
int fe_set_state(fe_handle* h, const float* qpos_host, const float* qvel_host);
/* Recorded starts, FurnitureEnv._init_qpos (furniture.py:121-130, :315-316, :1433-1434, :1505-1518, :1617): a bank of n_states
   get_env_state records, qpos (n_states, nq) and qvel (n_states, nv) from host memory, shared by the envs of the handle; n_states = 0 frees it.
   Non-finite values are refused.  Per env, field init_state is the bank index its resets start from (-1 = None: random placement).  Such a
   reset, an auto-reset included, plants the state instead of placing the parts and posing the robot: the parts start unwelded, the first
   `preassembled` recipe steps are connected without aligning the connectors, the state is planted again and 100 mj_steps settle it.
   Field init_pick = n > 0 is --load_init_states over the first n bank entries: before every reset, if rand() > 0.2, init_state = choice(n),
   drawn from the env's own numpy RandomState(seed + 2**20 + env) (init_mt_state / init_mt_pos), else the env keeps its start.  A reset
   after an unstable step sets init_state to -1 first (furniture.py:2895).  An index past the bank counts as None. */
int fe_set_init_states(fe_handle* h, const float* qpos_host, const float* qvel_host, int n_states);

/* Bits of `flags`.  A call ORs in the bits an env raised during it (the step kernels clear an env's bits when they set its controls
   and when they reset it); the field keeps them until the caller writes it. */
#define FE_FLAG_CONTACT_FULL 1 /* the contact capacity (fe_config.maxcon) was reached: the contacts past it were dropped */
#define FE_FLAG_NUMERIC 2      /* a NaN cost or gradient in a Newton solve, or a non-positive pivot in a part's 6x6 inertia or in the
                                  robot's mass or integration matrix */
#define FE_FLAG_NEWTON_PIVOT 4 /* a non-positive pivot in the Cholesky factor of a Newton solve's Hessian (replaced by a tiny one) */
#define FE_FLAG_DIVERGED 8     /* qpos or qvel NaN or beyond 1e6 after an mj_step: the episode is unstable (fe_env_step resets it) */

/* Columns of `stats`: counters of the env over the last call, zeroed at its start.  A constraint solve runs once per mj_step and per
   forward pass.  Cycles are clock64() / 16 of the env's warp; FE_STAT_KIN .. FE_STAT_WAIT_INTEGRATE are written by the env steps
   and fe_sim_step only. */
#define FE_STAT_PART_ITERS 0      /* Newton iterations of the per-part solver of free parts, max over the parts, summed over the solves */
#define FE_STAT_COUPLED 1         /* constraint solves whose coupled component holds a free part */
#define FE_STAT_NEWTON_SOLVES 2   /* Newton solves of the robot block or of the coupled component that had constraint rows */
#define FE_STAT_NEWTON_ITERS 3    /* Newton iterations of those solves, summed */
#define FE_STAT_KIN 4             /* cycles in kinematics and smooth dynamics */
#define FE_STAT_COLLIDE 5         /* cycles in collision detection */
#define FE_STAT_ASSEMBLE 6        /* cycles assembling the constraint rows */
#define FE_STAT_SOLVE 7           /* cycles in the constraint solve */
#define FE_STAT_INTEGRATE 8       /* cycles in integration */
#define FE_STAT_WAIT 9            /* cycles waiting at the block barriers ahead of the five phases above, all together */
#define FE_STAT_ROBOT_ONLY 10     /* constraint solves whose coupled component is the robot block alone (it touches something, no part is coupled) */
#define FE_STAT_SOLVE_MAX 11      /* cycles of the slowest constraint solve */
#define FE_STAT_WAIT_KIN 12       /* cycles waiting at the barrier ahead of kinematics */
#define FE_STAT_WAIT_COLLIDE 13   /* ... ahead of collision detection */
#define FE_STAT_WAIT_ASSEMBLE 14  /* ... ahead of the constraint rows */
#define FE_STAT_WAIT_SOLVE 15     /* ... ahead of the constraint solve */
#define FE_STAT_WAIT_INTEGRATE 16 /* ... ahead of integration */
/* cycles of a constraint solve whose coupled component fits the register solver (at most 32 dofs and 32 contacts): */
#define FE_STAT_SOLVE_PRE 17      /* finding the component: which parts are coupled, its dofs and its contacts */
#define FE_STAT_SOLVE_GROUPED 18  /* the per-part solver of the free parts outside it, and the robot's joint limits when the robot is outside it */
#define FE_STAT_SOLVE_COMP 19     /* the register solver of the component */
#define FE_STAT_RESERVED 20       /* never written */
/* cycles in the phases of the register solver of a component: */
#define FE_STAT_NEWTON_SETUP 21    /* set-up, once per solve */
#define FE_STAT_NEWTON_START 22    /* choosing the start: the smooth acceleration or the warm start */
#define FE_STAT_NEWTON_GRAD 23     /* per iteration: forces, J^T f, cost and gradient */
#define FE_STAT_NEWTON_HESSIAN 24  /* the Hessian rows */
#define FE_STAT_NEWTON_CHOL 25     /* Cholesky factor and solves */
#define FE_STAT_NEWTON_PRODUCTS 26 /* M s and J s along the search direction */
#define FE_STAT_NEWTON_LS 27       /* line search */
/* The shared-memory solver, which takes a component beyond 32 dofs or 32 contacts, adds its own phases to the same seven columns:
   set-up, choosing the start and the final forces (21); forces and J^T f (22); cost, gradient and stop test (23); the Hessian (24);
   the independent part blocks and, where the direction is not computed in registers, the Cholesky factor (25); the Newton
   direction (26); M s, J s and line search (27). */

/* ---- environment surface (FurnitureEnv / VecEnv) */
int fe_env_reset(fe_handle* h, const uint8_t* env_mask_dev /* NULL = all */, float* obs_dev, void* stream);
int fe_env_step(fe_handle* h, const float* actions_dev, float* obs_dev, float* reward_dev, uint8_t* done_dev, int32_t* info_dev,
                void* stream);
/* same step, results written by the kernel as rows of fe_packed_dim(h) floats: the send buffer of the observation all-gather over env
   shards (SURVEY.md 8e; the reference's counterpart is the pipe of util/subproc_vec_env.py:100-113 that carries (ob, reward, done, info)
   of every worker back to the caller).  A row is, in this order:
     obs           obs_dim floats, the row fe_env_step writes to obs
     reward, done  2 floats (done 0 or 1)
     info          FE_INFO_DIM = 6 floats holding the int32 bit patterns of the env's info row, so that they survive a float32 all-gather
                   exactly (read them through an int32 view)                                 -- with fe_set_packed_layout's info = 1
     dense_info    fe_dense_info_dim() floats, the step's row of field "dense_info"          -- with dense_info = 1
     terminal_obs  obs_dim floats, the row the step also writes to terminal_obs              -- with terminal_obs = 1
     step_info     6 floats: the step's row of field "reward_info" (NaN on a dense handle, which has no such row), then the 2 floats
                   it writes to "episode_info"                                              -- with fe_set_packed_step_info's step_info = 1
   The terminal slot and the last 2 floats of the step_info slot are valid where that step's done is 1 and are left untouched otherwise,
   exactly like terminal_obs and episode_info.  With the default layout the rows are [obs | reward | done], obs_dim + 2 floats, and
   nothing past them is written. */
int fe_env_step_packed(fe_handle* h, const float* actions_dev, float* packed_dev, int32_t* info_dev, void* stream);
/* What fe_env_step_packed writes after [obs | reward | done]: each flag 0 or 1, in effect from the next packed step.  Refused for a flag
   outside {0, 1}, for dense_info on a handle without the dense reward, and for a handle created without a scene blob. */
int fe_set_packed_layout(fe_handle* h, int info, int dense_info, int terminal_obs);
/* Whether fe_env_step_packed writes the step_info slot after the blocks of fe_set_packed_layout: 0 or 1, in effect from the next packed
   step.  Refused for a value outside {0, 1} and for a handle created without a scene blob. */
int fe_set_packed_step_info(fe_handle* h, int step_info);
/* floats per packed row under the handle's layout at its current obs_dim (it follows fe_set_obs_layout): obs_dim + 2 by default */
int fe_packed_dim(const fe_handle* h);
/* same call with host buffers: H2D of the actions and D2H of the results happen inside (pinned staging) */
int fe_env_step_host(fe_handle* h, const float* actions_host, float* obs_host, float* reward_host, uint8_t* done_host, int32_t* info_host);
/* FurnitureGym.set_max_episode_steps -> FurnitureEnv.set_max_episode_steps (furniture_gym.py:35-37, furniture.py:271-272):
   every env's field max_episode_steps and the handle's fe_config; takes effect from the next step */
int fe_set_max_episode_steps(fe_handle* h, int max_episode_steps);
/* Switch the handle to the dense reward; call before the first fe_env_reset.  The scene must carry a recipe, and dc->phase_ob must agree
 * with the scene (the one-hot phase is part of obs_dim).  Every env's row of field "dense_config" starts as dc (see fe_set_field).  fe_env_step then returns the dense reward / done / success, and field
 * "dense_info" holds (n_envs, fe_dense_info_dim()) float32 per step: phase, subtask, phase_bonus, ctrl_penalty, gripper_penalty,
 * move_other_part_penalty, drop_penalty, touch, drop_leg, table_moved, stable_grip_succ, skips (bit 0 to lift_leg, bit 1 to move_leg_fine). */
int fe_enable_dense_reward(fe_handle* h, const fe_dense_config* dc);
/* The observation flags of config/furniture.py (furniture.py:103-107, :215-252, :1344-1387), each 0 or 1; the defaults (1, 1, 1, 0) are the layout
 * of fe_create.  A row is [object_ob | subtask_ob | robot_ob | phase_ob], each entry present as its flag asks: object_ob holds 7 numbers
 * (pos, quat wxyz) per part, or with object_ob_all = 0 only those of the two parts of the env's current subtask, in part order (14 numbers,
 * zeros when no subtask is left); subtask_ob is [part1 + 1, part2 + 1] as float32.  The pair is the reference's _get_next_subtask
 * (furniture.py:2723-2736): the first weld in model order whose parts are not yet joined, recomputed after every connection and at the end
 * of every reset; with the dense reward, the recipe step's (leg, table) from each reset and from each move to the next subtask on, which the
 * observation shows from the following step (the observation of a step is taken before its reward, furniture_sawyer.py:66-84).  Field
 * "subtask_part" holds the pair.  Call before the first fe_env_reset or env step; it is refused after, and for a flag outside {0, 1}.
 * fe_obs_dim reports the new width, the obs buffer is reallocated (fe_obs_dev moves), and packed rows take the new width (fe_packed_dim). */
int fe_set_obs_layout(fe_handle* h, int robot_ob, int object_ob, int object_ob_all, int subtask_ob);
int fe_dense_info_dim(void);
/* device pointer of the internal obs buffer after the last step/reset: (n_envs, obs_dim) float32 */
const float* fe_obs_dev(const fe_handle* h);
/* What an episode left when it ended: the reference's FurnitureEnv.step returns the terminal observation with done (furniture.py:364-385),
 * while the env steps here reset a finished env in the same launch and return the next episode's first observation.  Every env step
 * (fe_env_step, fe_env_step_packed, fe_env_step_host, under every control type) writes, for each env whose step returns done = 1, the
 * observation row that step would have returned without the reset into terminal_obs (n_envs, obs_dim) float32, and its qpos / qvel into
 * terminal_qpos (n_envs, nq) / terminal_qvel (n_envs, nv) float32, before the auto-reset.  After an unstable step these hold the world of the
 * reset inside _do_simulation's except branch, which is what the reference's step returns (furniture.py:2889-2897).  A row is valid where
 * the last step's done is 1; the rows of the other envs, and every row after fe_env_reset, are left as they are.  The same arrays are the
 * read-only fields "terminal_obs", "terminal_qpos" and "terminal_qvel"; fe_set_obs_layout reallocates terminal_obs with obs (the pointer
 * moves).  A handle created without a scene blob has neither the fields nor the buffers: the accessors return NULL. */
const float* fe_terminal_obs_dev(const fe_handle* h);
const float* fe_terminal_qpos_dev(const fe_handle* h);
const float* fe_terminal_qvel_dev(const fe_handle* h);
/* The step's info dict of the reference (FurnitureEnv._compute_reward / _after_step, furniture.py:451-541), written by every env step
 * (fe_env_step, fe_env_step_packed, fe_env_step_host, under every control type):
 *   reward_info   (n_envs, 4) float32, on every step of a sparse-reward handle: success_reward, touch_reward, pick_reward, ctrl_penalty,
 *                 the terms the reward is made of (ctrl_penalty = -ctrl_penalty_coef * |a|^2, furniture.py:543-550).  On a step that is not
 *                 unstable ((success_reward + touch_reward) + pick_reward) + ctrl_penalty is the step's reward; on an unstable step the
 *                 reward adds the episode_unstable penalty.  A dense handle (fe_enable_dense_reward) has no such terms (they are
 *                 dense_info): its steps write no row, the field stays NaN and fe_reward_info_dev returns NULL.
 *   episode_info  (n_envs, 2) float32: episode_reward, episode_unstable of the episode the step ended -- the float32 sum of the episode's
 *                 rewards before the penalty, plus the penalty, and the penalty (-unstable_penalty_coef after an unstable step, else 0).
 *                 An unstable step resets the env inside the step first, as _do_simulation's except branch does (furniture.py:2889-2897),
 *                 so its episode reports that step's reward alone, with length 1, like the reference's.
 * A row of episode_info is valid where the last step's done is 1; the rows of the other envs are left as they are.  Rows no step has
 * written hold NaN.  The same arrays are the read-only fields "reward_info" and "episode_info"; a handle created without a scene blob has
 * neither the fields nor the buffers, and the accessors return NULL.  episode_time is a host clock and not part of the record. */
const float* fe_reward_info_dev(const fe_handle* h);
const float* fe_episode_info_dev(const fe_handle* h);

/* ---- test hook: the device _is_aligned on explicit site poses (float64), n independent cases */
int fe_is_aligned(fe_handle* h, int n, const double* p1, const double* m1, const double* p2, const double* m2, const double* angles /* (n,4) */,
                  const int32_t* nangles, const double* thr /* (n,4) */, uint8_t* aligned_host, double* target_quat_host /* (n,4) wxyz, NaN if unset */);

/* ---- test hook: the device reward machine on explicit poses.  Records [first[e], first[e] + count[e]) form episode e and are walked in
 * order by one thread; a record with reset != 0 starts the episode on the world it shows, at subtask reset - 1
 * (reset = 1 + the number of preassembled recipe steps).  Per record: site_pos (nsite,3), site_mat
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
 * velp 3, velr 3, q 7, qvel 7, Jx 21, Jr 21 (3 x 7 row-major), M 49.  Output: torques (7 doubles per record).
 * reset byte: 0 carries the controller on; 1 starts a new controller (nothing carried over); 2 calls Controller.reset() on the existing one, as
 * FurnitureEnv._reset does between episodes (the position controller keeps the orientation goal of its first policy step). */
int fe_ctl_eval(fe_handle* h, const fe_ctl_config* cc, int n_episodes, const int32_t* first, const int32_t* count, int n_records, const uint8_t* reset,
                const uint8_t* policy_step, const double* action, const double* readings, double* torques_host);

#ifdef __cplusplus
}
#endif
#endif
