// fe_dense_types.h -- data of the dense (phase-based) reward: the recipe block of fe_scene and the per-env state (see fe_dense.h)
#pragma once
#include <stdint.h>

#define FE_DENSE_MAXSUB 8
#define FE_DENSE_INFO 12 /* phase, subtask, phase_bonus, ctrl_penalty, gripper_penalty, move_other_part_penalty, drop_penalty, touch, drop_leg,
                            table_moved, stable_grip_succ, skips (bit 0: to lift_leg, bit 1: to move_leg_fine) */

// the assembly recipe (assets/recipes/<furniture>.yaml), resolved to ids by the host; part of fe_scene
typedef struct fe_dense_recipe {
  int32_t nsub, griptip_site, grip_site, pad_;
  double z_finedist;
  int32_t leg_part[FE_DENSE_MAXSUB], leg_site[FE_DENSE_MAXSUB], table_site[FE_DENSE_MAXSUB]; // recipe[i][0]; site_recipe[i][0], [1]
  int32_t gl_site[FE_DENSE_MAXSUB], gr_site[FE_DENSE_MAXSUB];                                 // "<leg>_ltgt_site<k>", "<leg>_rtgt_site<k>" claimed for subtask i
  int32_t n_allowed[FE_DENSE_MAXSUB], has_angle[FE_DENSE_MAXSUB], grip_init_len[FE_DENSE_MAXSUB]; // angles in the leg connector's name; site_recipe[i][2] given; 0 / 3 / 4
  double allowed_cos[FE_DENSE_MAXSUB][4], allowed_sin[FE_DENSE_MAXSUB][4];                    // cos / sin(angle / 180 * pi), host float64
  double angle_cos[FE_DENSE_MAXSUB], angle_sin[FE_DENSE_MAXSUB];
  double waypoint_z[FE_DENSE_MAXSUB], grip_init[FE_DENSE_MAXSUB][4];                          // waypoints[i][0][2]; grip_init_pos[i][0]
} fe_dense_recipe;

enum { FE_DP_INIT_EEF, FE_DP_ABOVE_LEG, FE_DP_EEF_LEG, FE_DP_GRASP, FE_DP_LIFT_Z, FE_DP_LIFT_XY, FE_DP_MOVE_POS, FE_DP_MOVE_UP, FE_DP_MOVE_FWD, FE_DP_PROJ_T, FE_DP_PROJ_L, FE_DP_N };
enum { FE_PH_INIT_EEF, FE_PH_ABOVE_LEG, FE_PH_LOWER_EEF, FE_PH_GRASP, FE_PH_LIFT, FE_PH_ALIGN, FE_PH_MOVE, FE_PH_FINE };

struct FeDenseState { // per env, in HBM; lane 0 reads and writes it once per step
  int32_t phase, subtask, dropped, table_moved, lifted, fine_aligned, success;
  int32_t diff_rew; // fe_dense_config.diff_rew of the env's row at the start of the episode
  double table_site0[3], leg0[3], lift_target[3], init_eef[3];
  double prev[FE_DP_N];
};

