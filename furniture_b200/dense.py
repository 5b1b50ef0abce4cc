"""Host side of the dense (phase-based) reward of FurnitureSawyerDenseRewardEnv (furniture/env/furniture_sawyer_dense.py).

The reward machine itself runs on the device (csrc/fe_dense.h); this module packs what it needs:
  * ``dense_config``      -> struct fe_dense_config: the coefficients of config/furniture_sawyer_dense.py:5-71 (defaults below)
  * ``pack_dense_recipe`` -> struct fe_dense_recipe: the assembly recipe (assets/recipes/<furniture>.yaml, kept in the composed scene as
                             ``meta["recipe_json"]``) resolved to site / part ids, with the grasp-target sites each subtask claims
                             (_update_reward_variables :202-207) and cos / sin of the recipe angles (transform_utils.rotate_vector :739-745)
"""
from __future__ import annotations

import ctypes as C

import numpy as np

i32, f64 = C.c_int32, C.c_double
MAXSUB = 8
INFO_KEYS = ["phase", "subtask", "phase_bonus", "ctrl_penalty", "gripper_penalty", "move_other_part_penalty", "drop_penalty", "touch", "drop_leg", "table_moved",
             "stable_grip_succ", "skips"]
PHASES = ["init_eef", "move_eef_above_leg", "lower_eef", "grasp_leg", "lift_leg", "align_leg", "move_leg", "move_leg_fine"]  # furniture_sawyer_dense.py:87-96

_COEFS = ["phase_bonus", "ctrl_penalty_coef", "eef_forward_dist_coef", "eef_up_dist_coef", "eef_rot_threshold", "gripper_penalty_coef",
          "move_other_part_penalty_coef", "drop_penalty_coef", "init_eef_pos_dist_coef", "move_eef_pos_dist_coef", "lower_eef_pos_dist_coef", "grasp_dist_coef",
          "lift_z_dist_coef", "lift_xy_dist_coef", "lift_z_pos_threshold", "lift_xy_pos_threshold", "align_pos_dist_coef", "align_rot_dist_coef",
          "align_pos_threshold", "align_rot_threshold", "move_pos_dist_coef", "move_rot_dist_coef", "move_pos_threshold", "move_rot_threshold",
          "move_fine_pos_exp_coef", "move_fine_pos_dist_coef", "move_fine_rot_dist_coef", "aligned_bonus_coef"]
_FLAGS = ["diff_rew", "early_termination", "phase_ob", "reset_robot_after_attach"]
# what each env of a dense handle may hold on its own (Engine.set_dense_options): everything but phase_ob, which sets the obs width
PER_ENV_KEYS = tuple(_COEFS) + ("diff_rew", "early_termination", "reset_robot_after_attach")

DENSE_DEFAULTS = dict(
    diff_rew=True, early_termination=False, phase_ob=False, reset_robot_after_attach=False,
    phase_bonus=5000.0, ctrl_penalty_coef=1e-3, eef_forward_dist_coef=2.0, eef_up_dist_coef=4.0, eef_rot_threshold=0.95, gripper_penalty_coef=1.0,
    move_other_part_penalty_coef=50.0, drop_penalty_coef=20.0, init_eef_pos_dist_coef=100.0, move_eef_pos_dist_coef=100.0, lower_eef_pos_dist_coef=1000.0,
    grasp_dist_coef=200.0, lift_z_dist_coef=500.0, lift_xy_dist_coef=250.0, lift_z_pos_threshold=0.02, lift_xy_pos_threshold=0.05, align_pos_dist_coef=100.0,
    align_rot_dist_coef=50.0, align_pos_threshold=0.2, align_rot_threshold=0.85, move_pos_dist_coef=300.0, move_rot_dist_coef=50.0, move_pos_threshold=0.06,
    move_rot_threshold=0.85, move_fine_pos_exp_coef=-25.0, move_fine_pos_dist_coef=500.0, move_fine_rot_dist_coef=200.0, aligned_bonus_coef=10.0)

# what else config/furniture_sawyer_dense.py:5-14 changes with respect to the base env
DENSE_ENV_DEFAULTS = dict(max_episode_steps=150, furniture_name="table_lack_0825", auto_align=False, alignment_pos_dist=0.02, alignment_rot_dist_up=0.99,
                          alignment_rot_dist_forward=0.99, alignment_project_dist=0.0)


class FeDenseConfig(C.Structure):
    _fields_ = [("struct_bytes", i32)] + [(k, i32) for k in _FLAGS] + [("pad_", i32)] + [(k, f64) for k in _COEFS]


class FeDenseRecipe(C.Structure):
    _fields_ = [
        ("nsub", i32), ("griptip_site", i32), ("grip_site", i32), ("pad_", i32), ("z_finedist", f64),
        ("leg_part", i32 * MAXSUB), ("leg_site", i32 * MAXSUB), ("table_site", i32 * MAXSUB), ("gl_site", i32 * MAXSUB), ("gr_site", i32 * MAXSUB),
        ("n_allowed", i32 * MAXSUB), ("has_angle", i32 * MAXSUB), ("grip_init_len", i32 * MAXSUB),
        ("allowed_cos", (f64 * 4) * MAXSUB), ("allowed_sin", (f64 * 4) * MAXSUB), ("angle_cos", f64 * MAXSUB), ("angle_sin", f64 * MAXSUB),
        ("waypoint_z", f64 * MAXSUB), ("grip_init", (f64 * 4) * MAXSUB),
    ]


def dense_config(**kw) -> FeDenseConfig:
    vals = dict(DENSE_DEFAULTS)
    for k, v in kw.items():
        if k not in vals:
            raise KeyError(k)
        vals[k] = v
    c = FeDenseConfig()
    c.struct_bytes = C.sizeof(FeDenseConfig)
    for k in _FLAGS:
        setattr(c, k, int(bool(vals[k])))
    for k in _COEFS:
        setattr(c, k, float(vals[k]))
    return c


def pack_dense_recipe(recipe: dict, site_id, part_id, griptip_site: int, grip_site: int) -> FeDenseRecipe:
    """`site_id(name)` / `part_id(name)` return the index the device will use, or None if the scene has no such site."""
    rc = FeDenseRecipe()
    n = len(recipe["recipe"])
    if n > MAXSUB:
        raise ValueError("recipe has %d subtasks, the device table holds %d" % (n, MAXSUB))
    rc.nsub, rc.griptip_site, rc.grip_site = n, griptip_site, grip_site
    rc.z_finedist = float(recipe["z_finedist"])
    grip_init = recipe.get("grip_init_pos")
    used = set()
    for s in range(n):
        leg = recipe["recipe"][s][0]
        sr = recipe["site_recipe"][s]
        rc.leg_part[s] = part_id(leg)
        for field, name in (("leg_site", sr[0]), ("table_site", sr[1])):
            sid = site_id(name)
            if sid is None:
                raise KeyError("recipe names site %r, which the scene does not have" % name)
            getattr(rc, field)[s] = sid
        # the first pair of grasp-target sites of the leg not yet claimed by an earlier subtask; the last pair looked at if all are taken
        for k in range(n):
            pair = ("%s_ltgt_site%d" % (leg, k), "%s_rtgt_site%d" % (leg, k))
            if pair[0] not in used and pair[1] not in used:
                used.update(pair)
                break
        ids = [site_id(p) for p in pair]
        if None in ids:
            raise KeyError("the dense reward needs the grasp-target sites %s / %s" % pair)
        rc.gl_site[s], rc.gr_site[s] = ids
        allowed = [float(x) for x in sr[0].split(",")[1:-1] if x]
        rc.n_allowed[s] = len(allowed)
        for k, a in enumerate(allowed):
            r = a / 180 * np.pi
            rc.allowed_cos[s][k], rc.allowed_sin[s][k] = float(np.cos(r)), float(np.sin(r))
        if len(sr) == 3:
            r = sr[2] / 180 * np.pi
            rc.has_angle[s], rc.angle_cos[s], rc.angle_sin[s] = 1, float(np.cos(r)), float(np.sin(r))
        rc.waypoint_z[s] = float(recipe["waypoints"][s][0][2])
        g = grip_init[s][0] if (grip_init is not None and grip_init[s] is not None) else None
        if g is not None:
            rc.grip_init_len[s] = len(g)
            for k, v in enumerate(g):
                rc.grip_init[s][k] = float(v)
    return rc
