"""ctypes binding of the C-ABI in include/furniture_b200.h plus the env-level scene table (struct fe_scene).

``Engine`` mirrors the part of ``mujoco_py.MjSim`` the reference touches (forward/step, named data views,
get/set state) for a whole batch of envs, and the batched FurnitureEnv entry points (reset/step).
The CUDA library is mandatory: if ``libfurniture_b200.so`` is missing or no CUDA device is present the constructor
raises -- there is no CPU fallback.  (Tests may pass ``lib_path`` to load the lane-emulated harness build.)
"""
from __future__ import annotations

import ctypes as C
import math
import os

import numpy as np

from . import mjcf
from .dense import PER_ENV_KEYS as DENSE_KEYS, FeDenseConfig, FeDenseRecipe, dense_config, pack_dense_recipe
from .engine_model import MAXEQ, MAXPART, MAXRDOF, MAXSITE, MAXU, EngineModel

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, "libfurniture_b200.so")
MAXCONN = 48
SCENE_MAGIC = 0x46455344
INFO_DIM = 6
# the step's info dict of the reference (FurnitureEnv._compute_reward / _after_step, furniture.py:451-541): fields "reward_info" and
# "episode_info" (include/furniture_b200.h) in this column order
REWARD_INFO_KEYS = ("success_reward", "touch_reward", "pick_reward", "ctrl_penalty")
EPISODE_INFO_KEYS = ("episode_reward", "episode_unstable")
# bits of the `flags` field and columns of the `stats` field: FE_FLAG_* / FE_STAT_* of include/furniture_b200.h, which says what each means
FLAG_CONTACT_FULL, FLAG_NUMERIC, FLAG_NEWTON_PIVOT, FLAG_DIVERGED = 1, 2, 4, 8
STAT_PART_ITERS, STAT_COUPLED, STAT_NEWTON_SOLVES, STAT_NEWTON_ITERS = 0, 1, 2, 3
STAT_KIN, STAT_COLLIDE, STAT_ASSEMBLE, STAT_SOLVE, STAT_INTEGRATE, STAT_WAIT, STAT_ROBOT_ONLY, STAT_SOLVE_MAX = 4, 5, 6, 7, 8, 9, 10, 11
STAT_WAIT_KIN, STAT_WAIT_COLLIDE, STAT_WAIT_ASSEMBLE, STAT_WAIT_SOLVE, STAT_WAIT_INTEGRATE = 12, 13, 14, 15, 16
STAT_SOLVE_PRE, STAT_SOLVE_GROUPED, STAT_SOLVE_COMP, STAT_RESERVED = 17, 18, 19, 20
STAT_NEWTON_SETUP, STAT_NEWTON_START, STAT_NEWTON_GRAD, STAT_NEWTON_HESSIAN, STAT_NEWTON_CHOL, STAT_NEWTON_PRODUCTS, STAT_NEWTON_LS = 21, 22, 23, 24, 25, 26, 27
i32, f32, f64 = C.c_int32, C.c_float, C.c_double
# the observation flags of config/furniture.py:228-258 and their defaults; other values go to fe_set_obs_layout
OBS_DEFAULTS = dict(robot_ob=True, object_ob=True, object_ob_all=True, subtask_ob=False)
# the per-env options of config/furniture.py by their key names -> (per-env field, column, converter from the caller's value to the field's,
# or None); Engine._set_options writes them.  The reset options (:116-127, :169-174, :307-312), the sim options (:71-73, :304-306) and the
# task options (:95-100, :163-168, :177-194, :203-226, :291-295).
OPTIONS = dict(
    fix_init=("fix_init", 0, None), fix_init_parts=("fix_init_parts", 0, lambda eng, parts: eng.part_mask(parts)),
    reset_robot_after_attach=("reset_robot_after_attach", 0, None), assembled=("assembled", 0, None),
    control_freq=("substeps", 0, lambda eng, freq: eng.substeps(freq)), no_collision=("no_collision", 0, lambda eng, v: np.asarray(v, dtype=bool)),
    alignment_pos_dist=("alignment", 0, None), alignment_rot_dist_up=("alignment", 1, None), alignment_rot_dist_forward=("alignment", 2, None),
    alignment_project_dist=("alignment", 3, None), auto_align=("auto_align", 0, None), furn_xyz_rand=("placement_rand", 0, None),
    furn_rot_rand=("placement_rand", 1, None), agent_xyz_rand=("placement_rand", 2, None), success_reward=("reward_coef", 0, None),
    touch_reward=("reward_coef", 1, None), pick_reward=("reward_coef", 2, None), ctrl_penalty_coef=("reward_coef", 3, None),
    unstable_penalty_coef=("reward_coef", 4, None), max_episode_steps=("max_episode_steps", 0, None))
# the dense reward's per-env options (config/furniture_sawyer_dense.py:23-70): members of each env's fe_dense_config row, field dense_config;
# Engine.set_dense_options writes them through the same path.  Two keys share a name with an OPTIONS key, hence a table of their own.
DENSE_OPTIONS = {k: ("dense_config", k, None) for k in DENSE_KEYS}


class FeConfig(C.Structure):
    _fields_ = [
        ("struct_bytes", i32), ("maxcon", i32), ("newton_iters", i32), ("ls_iters", i32), ("tolerance", f32), ("nsub", i32),
        ("max_episode_steps", i32), ("discrete_grip", i32), ("rescale_actions", i32), ("auto_align", i32),
        ("alignment_pos_dist", f64), ("alignment_rot_dist_up", f64), ("alignment_rot_dist_forward", f64), ("alignment_project_dist", f64),
        ("ctrl_penalty_coef", f32), ("unstable_penalty_coef", f32), ("success_reward", f32), ("touch_reward", f32), ("pick_reward", f32),
        ("furn_xyz_rand", f32), ("furn_rot_rand", f32), ("agent_xyz_rand", f32), ("furn_size_rand", f32), ("seed", C.c_uint64),
    ]


# the task options (set_task_options): the per-env options that start from the FeConfig member of the same name
TASK_OPTIONS = tuple(k for k in OPTIONS if hasattr(FeConfig, k))


class FeScene(C.Structure):
    _fields_ = [
        ("magic", i32), ("struct_bytes", i32),
        ("obs_dim", i32), ("act_dim", i32), ("robot_ob_dim", i32), ("nconn", i32), ("npart", i32), ("narm", i32), ("ngrip", i32), ("narms", i32),
        ("act_src", i32 * MAXU), ("act_sign", f32 * MAXU), ("grip_action_index", i32), ("connect_action_index", i32),
        ("conn_site", i32 * MAXCONN), ("conn_part", i32 * MAXCONN), ("conn_a", i32 * MAXCONN), ("conn_b", i32 * MAXCONN), ("conn_nangles", i32 * MAXCONN),
        ("conn_cos", (f64 * 4) * MAXCONN), ("conn_sin", (f64 * 4) * MAXCONN),
        ("eq_part1", i32 * MAXEQ), ("eq_part2", i32 * MAXEQ),
        ("part_site_start", i32 * (MAXPART + 1)), ("part_sites", i32 * MAXSITE),
        ("eef_site", i32 * 2), ("hand_link", i32 * 2), ("hand_quat", (f32 * 4) * 2),
        ("arm_dof", i32 * MAXRDOF), ("grip_dof", i32 * 8),
        ("robot_init_qpos", f32 * MAXRDOF),
        ("part_init_pos", (f32 * 3) * MAXPART), ("part_init_quat", (f32 * 4) * MAXPART), ("part_radius", f32 * MAXPART),
        ("phase_ob", i32), ("obs_layout", i32), ("dense", FeDenseRecipe),
    ]


def default_config(**kw):
    """Reference defaults: config/furniture.py:16-312 (control_freq 10 => 50 mj_steps per env step)."""
    c = FeConfig()
    c.struct_bytes = C.sizeof(FeConfig)
    c.maxcon, c.newton_iters, c.ls_iters, c.tolerance = 0, 30, 20, 1e-6  # maxcon 0: sized from the model (auto_maxcon)
    c.nsub, c.max_episode_steps = 50, 2000
    c.discrete_grip, c.rescale_actions, c.auto_align = 1, 1, 1
    c.alignment_pos_dist, c.alignment_rot_dist_up, c.alignment_rot_dist_forward, c.alignment_project_dist = 0.1, 0.9, 0.9, 0.3
    c.ctrl_penalty_coef, c.unstable_penalty_coef, c.success_reward, c.touch_reward, c.pick_reward = 1e-3, 100, 100, 10, 100
    c.furn_xyz_rand, c.furn_rot_rand, c.agent_xyz_rand, c.furn_size_rand = 0.02, 3, 0.001, 0.0
    c.seed = 123
    for k, v in kw.items():
        if not hasattr(c, k):
            raise KeyError(k)
        setattr(c, k, v)
    return c


def substep_count(control_freq, timestep):
    """mj_steps of one env step at `control_freq` (a positive number, or an array of them): the bound of _do_simulation's loop,
    int((1.0 / control_freq) / model.opt.timestep) (furniture.py:2855, :2878), in float64 with the model's float64 timestep as MuJoCo
    holds it (a float32 timestep would give 49 at 10 Hz).  A frequency whose count is 0 (above 1 / timestep) is a ValueError."""
    cf = np.asarray(control_freq, dtype=np.float64)
    if not np.all(np.isfinite(cf)) or np.any(cf <= 0):
        raise ValueError("control_freq must be a positive number, got %r" % (control_freq,))
    dt = float(timestep)
    n = np.array([int((1.0 / float(f)) / dt) for f in cf.ravel()], dtype=np.int64).reshape(cf.shape)
    if np.any(n < 1):
        raise ValueError("control_freq %r runs no mj_step per env step (timestep %g s: at most %g Hz)" % (control_freq, dt, 1.0 / dt))
    return n


def auto_maxcon(em: EngineModel) -> int:
    """Contact capacity per env when the config leaves it open.  The reference runs with nconmax=5000 (base.xml:5), i.e.
    never full; the engine keeps contacts in the env's shared-memory slice, so capacity is sized from the scene: four
    contacts per colliding part geom (a box resting on a face) plus 16 for the robot, at least 44, at most 128.  An env
    that still overflows raises FLAG_CONTACT_FULL in its `flags` field (never silently dropped)."""
    fm = em.fm
    part_geoms = sum(1 for g in range(fm.ngeom) if (fm.geom_tag[g] >> 8) & 0x3FFFFF)
    return int(min(128, max(44, 4 * part_geoms + 16)))


def build_scene(m: mjcf.Model, em: EngineModel, phase_ob: bool = False) -> FeScene:
    """Integer tables for the connect logic, pre-compiled from the site names (SURVEY.md a6), the obs layout and the
    reset placements; the assembly recipe of the dense reward when the furniture has one.  `phase_ob` appends the dense reward's
    8-way one-hot phase to the observation (furniture_sawyer_dense.py:100-117)."""
    meta = m.meta
    sc = FeScene()
    sc.magic, sc.struct_bytes = SCENE_MAGIC, C.sizeof(FeScene)
    parts = em.part_names
    npart = len(parts)
    narm, ngrip = len(meta.get("robot_joints", [])), len(meta.get("gripper_joints", []))
    sc.npart, sc.narm, sc.ngrip = npart, narm, ngrip
    has_robot = narm > 0
    narms = (2 if meta.get("eef_site2") else 1) if has_robot else 0
    sc.narms = narms
    # per arm: qpos 7, qvel 7, gripper 2, eef pos 3, quat 4, velp 3, velr 3 (furniture_sawyer.py:40, furniture_baxter.py:36-42)
    sc.robot_ob_dim = narms * (2 * (narm // narms) + ngrip // narms + 3 + 4 + 3 + 3) if has_robot else 0
    sc.obs_dim = 7 * npart + sc.robot_ob_dim
    sc.act_dim = (narm + narms + 1) if has_robot else 1  # arm joints, one gripper action per arm, connect
    sc.eef_site[0] = sc.eef_site[1] = -1
    sc.hand_link[0] = sc.hand_link[1] = -1
    if has_robot:
        jdof = lambda name: int(m.jnt_dofadr[m.names["jnt"].index(name)])
        for i, jn in enumerate(meta["robot_joints"]):
            sc.arm_dof[i] = jdof(jn)
        for i, jn in enumerate(meta["gripper_joints"]):
            sc.grip_dof[i] = jdof(jn)
        # _setup_action (furniture.py:3332-3367): arm actions straight through; every gripper takes one action, fanned out over its
        # two actuators as [g, -g] in actuator order (two_finger_gripper.py:67-72)
        assert m.nu == narm + ngrip
        seen = {}
        for u in range(m.nu):
            jn = m.names["jnt"][int(m.actuator_jntid[u])]
            if jn in meta["robot_joints"]:
                sc.act_src[u], sc.act_sign[u] = meta["robot_joints"].index(jn), 1.0
            else:
                g = meta["gripper_joints"].index(jn) // (ngrip // narms)  # which gripper: right first, then left
                sc.act_src[u], sc.act_sign[u] = narm + g, (1.0 if seen.get(g, 0) == 0 else -1.0)
                seen[g] = seen.get(g, 0) + 1
        # FurnitureSawyerEnv._step discretises its gripper action (furniture_sawyer.py:73-74); FurnitureBaxterEnv does not
        sc.grip_action_index = narm if narms == 1 else -1
        sc.connect_action_index = narm + narms
        init = np.concatenate([meta["robot_init_qpos"], meta["gripper_init_qpos"]])
        for d, v in enumerate(init):
            sc.robot_init_qpos[d] = v
        kin = mjcf.kinematics_np(m, m.qpos0)
        for arm, (sk, hk) in enumerate((("eef_site", "hand_body"), ("eef_site2", "hand_body2"))[:narms]):
            sc.eef_site[arm] = m.names["site"].index(meta[sk])
            hb = m.names["body"].index(meta[hk])
            hl = em.weld_link(hb)
            lb = em.link_body[hl]
            sc.hand_link[arm] = hl
            sc.hand_quat[arm][:] = list(mjcf.q_norm(mjcf.q_mul(mjcf.q_conj(kin["xquat"][lb]), kin["xquat"][hb])))
    else:
        sc.grip_action_index, sc.connect_action_index = 0, 0
    # connector sites (name contains "conn_site"), model site-id order
    names = {}
    conn = [s for s in range(m.nsite) if "conn_site" in m.names["site"][s]]
    assert len(conn) <= MAXCONN
    sc.nconn = len(conn)
    for i, s in enumerate(conn):
        nm = m.names["site"][s]
        pair = nm.split(",")[0].split("-")
        assert len(pair) == 2, nm
        a, b = (names.setdefault(x, len(names)) for x in pair)
        angles = [float(x) for x in nm.split(",")[1:-1] if x]
        assert len(angles) <= 4
        sc.conn_site[i], sc.conn_a[i], sc.conn_b[i], sc.conn_nangles[i] = s, a, b, len(angles)
        sc.conn_part[i] = parts.index(m.names["body"][m.site_bodyid[s]])
        for k, ang in enumerate(angles):
            r = ang / 180 * np.pi  # transform_utils.py:743
            sc.conn_cos[i][k], sc.conn_sin[i][k] = float(np.cos(r)), float(np.sin(r))
    for e in range(m.neq):
        sc.eq_part1[e] = parts.index(m.names["body"][m.eq_obj1id[e]])
        sc.eq_part2[e] = parts.index(m.names["body"][m.eq_obj2id[e]])
    k = 0
    for p, name in enumerate(parts):
        sc.part_site_start[p] = k
        b = m.names["body"].index(name)
        for s in range(m.nsite):
            if m.site_bodyid[s] == b:
                sc.part_sites[k] = s
                k += 1
        q = meta.get("part_init_qpos", {}).get(name)
        if q is None:
            q = np.concatenate([m.body_pos[b], m.body_quat[b]])
        sc.part_init_pos[p][:] = list(q[:3])
        sc.part_init_quat[p][:] = list(q[3:7])
        sc.part_radius[p] = meta.get("part_radius", {}).get(name, 0.0)
    sc.part_site_start[npart] = k
    if meta.get("recipe_json") and narms == 1:
        import json

        sites = m.names["site"]
        sid = lambda name: sites.index(name) if name in sites else None
        try:
            sc.dense = pack_dense_recipe(json.loads(meta["recipe_json"]), sid, parts.index, sid("griptip_site"), sid("grip_site"))
        except (KeyError, ValueError, TypeError):  # a recipe the scene cannot serve (no grasp-target sites ...): dense reward unavailable, nsub stays 0
            sc.dense = FeDenseRecipe()
    if phase_ob:
        sc.phase_ob = 1
        sc.obs_dim += 8
    return sc


def obs_columns(scene, robot_skip=0, robot_ob=True, object_ob=True, object_ob_all=True, subtask_ob=False):
    """Where each entry of the obs dict sits in a device row, in the reference's key order: object_ob, subtask_ob (FurnitureEnv._get_obs,
    furniture.py:1344-1387), robot_ob (the agent's, furniture_sawyer.py:103-155, furniture_baxter.py:98-155), phase_ob (the dense env's).
    An OrderedDict of key -> slice, or of index array for the robot_ob of two arms that drop their `robot_skip` joint columns each (the IK and
    controller control types, furniture_baxter.py:137-160)."""
    from collections import OrderedDict

    cols, o = OrderedDict(), 0
    if object_ob:
        w = 7 * scene.npart if object_ob_all else 14
        cols["object_ob"], o = slice(o, o + w), o + w
    if subtask_ob:
        cols["subtask_ob"], o = slice(o, o + 2), o + 2
    if robot_ob:
        narms, dim = max(1, int(scene.narms)), int(scene.robot_ob_dim)
        per = dim // narms
        if robot_skip and narms > 1:
            cols["robot_ob"] = np.array([o + a * per + k for a in range(narms) for k in range(robot_skip, per)])
        else:
            cols["robot_ob"] = slice(o + robot_skip, o + dim)
        o += dim
    if scene.phase_ob:
        cols["phase_ob"], o = slice(o, o + 8), o + 8
    return cols


def packed_columns(obs_dim, info=False, dense_info=False, terminal_obs=False, step_info=False):
    """Where each block of a packed row of fe_env_step_packed sits (include/furniture_b200.h): an OrderedDict name -> slice of the row, in
    its order obs, reward, done, then info (INFO_DIM int32 bit patterns), dense_info (DENSE_INFO_DIM floats), terminal_obs (obs_dim
    floats), reward_info (the 4 REWARD_INFO_KEYS, NaN on a dense handle) and episode_info (the 2 EPISODE_INFO_KEYS, valid where done) where
    the layout has them; step_info gives the last two together.  The end of the last slice is the row's stride.  The step kernel fills the blocks of a handle's
    layout; ShardedFurnitureEnv fills the same blocks on the host for a shard without that kernel."""
    from collections import OrderedDict

    from .dense import INFO_KEYS as DENSE_INFO_KEYS

    blocks = [("obs", obs_dim, True), ("reward", 1, True), ("done", 1, True), ("info", INFO_DIM, info),
              ("dense_info", len(DENSE_INFO_KEYS), dense_info), ("terminal_obs", obs_dim, terminal_obs),
              ("reward_info", len(REWARD_INFO_KEYS), step_info), ("episode_info", len(EPISODE_INFO_KEYS), step_info)]
    cols, o = OrderedDict(), 0
    for name, w, present in blocks:
        if present:
            cols[name], o = slice(o, o + w), o + w
    return cols


class Engine:
    def __init__(self, model: mjcf.Model, n_envs: int, device: int = 0, config: FeConfig | None = None, lib_path: str | None = None,
                 dense: FeDenseConfig | None = None, ik=None, controller=None, obs_layout=None, fix_init=False, fix_init_parts=None,
                 reset_robot_after_attach=None, assembled=False):
        """`fix_init`, `fix_init_parts`, `reset_robot_after_attach`, `assembled`: the keys of config/furniture.py:116-127, :169-174, :307-312
        for every env of the handle (set_reset_options changes them per env).  In a dense handle the dense reward's reset_robot_after_attach decides (None: follow it)."""
        path = lib_path or DEFAULT_LIB
        if not os.path.exists(path):
            raise RuntimeError(
                "furniture_b200: CUDA extension %s not built (run `python -c 'import __graft_entry__ as g; g.build()'`); there is no CPU fallback" % path
            )
        L = C.CDLL(path)
        self.L = L
        L.fe_last_error.restype = C.c_char_p
        L.fe_last_error.argtypes = [C.c_void_p]
        L.fe_field_dtype.restype = C.c_char_p
        L.fe_field_dtype.argtypes = [C.c_void_p, C.c_char_p]
        for f in ("fe_model_sizeof", "fe_scene_sizeof", "fe_config_sizeof"):
            getattr(L, f).restype = C.c_size_t
        for f in ("fe_obs_dev", "fe_terminal_obs_dev", "fe_terminal_qpos_dev", "fe_terminal_qvel_dev", "fe_reward_info_dev", "fe_episode_info_dev"):
            getattr(L, f).restype = C.c_void_p
            getattr(L, f).argtypes = [C.c_void_p]
        self.is_cuda = bool(L.fe_is_cuda())
        if lib_path is None and not self.is_cuda:
            raise RuntimeError("furniture_b200: default library is not a CUDA build")
        self.model = model
        self.em = EngineModel(model)
        self.scene = build_scene(model, self.em, phase_ob=bool(dense is not None and dense.phase_ob))
        self.cfg = config or default_config()
        if self.cfg.maxcon <= 0:
            self.cfg.maxcon = auto_maxcon(self.em)
        for fn, cls in (("fe_model_sizeof", type(self.em.fm)), ("fe_scene_sizeof", FeScene), ("fe_config_sizeof", FeConfig)):
            if getattr(L, fn)() != C.sizeof(cls):
                raise RuntimeError("furniture_b200: %s = %d but python layout has %d bytes" % (fn, getattr(L, fn)(), C.sizeof(cls)))
        self.h = C.c_void_p()
        rc = L.fe_create(C.byref(self.em.fm), C.c_size_t(C.sizeof(self.em.fm)), C.byref(self.scene), C.c_size_t(C.sizeof(self.scene)), C.byref(self.cfg),
                         int(n_envs), int(device), C.byref(self.h))  # (fe_create_from_file does the same from a compiled/*.feb scene file)
        if rc != 0:
            raise RuntimeError("fe_create failed (%d): %s" % (rc, L.fe_last_error(None).decode()))
        self.N = int(n_envs)
        self.obs_dim, self.act_dim = self.scene.obs_dim, self.scene.act_dim
        for f in ("fe_env_reset", "fe_env_step"):
            getattr(L, f).argtypes = None
        self.ik = ik
        if ik is not None:  # control_type="ik" (furniture_b200/ik.py: FeIkConfig): actions become (move 3, rotate 3, gripper, connect)
            self._chk(L.fe_enable_ik(self.h, C.byref(ik)))
            self.act_dim = int(L.fe_action_dim(self.h))
        self.controller = controller
        if controller is not None:  # one of the NEW_CONTROLLERS (furniture_b200/controllers.py: FeCtlConfig) on the torque-actuated robot
            self._chk(L.fe_enable_controller(self.h, C.byref(controller)))
            self.act_dim = int(L.fe_action_dim(self.h))
        self.obs_flags = dict(OBS_DEFAULTS)
        self.packed_flags = dict(info=False, dense_info=False, terminal_obs=False, step_info=False)  # set_packed_layout, set_packed_step_info
        if obs_layout is not None and {**OBS_DEFAULTS, **obs_layout} != OBS_DEFAULTS:  # `obs_layout`: overrides of OBS_DEFAULTS
            self.set_obs_layout(**obs_layout)
        self._bank, self._n_pick = [], 0  # host copy of the bank of recorded starts; its first _n_pick entries are the load_init_states list
        self.dense = dense
        if dense is not None:  # FurnitureSawyerDenseRewardEnv: the phase machine replaces the sparse reward inside fe_env_step
            self._chk(L.fe_enable_dense_reward(self.h, C.byref(dense)))
        # _load_model (furniture.py:2013-2021): init_pos / init_quat start as the XML's *_initpos numerics, or None when it lists none
        xml = mjcf.xml_init_poses(model.meta)
        self._xml_listed = set(xml or ())
        if xml is not None and self._xml_listed == set(self.em.part_names):
            self.set("fix_pose", np.concatenate([xml[n] for n in self.em.part_names])[None, :])
            self.set("fix_have", 1)
        rra = reset_robot_after_attach
        if dense is not None:  # fe_enable_dense_reward has set it from the dense reward's
            if rra is not None and bool(rra) != bool(dense.reset_robot_after_attach):
                raise ValueError("reset_robot_after_attach=%r disagrees with the dense reward's %r, which drives the phase machine and the arm"
                                 % (rra, bool(dense.reset_robot_after_attach)))
            rra = None
        if fix_init or fix_init_parts or rra or assembled:
            self.set_reset_options(fix_init=fix_init, fix_init_parts=fix_init_parts, reset_robot_after_attach=rra, assembled=assembled or None)

    @staticmethod
    def _part_names(parts):
        return [n for n in (parts.split(",") if isinstance(parts, str) else list(parts or ())) if n]

    def part_mask(self, parts):
        """fix_init_parts (config/furniture.py:122-127: a set of part names, or the comma string str2set reads) -> bit mask over the parts in
        XML order; an unknown name is a ValueError"""
        names = self._part_names(parts)
        unknown = sorted(set(names) - set(self.em.part_names))
        if unknown:
            raise ValueError("fix_init_parts names %s, which %s does not have (parts: %s)" % (unknown, self.model.meta.get("furniture"), list(self.em.part_names)))
        return sum(1 << self.em.part_names.index(n) for n in set(names))

    def set_reset_options(self, fix_init=None, fix_init_parts=None, reset_robot_after_attach=None, envs=None, assembled=None):
        """fix_init (the furniture starts every episode where the env's first random placement, or the XML, put it: furniture.py:1519-1532),
        fix_init_parts (only those parts do, the sampler places the others around them: :1389-1404), reset_robot_after_attach (the arm goes
        back to its start pose after every connection: :916-924) and assembled (every weld on, the parts left at the model's qpos0 -- the
        furniture as assembled -- in one group: :1501-1532), for the envs in `envs` (default: all); None leaves an option as it is.
        They act from the env's next reset or connection on, inside the kernels."""
        if assembled is not None and self.model.meta.get("agent") == "Cursor":
            raise ValueError("assembled is built for the robot envs; the Cursor env's reset is host logic (cursor_env.FurnitureCursorEnvB200)")
        partial = self._xml_listed and self._xml_listed != set(self.em.part_names)
        if partial and (np.any(fix_init) or set(self._part_names(fix_init_parts)) - self._xml_listed):  # init_pos[body]: the reference's KeyError
            raise ValueError("the XML of %s lists init poses for some parts only: fix_init, and fix_init_parts beyond %s, are undefined there"
                             % (self.model.meta.get("furniture"), sorted(self._xml_listed)))
        self._set_options(envs, dict(fix_init=fix_init, fix_init_parts=fix_init_parts, reset_robot_after_attach=reset_robot_after_attach,
                                     assembled=assembled))

    def substeps(self, control_freq):
        """substep_count at this model's timestep"""
        return substep_count(control_freq, self.model.opt_timestep)

    def set_sim_options(self, control_freq=None, no_collision=None, envs=None):
        """control_freq (config/furniture.py: mj_steps per env step, see substeps) and no_collision (the agent's contype = conaffinity = 0,
        furniture.py:1962-1965) for the envs in `envs` (default: all), each a scalar or one value per env of `envs`; None leaves an option as
        it is.  A new control_freq takes effect from the env's next step; no_collision changes the env's masks at once (back to the
        model's compiled masks when it turns off)."""
        if self.model.meta.get("agent") == "Cursor":
            raise ValueError("the Cursor env takes its own control_freq (cursor_env.FurnitureCursorEnvB200); control_freq and no_collision "
                             "are options of the robot envs")
        self._set_options(envs, dict(control_freq=control_freq, no_collision=no_collision))

    def set_task_options(self, envs=None, **values):
        """the task options of config/furniture.py for the envs in `envs` (default: all), each a scalar or one value per env of `envs`, by the
        reference's key names (TASK_OPTIONS): the alignment thresholds and auto_align, from the env's next step; furn_xyz_rand, furn_rot_rand
        and agent_xyz_rand, from its next reset (agent_xyz_rand also from its next connection under reset_robot_after_attach); success_reward,
        touch_reward, pick_reward, ctrl_penalty_coef and unstable_penalty_coef, from its next step; max_episode_steps at once.  A dense handle
        takes unstable_penalty_coef only among the coefficients: its phase machine replaces the other terms."""
        if self.model.meta.get("agent") == "Cursor":
            raise ValueError("the Cursor env's reward and connection logic is host code (cursor_env.FurnitureCursorEnvB200); the task options "
                             "are options of the robot envs")
        unknown = sorted(set(values) - set(TASK_OPTIONS))
        if unknown:
            raise ValueError("unknown task options %s (known: %s)" % (unknown, sorted(TASK_OPTIONS)))
        self._set_options(envs, values)

    def set_dense_options(self, envs=None, **values):
        """the dense reward's coefficients, thresholds (config/furniture_sawyer_dense.py:23-70, ctrl_penalty_coef included), diff_rew,
        early_termination and reset_robot_after_attach for the envs in `envs` (default: all), each a scalar or one value per env of
        `envs`, so that one batch can run a sweep or a curriculum over them.  They act from the env's next step; diff_rew from its next
        reset, since an episode's shaped terms difference against what they kept in its mode; reset_robot_after_attach, which the arm follows
        too, from its next connection.  phase_ob sets the obs width and stays the handle's."""
        if self.model.meta.get("agent") == "Cursor":
            raise ValueError("the Cursor env's reward is host code (cursor_env.FurnitureCursorEnvB200); it has no dense reward")
        if self.dense is None:
            raise ValueError("this handle runs the sparse reward: the dense options need a handle built with the dense reward")
        unknown = sorted(set(values) - set(DENSE_OPTIONS))
        if unknown:
            raise ValueError("unknown dense options %s (known: %s; phase_ob is one per handle)" % (unknown, sorted(DENSE_OPTIONS)))
        self._set_options(envs, values, DENSE_OPTIONS)

    def dense_rows(self):
        """(N,) record array of every env's fe_dense_config row (a host copy of field dense_config)"""
        return self.get("dense_config")[:, 0].view(np.dtype(FeDenseConfig))

    def _set_options(self, envs, values, table=OPTIONS):
        """writes `values` (keys of `table` -> a scalar or one value per env of `envs`; None leaves an option as it is) for the envs in `envs`
        (default: all).  A column is an index into the field's row, or the name of a member of its struct-valued row.  Every value is
        checked and converted before any field is written, and each field touched is written once."""
        idx = np.arange(self.N) if envs is None else np.asarray(envs, dtype=np.int64).ravel()
        if idx.size and (idx.min() < 0 or idx.max() >= self.N):
            raise IndexError("envs must lie in [0, %d), got %s" % (self.N, idx.tolist()))
        columns = {}
        for key, v in values.items():
            if v is None:
                continue
            name, col, convert = table[key]
            v = np.asarray(v if convert is None else convert(self, v))
            if v.ndim > 1 or (v.ndim == 1 and v.shape != idx.shape):
                raise ValueError("%s takes a scalar or one value per env of `envs` (%d), got shape %s" % (key, idx.size, v.shape))
            columns.setdefault(name, []).append((col, v))
        for name, cols in columns.items():
            cur = self.get(name)
            for col, v in cols:
                if isinstance(col, str):
                    rows = cur[:, 0].view(np.dtype(FeDenseConfig))  # a view: writing its member writes `cur`
                    rows[col][idx] = v.astype(rows.dtype[col])
                else:
                    cur[idx, col] = v.astype(cur.dtype)
            self.set(name, cur)

    def close(self):
        if getattr(self, "h", None) and self.h.value:
            self.L.fe_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, rc):
        if rc != 0:
            raise RuntimeError("furniture_b200 error %d: %s" % (rc, self.L.fe_last_error(self.h).decode()))

    # ---- simulator surface
    def field_info(self, name):
        d, e = C.c_int(), C.c_int()
        self._chk(self.L.fe_field_dim(self.h, name.encode(), C.byref(d), C.byref(e)))
        return d.value, e.value

    def _dtype(self, name):
        """the field's element type as the library registers it (after field_info, which refuses an unknown name)"""
        return np.dtype(self.L.fe_field_dtype(self.h, name.encode()).decode())

    def get(self, name):
        dim, _ = self.field_info(name)
        out = np.empty((self.N, dim), dtype=self._dtype(name))
        self._chk(self.L.fe_get_field(self.h, name.encode(), out.ctypes.data_as(C.c_void_p), C.c_size_t(out.nbytes)))
        return out

    def set(self, name, value):
        dim, _ = self.field_info(name)
        v = np.ascontiguousarray(np.broadcast_to(np.asarray(value, dtype=self._dtype(name)), (self.N, dim)))
        self._chk(self.L.fe_set_field(self.h, name.encode(), v.ctypes.data_as(C.c_void_p), C.c_size_t(v.nbytes)))

    def get_state(self):
        """(qpos, qvel) of every env through fe_get_state: get_env_state, furniture.py:1781-1792"""
        q = np.empty((self.N, self.model.nq), np.float32)
        v = np.empty((self.N, self.model.nv), np.float32)
        self._chk(self.L.fe_get_state(self.h, q.ctypes.data_as(C.c_void_p), v.ctypes.data_as(C.c_void_p)))
        return q, v

    def set_state(self, qpos, qvel):
        """fe_set_state: set_env_state / sim.set_state, furniture.py:1794-1803, :3095-3105 (call forward() afterwards, as the reference does)"""
        q = np.ascontiguousarray(np.broadcast_to(np.asarray(qpos, np.float32), (self.N, self.model.nq)))
        v = np.ascontiguousarray(np.broadcast_to(np.asarray(qvel, np.float32), (self.N, self.model.nv)))
        self._chk(self.L.fe_set_state(self.h, q.ctypes.data_as(C.c_void_p), v.ctypes.data_as(C.c_void_p)))

    def forward(self, stream=None):
        self._chk(self.L.fe_sim_forward(self.h, C.c_void_p(stream or 0)))

    def step(self, nsub=1, stream=None):
        self._chk(self.L.fe_sim_step(self.h, int(nsub), C.c_void_p(stream or 0)))

    # ---- env surface with host buffers (numpy); torch-tensor variants live in furniture_b200/env.py
    def env_reset(self, mask_dev=None, obs_dev=None, stream=None):
        self._chk(self.L.fe_env_reset(self.h, C.c_void_p(mask_dev or 0), C.c_void_p(obs_dev or 0), C.c_void_p(stream or 0)))

    def env_step_dev(self, actions_dev, obs_dev, reward_dev, done_dev, info_dev, stream=None):
        self._chk(self.L.fe_env_step(self.h, C.c_void_p(actions_dev), C.c_void_p(obs_dev or 0), C.c_void_p(reward_dev or 0), C.c_void_p(done_dev or 0),
                                     C.c_void_p(info_dev or 0), C.c_void_p(stream or 0)))

    def env_step_packed(self, actions_dev, packed_dev, info_dev=None, stream=None):
        """fe_env_step_packed: the kernel writes rows [obs | reward | done] straight into `packed_dev` (the all-gather send buffer)"""
        self._chk(self.L.fe_env_step_packed(self.h, C.c_void_p(actions_dev), C.c_void_p(packed_dev), C.c_void_p(info_dev or 0), C.c_void_p(stream or 0)))

    def set_packed_layout(self, info=False, dense_info=False, terminal_obs=False):
        """fe_set_packed_layout: what env_step_packed writes after [obs | reward | done] in each row, from the next packed step on: the info
        row (int32 bit patterns), the dense reward's dense_info row (a dense handle only) and the terminal observation (valid where done)"""
        flags = dict(info=info, dense_info=dense_info, terminal_obs=terminal_obs)
        self._chk(self.L.fe_set_packed_layout(self.h, *[int(v) if isinstance(v, (bool, np.bool_)) else v for v in flags.values()]))
        self.packed_flags.update((k, bool(v)) for k, v in flags.items())

    def set_packed_step_info(self, step_info=True):
        """fe_set_packed_step_info: whether env_step_packed writes the step-info block [reward_info | episode_info] after the blocks of
        set_packed_layout, from the next packed step on"""
        self._chk(self.L.fe_set_packed_step_info(self.h, int(step_info) if isinstance(step_info, (bool, np.bool_)) else step_info))
        self.packed_flags["step_info"] = bool(step_info)

    def packed_dim(self):
        """fe_packed_dim: floats per packed row under the current layout and obs_dim"""
        return int(self.L.fe_packed_dim(self.h))

    def packed_columns(self):
        """name -> slice of a packed row under this handle's layout (the module's packed_columns)"""
        return packed_columns(self.obs_dim, **self.packed_flags)

    def env_step_host(self, actions):
        a = np.ascontiguousarray(actions, dtype=np.float32)
        assert a.shape == (self.N, self.act_dim), a.shape
        obs = np.empty((self.N, self.obs_dim), np.float32)
        rew = np.empty(self.N, np.float32)
        done = np.empty(self.N, np.uint8)
        info = np.empty((self.N, INFO_DIM), np.int32)
        self._chk(self.L.fe_env_step_host(self.h, a.ctypes.data_as(C.c_void_p), obs.ctypes.data_as(C.c_void_p), rew.ctypes.data_as(C.c_void_p),
                                          done.ctypes.data_as(C.c_void_p), info.ctypes.data_as(C.c_void_p)))
        return obs, rew, done, info

    def set_obs_layout(self, robot_ob=True, object_ob=True, object_ob_all=True, subtask_ob=False):
        """fe_set_obs_layout: the observation flags of config/furniture.py (furniture.py:103-107), before the first reset"""
        flags = dict(robot_ob=robot_ob, object_ob=object_ob, object_ob_all=object_ob_all, subtask_ob=subtask_ob)
        self._chk(self.L.fe_set_obs_layout(self.h, *[int(v) if isinstance(v, (bool, np.bool_)) else v for v in flags.values()]))
        self.obs_flags = {k: bool(v) for k, v in flags.items()}
        self.obs_dim = self.scene.obs_dim = int(self.L.fe_obs_dim(self.h))
        self.scene.obs_layout = (0 if robot_ob else 1) | (0 if object_ob else 2) | (0 if object_ob_all else 4) | (8 if subtask_ob else 0)

    def obs_columns(self):
        """(key -> columns of a device row, key -> width) of the obs dict under this handle's flags (the module's obs_columns); the widths of
        object_ob, subtask_ob, robot_ob and phase_ob are 0 where the dict has no such entry.  Under the IK and controller control types robot_ob
        drops each arm's 14 joint positions and velocities (furniture_sawyer.py:110-125, furniture_baxter.py:137-160)."""
        skip = 0 if self.ik is None and self.controller is None else 14
        cols = obs_columns(self.scene, skip, **self.obs_flags)
        widths = {k: len(np.arange(self.obs_dim)[cols[k]]) if k in cols else 0 for k in ("object_ob", "subtask_ob", "robot_ob", "phase_ob")}
        return cols, widths

    def set_max_episode_steps(self, n):
        self._chk(self.L.fe_set_max_episode_steps(self.h, int(n)))
        self.cfg.max_episode_steps = int(n)

    def set_subtask(self, subtask, num_connects=None):
        """FurnitureEnv.set_subtask (furniture.py:204-207), per env: `subtask` recipe steps are connected by the env's next reset (an
        auto-reset included) and the episode then succeeds after `num_connects` more connections (None: when every part is connected).
        Each is a scalar or an (N,) array; num_connects < 0 in an array stands for None."""
        k = np.broadcast_to(np.asarray(subtask, dtype=np.int64), (self.N,))
        nc = np.broadcast_to(np.asarray(-1 if num_connects is None else num_connects, dtype=np.int64), (self.N,))
        nsub = int(self.scene.dense.nsub)
        if k.any() and nsub == 0:
            raise NotImplementedError("preassembled starts follow the furniture's assembly recipe, and this scene packs none (a furniture without "
                                      "recipes/<name>.yaml, or a two-arm agent)")
        last = nsub - 1 if (self.dense is not None and nsub > 0) else nsub  # the dense reward needs a subtask left to work on
        if k.min() < 0 or k.max() > last:
            raise ValueError("subtask must lie in [0, %d] for this env, got %s" % (last, np.unique(k).tolist()))
        self.set("preassembled", k[:, None])
        self.set("num_connects", np.maximum(nc, -1)[:, None])

    def num_subtask(self):
        """FurnitureEnv.num_subtask (furniture.py:209-213) per env: num_connects where it is set, else the number of parts - 1"""
        nc = self.get("num_connects")[:, 0]
        return np.where(nc >= 0, nc, self.scene.npart - 1)

    # ---- recorded starts: _init_qpos, --load_init_states, --load_demo (furniture.py:121-130, :315-316, :1433-1434)
    def _state_arrays(self, state):
        """a get_env_state dict -> (qpos, qvel) float32 of this handle's model, or ValueError"""
        try:
            q = np.asarray(state["qpos"], dtype=np.float64).ravel()
            v = np.asarray(state["qvel"], dtype=np.float64).ravel()
        except (KeyError, TypeError, ValueError) as e:
            raise ValueError("a state is a dict with numeric 'qpos' and 'qvel' (get_env_state), got %r" % (type(state),)) from e
        if q.size != self.model.nq or v.size != self.model.nv:
            raise ValueError("state has qpos / qvel of length %d / %d, this model has nq = %d, nv = %d" % (q.size, v.size, self.model.nq, self.model.nv))
        if not (np.isfinite(q).all() and np.isfinite(v).all()):
            raise ValueError("state holds non-finite qpos / qvel")
        return q.astype(np.float32), v.astype(np.float32)

    def set_init_states(self, states):
        """fe_set_init_states: the bank of recorded starts every env of the handle indexes with its `init_state` / `init_pick` fields, a list
        of get_env_state dicts ([] or None frees it).  The fields are left as they are; set_init_qpos and load_init_states manage both."""
        arrs = [self._state_arrays(st) for st in (states or [])]
        self._upload_bank(arrs)
        self._n_pick = min(self._n_pick, len(arrs))

    def _upload_bank(self, arrs):
        nq, nv = self.model.nq, self.model.nv
        q = np.ascontiguousarray(np.array([a[0] for a in arrs], np.float32).reshape(len(arrs), nq))
        v = np.ascontiguousarray(np.array([a[1] for a in arrs], np.float32).reshape(len(arrs), nv))
        self._chk(self.L.fe_set_init_states(self.h, q.ctypes.data_as(C.c_void_p), v.ctypes.data_as(C.c_void_p), len(arrs)))
        self._bank = list(arrs)

    def _rebank(self, head, extra):
        """bank = head (the pick list) + every other entry an env starts from + extra; remaps init_state and returns the index of extra[0]"""
        cur = self.get("init_state")[:, 0]
        used = sorted({int(s) for s in cur if s >= 0})
        keep = [s for s in used if head is not None or s >= self._n_pick]  # a new list keeps every start in use, wherever it sat
        head_arrs = self._bank[: self._n_pick] if head is None else head
        remap = {s: s for s in used if s not in keep}
        remap.update({s: len(head_arrs) + i for i, s in enumerate(keep)})
        self._upload_bank(list(head_arrs) + [self._bank[s] for s in keep] + list(extra))
        self.set("init_state", np.array([remap.get(int(s), -1) for s in cur], np.int32)[:, None])
        return len(head_arrs) + len(keep)

    def set_init_qpos(self, states):
        """FurnitureEnv.set_init_qpos (furniture.py:315-316) per env: `states` is one get_env_state dict or None for every env, or a list of
        N such entries.  From its next reset on (an auto-reset included) an env with a state starts from it, and None goes back to random
        placement; a load_init_states pick may later replace it, an unstable step clears it."""
        per_env = isinstance(states, (list, tuple))
        if per_env and len(states) != self.N:
            raise ValueError("set_init_qpos takes one state or None for all envs, or a list of %d (one per env), got %d" % (self.N, len(states)))
        entries = list(states) if per_env else [states] * self.N
        distinct, slot = [], {}
        for st in entries:  # the same dict given to many envs is one bank entry
            if st is not None and id(st) not in slot:
                slot[id(st)] = len(distinct)
                distinct.append(self._state_arrays(st))
        self.set("init_state", np.full((self.N, 1), -1, np.int32))
        first = self._rebank(None, distinct)
        self.set("init_state", np.array([-1 if st is None else first + slot[id(st)] for st in entries], np.int32)[:, None])

    def load_init_states(self, states, envs=None):
        """--load_init_states (furniture.py:127-130, :1433-1434): the handle's list of recorded starts, a list of get_env_state dicts.  Before
        each of its resets an env in `envs` (default: all) keeps its start with probability 0.2 and otherwise picks one from the list
        uniformly, drawing from its own numpy RandomState(seed + 2**20 + env); the other envs do not pick.  [] or None ends the picking."""
        arrs = [self._state_arrays(st) for st in (states or [])]
        idx = np.arange(self.N) if envs is None else np.asarray(envs, dtype=np.int64).ravel()
        if idx.size and (idx.min() < 0 or idx.max() >= self.N):
            raise ValueError("envs must index the %d envs of this handle, got %s" % (self.N, idx.tolist()))
        self._rebank(arrs, [])
        self._n_pick = len(arrs)
        pick = np.zeros(self.N, np.int32)
        pick[idx] = len(arrs)
        self.set("init_pick", pick[:, None])

    def init_states(self):
        """the bank of recorded starts as the device holds it: (qpos (S, nq), qvel (S, nv)) float32, and the length of the pick list"""
        nq, nv = self.model.nq, self.model.nv
        return (np.array([a[0] for a in self._bank], np.float32).reshape(-1, nq), np.array([a[1] for a in self._bank], np.float32).reshape(-1, nv), self._n_pick)

    def dense_eval(self, dc, recipe, thr, n_goal, first, count, site_pos, site_mat, part_pos, touch, reset, connected, ac):
        """test hook fe_dense_eval: the device reward machine on explicit poses, episodes [first[e], first[e] + count[e]); a record with
        reset = 1 + k starts its episode at subtask k"""
        R, nsite = site_pos.shape[:2]
        npart, act_dim = part_pos.shape[1], ac.shape[1]
        f = lambda a, dt: np.ascontiguousarray(a, dtype=dt)
        first, count = f(first, np.int32), f(count, np.int32)
        arrs = [f(site_pos, np.float64), f(site_mat, np.float64), f(part_pos, np.float64), f(touch, np.uint8), f(reset, np.uint8), f(connected, np.uint8), f(ac, np.float64)]
        thr = f(thr, np.float64)
        rew = np.zeros(R, np.float64)
        done = np.zeros(R, np.uint8)
        info = np.zeros((R, self.L.fe_dense_info_dim()), np.float64)
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        self._chk(self.L.fe_dense_eval(self.h, C.byref(dc), C.byref(recipe), C.c_size_t(C.sizeof(recipe)), p(thr), int(n_goal), len(first), p(first), p(count), int(R),
                                       int(nsite), int(npart), int(act_dim), *[p(a) for a in arrs], p(rew), p(done), p(info)))
        return rew, done, info

    def ctl_eval(self, cc, first, count, reset, policy_step, action, readings):
        """test hook fe_ctl_eval: the device controller arithmetic on explicit simulator readings (R, 123), episodes [first[e], first[e] + count[e])"""
        f = lambda a, dt: np.ascontiguousarray(a, dtype=dt)
        first, count, reset, policy_step = f(first, np.int32), f(count, np.int32), f(reset, np.uint8), f(policy_step, np.uint8)
        action, readings = f(action, np.float64), f(readings, np.float64)
        assert readings.shape[1] == 123 and action.shape[1] == 7
        tau = np.zeros((len(readings), 7), np.float64)
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        self._chk(self.L.fe_ctl_eval(self.h, C.byref(cc), len(first), p(first), p(count), len(readings), p(reset), p(policy_step), p(action), p(readings), p(tau)))
        return tau

    def obs_dev_ptr(self):
        return self.L.fe_obs_dev(self.h)

    # ---- what a finished episode left (the terminal `ob` of FurnitureEnv.step, furniture.py:364-385): the step that returns done = 1 for an
    # env writes its last observation row and qpos / qvel before the auto-reset; other envs' rows keep what they held
    def terminal_obs(self):
        """(N, obs_dim) float32 host copy of the terminal observation rows, valid where the last step's done is 1"""
        return self.get("terminal_obs")

    def terminal_state(self):
        """(qpos (N, nq), qvel (N, nv)) float32 host copies of the terminal state, valid where the last step's done is 1"""
        return self.get("terminal_qpos"), self.get("terminal_qvel")

    def terminal_dev_ptrs(self):
        """device pointers of the terminal buffers: (obs (N, obs_dim), qpos (N, nq), qvel (N, nv)), float32, env-major; the obs pointer moves
        with set_obs_layout"""
        return self.L.fe_terminal_obs_dev(self.h), self.L.fe_terminal_qpos_dev(self.h), self.L.fe_terminal_qvel_dev(self.h)

    # ---- the step's info dict (furniture.py:451-541): fields "reward_info" and "episode_info", written by every env step
    def reward_info(self):
        """(N, 4) float32 host copy of the last step's reward terms in the order of REWARD_INFO_KEYS (a sparse-reward handle only: a dense
        handle has no such terms: its steps write none, and this raises)"""
        if self.dense is not None:
            raise RuntimeError("this handle runs the dense reward: its reward terms are the field dense_info")
        return self.get("reward_info")

    def episode_info(self):
        """(N, 2) float32 host copy of the episode record in the order of EPISODE_INFO_KEYS, valid where the last step's done is 1; rows no
        step has written are NaN"""
        return self.get("episode_info")

    def step_info_dev_ptrs(self):
        """device pointers of (reward_info (N, 4), episode_info (N, 2)), float32, env-major; reward_info is None on a dense handle"""
        return self.L.fe_reward_info_dev(self.h), self.L.fe_episode_info_dev(self.h)

    def is_aligned(self, p1, m1, p2, m2, angles, nangles, thr):
        n = len(p1)
        arrs = [np.ascontiguousarray(x, dtype=np.float64) for x in (p1, m1, p2, m2, angles, thr)]
        na = np.ascontiguousarray(nangles, dtype=np.int32)
        al = np.empty(n, np.uint8)
        tq = np.empty((n, 4), np.float64)
        self._chk(self.L.fe_is_aligned(self.h, n, arrs[0].ctypes.data_as(C.c_void_p), arrs[1].ctypes.data_as(C.c_void_p), arrs[2].ctypes.data_as(C.c_void_p),
                                       arrs[3].ctypes.data_as(C.c_void_p), arrs[4].ctypes.data_as(C.c_void_p), na.ctypes.data_as(C.c_void_p),
                                       arrs[5].ctypes.data_as(C.c_void_p), al.ctypes.data_as(C.c_void_p), tq.ctypes.data_as(C.c_void_p)))
        return al.astype(bool), tq
