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
from .dense import FeDenseConfig, FeDenseRecipe, dense_config, pack_dense_recipe
from .engine_model import MAXEQ, MAXPART, MAXRDOF, MAXSITE, MAXU, EngineModel

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, "libfurniture_b200.so")
MAXCONN = 48
SCENE_MAGIC = 0x46455344
INFO_DIM = 6
# bits of the `flags` field and columns of the `stats` field: FE_FLAG_* / FE_STAT_* of include/furniture_b200.h, which says what each means
FLAG_CONTACT_FULL, FLAG_NUMERIC, FLAG_NEWTON_PIVOT, FLAG_DIVERGED = 1, 2, 4, 8
STAT_PART_ITERS, STAT_COUPLED, STAT_NEWTON_SOLVES, STAT_NEWTON_ITERS = 0, 1, 2, 3
STAT_KIN, STAT_COLLIDE, STAT_ASSEMBLE, STAT_SOLVE, STAT_INTEGRATE, STAT_WAIT, STAT_ROBOT_ONLY, STAT_SOLVE_MAX = 4, 5, 6, 7, 8, 9, 10, 11
STAT_WAIT_KIN, STAT_WAIT_COLLIDE, STAT_WAIT_ASSEMBLE, STAT_WAIT_SOLVE, STAT_WAIT_INTEGRATE = 12, 13, 14, 15, 16
STAT_SOLVE_PRE, STAT_SOLVE_GROUPED, STAT_SOLVE_COMP, STAT_RESERVED = 17, 18, 19, 20
STAT_NEWTON_SETUP, STAT_NEWTON_START, STAT_NEWTON_GRAD, STAT_NEWTON_HESSIAN, STAT_NEWTON_CHOL, STAT_NEWTON_PRODUCTS, STAT_NEWTON_LS = 21, 22, 23, 24, 25, 26, 27
i32, f32, f64 = C.c_int32, C.c_float, C.c_double


class FeConfig(C.Structure):
    _fields_ = [
        ("struct_bytes", i32), ("maxcon", i32), ("newton_iters", i32), ("ls_iters", i32), ("tolerance", f32), ("nsub", i32),
        ("max_episode_steps", i32), ("discrete_grip", i32), ("rescale_actions", i32), ("auto_align", i32),
        ("alignment_pos_dist", f64), ("alignment_rot_dist_up", f64), ("alignment_rot_dist_forward", f64), ("alignment_project_dist", f64),
        ("ctrl_penalty_coef", f32), ("unstable_penalty_coef", f32), ("success_reward", f32), ("touch_reward", f32), ("pick_reward", f32),
        ("furn_xyz_rand", f32), ("furn_rot_rand", f32), ("agent_xyz_rand", f32), ("furn_size_rand", f32), ("seed", C.c_uint64),
    ]


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
        ("phase_ob", i32), ("pad_", i32), ("dense", FeDenseRecipe),
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


class Engine:
    def __init__(self, model: mjcf.Model, n_envs: int, device: int = 0, config: FeConfig | None = None, lib_path: str | None = None,
                 dense: FeDenseConfig | None = None, ik=None, controller=None):
        path = lib_path or DEFAULT_LIB
        if not os.path.exists(path):
            raise RuntimeError(
                "furniture_b200: CUDA extension %s not built (run `python -c 'import __graft_entry__ as g; g.build()'`); there is no CPU fallback" % path
            )
        L = C.CDLL(path)
        self.L = L
        L.fe_last_error.restype = C.c_char_p
        L.fe_last_error.argtypes = [C.c_void_p]
        for f in ("fe_model_sizeof", "fe_scene_sizeof", "fe_config_sizeof"):
            getattr(L, f).restype = C.c_size_t
        L.fe_obs_dev.restype = C.c_void_p
        L.fe_obs_dev.argtypes = [C.c_void_p]
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
        self.dense = dense
        if dense is not None:  # FurnitureSawyerDenseRewardEnv: the phase machine replaces the sparse reward inside fe_env_step
            self._chk(L.fe_enable_dense_reward(self.h, C.byref(dense)))

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

    _INT = {"order", "geom_contype", "geom_conaffinity", "eq_active", "touch", "flags", "ncon", "niter", "stats", "con_geom", "con_state", "group", "site_connected",
            "num_connected", "prev_num_connected", "touched", "picked", "episode_length", "done", "mt_pos"}

    def get(self, name):
        dim, eb = self.field_info(name)
        dt = np.uint8 if eb == 1 else np.uint64 if eb == 8 else (np.uint32 if name == "mt_state" else (np.int32 if name in self._INT else np.float32))
        out = np.empty((self.N, dim), dtype=dt)
        self._chk(self.L.fe_get_field(self.h, name.encode(), out.ctypes.data_as(C.c_void_p), C.c_size_t(out.nbytes)))
        return out

    def set(self, name, value):
        dim, eb = self.field_info(name)
        dt = np.uint8 if eb == 1 else np.uint64 if eb == 8 else (np.uint32 if name == "mt_state" else (np.int32 if name in self._INT else np.float32))
        v = np.ascontiguousarray(np.broadcast_to(np.asarray(value, dtype=dt), (self.N, dim)))
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

    def set_max_episode_steps(self, n):
        self._chk(self.L.fe_set_max_episode_steps(self.h, int(n)))
        self.cfg.max_episode_steps = int(n)

    def dense_eval(self, dc, recipe, thr, n_goal, first, count, site_pos, site_mat, part_pos, touch, reset, connected, ac):
        """test hook fe_dense_eval: the device reward machine on explicit poses, episodes [first[e], first[e] + count[e])"""
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
