"""CPU ORACLE for episodes that start part-way through the assembly (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

The env oracles of oracle/ref_env.py with the reference's `preassembled` / `set_subtask` on top, restated with line cites:

  project_connector_quat   <- FurnitureEnv._project_connector_quat   furniture/env/furniture.py:1201-1222  (tests/golden/preassembled.npz, bit for bit)
  set_subtask / num_subtask <- FurnitureEnv.set_subtask / num_subtask :204-213
  reset                    <- FurnitureEnv._reset with its preassembly :1406-1663 (:1477-1481 the success count, :1542-1566 the connections
                              and the second settle loop)
  connected                <- FurnitureEnv._connected :392, :911, :1468, :1557

PreassembledEnv is the sparse-reward Sawyer env, PreassembledDenseEnv the dense-reward one (its DenseOracle starts at subtask k,
furniture_sawyer_dense.py:128-139).  With nothing preassembled both reset exactly like their parents: for a furniture with a recipe the
reference runs the second settle loop even then, these envs and the device do not.
"""
import json

import numpy as np

from . import assembly_oracle as A
from .ref_env import OracleDenseEnv, OracleFurnitureEnv


def project_connector_quat(m1, m2, angle=None):
    """connector2's xquat (wxyz) when aligned with connector1 at `angle` degrees, or at the nearer of the two rotations that bring the forward
    vectors together when `angle` is None.  m*: site world rotation (3,3)."""
    m1, m2 = np.asarray(m1, dtype=np.float64).reshape(3, 3), np.asarray(m2, dtype=np.float64).reshape(3, 3)
    up1, f1, f2 = m1[:, 2].copy(), m1[:, 1].copy(), m2[:, 1].copy()
    if angle is None:
        c = A.cos_siml(f1, f2)
        fp = A.rotate_vector_cos_siml(f1, up1, c, 1)
        fn = A.rotate_vector_cos_siml(f1, up1, c, -1)
        fr = fp if A.cos_siml(fp, f2) > A.cos_siml(fn, f2) else fn
    else:
        fr = A.rotate_vector(f1, up1, angle)
    return A.lookat_to_quat(up1, fr)[[3, 0, 1, 2]]


class PreassembledEnv(OracleFurnitureEnv):
    def __init__(self, model, cfg=None):
        super().__init__(model, cfg)
        self.preassembled, self.num_connects = 0, None
        self.success_num_conn = self.npart - 1
        self.connected = False  # _connected: a connection was made during the current step

    def set_subtask(self, subtask, num_connects=None):  # :204-207: _preassembled = range(subtask), from the next reset on
        self.preassembled, self.num_connects = int(subtask), num_connects

    def num_subtask(self):  # :209-213
        return self.num_connects if self.num_connects is not None else self.npart - 1

    def _stabilise(self):  # :1535-1540, :1560-1566
        for _ in range(10):
            for p in range(self.npart):
                self._stop(p, 0)
            for _ in range(10):
                self._fwd_step()
                for p in range(self.npart):
                    self._slow(p)

    def _preassemble(self):
        """:1542-1558: connect the first steps of the recipe.  _connect(site2_id, site1_id, auto_align=True): the table's site is _connect's
        site1, so the leg's group moves, and the connectors are aligned whatever the config says.  No random draw is made."""
        m, sim = self.m, self.sim
        names = m.names["site"]
        mat = lambda s: sim.site_xmat[9 * s : 9 * s + 9]
        auto_align, self.cfg.auto_align = self.cfg.auto_align, True
        for sr in json.loads(m.meta["recipe_json"])["site_recipe"][: self.preassembled]:
            leg_site, table_site = names.index(sr[0]), names.index(sr[1])
            self.target_quat = project_connector_quat(mat(table_site), mat(leg_site), sr[2] if len(sr) == 3 else None)
            self._connect(table_site, leg_site)
            self.connected = False
            self.connected_body1 = None
        self.cfg.auto_align = auto_align

    def reset(self):
        """OracleFurnitureEnv.reset with the preassembly between the settled furniture and the robot's pose"""
        sim, cfg = self.sim, self.cfg
        if cfg.furn_size_rand != 0:  # :1428-1431 (edits the XML tree only)
            self.rng.uniform(-cfg.furn_size_rand, cfg.furn_size_rand, 1)
        sim.reset()
        saved = {g: (sim.geom_contype[g], sim.geom_conaffinity[g]) for g in self.robot_geoms}
        for g in self.robot_geoms:
            sim.geom_contype[g] = 0; sim.geom_conaffinity[g] = 0
        for g in self.part_col_geoms:
            sim.geom_contype[g] = 1; sim.geom_conaffinity[g] = 1
        self.group = list(range(self.npart))
        self.connected_sites = set()
        self.num_connected = self.prev_num_connected = 0
        self.success_num_conn = self.npart - 1 if self.num_connects is None else self.num_connects + self.preassembled  # :1477-1481
        self.touched = [False] * self.npart
        self.picked = [False] * self.npart
        sim.eq_active[:] = 0
        for p, (pos, quat) in enumerate(self.place()):
            self._set_qpos(p, pos, quat)
        self._stabilise()
        if self.preassembled:
            self._preassemble()
            self._stabilise()
        self._grav_comp()
        self._init_robot()
        self._fwd_step()
        for g, (ct, ca) in saved.items():
            sim.geom_contype[g] = ct; sim.geom_conaffinity[g] = ca
        self._grav_comp()
        for _ in range(100):
            self._init_robot()
            self._fwd_step()
        sim.ctrl[:] = 0; sim.qfrc_applied[:] = 0; sim.xfrc_applied[:] = 0; sim.qacc[:] = 0; sim.qacc_warmstart[:] = 0
        sim.forward()
        self._grav_comp()
        for _ in range(100):
            self._fwd_step()
        self.episode_len = 0
        self.connected_body1 = None
        self.connected = False  # :1468
        return self.obs()

    def _connect(self, s1, s2):
        super()._connect(s1, s2)
        self.connected = True  # :911

    def step(self, action):
        self.connected = False  # :392
        return super().step(action)

    def _compute_reward(self, raw, fail):
        reward, _, _ = super()._compute_reward(raw, fail)
        success = self.num_connected == self.success_num_conn and self.npart > 1  # furniture.py:438-445
        return reward, success, success


class PreassembledDenseEnv(OracleDenseEnv, PreassembledEnv):
    def reset(self):
        PreassembledEnv.reset(self)
        self.dense.preassembled, self.dense.n_goal = list(range(self.preassembled)), self.success_num_conn
        self.dense.begin_episode()
        return self.obs()

    def _compute_reward(self, raw, fail):
        self.prev_num_connected = self.num_connected
        reward, done, self.dense_info = self.dense.step(np.asarray(raw, dtype=np.float64), self.connected)  # the preassembled legs are not a connection
        base_done = self.num_connected == self.success_num_conn and self.npart > 1
        return reward, bool(done or base_done), self.dense.success
