"""CPU ORACLE for episodes that start from recorded states (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

The env oracles of oracle/preassembled_oracle.py with the reference's `_init_qpos` on top, restated with line cites:

  set_init_qpos     <- FurnitureEnv.set_init_qpos                        furniture/env/furniture.py:315-316
  load_init_states  <- --load_init_states and the pick before each reset  :127-130, :1433-1434
  set_env_state     <- FurnitureEnv.set_env_state                        :1794-1798
  reset             <- FurnitureEnv._reset, both branches of `if self._init_qpos:`  :1406-1663
  _do_simulation    <- its except branch clears the start                 :2889-2897

The reference draws the pick from the process-global np.random, which nothing seeds; here it is a RandomState(seed + 2**20) of the env's own
(cfg.seed = seed + env gives the generator the device seeds for env `env`), so that the sampler stream (self.rng) stays draw for draw on the
reference's _rng.  The settle loop after the preassembly (:1560-1566) runs as written, although the second set_env_state overwrites what it
does.
"""
import json

import numpy as np

from .preassembled_oracle import PreassembledDenseEnv, PreassembledEnv, project_connector_quat


class InitStateEnv(PreassembledEnv):
    def __init__(self, model, cfg=None):
        super().__init__(model, cfg)
        self.init_qpos = None    # _init_qpos
        self.init_states = None  # _load_init_states
        self.pick_rng = np.random.RandomState(self.cfg.seed + 2**20)

    def set_init_qpos(self, init_qpos):  # :315-316
        self.init_qpos = init_qpos

    def load_init_states(self, states):  # :127-130
        self.init_states = list(states) if states else None

    def _pick(self):  # :1433-1434: np.random.choice(list) draws randint(0, len(list))
        if self.init_states and self.pick_rng.rand() > 0.2:
            self.set_init_qpos(self.init_states[self.pick_rng.choice(len(self.init_states))])

    def _set_env_state(self):  # :1794-1798
        sim = self.sim
        for p in range(self.npart):
            self._stop(p, 0)
        sim.qpos[:] = self.init_qpos["qpos"]
        sim.qvel[:] = self.init_qpos["qvel"]
        sim.ctrl[:] = 0

    def _preassemble_unaligned(self):
        """:1542-1558 with auto_align = self._init_qpos is None = False: the parts are connected where the recorded state has them"""
        m, sim = self.m, self.sim
        names = m.names["site"]
        mat = lambda s: sim.site_xmat[9 * s : 9 * s + 9]
        auto_align, self.cfg.auto_align = self.cfg.auto_align, False
        for sr in json.loads(m.meta["recipe_json"])["site_recipe"][: self.preassembled]:
            leg_site, table_site = names.index(sr[0]), names.index(sr[1])
            self.target_quat = project_connector_quat(mat(table_site), mat(leg_site), sr[2] if len(sr) == 3 else None)
            self._connect(table_site, leg_site)
            self.connected = False
            self.connected_body1 = None
        self.cfg.auto_align = auto_align

    def reset(self):
        cfg, sim = self.cfg, self.sim
        self._pick()  # after the size-factor draw in the reference; the two generators are independent
        if self.init_qpos is None:
            return super().reset()
        if cfg.furn_size_rand != 0:  # :1428-1431
            self.rng.uniform(-cfg.furn_size_rand, cfg.furn_size_rand, 1)
        sim.reset()  # :1437-1503
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
        sim.eq_active[:] = 0  # :1501-1503: a recorded mid-assembly state starts unwelded
        self._set_env_state()  # :1505-1518: robot collisions back on, forward; no placement, no settle loop, no draw
        for g, (ct, ca) in saved.items():
            sim.geom_contype[g] = ct; sim.geom_conaffinity[g] = ca
        sim.forward()
        if self.preassembled:  # :1542-1566
            self._preassemble_unaligned()
            self._stabilise()
        sim.forward()  # :1568
        self._set_env_state()  # :1617
        sim.ctrl[:] = 0; sim.qfrc_applied[:] = 0; sim.xfrc_applied[:] = 0; sim.qacc[:] = 0; sim.qacc_warmstart[:] = 0  # :1620-1628
        sim.forward()
        self._grav_comp()
        for _ in range(100):  # :1639-1641
            self._fwd_step()
        self.episode_len = 0
        self.connected_body1 = None
        self.connected = False
        return self.obs()

    def _simulate(self, raw):
        fail, reset_now = super()._simulate(raw)
        if fail:  # :2895: set_init_qpos(None) before the except branch's reset; the VecEnv worker's reset after `done` starts from None too
            self.set_init_qpos(None)
        return fail, reset_now


class InitStateDenseEnv(PreassembledDenseEnv, InitStateEnv):
    def reset(self):
        InitStateEnv.reset(self)
        self.dense.preassembled, self.dense.n_goal = list(range(self.preassembled)), self.success_num_conn
        self.dense.begin_episode()
        return self.obs()
