"""CPU ORACLE for the reset options fix_init, fix_init_parts and reset_robot_after_attach (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

A mixin over the env oracles of oracle/ (ref_env.py, preassembled_oracle.py, init_state_oracle.py), in the way oracle/obs_layout_oracle.py
is one; those files are unchanged.  Restated with line cites:

  init_pos / init_quat  <- FurnitureEnv._load_model: the XML's *_initpos numerics, or None     furniture/env/furniture.py:2013-2021
  place                 <- _reset's random-placement branch: sample, update or keep init_pos  :1519-1532
  _place_objects        <- the fixed parts frozen once, then UniformRandomSampler.sample       :1389-1404, placement_sampler.py:137-190
  _connect              <- its tail: _initialize_robot_pos, and sync_state for IK              :916-924, sawyer_ik_controller.py:90-102

A recorded start (`if self._init_qpos:`) never calls place, so it ignores fix_init and fix_init_parts as the reference does.  The IK target is
re-seeded from the hand pose of the next command (after the re-pin step's forward pass), where the device re-seeds it.
"""
import numpy as np

from furniture_b200.mjcf import xml_init_poses
from oracle import assembly_oracle as A
from oracle.init_state_oracle import InitStateEnv
from oracle.preassembled_oracle import PreassembledDenseEnv, PreassembledEnv
from oracle.ref_env import IKMixin


class ResetOptionsMixin:
    def __init__(self, *a, fix_init=False, fix_init_parts=None, reset_robot_after_attach=False, **kw):
        super().__init__(*a, **kw)
        self.fix_init = bool(fix_init)
        names = [n for n in (fix_init_parts.split(",") if isinstance(fix_init_parts, str) else list(fix_init_parts or ())) if n]
        if set(names) - set(self.parts):
            raise KeyError(sorted(set(names) - set(self.parts)))  # init_pos[part] (:1400)
        self.fix_init_parts = set(names)
        self.reset_robot_after_attach = bool(reset_robot_after_attach)
        xml = xml_init_poses(self.m.meta)
        self.init_pos = None if xml is None else {n: list(xml[n][:3]) for n in self.parts}
        self.init_quat = None if xml is None else {n: np.array(xml[n][3:7]) for n in self.parts}
        self.fixed_parts = []    # :117
        self.arm_resync = False  # a connection sent the arm home: the next IK command re-seeds its position target
        self.tries = []          # x, y tries of every part of the last sampled placement (0 for a fixed part)
        self.rejected = []       # "part<rejecter" for every rejected try of the last sampled placement

    def _place_objects(self):
        """:1389-1404: the named parts frozen at init_pos the first time there is one; UniformRandomSampler.sample with them as placed objects"""
        m, cfg, rng = self.m, self.cfg, self.rng
        if self.fix_init_parts and not self.fixed_parts and self.init_pos:
            for n in sorted(self.fix_init_parts, key=self.parts.index):
                self.fixed_parts.append((n, m.meta["part_radius"][n], np.array(self.init_pos[n], dtype=np.float64), np.array(self.init_quat[n], dtype=np.float64)))
        pos_arr, quat_arr, placed = {}, {}, []
        for n, r, pos, quat in self.fixed_parts:  # placement_sampler.py:150-158: at their pose, z included, no draw
            pos_arr[n], quat_arr[n] = pos.copy(), quat.copy()
            placed.append((n, pos[0], pos[1], r))
        fixed = {f[0] for f in self.fixed_parts}
        self.tries, self.rejected = [], []
        for name in self.parts:
            if name in fixed:
                self.tries.append(0)
                continue
            init, r = m.meta["part_init_qpos"][name], m.meta["part_radius"][name]
            for t in range(10000):
                x = init[0] + rng.uniform(-cfg.furn_xyz_rand, cfg.furn_xyz_rand)
                y = init[1] + rng.uniform(-cfg.furn_xyz_rand, cfg.furn_xyz_rand)
                hit = next((pn for pn, px, py, pr in placed if np.linalg.norm([x - px, y - py], 2) <= pr + r), None)  # :165-171, first overlap
                if hit is None:
                    break
                self.rejected.append("%s<%s" % (name, hit))
            self.tries.append(t + 1)
            rot = rng.uniform(high=cfg.furn_rot_rand, low=cfg.furn_rot_rand)
            placed.append((name, x, y, r))
            pos_arr[name] = np.array([x, y, init[2] + 0.01])
            quat_arr[name] = np.asarray(A.euler_to_quat([rot, 0, 0], init[3:7]), dtype=np.float64)
        return pos_arr, quat_arr

    def place(self):
        """:1519-1532: the first placement is sampled unless the XML gave one; later ones are sampled and remembered, or, under fix_init, kept"""
        if self.init_pos is None:
            self.init_pos, self.init_quat = self._place_objects()
        elif not self.fix_init:
            pos, quat = self._place_objects()
            self.init_pos.update(pos)
            self.init_quat.update(quat)
        else:
            self.tries, self.rejected = [0] * self.npart, []
        return [(np.asarray(self.init_pos[n], dtype=np.float64), np.asarray(self.init_quat[n], dtype=np.float64)) for n in self.parts]

    def _connect(self, s1, s2):
        super()._connect(s1, s2)
        if self.reset_robot_after_attach:  # :919-924
            self._init_robot()
            self.arm_resync = True


class ResetOptionsEnv(ResetOptionsMixin, PreassembledEnv):
    pass


class ResetOptionsIKEnv(ResetOptionsMixin, IKMixin, PreassembledEnv):
    def __init__(self, model, cfg=None, **kw):
        ik_kw = {k: kw.pop(k) for k in list(kw) if k not in ("fix_init", "fix_init_parts", "reset_robot_after_attach")}
        super().__init__(model, cfg, **kw)
        self._ik_setup(**ik_kw)

    def reset(self):
        ob = super().reset()
        self._ik_sync()
        self.arm_resync = False
        return ob

    def _simulate(self, raw):
        if self.arm_resync:  # controller.sync_state(): the position target only, _initial_<arm>_hand_quat stays
            for a, ik in enumerate(self.iks):
                s = ik.s
                ik.sync(*self._hand(a))
                ik.s = s
            self.arm_resync = False
        return super()._simulate(raw)


class ResetOptionsInitStateEnv(ResetOptionsMixin, InitStateEnv):
    pass


class ResetOptionsDenseEnv(ResetOptionsMixin, PreassembledDenseEnv):
    pass
