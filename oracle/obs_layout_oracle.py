"""CPU ORACLE for the observation flags robot_ob / object_ob / object_ob_all / subtask_ob (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

A mixin over the env oracles of oracle/ref_env.py, oracle/preassembled_oracle.py and oracle/init_state_oracle.py that tracks the reference's
current subtask and lays the observation out as its flags ask, restated with line cites:

  flags              <- FurnitureEnv.__init__                          furniture/env/furniture.py:103-107
  obs_dict / space   <- FurnitureEnv._get_obs / observation_space      :1344-1387, :215-252; robot_ob furniture_sawyer.py:27-48, :103-155,
                                                                         furniture_baxter.py:27-48, :98-155; phase_ob furniture_sawyer_dense.py:99-117
  _get_next_subtask  <- the first weld whose parts are in different groups   :2723-2736 (_find_group / _merge_groups :2738-2759)
                        called at the end of _connect (:917) and of _reset (:1653)
  dense pair         <- _update_reward_variables                       furniture_sawyer_dense.py:149-162 (from _reset_reward_variables :128-139
                                                                         and _set_next_subtask :141-147)

Timing: FurnitureSawyerEnv._step takes `ob` from FurnitureEnv._step before _compute_reward (furniture_sawyer.py:66-84), so a step's object_ob and
subtask_ob show the pair the connect scan left, and only phase_ob follows the reward (furniture_sawyer_dense.py:119-126).  `obs()` is the
device's row ([object_ob | subtask_ob | robot_ob (all joints) | phase_ob]); `obs_dict(row, control_type)` splits it as the host does.
"""
from collections import OrderedDict

import numpy as np

from .init_state_oracle import InitStateDenseEnv, InitStateEnv
from .ref_env import OracleIKEnv

DEFAULTS = dict(robot_ob=True, object_ob=True, object_ob_all=True, subtask_ob=False)  # config/furniture.py:228-258


class ObsLayoutMixin:
    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.flags = dict(DEFAULTS)
        self.subtask_part1 = self.subtask_part2 = -1
        self._ob_pair = None  # the pair the step's observation shows, taken before the reward
        dense = getattr(self, "dense", None)
        if dense is not None:
            begin_subtask = dense.begin_subtask

            def update_reward_variables():  # furniture_sawyer_dense.py:149-162
                begin_subtask()
                st = dense.sub[dense.subtask]
                self.subtask_part1, self.subtask_part2 = self.parts.index(st.leg), self.parts.index(st.table)

            dense.begin_subtask = update_reward_variables
            begin_episode = dense.begin_episode

            def reset_reward_variables():  # FurnitureEnv._reset ends with _get_next_subtask (:1653) before the dense _reset runs
                self._get_next_subtask()
                begin_episode()

            dense.begin_episode = reset_reward_variables

    def set_obs_layout(self, **flags):
        self.flags = dict(DEFAULTS, **flags)

    def _get_next_subtask(self):  # :2723-2736
        m = self.m
        for b1, b2 in zip(m.eq_obj1id, m.eq_obj2id):
            p1, p2 = self._part_of_body(b1), self._part_of_body(b2)
            if self._find(p1) != self._find(p2):
                self.subtask_part1, self.subtask_part2 = p1, p2
                return
        self.subtask_part1 = self.subtask_part2 = -1

    def _connect(self, s1, s2):
        super()._connect(s1, s2)
        self._get_next_subtask()  # :917

    def reset(self):
        super().reset()
        if getattr(self, "dense", None) is None:
            self._get_next_subtask()  # :1653 (the dense env ran it ahead of its reward variables)
        return self.obs()

    def _compute_reward(self, raw, fail):
        self._ob_pair = (self.subtask_part1, self.subtask_part2)
        return super()._compute_reward(raw, fail)

    def step(self, action):
        try:
            return super().step(action)
        finally:
            self._ob_pair = None

    def obs(self):
        """the device row under the flags"""
        base = np.asarray(super().obs(), dtype=np.float64)
        n_obj = 7 * self.npart
        phase = 8 if (getattr(self, "dense", None) is not None and self.dense.c["phase_ob"]) else 0
        robot, ph = base[n_obj : len(base) - phase], base[len(base) - phase :]
        p1, p2 = self._ob_pair if self._ob_pair is not None else (self.subtask_part1, self.subtask_part2)
        f, row = self.flags, []
        if f["object_ob"]:
            if f["object_ob_all"]:
                row.append(base[:n_obj])
            else:  # :1364-1377: the pair's parts in part order, or the 14 zeros of "dummy"
                keep = [base[7 * i : 7 * i + 7] for i in range(self.npart) if i in (p1, p2)]
                row += keep + ([np.zeros(14)] if p1 == -1 else [])
        if f["subtask_ob"]:
            row.append(np.array([p1 + 1, p2 + 1], dtype=np.float64))  # :1379-1382
        if f["robot_ob"]:
            row.append(robot)
        row.append(ph)
        return np.concatenate(row) if row else np.zeros(0)

    def obs_dict(self, row, control_type="impedance"):
        """the row as the host splits it into the reference's keys (the IK control types keep the 15-number tail of each arm's robot block)"""
        f, d, o = self.flags, OrderedDict(), 0
        if f["object_ob"]:
            w = 7 * self.npart if f["object_ob_all"] else 14
            d["object_ob"], o = row[o : o + w], o + w
        if f["subtask_ob"]:
            d["subtask_ob"], o = row[o : o + 2], o + 2
        if f["robot_ob"]:
            per = (2 * (self.narm // self.narms) + self.ngrip // self.narms + 13)
            skip = 0 if control_type == "impedance" else 14
            d["robot_ob"] = np.concatenate([row[o + a * per + skip : o + (a + 1) * per] for a in range(self.narms)])
            o += per * self.narms
        if len(row) > o:
            d["phase_ob"] = row[o:]
        return d


class ObsLayoutEnv(ObsLayoutMixin, InitStateEnv):
    """the sparse Sawyer / Baxter env with preassembled and recorded starts"""


class ObsLayoutDenseEnv(ObsLayoutMixin, InitStateDenseEnv):
    """FurnitureSawyerDenseRewardEnv with preassembled and recorded starts"""


class ObsLayoutIKEnv(ObsLayoutMixin, OracleIKEnv):
    """control_type="ik" over the sparse env"""
