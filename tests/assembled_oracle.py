"""CPU ORACLE for the reset option `assembled` (TEST INFRASTRUCTURE, NOT PRODUCT CODE).

A mixin over the reset-options oracles of tests/reset_options_oracle.py, which are unchanged, as that file is one over oracle/.  Restated
with line cites of furniture/env/furniture.py:

  welds      <- `eq_active[i] = 1 if assembled else 0` for every weld, on both branches of `if self._init_qpos:`          :1501-1503
  eq_data    <- a model array: sim.reset() (mj_resetData) leaves it as the last _activate_weld wrote it                   :1437, :2761-2776
  place      <- _place_objects still draws and init_pos is still updated, but no part is _set_qpos'd: the parts stay at
                sim.reset()'s qpos0 and every _object_group[i] becomes 0 (a recorded start merges no group)              :1519-1532
  subtask    <- _get_next_subtask: the first weld whose parts lie in different groups, (-1, -1) when none does            :2723-2736

The oracle's simulator copies the model's eq_data back on every reset; the mixin keeps the env's instead, as MuJoCo does.
"""
from reset_options_oracle import ResetOptionsDenseEnv, ResetOptionsIKEnv, ResetOptionsInitStateEnv


class AssembledMixin:
    def __init__(self, *a, assembled=False, **kw):
        super().__init__(*a, **kw)
        self.assembled = bool(assembled)
        self.moved = []  # the parts the last random-placement reset planted (_set_qpos)

    def reset(self):
        sim = self.sim
        keep = sim.eq_data.copy()
        reset = sim.reset

        def sim_reset():  # mj_resetData: data only, the model's eq_data stays
            reset()
            sim.eq_data[:] = keep

        sim.reset = sim_reset
        try:
            return super().reset()
        finally:
            del sim.reset

    def place(self):
        placed = super().place()
        if not self.assembled:
            self.moved = list(range(self.npart))
            return placed
        self.sim.eq_active[:] = 1
        self.group = [0] * self.npart
        self.moved = []
        return [(self._qpos(p)[:3], self._qpos(p)[3:]) for p in range(self.npart)]  # where sim.reset() left them: planting them moves nothing

    def _set_env_state(self):
        super()._set_env_state()
        if self.assembled:  # the recorded-start branch: every weld on, the groups as they are
            self.sim.eq_active[:] = 1

    def subtask_pair(self):
        m = self.m
        for e in range(m.neq):
            a, b = self._part_of_body(m.eq_obj1id[e]), self._part_of_body(m.eq_obj2id[e])
            if self._find(a) != self._find(b):
                return a, b
        return -1, -1


class AssembledIKEnv(AssembledMixin, ResetOptionsIKEnv):
    pass


class AssembledInitStateEnv(AssembledMixin, ResetOptionsInitStateEnv):
    pass


class AssembledDenseEnv(AssembledMixin, ResetOptionsDenseEnv):
    pass
