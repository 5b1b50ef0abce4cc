"""Golden vectors for episodes that start from recorded states, made by running the REFERENCE'S OWN Python, unmodified.

Runs only where the reference checkout is (make_golden_assembly.REF); writes tests/golden/init_states.npz, which travels.
What is executed from the reference:
  * furniture/env/furniture.py  FurnitureEnv._reset (:1406-1663), with set_init_qpos (:315-316) and set_env_state (:1794-1798), on a
    recording stand-in: `sim` records reset / forward / step (each with whether the robot's collisions are on at that moment), its
    `data` records which state set_env_state plants and the gravity compensation of the arm; _place_objects, _initialize_robot_pos,
    _stop_objects, _slow_objects, _connect (with its auto_align argument) and _merge_groups are recorders.  The module's np.random is
    replaced by a seeded RandomState while _reset runs.
    Cases: start None / fixed / a bank of 3 (np.random seeded for env 0, whose first draw keeps None, and env 1, whose draw picks), x k = 0, 1, 2
    preassembled steps, x the table_lack_0825 recipe or none.
  * the pick alone: 20 resets with a bank of S = 1, 3, 7 states, np.random seeded as the device seeds env 0..7
    (RandomState(123 + 2**20 + env)); recorded: the bank index of _init_qpos after each reset (-1 = None).
  * FurnitureEnv._do_simulation (:2857-2897) with a sim.step that raises: what _init_qpos is when the except branch calls reset().
A state's qpos is filled with its tag (bank index, 100 for the fixed start), so that the trace names the state set_env_state plants.
"""
import os
import sys
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_assembly import import_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
SEED = 123  # default_config's seed
FIXED = 100


class Data:
    """sim.data of the stand-in: records the qpos set_env_state plants and the arm's gravity compensation"""

    def __init__(self, env, log):
        self.env, self.log = env, log
        self.time = 0

    def __getattr__(self, name):
        if name in ("qpos", "qvel", "ctrl", "qfrc_applied", "xfrc_applied", "qacc", "qacc_warmstart", "qfrc_bias"):
            return Watch(name, self)
        raise AttributeError(name)


class Watch:
    def __init__(self, name, data):
        self.name, self.data = name, data

    def __setitem__(self, idx, val):
        if self.name == "qpos":
            self.data.log.append("set_state(%d)" % int(np.ravel(val)[0]))
        elif self.name == "qfrc_applied" and idx is self.data.env._ref_joint_vel_indexes_all:
            self.data.log.append("grav_comp")

    def __getitem__(self, idx):
        return 0.0


class Sim:
    """MjSim stand-in: two geoms, a robot one (whose collision flag every event reports) and a part's collision geom"""

    def __init__(self, env, log, sites):
        self.log, self.env = log, env
        m = types.SimpleNamespace()
        m.geom_bodyid = [0, 1]
        m.body_names = ["right_l0", "part0"]
        m.geom_id2name = lambda g: ["right_l0_collision", "part0_collision"][g]
        m.geom_contype = np.array([1, 0])
        m.geom_conaffinity = np.array([1, 0])
        m.eq_obj1id, m.eq_obj2id = np.array([1, 1]), np.array([1, 1])
        m.eq_active = np.array([0, 0])
        m.site_name2id = sites.index
        self.model = m
        self.data = Data(env, log)

    def _rc(self):
        return int(self.model.geom_contype[0] != 0)

    def reset(self):
        self.log.append("reset")

    def forward(self):
        self.log.append("forward:rc%d" % self._rc())

    def step(self):
        self.log.append("step:rc%d" % self._rc())


def stand_in(FurnitureEnv, recipe, k, init_qpos, bank):
    class StandIn(FurnitureEnv):
        _right_hand_quat = None  # a property of the reference that reads the simulator

    env = object.__new__(StandIn)
    log = []
    sites = sorted({s for row in (recipe or {}).get("site_recipe", []) for s in row[:2]})
    env.sim = Sim(env, log, sites)
    env._config = types.SimpleNamespace(furniture_name="table_lack_0825", furn_size_rand=0, assembled=False, fix_init=False, background=None)
    env._furniture_id, env._manual_resize = 0, None
    env._load_init_states, env._init_qpos = bank, init_qpos
    env._object_names, env._object_body_ids = ["part0"], [1]
    env._object_body_id2name = {1: "part0"}
    env.mujoco_robot = types.SimpleNamespace(is_robot_part=lambda name: name.startswith("right_"))
    env._agent_type, env._control_type = "Sawyer", "impedance"
    env._num_connects, env._preassembled = None, list(range(k))
    env._recipe = recipe
    env.init_pos = None
    env._ref_joint_vel_indexes_all, env._ref_gripper_joint_vel_indexes_all = [0], [1]
    env._record_demo, env._unity = False, None
    env._place_objects = lambda: (log.append("place_objects"), ({"part0": [0, 0, 0]}, {"part0": [1, 0, 0, 0]}))[1]
    env._set_qpos = lambda *a: None
    env._stop_objects = lambda gravity=1: log.append("stop_objects(%d)" % gravity)
    env._slow_objects = lambda: log.append("slow_objects")
    env._initialize_robot_pos = lambda: log.append("initialize_robot_pos")
    env._project_connector_quat = lambda *a: np.array([1.0, 0, 0, 0])
    env._connect = lambda s1, s2, auto_align=True: log.append("connect(%s,%s,auto_align=%d):rc%d" % (sites[s1], sites[s2], int(auto_align), env.sim._rc()))
    env._merge_groups = lambda a, b: log.append("merge_groups")
    env._get_next_subtask = lambda: None
    env._unity = None
    return env, log


def state(tag, nq=4):
    return {"qpos": np.full(nq, float(tag)), "qvel": np.zeros(nq)}


class NpWithRandom(types.ModuleType):
    """numpy with `random` replaced by one seeded RandomState, for the module global `np` of furniture.py"""

    def __init__(self, rs):
        super().__init__("numpy")
        self.random = rs

    def __getattr__(self, name):
        return getattr(np, name)


def run_reset(FurnitureEnv, env, rs):
    g = FurnitureEnv._reset.__globals__
    saved = g["np"]
    g["np"] = NpWithRandom(rs)
    try:
        env._reset()
    finally:
        g["np"] = saved


def main():
    T, FurnitureEnv = import_reference()
    from furniture.env.models import furniture_name2id

    probe = object.__new__(FurnitureEnv)
    probe._furniture_id = furniture_name2id["table_lack_0825"]
    FurnitureEnv._load_recipe(probe)
    recipe = probe._recipe
    probe._unity = None
    cases = dict(start=[], env=[], k=[], recipe=[], trace=[], pick=[])
    for start, e in (("none", 0), ("fixed", 0), ("bank", 0), ("bank", 1)):  # env 0's first draw keeps None, env 1's picks
        for k in (0, 1, 2):
            for with_recipe in (True, False):
                bank = [state(i) for i in range(3)] if start == "bank" else None
                env, log = stand_in(FurnitureEnv, recipe if with_recipe else None, k, state(FIXED) if start == "fixed" else None, bank)
                run_reset(FurnitureEnv, env, np.random.RandomState(SEED + 2**20 + e))
                cases["start"].append(start); cases["env"].append(e); cases["k"].append(k); cases["recipe"].append(with_recipe)
                cases["trace"].append("\n".join(log))
                cases["pick"].append(-1 if env._init_qpos is None else int(env._init_qpos["qpos"][0]))
    picks = dict(S=[], env=[], picks=[])
    for S in (1, 3, 7):
        for e in range(8):
            env, log = stand_in(FurnitureEnv, None, 0, None, [state(i) for i in range(S)])
            rs = np.random.RandomState(SEED + 2**20 + e)
            out = []
            for _ in range(20):
                run_reset(FurnitureEnv, env, rs)
                out.append(-1 if env._init_qpos is None else int(env._init_qpos["qpos"][0]))
            picks["S"].append(S); picks["env"].append(e); picks["picks"].append(out)
    # _do_simulation's except branch: the start it resets from
    env, log = stand_in(FurnitureEnv, None, 0, state(FIXED), None)
    env._control_timestep, env._model_timestep, env._cur_time = 0.1, 0.002, 0.0

    def boom():
        raise RuntimeError("unstable")

    env.sim.step = boom
    seen = []
    env.reset = lambda *a, **kw: seen.append(-1 if env._init_qpos is None else int(env._init_qpos["qpos"][0]))
    FurnitureEnv._do_simulation(env, None)
    assert seen and env._fail
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, "init_states.npz"), **{"case_" + k: np.array(v) for k, v in cases.items()},
                        **{"pick_" + k: np.array(v) for k, v in picks.items()}, except_reset_start=np.array(seen), except_fail=np.array(bool(env._fail)),
                        fixed_tag=np.array(FIXED), seed=np.array(SEED),
                        source="reference FurnitureEnv._reset / set_init_qpos / set_env_state / _do_simulation run unmodified on a recording "
                               "stand-in (tools/make_golden_init_states.py)")
    for s, e, k, r, t, pk in zip(cases["start"], cases["env"], cases["k"], cases["recipe"], cases["trace"], cases["pick"]):
        print(s, e, k, r, len(t.split("\n")), pk)


if __name__ == "__main__":
    main()
