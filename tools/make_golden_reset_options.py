"""Golden vectors for fix_init / fix_init_parts / reset_robot_after_attach, made by running the REFERENCE'S OWN Python, unmodified.

Runs only where the reference checkout is (make_golden_assembly.REF); writes tests/golden/reset_options.npz, which travels.
What is executed from the reference, on the recording stand-in of make_golden_init_states.py:
  * furniture/env/furniture.py  FurnitureEnv._reset (:1406-1663) with _init_qpos None, FurnitureEnv._place_objects (:1389-1404),
    models/tasks/floor_task.py FloorTask.place_objects (:79-81) and models/tasks/placement_sampler.py UniformRandomSampler.setup / sample
    (:66-190) with the env's numpy RandomState(123).  init_pos / init_quat start as _load_model leaves them (:2013-2021): the XML's
    *_initpos numerics as the reference's own MujocoXMLObject.get_init_qpos (models/objects/objects.py:149-164) reads them, or None for a
    model whose XML lists none.  Recorded per reset: the pose _reset plants for every part, the draws the reset consumed (32-bit words; the
    stand-in's _initialize_robot_pos draws nothing here), the x / y tries of the reset (one sample_x call each), init_pos after it, and for
    every rejected try which placed object rejected it (the sampler's placed-objects list records what it hands out).
    Cases: fix_init x fix_init_parts (none, one leg, two legs, the table top 4_part4, whose 0.18 m radius rejects tries of the legs placed
    before it in XML order) x table_lack_0825 (XML poses) and table_klubbo_0740 (none) x furn_xyz_rand 0.02 and 0.3, 4 consecutive resets.
  * FurnitureEnv._connect (:847-924) with reset_robot_after_attach on, the real _initialize_robot_pos (:1761-1779) and _init_random
    (:336-349) on the Sawyer's init qpos; the simulator, _align_connectors, _get_bounding_box, _activate_weld and the IK controller's
    sync_state are recorders.  Recorded: the calls after the weld, the words they draw and the arm / gripper qpos they write, for a policy
    connection (impedance, ik), and the calls and words of a whole _reset (:1406-1663) that preassembles 2 recipe steps, after random
    placement and from a recorded start.
"""
import collections
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
import make_golden_assembly as G  # noqa: E402
from make_golden_init_states import stand_in  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden")
ASSETS = os.path.join(G.REF, "furniture", "env", "models", "assets")
SEED = 123
NRESET = 4


def words(s0, s1):
    """32-bit words a RandomState consumed between states s0 and s1, replayed one word at a time"""
    rs = np.random.RandomState()
    rs.set_state(s0)
    n = 0
    while not (rs.get_state()[2] == s1[2] and np.array_equal(rs.get_state()[1], s1[1])):
        rs.bytes(4)
        n += 1
    return n


class PlacedList(list):
    """the sampler's placed-objects list (copy.copy of fixed_parts keeps the type): logs the name of every entry the overlap test reads, and
    every append, so that the last name read before a new try is the object that rejected the try before it"""
    log = None

    def __iter__(self):
        for item in list.__iter__(self):
            if PlacedList.log is not None:
                PlacedList.log.append(("read", item[0]))
            yield item

    def append(self, item):
        if PlacedList.log is not None:
            PlacedList.log.append(("append", item[0]))
        list.append(self, item)


def rejections(log, names):
    """sampler events -> "part<rejecter" for every rejected try, in order: a try that another try follows was rejected by the last object it
    read; an append ends the tries of the part it places"""
    out, pending, reads = [], [], None
    for ev, name in log:
        if ev == "try":
            if reads is not None:
                pending.append(reads[-1])
            reads = []
        elif ev == "read" and reads is not None:
            reads.append(name)
        elif ev == "append":
            out += ["%s<%s" % (name, r) for r in pending]
            pending, reads = [], None
    return ";".join(out)


def placement_env(FurnitureEnv, furniture, fix_init, parts, xyz):
    from furniture.env.models.objects import MujocoXMLObject
    from furniture.env.models.tasks.floor_task import FloorTask
    from furniture.env.models.tasks.placement_sampler import UniformRandomSampler
    from furniture.util import Qpos

    from furniture_b200 import mjcf

    m = mjcf.load_scene("Sawyer", furniture)
    meta, names = m.meta, list(m.meta["part_names"])
    xml = mjcf.xml_init_poses(meta)

    class FakeObject:  # the MujocoXMLObject queries the sampler and _place_objects make
        def get_horizontal_radius(self, name):
            return meta["part_radius"][name]

    objs = collections.OrderedDict((n, FakeObject()) for n in names)
    env, log = stand_in(FurnitureEnv, None, 0, None, None)
    rng = np.random.RandomState(SEED)
    base = {n: Qpos(q[0], q[1], q[2], G.Quaternion(q[3], q[4], q[5], q[6])) for n, q in meta["part_init_qpos"].items()}
    sampler = UniformRandomSampler(rng, r_xyz=xyz, r_rot=3, init_qpos=base)  # floor_task.py:33-34
    sampler.setup(objs, (0, 0, 0), (0.7, 0.7, 0))                           # floor_task.py:37
    tries = []
    sample_x = sampler.sample_x

    def logged_x(r):
        tries.append(1)
        if PlacedList.log is not None:
            PlacedList.log.append(("try", None))
        return sample_x(r)

    sampler.sample_x = logged_x
    env._config.fix_init, env._config.fix_init_parts = fix_init, set(parts) if parts else None
    env._object_names = names
    env.mujoco_objects = objs
    env.mujoco_model = types.SimpleNamespace(initializer=sampler)
    env.mujoco_model.place_objects = lambda fixed_parts=None: FloorTask.place_objects(env.mujoco_model, fixed_parts)
    env.fixed_parts = PlacedList()
    FurnitureEnv._load_model  # where init_pos starts (:2013-2021), read here with the reference's own reader of the XML
    ref_xml = MujocoXMLObject(os.path.join(ASSETS, "objects", furniture + ".xml")).get_init_qpos(names)
    assert (ref_xml is None) == (xml is None)
    env.init_pos = None if ref_xml is None else {n: [q.x, q.y, q.z] for n, q in ref_xml.items()}
    env.init_quat = None if ref_xml is None else {n: q.quat for n, q in ref_xml.items()}
    env._place_objects = types.MethodType(FurnitureEnv._place_objects, env)
    planted = {}
    env._set_qpos = lambda body, pos, quat: planted.__setitem__(body, (np.asarray(pos, np.float64), np.asarray(list(quat), np.float64)))
    return env, rng, names, planted, tries


def connect_env(FurnitureEnv, ctl, recipe=None, k=0, init_qpos=None):
    """the stand-in with the reference's own _connect, _initialize_robot_pos and _init_random; `calls` records what matters here"""
    from furniture_b200 import mjcf

    sites = sorted({s for row in (recipe or {}).get("site_recipe", []) for s in row[:2]}) or ["a", "b"]
    env, log = stand_in(FurnitureEnv, recipe, k, init_qpos, None)
    calls = []
    env._rng = np.random.RandomState(SEED)
    env._config.reset_robot_after_attach = True
    env._config.agent_xyz_rand = 0.001
    env._control_type = ctl
    env._arms = ["right"]
    env.mujoco_robot = types.SimpleNamespace(init_qpos=mjcf.SAWYER_INIT_QPOS.copy(), is_robot_part=lambda name: name.startswith("right_"))
    env.gripper = {"right": types.SimpleNamespace(init_qpos=mjcf.GRIPPER_INIT_QPOS.copy())}
    env._ref_joint_pos_indexes_all, env._ref_gripper_joint_pos_indexes = list(range(7)), {"right": [7, 8]}
    qpos = np.zeros(9)

    class Data:
        def __getattr__(self, name):
            if name == "qpos":
                return qpos
            return env_data.__getattr__(name)

    env_data = env.sim.data
    env.sim.data = Data()
    m = env.sim.model
    m.site_names, m.site_bodyid = sites, [1] * len(sites)
    m.site_name2id = sites.index
    m.body_id2name = lambda b: ["right_l0", "part0"][b]
    m.body_names = ["right_l0", "part0"]
    env._connected_sites, env._num_connected, env._gravity_compensation = set(), 0, 0
    env._find_group = lambda body: 0
    env._align_connectors = lambda *a, **kw: None
    env._get_bounding_box = lambda body: (np.zeros(3), np.zeros(3))
    env._activate_weld = lambda *a: calls.append("activate_weld")
    env._get_qpos = lambda body: np.zeros(7)
    env._get_next_subtask = lambda: calls.append("get_next_subtask")
    env._controller = types.SimpleNamespace(sync_state=lambda: calls.append("sync_state"))
    init_robot = types.MethodType(FurnitureEnv._initialize_robot_pos, env)
    env._initialize_robot_pos = lambda: (calls.append("initialize_robot_pos"), init_robot())[1]
    connect = types.MethodType(FurnitureEnv._connect, env)
    env._connect = lambda s1, s2, auto_align=True: (calls.append("connect"), connect(s1, s2, auto_align=auto_align))[1]
    return env, calls, qpos, sites


def connect_cases(FurnitureEnv):
    from furniture.env.models import furniture_name2id

    probe = object.__new__(FurnitureEnv)
    probe._furniture_id = furniture_name2id["table_lack_0825"]
    FurnitureEnv._load_recipe(probe)
    recipe = probe._recipe
    probe._unity = None
    out = collections.defaultdict(list)
    for case, ctl in (("policy", "impedance"), ("policy", "ik"), ("preassembly_random", "impedance"), ("preassembly_init_state", "impedance")):
        init = {"qpos": np.zeros(9), "qvel": np.zeros(9)} if case == "preassembly_init_state" else None
        env, calls, qpos, sites = connect_env(FurnitureEnv, ctl, recipe if case != "policy" else None, 2 if case != "policy" else 0, init)
        s0 = env._rng.get_state()
        if case == "policy":
            env._connect(0, 1)
        else:
            env._reset()
        out["case"].append(case); out["control"].append(ctl); out["calls"].append(";".join(calls))
        out["words"].append(words(s0, env._rng.get_state())); out["qpos"].append(qpos.copy())
        print(case, ctl, ";".join(calls)[:200], words(s0, env._rng.get_state()))
    return out


def main():
    T, FurnitureEnv = G.import_reference()
    cases = collections.defaultdict(list)
    pos, quat, draws, tries, init_pos, rejects = [], [], [], [], [], []
    P = 16
    for furniture in ("table_lack_0825", "table_klubbo_0740"):
        for xyz in (0.02, 0.3):
            for fix_init in (False, True):
                for parts in ((), ("1_part1",), ("1_part1", "3_part3"), ("4_part4",)):
                    env, rng, names, planted, tlog = placement_env(FurnitureEnv, furniture, fix_init, parts, xyz)
                    cp, cq, cd, ct, ci, cr = [], [], [], [], [], []
                    for r in range(NRESET):
                        s0 = rng.get_state()
                        tlog.clear()
                        PlacedList.log = []
                        env._reset()
                        cr.append(rejections(PlacedList.log, names))
                        PlacedList.log = None
                        s1 = rng.get_state()
                        cp.append(np.zeros((P, 3))); cq.append(np.zeros((P, 4))); ci.append(np.zeros((P, 7)))
                        for k, n in enumerate(names):
                            cp[-1][k], cq[-1][k] = planted[n]
                            ci[-1][k, :3] = np.asarray(env.init_pos[n], np.float64)
                            ci[-1][k, 3:] = np.asarray(list(env.init_quat[n]), np.float64)
                        cd.append(words(s0, s1))
                        ct.append(len(tlog))
                    pos.append(cp); quat.append(cq); draws.append(cd); tries.append(ct); init_pos.append(ci); rejects.append(cr)
                    cases["furniture"].append(furniture); cases["xyz"].append(xyz); cases["fix_init"].append(fix_init)
                    cases["parts"].append(",".join(parts)); cases["npart"].append(len(names))
                    print(furniture, xyz, fix_init, parts, "draws", cd, "tries", ct, "rejected", cr)
    conn = connect_cases(FurnitureEnv)
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, "reset_options.npz"), **{"case_" + k: np.array(v) for k, v in cases.items()},
                        pos=np.array(pos), quat=np.array(quat), draws=np.array(draws), tries=np.array(tries), init_pos=np.array(init_pos),
                        rejected=np.array(rejects), **{"connect_" + k: np.array(v) for k, v in conn.items()}, seed=np.array(SEED),
                        source="reference FurnitureEnv._reset / _place_objects / _connect / _initialize_robot_pos, FloorTask.place_objects, "
                               "UniformRandomSampler run unmodified "
                               "on a recording stand-in (tools/make_golden_reset_options.py)")


if __name__ == "__main__":
    main()
