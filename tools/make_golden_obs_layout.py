"""Golden vectors for the observation flags robot_ob / object_ob / object_ob_all / subtask_ob, made by running the REFERENCE'S OWN Python,
unmodified.

Runs only where the reference checkout is (make_golden_assembly.REF); writes tests/golden/obs_layout.npz, which travels.
What is executed from the reference:
  * FurnitureEnv._get_obs (furniture.py:1344-1387) and observation_space (:215-252) through the agents' FurnitureSawyerEnv /
    FurnitureBaxterEnv._get_obs and observation_space (furniture_sawyer.py:27-48, :103-155; furniture_baxter.py:27-48, :98-175), on a stand-in
    whose _get_pos / _get_quat return tagged part poses (part i: pos 100 i + (1, 2, 3), quat 100 i + (4 .. 7)) and whose sim.data returns tagged
    robot readings; gym.spaces.Box is a stub that records shapes.  Cases: the 16 flag combinations x control_type impedance / ik x the pairs
    the merges below produce, for Sawyer + table_lack_0825, Baxter + chair_ingolf_0650 and Sawyer + block (two parts).
  * _get_next_subtask, _find_group and _merge_groups (:2723-2759) over the welds of the compiled scene (eq_obj1id / eq_obj2id and body names
    from furniture_b200/compiled): scripted merge sequences, in weld order, out of it, and to the finished assembly (-1 / -1).
  * FurnitureSawyerDenseRewardEnv._update_reward_variables (furniture_sawyer_dense.py:149-219) for every recipe step of table_lack_0825:
    the pair it sets.
"""
import itertools
import os
import sys
import types
from collections import OrderedDict

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden_assembly import import_reference  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden")
FLAGS = ("robot_ob", "object_ob", "object_ob_all", "subtask_ob")
SCENES = (("Sawyer", "table_lack_0825"), ("Baxter", "chair_ingolf_0650"), ("Sawyer", "block"))
# merge sequences by part index (the pair _connect merges); table_lack_0825: 0..3 legs, 4 table; chair_ingolf_0650 and block as compiled
MERGES = {
    "table_lack_0825": [[], [(0, 4)], [(2, 4)], [(2, 4), (0, 4)], [(3, 4), (1, 4), (0, 4)], [(0, 4), (1, 4), (2, 4), (3, 4)]],
    "chair_ingolf_0650": None,  # every weld in model order, then in reverse
    "block": [[], [(0, 1)]],
}


class Box:
    """gym.spaces.Box stand-in: records the shape"""

    def __init__(self, low=None, high=None, shape=None, dtype=None):
        self.shape = tuple(shape)


class Spaces(types.ModuleType):
    Box = Box

    @staticmethod
    def Dict(d):
        return types.SimpleNamespace(spaces=d)


class Data:
    """sim.data with tagged robot readings: qpos[x] = 1000 + x, qvel[x] = 2000 + x, site_xpos[s] = 3000 + 10 s + (0, 1, 2), hand xquat
    (wxyz) = 4000 + 10 h + (0 .. 3), site_xvelp / xvelr = 5000 / 6000 + 10 s + (0, 1, 2)"""

    def __init__(self):
        self.qpos = 1000.0 + np.arange(200)
        self.qvel = 2000.0 + np.arange(200)
        self.site_xpos = 3000.0 + 10 * np.arange(8)[:, None] + np.arange(3)
        self.site_xvelp = 5000.0 + 10 * np.arange(8)[:, None] + np.arange(3)
        self.site_xvelr = 6000.0 + 10 * np.arange(8)[:, None] + np.arange(3)

    def get_body_xquat(self, name):
        return 4000.0 + 10 * ("left" in name) + np.arange(4)


def scene_welds(agent, furniture):
    from furniture_b200 import mjcf

    m = mjcf.load_scene(agent, furniture)
    return m, list(m.meta["part_names"]), [int(b) for b in m.eq_obj1id], [int(b) for b in m.eq_obj2id]


def stand_in(cls, m, parts, eq1, eq2, flags, control_type):
    env = object.__new__(cls)
    env._unity = None
    env._visual_ob = env._segmentation_ob = env._depth_ob = False
    env._camera_ids = []
    env._robot_ob, env._object_ob, env._object_ob_all, env._subtask_ob = (flags[k] for k in FLAGS)
    env._control_type = control_type
    env._config = types.SimpleNamespace(phase_ob=False)
    env._object_names = list(parts)
    env.n_objects = len(parts)
    env._object_name2id = {k: i for i, k in enumerate(parts)}
    env._object_body_id2name = {b: m.names["body"][b] for b in set(eq1) | set(eq2)}
    env._object_group = list(range(len(parts)))
    env._subtask_part1 = env._subtask_part2 = -1
    env._get_pos = lambda name: 100.0 * parts.index(name) + np.array([1.0, 2.0, 3.0])
    env._get_quat = lambda name: 100.0 * parts.index(name) + np.array([4.0, 5.0, 6.0, 7.0])
    model = types.SimpleNamespace(eq_obj1id=np.array(eq1), eq_obj2id=np.array(eq2))
    env.sim = types.SimpleNamespace(model=model, data=Data())
    env._ref_joint_pos_indexes = {"right": list(range(0, 7)), "left": list(range(20, 27))}
    env._ref_joint_vel_indexes = {"right": list(range(0, 7)), "left": list(range(20, 27))}
    env._ref_gripper_joint_pos_indexes = {"right": [7, 8], "left": [27, 28]}
    env.eef_site_id = {"right": 1, "left": 2}
    env._arms = ["right", "left"]
    return env


def main():
    T, FurnitureEnv = import_reference()
    sys.modules["gym"].spaces = Spaces("gym.spaces")
    sys.modules["gym.spaces"] = sys.modules["gym"].spaces
    from furniture.env.furniture_baxter import FurnitureBaxterEnv
    from furniture.env.furniture_sawyer import FurnitureSawyerEnv
    from furniture.env.furniture_sawyer_dense import FurnitureSawyerDenseRewardEnv
    from furniture.env.models import furniture_name2id

    agents = {"Sawyer": FurnitureSawyerEnv, "Baxter": FurnitureBaxterEnv}
    out = OrderedDict((k, []) for k in ("furniture", "agent", "merges", "pair", "flags", "control", "keys", "shapes", "space", "row"))
    for agent, furniture in SCENES:
        m, parts, eq1, eq2 = scene_welds(agent, furniture)
        seqs = MERGES[furniture]
        if seqs is None:
            pairs = [(parts.index(m.names["body"][a]), parts.index(m.names["body"][b])) for a, b in zip(eq1, eq2)]
            seqs = [pairs[:k] for k in range(len(pairs) + 1)] + [list(reversed(pairs))[:k] for k in range(1, len(pairs))]
        for merges in seqs:
            for bits in itertools.product((0, 1), repeat=4):
                flags = dict(zip(FLAGS, map(bool, bits)))
                for control in ("impedance", "ik"):
                    env = stand_in(agents[agent], m, parts, eq1, eq2, flags, control)
                    for a, b in merges:  # _connect's _activate_weld merges the two groups (:2772-2775), then _get_next_subtask (:917)
                        FurnitureEnv._merge_groups(env, a, b)
                        FurnitureEnv._get_next_subtask(env)
                    FurnitureEnv._get_next_subtask(env)  # _reset's call (:1653); no merge changes the answer after the last _connect
                    ob = agents[agent]._get_obs(env)
                    space = agents[agent].observation_space.fget(env).spaces
                    out["furniture"].append(furniture); out["agent"].append(agent)
                    out["merges"].append(";".join("%d-%d" % ab for ab in merges))
                    out["pair"].append([env._subtask_part1, env._subtask_part2])
                    out["flags"].append(list(bits)); out["control"].append(control)
                    out["keys"].append(",".join(ob.keys()))
                    out["shapes"].append(",".join(str(len(np.ravel(v))) for v in ob.values()))
                    out["space"].append(",".join("%s:%d" % (k, v.shape[0]) for k, v in space.items()))
                    out["row"].append(";".join(",".join(repr(float(x)) for x in np.ravel(v)) for v in ob.values()))
    # the dense env's pair for every recipe step (furniture_sawyer_dense.py:149-162)
    m, parts, eq1, eq2 = scene_welds("Sawyer", "table_lack_0825")
    probe = object.__new__(FurnitureSawyerDenseRewardEnv)
    probe._unity = None
    probe._furniture_id = furniture_name2id["table_lack_0825"]
    FurnitureEnv._load_recipe(probe)
    dense_pairs = []
    for k in range(len(probe._recipe["recipe"])):
        env = stand_in(FurnitureSawyerDenseRewardEnv, m, parts, eq1, eq2, dict(zip(FLAGS, (1, 1, 0, 1))), "impedance")
        env._recipe, env._site_recipe = probe._recipe, probe._site_recipe
        env._subtask_step, env._used_sites = k, set()
        env._config = types.SimpleNamespace(phase_ob=False, reset_robot_after_attach=False)
        env._diff_rew = False
        env._get_pos = lambda name: np.zeros(3)
        FurnitureSawyerDenseRewardEnv._update_reward_variables(env)
        dense_pairs.append([env._subtask_part1, env._subtask_part2])
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, "obs_layout.npz"), **{"case_" + k: np.array(v) for k, v in out.items()}, dense_pairs=np.array(dense_pairs),
                        dense_furniture=np.array("table_lack_0825"),
                        source="reference FurnitureEnv / FurnitureSawyerEnv / FurnitureBaxterEnv _get_obs and observation_space, _get_next_subtask, "
                               "_find_group, _merge_groups and FurnitureSawyerDenseRewardEnv._update_reward_variables run unmodified on a recording "
                               "stand-in (tools/make_golden_obs_layout.py)")
    print(len(out["row"]), "cases; dense pairs", dense_pairs)


if __name__ == "__main__":
    main()
