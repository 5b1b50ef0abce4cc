"""Golden vectors for `assembled` (config/furniture.py:307-312), made by running the REFERENCE'S OWN Python, unmodified.

Runs only where the reference checkout is (make_golden_assembly.REF); writes tests/golden/assembled.npz, which travels.
What is executed from the reference, on the recording stand-in of make_golden_init_states.py / make_golden_reset_options.py with the
scene's real names (bodies, geoms, sites, welds) and masks:
  * furniture/env/furniture.py  FurnitureEnv._reset (:1406-1663), _place_objects (:1389-1404) with FloorTask.place_objects and
    UniformRandomSampler (the env's numpy RandomState(123)), _connect (:847-924), _activate_weld (:2761-2776), _find_group / _merge_groups
    (:2738-2759) and _get_next_subtask (:2723-2736).  The simulator does not move anything: sim.reset() puts every part at the scene's
    qpos0, _set_qpos writes the pose table (and is recorded), _get_qpos reads it; _align_connectors, _get_bounding_box (a box above the
    floor), _initialize_robot_pos, _stop_objects and _slow_objects are recorders.  eq_data is a model array: nothing resets it.
  Recorded after every reset: eq_active, eq_data, _object_group, which parts were _set_qpos'd, the 32-bit words the reset drew, init_pos /
  init_quat, every geom's contype / conaffinity, _num_connected, _success_num_conn and (_subtask_part1, _subtask_part2).
  Cases (assembled on unless named): table_lack_0825 x {random placement, fix_init over two resets, fix_init_parts 1_part1 + 3_part3, a
  recorded start} x k = 0, 1, 2 preassembled recipe steps; k = 0 on a furniture without a recipe and on Baxter + chair_ingolf_0650; and an
  episode of connections (a reset with k = 2, assembled off) followed by an assembled reset, whose eq_data is the one the connections left.
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
from make_golden_reset_options import placement_env, words  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden")
NORECIPE = "table_klubbo_0740"
# case: (agent, furniture, start, k, assembled per reset)
CASES = ([("Sawyer", "table_lack_0825", s, k, (True,) * (2 if s == "fix_init" else 1)) for s in ("random", "fix_init", "fix_init_parts", "init_state")
          for k in (0, 1, 2)]
         + [("Sawyer", NORECIPE, "random", 0, (True,)), ("Baxter", "chair_ingolf_0650", "random", 0, (True,)),
            ("Sawyer", "table_lack_0825", "random", 2, (False, True))])
R, P, NG, NE = 2, 16, 64, 16  # resets, parts, geoms, welds (padded)


def recipe_of(FurnitureEnv, furniture):
    from furniture.env.models import furniture_name2id

    probe = object.__new__(FurnitureEnv)
    probe._furniture_id, probe._unity = furniture_name2id[furniture], None
    FurnitureEnv._load_recipe(probe)
    return probe._recipe


def case_env(FurnitureEnv, agent, furniture, start, k):
    from furniture_b200 import mjcf

    m = mjcf.load_scene(agent, furniture)
    names = list(m.meta["part_names"])
    recipe = recipe_of(FurnitureEnv, furniture) if agent == "Sawyer" else None  # the two-arm scenes pack no recipe
    env, rng, names, planted, _ = placement_env(FurnitureEnv, furniture, start == "fix_init", ("1_part1", "3_part3") if start == "fix_init_parts" else (), 0.02)
    if agent != "Sawyer":  # placement_env composes the Sawyer scene of the furniture; the sampler only needs its part names and radii
        assert names == list(m.meta["part_names"])
    init_qpos = {"qpos": np.zeros(m.nq), "qvel": np.zeros(m.nv)} if start == "init_state" else None
    shell, _ = stand_in(FurnitureEnv, recipe, k, init_qpos, None)
    shell._unity = None
    env.sim = shell.sim
    env._recipe, env._preassembled, env._init_qpos, env._load_init_states = recipe, list(range(k)), init_qpos, None
    env._config.assembled, env._config.reset_robot_after_attach = False, False
    # the scene's names and masks in place of the stand-in's two geoms
    bn, gn, sn = m.names["body"], m.names["geom"], m.names["site"]
    sm = env.sim.model
    sm.body_names, sm.geom_bodyid = bn, list(m.geom_bodyid)
    sm.geom_id2name, sm.body_id2name, sm.body_name2id = (lambda g: gn[g]), (lambda b: bn[b]), bn.index
    sm.site_names, sm.site_bodyid, sm.site_name2id = sn, list(m.site_bodyid), sn.index
    sm.geom_contype, sm.geom_conaffinity = np.array(m.geom_contype, dtype=np.int64), np.array(m.geom_conaffinity, dtype=np.int64)
    sm.eq_obj1id, sm.eq_obj2id = np.array(m.eq_obj1id), np.array(m.eq_obj2id)
    sm.eq_active, sm.eq_data = np.zeros(m.neq, np.int64), np.array(m.eq_data, np.float64).reshape(m.neq, 7)
    robot_prefix = ("right_", "left_", "r_", "l_", "base", "pedestal", "head", "torso")
    env.mujoco_robot = types.SimpleNamespace(is_robot_part=lambda name: bool(name) and name.startswith(robot_prefix))
    env._object_body_ids = [bn.index(n) for n in names]
    env._object_body_id2name = {bn.index(n): n for n in names}
    env._object_name2id = {n: i for i, n in enumerate(names)}
    env._agent_type = "Sawyer"  # the two-arm env's _reset differs only in the hand quaternion it reads at the end, which the stand-in has not
    # the pose table the stand-in simulator holds: sim.reset() puts every part at qpos0
    qpos0 = {n: np.array(m.qpos0[int(m.jnt_qposadr[m.names["jnt"].index(n)]) :][:7], np.float64) for n in names}
    poses = {}
    reset = env.sim.reset

    def sim_reset():
        reset()
        poses.update({n: q.copy() for n, q in qpos0.items()})

    env.sim.reset = sim_reset
    moved = []

    def set_qpos(body, pos, quat=(1, 0, 0, 0)):
        moved.append(body)
        planted[body] = (np.asarray(pos, np.float64), np.asarray(list(quat), np.float64))
        poses[body] = np.concatenate([np.asarray(pos, np.float64), np.asarray(list(quat), np.float64)])

    env._set_qpos = set_qpos
    env._get_qpos = lambda name: poses[name].copy()
    for f in ("_connect", "_activate_weld", "_find_group", "_merge_groups", "_get_next_subtask"):
        setattr(env, f, types.MethodType(getattr(FurnitureEnv, f), env))
    env._align_connectors = lambda *a, **kw: None
    env._get_bounding_box = lambda body: (np.zeros(3), np.ones(3))
    env._gravity_compensation = 0
    env._connected_sites = set()
    return env, rng, m, names, moved


def main():
    T, FurnitureEnv = G.import_reference()
    assert recipe_of(FurnitureEnv, NORECIPE) is None
    out = collections.defaultdict(list)
    for agent, furniture, start, k, assembled in CASES:
        env, rng, m, names, moved = case_env(FurnitureEnv, agent, furniture, start, k)
        rec = collections.defaultdict(list)
        for r in range(R):
            if r < len(assembled):
                env._config.assembled = assembled[r]
                del moved[:]
                s0 = rng.get_state()
                eq_before = np.array(env.sim.model.eq_data, np.float64)
                env._reset()
                rec["words"].append(words(s0, rng.get_state()))
                rec["moved"].append([n in moved for n in names] + [False] * (P - len(names)))
                rec["group"].append(list(env._object_group) + [-9] * (P - len(names)))
                rec["eq_active"].append(list(env.sim.model.eq_active) + [-9] * (NE - m.neq))
                rec["eq_data"].append(np.vstack([env.sim.model.eq_data, np.zeros((NE - m.neq, 7))]))
                rec["eq_data_before"].append(np.vstack([eq_before, np.zeros((NE - m.neq, 7))]))
                ip = np.zeros((P, 7))
                for i, n in enumerate(names):
                    ip[i, :3], ip[i, 3:] = np.asarray(env.init_pos[n], np.float64), np.asarray(list(env.init_quat[n]), np.float64)
                rec["init_pos"].append(ip)
                masks = np.full((NG, 2), -9, np.int64)
                masks[: m.ngeom, 0], masks[: m.ngeom, 1] = env.sim.model.geom_contype, env.sim.model.geom_conaffinity
                rec["masks"].append(masks)
                rec["num_connected"].append(env._num_connected)
                rec["success_num_conn"].append(env._success_num_conn)
                rec["subtask"].append([env._subtask_part1, env._subtask_part2])
            else:  # padding
                for key in list(rec):
                    rec[key].append(np.zeros_like(np.asarray(rec[key][-1])) - 9)
        for key, v in rec.items():
            out[key].append(np.array(v))
        out["case_agent"].append(agent); out["case_furniture"].append(furniture); out["case_start"].append(start); out["case_k"].append(k)
        out["case_assembled"].append(list(assembled) + [False] * (R - len(assembled))); out["case_nreset"].append(len(assembled))
        print(agent, furniture, start, k, assembled, "words", rec["words"], "group", [g[: len(names)] for g in rec["group"]][:len(assembled)],
              "subtask", rec["subtask"][: len(assembled)], "conn", rec["num_connected"][: len(assembled)])
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, "assembled.npz"), **{k: np.array(v) for k, v in out.items()},
                        source="reference FurnitureEnv._reset / _place_objects / _connect / _activate_weld / _get_next_subtask, FloorTask."
                               "place_objects, UniformRandomSampler run unmodified on a recording stand-in (tools/make_golden_assembled.py)")


if __name__ == "__main__":
    main()
