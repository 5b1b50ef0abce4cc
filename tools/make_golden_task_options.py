"""Golden vectors for the sparse reward and the episode end under several reward coefficients and episode lengths, made by running the
REFERENCE'S OWN Python, unmodified.

Runs only where the reference checkout is (make_golden_assembly.REF); writes tests/golden/task_options.npz, which travels.
What is executed from the reference: furniture/env/furniture.py FurnitureEnv._compute_reward and _ctrl_penalty (:482-550), then
FurnitureEnv._after_step (:451-480), as FurnitureEnv.step chains them (:364-385: reward += penalty).  The simulator is a stand-in whose
contact list the script fills: per step and per part, a contact of the part with the left finger, the right finger and the floor.  The
script also sets the connection count; the `done` that _step passes to _after_step is its success test (:438-445, restated here:
every part connected).  A failed step (_do_simulation's except branch, :2889-2897) is shown as the reset it triggers: the episode's
counters start again, no finger touches anything, and _fail is set.
Recorded per step: case, coefficient set, episode length, per-part touch bits (1 left finger, 2 right finger, 4 floor), num_connected,
fail, the action, and the reference's reward (penalty included), done and episode length.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_assembly as G  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden")
NPART, DOF, STEPS = 5, 9, 24  # Sawyer impedance (7 joints, gripper, connect) + table_lack_0825's five parts
# success_reward, touch_reward, pick_reward, ctrl_penalty_coef, unstable_penalty_coef: the defaults of config/furniture.py:291-295 first
COEFS = np.array([[100.0, 10.0, 100.0, 1e-3, 100.0], [50.0, 2.5, 7.0, 1e-2, 30.0], [0.0, 0.0, 0.0, 0.0, 0.0], [1.0, 0.5, 0.25, 0.5, 1000.0]])
LENGTHS = np.array([2, 3, 5, 2000])
FLOOR, LF, RF = 0, (10, 11), (12, 13)  # geom ids of the stand-in: floor, left / right finger geoms; part p's geom is 20 + p on body 1 + p


def main():
    _, FurnitureEnv = G.import_reference()
    bodyid = np.zeros(20 + NPART, np.int64)
    bodyid[20:] = 1 + np.arange(NPART)
    model = types.SimpleNamespace(geom_bodyid=bodyid, geom_name2id=lambda name: {"FLOOR": FLOOR}[name])
    rng = np.random.RandomState(20261017)
    rec = {k: [] for k in ("case", "coef", "length", "bits", "num_connected", "fail", "ac", "reward", "done", "episode_length")}
    case = 0
    for c, coef in enumerate(COEFS):
        for L in LENGTHS:
            env = object.__new__(FurnitureEnv)
            env._agent_type, env._arms, env._unity = "Sawyer", ["right"], None
            env._object_body_ids = list(1 + np.arange(NPART))
            env.l_finger_geom_ids, env.r_finger_geom_ids = {"right": list(LF)}, {"right": list(RF)}
            env._config = types.SimpleNamespace(success_reward=coef[0], touch_reward=coef[1], pick_reward=coef[2], ctrl_penalty_coef=coef[3],
                                                unstable_penalty_coef=coef[4])
            env._max_episode_steps = int(L)
            env.get_env_state = lambda: None

            def new_episode(env=env):
                env._touched = {b: False for b in env._object_body_ids}
                env._picked = {b: False for b in env._object_body_ids}
                env._num_connected = env._prev_num_connected = 0
                env._episode_reward, env._episode_length, env._episode_time = 0, 0, 0.0
                env._success, env._fail = False, False

            new_episode()
            for _ in range(STEPS):
                fail = rng.uniform() < 0.08
                bits = np.zeros(NPART, np.int64)
                if fail:
                    new_episode()
                    env._fail = True
                else:
                    for p in range(NPART):
                        u = rng.uniform(size=3)
                        bits[p] = (1 if u[0] < 0.35 else 0) | (2 if u[1] < 0.35 else 0) | (4 if u[2] < 0.5 else 0)
                    if rng.uniform() < 0.55:
                        env._num_connected = min(env._num_connected + 1, NPART - 1)
                contacts = []
                for p in range(NPART):
                    for bit, g in ((1, LF[p % 2]), (2, RF[p % 2]), (4, FLOOR)):
                        if bits[p] & bit:
                            contacts.append(types.SimpleNamespace(geom1=20 + p, geom2=g) if p % 2 else types.SimpleNamespace(geom1=g, geom2=20 + p))
                env.sim = types.SimpleNamespace(model=model, data=types.SimpleNamespace(ncon=len(contacts), contact=contacts))
                ac = rng.uniform(-1, 1, DOF)
                ac[-1] = -1.0  # no connect request: the connection count is the script's
                num_connected = env._num_connected
                env._success = num_connected == NPART - 1
                reward, _, info = FurnitureEnv._compute_reward(env, ac)
                done, _, penalty = FurnitureEnv._after_step(env, reward, env._success, info)
                reward += penalty
                for k, v in (("case", case), ("coef", c), ("length", L), ("bits", bits), ("num_connected", num_connected), ("fail", fail),
                             ("ac", ac), ("reward", reward), ("done", done), ("episode_length", env._episode_length)):
                    rec[k].append(v)
                if done:  # the VecEnv worker resets a finished env (subproc_vec_env.py:16-20)
                    new_episode()
            case += 1
    out = {k: np.array(v) for k, v in rec.items()}
    out.update(coefs=COEFS, lengths=LENGTHS, source="reference FurnitureEnv._compute_reward / _ctrl_penalty / _after_step run unmodified on a "
                                                     "scripted contact stand-in (tools/make_golden_task_options.py)")
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, "task_options.npz"), **out)
    print("steps", len(rec["reward"]), "done", int(out["done"].sum()), "fail", int(out["fail"].sum()), "touch steps", int((out["bits"] & 3 == 3).any(1).sum()))


if __name__ == "__main__":
    main()
