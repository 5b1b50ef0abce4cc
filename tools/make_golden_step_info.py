"""Golden vectors for the info dict of every env step: the sparse reward's four terms and the episode record, made by running the
REFERENCE'S OWN Python, unmodified.

Runs only where the reference checkout is (make_golden_assembly.REF); writes tests/golden/step_info.npz, which travels.
What is executed from the reference: furniture/env/furniture.py FurnitureEnv._compute_reward and _ctrl_penalty (:482-550), then
FurnitureEnv._after_step (:451-480), as FurnitureEnv.step chains them (:364-385: reward += penalty), and FurnitureEnv._after_reset
(:351-362) for every reset.  The simulator is the contact stand-in of make_golden_task_options.py, here with one arm (_arms = ["right"])
or two (["right", "left"], each with its own finger geoms): per step and per part, a contact of the part with arm 0's left / right finger,
arm 1's left / right finger and the floor.  The script sets the connection count; the `done` that _step passes to _after_step is its
success test (:438-445, restated here).  A failed step is _do_simulation's except branch (:2889-2897) in its order: reset() (the
episode's counters and the touched / picked flags start again, _after_reset runs), then _fail = True; no finger touches anything.
On the two-arm env FurnitureBaxterEnv._step adds info["ac"] = a (furniture_baxter.py:75), restated here.
Recorded per step: case, arms, coefficient set, episode length, per-part touch bits (1 / 2 arm 0's left / right finger, 4 floor, 8 / 16
arm 1's left / right finger), num_connected, fail, the action, the reference's reward (penalty included), done, the env's episode length,
and its info dict: every key (joined with ","), the four reward terms and, where the step ends the episode, the episode keys
(episode_time, a wall clock, is not recorded; NaN / -1 elsewhere).
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_assembly as G  # noqa: E402
from make_golden_controllers import savez  # noqa: E402
from make_golden_task_options import COEFS, FLOOR, LENGTHS, LF, NPART, RF, STEPS  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden")
LF2, RF2 = (14, 15), (16, 17)  # arm 1's finger geoms in the stand-in
TERMS = ("success_reward", "touch_reward", "pick_reward", "ctrl_penalty")
EPISODE = ("episode_success", "episode_reward", "episode_length", "episode_unstable", "episode_num_connected")
# scripted touch bits of the first steps of every case, before the random ones: one arm's fingers, both arms' fingers on one part, the
# fingers of different arms on one part, floor contact before and after a grasp
SCRIPT = [[1, 2, 0, 0, 0], [3 | 4, 0, 1 | 16, 0, 0], [3, 8 | 2, 24 | 4, 0, 0], [4, 0, 24, 3 | 24, 1 | 8]]


def main():
    _, FurnitureEnv = G.import_reference()
    bodyid = np.zeros(20 + NPART, np.int64)
    bodyid[20:] = 1 + np.arange(NPART)
    model = types.SimpleNamespace(geom_bodyid=bodyid, geom_name2id=lambda name: {"FLOOR": FLOOR}[name])
    rng = np.random.RandomState(20261019)
    cols = ("case", "arms", "coef", "length", "bits", "num_connected", "fail", "ac", "reward", "done", "episode_length", "keys", "terms",
            "episode", "success_state")
    rec = {k: [] for k in cols}
    case = 0
    for arms in (["right"], ["right", "left"]):
        two = len(arms) == 2
        dof = 17 if two else 9  # Baxter impedance: (7 + 1) x 2 + 1 (furniture_baxter.py:58-59); Sawyer: 7 + 1 + 1
        for c, coef in enumerate(COEFS):
            for L in LENGTHS:
                env = object.__new__(FurnitureEnv)
                env._agent_type, env._arms, env._unity = "Baxter" if two else "Sawyer", list(arms), None
                env._object_body_ids = list(1 + np.arange(NPART))
                env.l_finger_geom_ids = {"right": list(LF), "left": list(LF2)}
                env.r_finger_geom_ids = {"right": list(RF), "left": list(RF2)}
                env._config = types.SimpleNamespace(success_reward=coef[0], touch_reward=coef[1], pick_reward=coef[2], ctrl_penalty_coef=coef[3],
                                                    unstable_penalty_coef=coef[4])
                env._max_episode_steps = int(L)
                env.get_env_state = lambda: {"qpos": np.zeros(1), "qvel": np.zeros(1)}

                def reset(env=env):  # what FurnitureEnv.reset leaves of the reward's state (furniture.py:318-334, :1477-1481), then _after_reset
                    env._touched = {b: False for b in env._object_body_ids}
                    env._picked = {b: False for b in env._object_body_ids}
                    env._num_connected = env._prev_num_connected = 0
                    FurnitureEnv._after_reset(env)

                reset()
                for k in range(STEPS):
                    fail = k >= len(SCRIPT) and rng.uniform() < 0.08
                    bits = np.zeros(NPART, np.int64)
                    if fail:  # _do_simulation's except branch: self.reset(), then self._fail = True
                        reset()
                        env._fail = True
                    else:
                        if k < len(SCRIPT):
                            bits[:] = SCRIPT[k]
                        else:
                            for p in range(NPART):
                                u = rng.uniform(size=5)
                                bits[p] = (1 if u[0] < 0.35 else 0) | (2 if u[1] < 0.35 else 0) | (4 if u[2] < 0.5 else 0)
                                if two:
                                    bits[p] |= (8 if u[3] < 0.35 else 0) | (16 if u[4] < 0.35 else 0)
                        if not two:
                            bits &= 7
                        if k >= len(SCRIPT) - 1 and rng.uniform() < 0.5:
                            env._num_connected = min(env._num_connected + 1, NPART - 1)
                    contacts = []
                    for p in range(NPART):
                        for bit, g in ((1, LF[p % 2]), (2, RF[p % 2]), (4, FLOOR), (8, LF2[p % 2]), (16, RF2[p % 2])):
                            if bits[p] & bit:
                                contacts.append(types.SimpleNamespace(geom1=20 + p, geom2=g) if p % 2 else types.SimpleNamespace(geom1=g, geom2=20 + p))
                    env.sim = types.SimpleNamespace(model=model, data=types.SimpleNamespace(ncon=len(contacts), contact=contacts))
                    ac = rng.uniform(-1, 1, dof)
                    ac[-1] = -1.0  # no connect request: the connection count is the script's
                    num_connected = env._num_connected
                    env._success = num_connected == NPART - 1
                    reward, _, info = FurnitureEnv._compute_reward(env, ac)
                    if two:
                        info["ac"] = ac
                    done, info, penalty = FurnitureEnv._after_step(env, reward, env._success, info)
                    reward += penalty
                    ep = [np.nan] * len(EPISODE)
                    if done:
                        ep = [float(info[key]) for key in EPISODE]
                    for key, v in (("case", case), ("arms", len(arms)), ("coef", c), ("length", L), ("bits", bits), ("num_connected", num_connected),
                                   ("fail", fail), ("ac", np.pad(ac, (0, 17 - dof))), ("reward", reward), ("done", done),
                                   ("episode_length", env._episode_length), ("keys", ",".join(info)), ("terms", [float(info[t]) for t in TERMS]),
                                   ("episode", ep), ("success_state", "episode_success_state" in info)):
                        rec[key].append(v)
                    if done:  # the VecEnv worker resets a finished env (subproc_vec_env.py:16-20)
                        reset()
                case += 1
    out = {k: np.array(v) for k, v in rec.items()}
    out.update(coefs=COEFS, lengths=LENGTHS, terms_keys=np.array(TERMS), episode_keys=np.array(EPISODE),
               source=np.array("reference FurnitureEnv._compute_reward / _ctrl_penalty / _after_step / _after_reset run unmodified on a scripted "
                               "contact stand-in with one and two arms (tools/make_golden_step_info.py)"))
    os.makedirs(OUT, exist_ok=True)
    savez(os.path.join(OUT, "step_info.npz"), **out)
    print("steps", len(rec["reward"]), "done", int(out["done"].sum()), "fail", int(out["fail"].sum()), "success", int(out["success_state"].sum()))


if __name__ == "__main__":
    main()
