"""Golden vectors for episodes that start part-way through the assembly, made by running the REFERENCE'S OWN Python, unmodified.

Runs only where the reference checkout is (make_golden_assembly.REF); writes tests/golden/preassembled.npz, which travels.
What is executed from the reference:
  * furniture/env/furniture.py  FurnitureEnv._project_connector_quat (:1201-1222) on random connector poses, with and without an
    angle, including forwards so close to parallel / antiparallel that the cosine rounds past +-1 (the answer is then NaN, as it is there)
  * furniture/env/furniture.py  the `_success_num_conn` statement of FurnitureEnv._reset (:1477-1481), cut out of the method's source
    and executed as it stands
  * furniture/env/furniture_sawyer_dense.py  _reset_reward_variables (:128-139) with `_preassembled = range(k)` for every k the recipe
    allows, on the four recipes of tools/make_golden_dense.py, then the first _compute_reward with `_connected` False, which is
    how _reset leaves it (:1557) and how step() sets it (:392)
The simulator is a scripted world as in tools/make_golden_dense.py; here every grasp-target pair of a leg has its own position, so
that the pair a subtask claims shows in the numbers as well as in the recorded index.
"""
import ast
import inspect
import json
import os
import sys
import textwrap
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_assembly import import_reference, rand_rot, small_rot  # noqa: E402
from make_golden_dense import INFO_KEYS, MAXS, RECIPES  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
ANGLES = [None, 0, 90, 180, 270, 45]


def rot_z(deg):
    a = np.deg2rad(deg)
    return np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])


def success_num_conn_statement(FurnitureEnv):
    """the `if self._num_connects is not None: ... else: ...` statement of FurnitureEnv._reset, compiled from the reference's source"""
    fn = ast.parse(textwrap.dedent(inspect.getsource(FurnitureEnv._reset))).body[0]
    for node in ast.walk(fn):
        if isinstance(node, ast.If) and "_num_connects" in ast.dump(node.test):
            return compile(ast.Module(body=[node], type_ignores=[]), "furniture.py:_reset", "exec")
    raise RuntimeError("FurnitureEnv._reset no longer sets _success_num_conn the way this tool expects")


def main():
    T, FurnitureEnv = import_reference()
    from furniture.config import create_parser
    from furniture.env.furniture_sawyer import FurnitureSawyerEnv
    from furniture.env.furniture_sawyer_dense import FurnitureSawyerDenseRewardEnv as Dense
    from furniture.env.models import furniture_name2id

    rng = np.random.RandomState(20261016)
    # ---- _project_connector_quat
    q = dict(m1=[], m2=[], angle=[], has_angle=[], tq=[])
    for n in range(4000):
        angle = ANGLES[rng.randint(len(ANGLES))]
        R1 = rand_rot(rng)
        mode = rng.randint(5)
        if mode == 0:
            R2 = rand_rot(rng)
        elif mode == 1:  # a settled leg next to the table: same up within a few degrees, any yaw
            R2 = small_rot(rng, 6.0) @ R1 @ rot_z(rng.uniform(0, 360))
        elif mode == 2:  # forwards parallel to the last bits
            R2 = R1 @ rot_z(rng.choice([0.0, 1e-7, 1e-6, 1e-5]) * rng.choice([-1, 1]))
        elif mode == 3:  # antiparallel to the last bits
            R2 = R1 @ rot_z(180.0 + rng.choice([0.0, 1e-7, 1e-6, 1e-5]) * rng.choice([-1, 1]))
        else:  # the same matrix, or its forward and right flipped exactly
            R2 = R1.copy() if rng.rand() < 0.5 else R1 @ np.diag([-1.0, -1.0, 1.0])
        poses = {"c1": R1, "c2": R2}
        fake = types.SimpleNamespace(_get_up_vector=lambda nm: poses[nm][:, 2].copy(), _get_forward_vector=lambda nm: poses[nm][:, 1].copy())
        with np.errstate(invalid="ignore"):
            tq = FurnitureEnv._project_connector_quat(fake, "c1", "c2", angle)
        q["m1"].append(R1.ravel()); q["m2"].append(R2.ravel())
        q["angle"].append(0.0 if angle is None else float(angle)); q["has_angle"].append(angle is not None)
        q["tq"].append(np.asarray(tq, dtype=np.float64))

    # ---- _success_num_conn
    stmt = success_num_conn_statement(FurnitureEnv)
    goal = dict(nparts=[], k=[], num_connects=[], success_num_conn=[])
    for nparts in (2, 3, 5):
        for k in range(nparts - 1):
            for nc in (None, 1, 2):
                fake = types.SimpleNamespace(_num_connects=nc, _preassembled=range(k), _object_names=["p%d" % i for i in range(nparts)])
                exec(stmt, {}, {"self": fake})
                goal["nparts"].append(nparts); goal["k"].append(k); goal["num_connects"].append(-1 if nc is None else nc)
                goal["success_num_conn"].append(fake._success_num_conn)

    # ---- _reset_reward_variables from subtask k and the first reward
    argv, sys.argv = sys.argv, sys.argv[:1]
    base_cfg = create_parser("IKEASawyerDense-v0").parse_args([])
    sys.argv = argv
    FurnitureSawyerEnv.__init__ = lambda self, config: None  # no simulator: only the dense env's own attribute set-up runs
    keys = ("recipe", "k", "diff_rew", "reset_robot_after_attach", "num_connects", "leg_pos", "leg_site_pos", "leg_site_mat", "table_site_pos", "table_site_mat",
            "gl", "gr", "touch", "eef", "grip_mat", "ac", "subtask0", "phase0", "claimed", "reward", "done", "success", "phase", "subtask", "info")
    rec = {k: [] for k in keys}
    recipe_json = {}
    for ri, recipe_name in enumerate(RECIPES):
        for rep in range(6):
            cfg = types.SimpleNamespace(**vars(base_cfg))
            cfg.furniture_name = recipe_name
            cfg.diff_rew = bool(rep % 2 == 0)
            cfg.reset_robot_after_attach = bool(rep % 3 == 2)
            cfg.phase_ob = cfg.early_termination = False
            env = object.__new__(Dense)
            Dense.__init__(env, cfg)
            env._config, env._unity = cfg, None
            env._prev_grasp_dist = -1  # see tools/make_golden_dense.py
            env._furniture_id = furniture_name2id[recipe_name]
            FurnitureEnv._load_recipe(env)
            S = len(env._recipe["recipe"])
            recipe_json[recipe_name] = json.dumps(env._recipe)
            env._object_name2id = {}
            for leg, table in env._recipe["recipe"]:
                for nm in (leg, table):
                    env._object_name2id.setdefault(nm, len(env._object_name2id))
            for k in range(S):
                nc = [None, 1][rep % 2] if k + 1 < S else None
                leg_pos = rng.uniform(-0.3, 0.3, size=(S, 3)) + [0, 0, 0.05]
                leg_R = np.stack([small_rot(rng, 10.0) for _ in range(S)])
                table_pos = rng.uniform(-0.2, 0.2, size=(S, 3)) + [0, 0, 0.02]
                table_R = np.stack([small_rot(rng, 8.0) for _ in range(S)])
                site_off = rng.uniform(0.05, 0.15, size=S)
                gl = leg_pos[:, None, :] + rng.uniform(-0.05, 0.05, size=(S, MAXS, 3))  # [subtask whose leg it is][pair index]
                gr = gl + rng.uniform(0.02, 0.05, size=(S, MAXS, 3))
                grip_R = small_rot(rng, 10.0) @ np.array([[1.0, 0, 0], [0, -1, 0], [0, 0, -1]])
                touch = rng.rand(S) < 0.3
                names, asked = {}, []
                for s in range(S):
                    leg = env._recipe["recipe"][s][0]
                    names.setdefault(leg, ("leg", s))
                    names[env._site_recipe[s][0]] = ("leg_site", s)
                    names[env._site_recipe[s][1]] = ("table_site", s)
                    for i in range(S):
                        names.setdefault("%s_ltgt_site%d" % (leg, i), ("gl", names[leg][1], i))
                        names.setdefault("%s_rtgt_site%d" % (leg, i), ("gr", names[leg][1], i))
                eef = rng.uniform(-0.2, 0.2, size=3) + [0, 0, 0.35]

                def get_pos(nm):
                    asked.append(nm)
                    if nm == "griptip_site":
                        return eef.copy()
                    kind, s = names[nm][:2]
                    if kind == "leg":
                        return leg_pos[s].copy()
                    if kind == "leg_site":
                        return leg_pos[s] + leg_R[s][:, 2] * site_off[s]
                    if kind == "table_site":
                        return table_pos[s].copy()
                    return (gl if kind == "gl" else gr)[s, names[nm][2]].copy()

                def get_mat(nm):
                    if nm == "grip_site":
                        return grip_R
                    kind, s = names[nm][:2]
                    return leg_R[s] if kind == "leg_site" else table_R[s]

                env._get_pos = get_pos
                env._get_up_vector = lambda nm: get_mat(nm)[:, 2].copy()
                env._get_forward_vector = lambda nm: get_mat(nm)[:, 1].copy()
                env._site_xpos_xquat = lambda nm: np.hstack([get_pos(nm), [1, 0, 0, 0]])
                env._finger_contact = lambda leg: (bool(touch[names[leg][1]]), bool(touch[names[leg][1]]))
                env._preassembled = range(k)
                env._num_connects = nc
                env._object_names = list(env._object_name2id)
                exec(stmt, {}, {"self": env})
                env._max_episode_steps, env._episode_length, env._success = 150, 0, False
                env._connected = False  # FurnitureEnv._reset :1557, step :392
                env._reset_reward_variables()
                del asked[:]
                env._get_leg_grasp_vector()
                claimed = sorted(set(int(nm.rsplit("site", 1)[1]) for nm in asked))
                assert len(claimed) == 1 and names[asked[0]][1] == names[env._recipe["recipe"][k][0]][1]
                ac = rng.uniform(-1, 1, size=9)
                pad = lambda a: np.concatenate([a, np.zeros((MAXS - S,) + a.shape[1:])]) if S < MAXS else a
                rec["recipe"].append(ri); rec["k"].append(k); rec["diff_rew"].append(cfg.diff_rew); rec["reset_robot_after_attach"].append(cfg.reset_robot_after_attach)
                rec["num_connects"].append(-1 if nc is None else nc)
                rec["leg_pos"].append(pad(leg_pos)); rec["leg_site_pos"].append(pad(np.stack([leg_pos[s] + leg_R[s][:, 2] * site_off[s] for s in range(S)])))
                rec["leg_site_mat"].append(pad(leg_R.reshape(S, 9))); rec["table_site_pos"].append(pad(table_pos)); rec["table_site_mat"].append(pad(table_R.reshape(S, 9)))
                rec["gl"].append(pad(gl)); rec["gr"].append(pad(gr)); rec["touch"].append(pad(touch.astype(np.float64)).astype(bool))
                rec["eef"].append(eef.copy()); rec["grip_mat"].append(grip_R.ravel().copy()); rec["ac"].append(ac)
                rec["subtask0"].append(int(env._subtask_step)); rec["phase0"].append(int(env._phase_i)); rec["claimed"].append(claimed[0])
                reward, done, info = Dense._compute_reward(env, ac)
                rec["reward"].append(float(reward)); rec["done"].append(bool(done)); rec["success"].append(bool(env._success))
                rec["phase"].append(int(env._phase_i)); rec["subtask"].append(int(env._subtask_step))
                rec["info"].append(np.array([float(info.get(kk, 0.0)) for kk in INFO_KEYS]))
                rec.setdefault("success_num_conn", []).append(int(env._success_num_conn))
    coef_names = sorted(k for k, v in vars(base_cfg).items() if isinstance(v, (int, float, bool)) and ("coef" in k or "threshold" in k or k in (
        "phase_bonus", "alignment_pos_dist", "alignment_rot_dist_up", "alignment_rot_dist_forward", "alignment_project_dist")))
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, "preassembled.npz"), **{"q_" + k: np.array(v) for k, v in q.items()}, **{"goal_" + k: np.array(v) for k, v in goal.items()},
                        **{k: np.array(v) for k, v in rec.items()}, coef_names=np.array(coef_names), coefs=np.array([float(getattr(base_cfg, k)) for k in coef_names]),
                        recipes=np.array(RECIPES), recipe_json=np.array([recipe_json[r] for r in RECIPES]), info_keys=np.array(INFO_KEYS),
                        source="reference FurnitureEnv._project_connector_quat, the _success_num_conn statement of FurnitureEnv._reset and "
                               "FurnitureSawyerDenseRewardEnv._reset_reward_variables / _compute_reward run unmodified (tools/make_golden_preassembled.py)")
    tq = np.array(q["tq"])
    print("project_connector_quat: %d cases, %d NaN answers; starts: %d (k up to %d); first-step done %d" % (
        len(tq), int(np.isnan(tq).any(axis=1).sum()), len(rec["k"]), max(rec["k"]), int(np.sum(rec["done"]))))


if __name__ == "__main__":
    main()
