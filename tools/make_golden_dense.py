"""Golden vectors for the dense (phase-based) reward, made by running the REFERENCE'S OWN Python, unmodified.

Runs only in the build container (needs /root/reference); writes tests/golden/dense_reward.npz, which travels.
What is executed from the reference:
  * furniture/env/furniture_sawyer_dense.py  FurnitureSawyerDenseRewardEnv.__init__ (coefficient attributes only: the parent
    constructor that builds the MuJoCo sim is skipped), _reset_reward_variables, _update_reward_variables, _set_next_subtask,
    _collect_values, _compute_reward and every phase reward it calls (:18-1016)
  * furniture/env/furniture.py  FurnitureEnv._is_aligned (:1057-1153), _project_connector_forward (:1178-1199), _load_recipe (:2033-2044)
  * furniture/config  create_parser("IKEASawyerDense-v0") -> the reference's default coefficients
The simulator is replaced by a scripted world: per step the script supplies the positions / rotation matrices the reward code asks
for by name (_get_pos, _get_up_vector, _get_forward_vector, _finger_contact, _connected).  The script drives an episode through
the eight phases with random sloppiness and random accidents (dropped leg, moved table, early / wrong connections), so that every
branch of the phase machine is visited; what it records is the world it showed and what the reference answered.
"""
import os
import sys
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_assembly import import_reference, rand_rot, small_rot  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
RECIPES = ["table_lack_0825", "toy_table", "chair_agne_0007", "three_blocks"]
MAXS = 4  # subtasks recorded per step (padded)
INFO_KEYS = ["phase_bonus", "ctrl_penalty", "gripper_penalty", "move_other_part_penalty", "drop_penalty", "touch", "drop_leg", "table_moved",
             "stable_grip_succ", "skip_to_lift_leg", "skip_to_move_leg_fine"]


def orthonormal(M):
    u, _, vt = np.linalg.svd(M)
    R = u @ vt
    if np.linalg.det(R) < 0:
        u[:, -1] *= -1
        R = u @ vt
    return R


class World:
    """Everything the reward code can ask about, per subtask s: leg body position, leg / table connector site pose, the two grasp
    target sites of the leg, finger touches; plus the end effector (griptip position, grip_site rotation)."""

    def __init__(self, rng, S):
        self.S = S
        self.leg_pos = rng.uniform(-0.3, 0.3, size=(S, 3)) + [0, 0, 0.05]
        self.leg_R = np.stack([small_rot(rng, 10.0) for _ in range(S)])
        self.table_pos = rng.uniform(-0.2, 0.2, size=(S, 3)) + [0, 0, 0.02]
        self.table_R = np.stack([small_rot(rng, 8.0) @ np.diag([1.0, 1.0, 1.0]) for _ in range(S)])
        self.eef = rng.uniform(-0.2, 0.2, size=3) + [0, 0, 0.35]
        self.grip_R = small_rot(rng, 10.0) @ np.array([[1.0, 0, 0], [0, -1, 0], [0, 0, -1]])
        self.touchL = np.zeros(S, dtype=bool)
        self.touchR = np.zeros(S, dtype=bool)
        self.site_off = rng.uniform(0.05, 0.15, size=S)  # leg connector site sits this far along the leg's up axis

    def leg_site_pos(self, s):
        return self.leg_pos[s] + self.leg_R[s][:, 2] * self.site_off[s]

    def gl(self, s):
        return self.leg_pos[s] - self.leg_R[s][:, 0] * 0.02

    def gr(self, s):
        return self.leg_pos[s] + self.leg_R[s][:, 0] * 0.02


def reference_dense_env():
    """the reference's FurnitureSawyerDenseRewardEnv class with its parent constructor stubbed (no simulator), and its default config"""
    T, FurnitureEnv = import_reference()
    from furniture.env.furniture_sawyer import FurnitureSawyerEnv
    from furniture.env.furniture_sawyer_dense import FurnitureSawyerDenseRewardEnv as Dense
    from furniture.config import create_parser

    argv, sys.argv = sys.argv, sys.argv[:1]
    base_cfg = create_parser("IKEASawyerDense-v0").parse_args([])
    sys.argv = argv
    FurnitureSawyerEnv.__init__ = lambda self, config: None  # no simulator: only the dense env's own attribute set-up runs
    return Dense, FurnitureEnv, base_cfg


def draw_flags(rng, cfg):
    """the three flags and phase_ob of an episode"""
    cfg.diff_rew = bool(rng.rand() < 0.7)
    cfg.early_termination = bool(rng.rand() < 0.4)
    cfg.phase_ob = bool(rng.rand() < 0.25)
    cfg.reset_robot_after_attach = bool(rng.rand() < 0.3)


class Recorder:
    """runs scripted episodes of the reference's dense env and keeps what it showed and what the reference answered"""

    def __init__(self):
        self.Dense, self.FurnitureEnv, self.base_cfg = reference_dense_env()
        self.rec = {k: [] for k in ("episode", "is_reset", "leg_pos", "leg_site_pos", "leg_site_mat", "table_site_pos", "table_site_mat", "gl", "gr",
                                    "touchL", "touchR", "eef", "grip_mat", "connected", "ac", "reward", "done", "success", "phase", "subtask", "info")}
        self.eps = {k: [] for k in ("recipe", "diff_rew", "early_termination", "phase_ob", "reset_robot_after_attach", "nsub")}
        self.recipe_json = {}
        self.branch = {}
        self.n_ep = 0
        cfg = self.base_cfg
        self.coef_names = sorted(k for k, v in vars(cfg).items() if isinstance(v, (int, float, bool)) and ("coef" in k or "threshold" in k or k in (
            "phase_bonus", "alignment_pos_dist", "alignment_rot_dist_up", "alignment_rot_dist_forward", "alignment_project_dist")))

    def new_config(self, rng, configure=draw_flags):
        """the next episode's config: the reference's defaults for the next recipe, then `configure(rng, cfg)`"""
        cfg = types.SimpleNamespace(**vars(self.base_cfg))
        cfg.furniture_name = RECIPES[self.n_ep % len(RECIPES)]
        configure(rng, cfg)
        return cfg

    def episode(self, rng, cfg, record=True):
        """one scripted episode under `cfg`; with record=False nothing is kept and the episode's phase trace is returned"""
        from furniture.env.models import furniture_name2id

        Dense, FurnitureEnv = self.Dense, self.FurnitureEnv
        rec = self.rec if record else {k: [] for k in self.rec}
        recipe_name = cfg.furniture_name
        env = object.__new__(Dense)
        Dense.__init__(env, cfg)
        env._config = cfg
        env._unity = None
        # the reference initialises _prev_grasp_dist only when diff_rew is on, yet _grasp_leg_reward reads it in both modes (an
        # AttributeError in the reference when diff_rew=False reaches the grasp phase); the script provides the diff-mode initial value
        env._prev_grasp_dist = -1
        env._furniture_id = furniture_name2id[recipe_name]
        FurnitureEnv._load_recipe(env)
        S = len(env._recipe["recipe"])
        assert S <= MAXS
        import json
        self.recipe_json[recipe_name] = json.dumps(env._recipe)
        env._preassembled = []
        env._success_num_conn = S
        env._max_episode_steps = 150
        env._episode_length = 0
        env._connected = False
        env._success = False
        env._object_name2id = {}
        for leg, table in env._recipe["recipe"]:
            for nm in (leg, table):
                env._object_name2id.setdefault(nm, len(env._object_name2id))
        w = World(rng, S)
        names = {}
        for s in range(S):
            leg = env._recipe["recipe"][s][0]
            ls, ts = env._site_recipe[s][:2]
            names[leg] = ("leg", s)
            names[ls] = ("leg_site", s)
            names[ts] = ("table_site", s)
            for i in range(S):
                names["%s_ltgt_site%d" % (leg, i)] = ("gl", s)
                names["%s_rtgt_site%d" % (leg, i)] = ("gr", s)

        def get_pos(nm):
            if nm == "griptip_site":
                return w.eef.copy()
            kind, s = names[nm]
            if kind == "leg":
                return w.leg_pos[s].copy()
            if kind == "leg_site":
                return w.leg_site_pos(s)
            if kind == "table_site":
                return w.table_pos[s].copy()
            return w.gl(s) if kind == "gl" else w.gr(s)

        def get_mat(nm):
            if nm == "grip_site":
                return w.grip_R
            kind, s = names[nm]
            return w.leg_R[s] if kind == "leg_site" else w.table_R[s]

        env._get_pos = get_pos
        env._get_up_vector = lambda nm: get_mat(nm)[:, 2].copy()
        env._get_forward_vector = lambda nm: get_mat(nm)[:, 1].copy()
        env._site_xpos_xquat = lambda nm: np.hstack([get_pos(nm), [1, 0, 0, 0]])
        env._finger_contact = lambda leg: (bool(w.touchL[names[leg][1]]), bool(w.touchR[names[leg][1]]))

        def snapshot(is_reset, ac, out):
            pad = lambda a, shape: np.concatenate([a, np.zeros((MAXS - S,) + shape)]) if S < MAXS else a
            rec["episode"].append(self.n_ep)
            rec["is_reset"].append(is_reset)
            rec["leg_pos"].append(pad(w.leg_pos.copy(), (3,)))
            rec["leg_site_pos"].append(pad(np.stack([w.leg_site_pos(s) for s in range(S)]), (3,)))
            rec["leg_site_mat"].append(pad(w.leg_R.reshape(S, 9).copy(), (9,)))
            rec["table_site_pos"].append(pad(w.table_pos.copy(), (3,)))
            rec["table_site_mat"].append(pad(w.table_R.reshape(S, 9).copy(), (9,)))
            rec["gl"].append(pad(np.stack([w.gl(s) for s in range(S)]), (3,)))
            rec["gr"].append(pad(np.stack([w.gr(s) for s in range(S)]), (3,)))
            rec["touchL"].append(np.concatenate([w.touchL, np.zeros(MAXS - S, dtype=bool)]))
            rec["touchR"].append(np.concatenate([w.touchR, np.zeros(MAXS - S, dtype=bool)]))
            rec["eef"].append(w.eef.copy())
            rec["grip_mat"].append(w.grip_R.ravel().copy())
            rec["connected"].append(bool(env._connected))
            rec["ac"].append(ac)
            for k, v in out.items():
                rec[k].append(v)

        env._reset_reward_variables()
        snapshot(True, np.zeros(9), dict(reward=0.0, done=False, success=False, phase=env._phase_i, subtask=env._subtask_step, info=np.zeros(len(INFO_KEYS))))
        if record:
            for k in self.eps:
                self.eps[k].append(S if k == "nsub" else (RECIPES.index(recipe_name) if k == "recipe" else getattr(cfg, k)))
        sloppy = rng.choice([0.0, 0.002, 0.01, 0.04])
        speed = rng.choice([0.35, 0.6, 1.0])
        accident = rng.choice([0.0, 0.01, 0.04])
        table0 = w.table_pos.copy()
        for t in range(150):
            s = env._subtask_step
            ph = env._phase_i
            ac = rng.uniform(-1, 1, size=9) * rng.choice([0.05, 0.5, 1.0])
            ac[-2] = -1.0 if ph <= 2 else 1.0
            if rng.rand() < 0.1:
                ac[-2] = rng.uniform(-1, 1)
            ac[-1] = rng.uniform(-1, 1)
            env._connected = False
            grasp = (w.gl(s) + w.gr(s)) / 2
            a = speed if rng.rand() < 0.8 else 0.1

            def carry(target_leg_pos=None, target_R=None):
                # the leg moves rigidly with the gripper once held
                if target_R is not None:
                    w.leg_R[s] = orthonormal((1 - a) * w.leg_R[s] + a * target_R)
                if target_leg_pos is not None:
                    d = a * (target_leg_pos - w.leg_pos[s])
                    w.leg_pos[s] = w.leg_pos[s] + d
                w.eef = (w.gl(s) + w.gr(s)) / 2 + [0, 0, -0.01]

            grip_target = orthonormal(np.stack([np.cross(w.leg_R[s][:, 0], [0, 0, -1.0]), w.leg_R[s][:, 0], [0, 0, -1.0]], axis=1))
            w.grip_R = orthonormal((1 - a) * w.grip_R + a * grip_target + rng.normal(size=(3, 3)) * sloppy)
            if ph == 0:
                w.eef = w.eef + a * (env._init_eef_pos - w.eef)
            elif ph == 1:
                w.eef = w.eef + a * (grasp + [0, 0, 0.05] - w.eef)
            elif ph == 2:
                w.eef = w.eef + a * (grasp + [0, 0, -0.015] - w.eef)
            elif ph == 3:
                w.eef = w.eef + a * (grasp + [0, 0, -0.015] - w.eef)
                if rng.rand() < 0.6:
                    w.touchL[s] = w.touchR[s] = True
                elif rng.rand() < 0.3:
                    w.touchL[s] = True
            elif ph == 4:
                carry(target_leg_pos=env._lift_leg_pos + [0, 0, 0.005])
            elif ph in (5, 6, 7):
                # leg connector up anti-parallel... the reward wants cos(leg_up, table_up) -> 1 and forward (rotated) -> table forward
                tR = w.table_R[s].copy()
                ang = env._leg_table_angle
                if ang is not None:
                    c, sn = np.cos(np.deg2rad(-ang)), np.sin(np.deg2rad(-ang))
                    tR = tR @ np.array([[c, -sn, 0], [sn, c, 0], [0, 0, 1]])
                if ph == 5:
                    carry(target_leg_pos=env._lift_leg_pos, target_R=tR)
                else:
                    above = w.table_pos[s] + [0, 0, env._recipe["z_finedist"] if ph == 6 else 0.0]
                    tgt_leg = above - tR[:, 2] * w.site_off[s]
                    carry(target_leg_pos=tgt_leg, target_R=tR)
                    if ph == 7 and ac[-1] > 0 and rng.rand() < 0.7:
                        env._connected = True
            w.eef = w.eef + rng.normal(size=3) * sloppy
            if rng.rand() < 0.97:  # an exactly aligned pair makes the reference's sqrt(1 - cos^2) NaN about half of the time: keep that rare
                w.leg_R[s] = small_rot(rng, 0.3) @ w.leg_R[s]
            w.leg_pos[s] = w.leg_pos[s] + rng.normal(size=3) * sloppy * (0.3 if ph >= 4 else 0.02)
            # accidents
            if ph > 3 and rng.rand() < accident:
                w.touchL[s] = w.touchR[s] = False
            elif ph > 3 and rng.rand() < 0.5:
                w.touchL[s] = w.touchR[s] = True
            if rng.rand() < accident * 0.5:
                w.table_pos[s] = table0[s] + rng.normal(size=3) * 0.15
            elif rng.rand() < 0.3:
                w.table_pos[s] = table0[s] + rng.normal(size=3) * 0.002
            if rng.rand() < accident * 0.5 and ac[-1] > 0:
                env._connected = True  # a connection the phase machine did not expect
            if rng.rand() < 0.02 and ph < 3:  # early pick
                w.touchL[s] = w.touchR[s] = True
                w.eef = grasp + [0, 0, -0.02]
            reward, done, info = Dense._compute_reward(env, ac)
            env._episode_length += 1
            if record:
                key = (ph, bool(done), bool(env._success), int(env._subtask_step - s), int(env._phase_i))
                self.branch[key] = self.branch.get(key, 0) + 1
            snapshot(False, ac, dict(reward=float(reward), done=bool(done), success=bool(env._success), phase=int(env._phase_i), subtask=int(env._subtask_step),
                                     info=np.array([float(info.get(k, 0.0)) for k in INFO_KEYS])))
            if done:
                break
            if env._subtask_step != s:
                table0 = w.table_pos.copy()
        if record:
            self.n_ep += 1
        return rec["phase"]

    def arrays(self):
        """the records and the per-episode flags as the fixture stores them"""
        return dict({k: np.array(v) for k, v in self.rec.items()}, **{"ep_" + k: np.array(v) for k, v in self.eps.items()}, recipes=np.array(RECIPES),
                    recipe_json=np.array([self.recipe_json[r] for r in RECIPES]), info_keys=np.array(INFO_KEYS))

    def report(self, name):
        ph = np.array(self.rec["phase"])
        print("%s: %d records, %d episodes; final phases seen %s; successes %d; subtask max %d" % (
            name, len(ph), self.n_ep, np.bincount(ph, minlength=8).tolist(), int(np.sum(self.rec["success"])), int(np.max(self.rec["subtask"]))))
        print("branches (phase before, done, success, subtask advance, phase after):", len(self.branch))
        for k in sorted(self.branch):
            print("  ", k, self.branch[k])


def main():
    r = Recorder()
    rng = np.random.RandomState(20260924)
    while len(r.rec["reward"]) < 9000:
        r.episode(rng, r.new_config(rng))
    os.makedirs(OUT, exist_ok=True)
    a = r.arrays()
    coefs = np.array([float(getattr(r.base_cfg, k)) for k in r.coef_names])
    np.savez_compressed(os.path.join(OUT, "dense_reward.npz"), **{k: a[k] for k in r.rec}, **{"ep_" + k: a["ep_" + k] for k in r.eps},
                        coef_names=np.array(r.coef_names), coefs=coefs, recipes=a["recipes"], recipe_json=a["recipe_json"], info_keys=a["info_keys"],
                        source="reference furniture/env/furniture_sawyer_dense.py _compute_reward run unmodified on a scripted world (tools/make_golden_dense.py)")
    r.report("dense_reward")


if __name__ == "__main__":
    main()
