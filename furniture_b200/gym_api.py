"""Single-environment gym-shaped surface (numpy in / numpy out) over the engine: the call surface of the reference's
`FurnitureGym` (furniture/env/furniture_gym.py:11-80) and of `FurnitureEnv.step()/reset()` behind it.

  env = FurnitureGymB200(name="FurnitureSawyerEnv", furniture_name="table_lack_0825", seed=123)
  ob = env.reset()                                  # OrderedDict(object_ob (7 n_objects,), robot_ob (29,)); see the observation flags
  ob, reward, done, info = env.step(action)         # action: (dof,) array or {"default": array}

It is the batched engine with one env (the batch entry point `furniture_b200.env.make_vec_env` is the one to use for
throughput).  The step kernel resets a finished env on the device in the same launch, like a `SubprocVecEnv` worker
does (subproc_vec_env.py:16-20).  The `reset()` the caller issues after `done` returns the first observation of the
episode the device has already started and does not reset a second time, so the env consumes exactly one reset's worth
of numpy random draws per episode, like the reference (furniture.py:72).  What `step` returns with `done=True` depends
on the keyword `terminal_observation`:
  * False (the default): the first observation of the next episode, not the terminal one, and `get_env_state()` gives
    the state of that next episode -- the difference from the reference's `FurnitureEnv.step`;
  * True: the terminal observation, as the reference's `FurnitureEnv.step` returns it (furniture.py:364-385), and
    `get_env_state()` gives the terminal state until the caller's `reset()`.  The step kernel writes both before its
    auto-reset; after an unstable step they are those of the reset inside `_do_simulation`'s except branch
    (furniture.py:2889-2897), as in the reference.
`info` carries the reference's episode keys at the end of an episode (`_after_step`, furniture.py:451-480).  With the keyword
`step_info=True` it is the reference's whole `info` dict: the sparse env adds `_compute_reward`'s four terms on every step
(furniture.py:535-540), the two-arm env adds `ac` (furniture_baxter.py:75), `episode_reward` and `episode_unstable` come from the
record the step kernel keeps, and a successful episode adds `episode_success_state`.  The default keeps the info described above.
"""
from __future__ import annotations

import time
from collections import OrderedDict

import numpy as np


class FurnitureGymB200:
    metadata = {"render.modes": []}

    def __init__(self, name="FurnitureSawyerEnv", furniture_name=None, device=0, lib_path=None, id=None, terminal_observation=False,
                 step_info=False, **config):
        """`id`, `name` and the remaining keywords are what gym passes from the registration (env/__init__.py:19-114: id, name,
        furniture_name / furniture_id, background, port ...); options of the renderer are ignored, see env.split_config.
        `terminal_observation`: step returns the terminal observation with done=True, as the reference's FurnitureEnv.step does (see the
        module's docstring).  `step_info`: step returns the reference's whole info dict (see the module's docstring)"""
        from .env import ENV_IDS, build_engine, env_options

        ids = dict(ENV_IDS, Sawyer=ENV_IDS["FurnitureSawyerEnv"], Baxter=ENV_IDS["FurnitureBaxterEnv"])  # and the bare agent names
        if name not in ids:
            raise ValueError("unknown env %s (this build accelerates %s)" % (name, sorted(ids)))
        if furniture_name is not None:
            config["furniture_name"] = furniture_name
        agent, dense_reward = ids[name]
        furniture_name, options, self.ignored_config = env_options(config, dense_reward)
        self.engine = e = build_engine(agent, furniture_name, 1, device=device, lib_path=lib_path, **options)
        self.model, self.cfg, self.dense_cfg, self.ik_cfg, self.ctl_cfg = e.model, e.cfg, e.dense, e.ik, e.controller
        self.control_type, self.obs_flags, self.n_objects, self.dof = e.control_type, e.obs_flags, e.scene.npart, e.act_dim
        cols, widths = e.obs_columns()
        self._cols = OrderedDict((k, np.arange(e.obs_dim)[c]) for k, c in cols.items())  # the row's columns of each obs entry
        self.object_ob_dim, self.subtask_ob_dim, self.robot_ob_dim, self.phase_ob_dim = (widths[k] for k in ("object_ob", "subtask_ob", "robot_ob", "phase_ob"))
        self._max_episode_steps = self.cfg.max_episode_steps
        self._pending_ob = None  # observation of an episode the device has already started
        self._terminal = bool(terminal_observation)
        self._step_info = bool(step_info)
        self._terminal_state = None  # with terminal_observation: the state the finished episode ended in, until reset()
        self._episode_reward = 0.0
        self._episode_time = time.time()

    # ---- spaces (furniture.py:215-252, :293-310): plain shape / bound records, gym.spaces objects when gym is installed
    @property
    def observation_space(self):
        shapes = OrderedDict((k, (len(c),)) for k, c in self._cols.items())  # object_ob, subtask_ob, robot_ob, phase_ob as the flags ask
        try:
            import gym.spaces as sp

            return sp.Dict(OrderedDict((k, sp.Box(low=-np.inf, high=np.inf, shape=v)) for k, v in shapes.items()))
        except Exception:
            return shapes

    @property
    def action_space(self):
        try:
            import gym.spaces as sp

            return sp.Dict([("default", sp.Box(shape=(self.dof,), low=-1, high=1, dtype=np.float32))])
        except Exception:
            return OrderedDict(default=dict(shape=(self.dof,), low=-1.0, high=1.0))

    def _ob(self, obs_row):
        return OrderedDict((k, obs_row[c].astype(np.float64)) for k, c in self._cols.items())

    def reset(self):
        self._terminal_state = None
        if self._pending_ob is not None:
            ob, self._pending_ob = self._pending_ob, None
        else:
            self.engine.env_reset()
            ob = self._ob(self.engine.get("obs")[0])
        self._episode_reward = 0.0
        self._episode_time = time.time()
        return ob

    def step(self, action):
        if isinstance(action, dict):
            action = np.concatenate([np.asarray(v, dtype=np.float32).ravel() for v in action.values()])
        a = np.asarray(action, dtype=np.float32).reshape(1, self.dof)
        if self._pending_ob is not None:  # stepping on after `done` without reset(): the device is already in the next episode
            self._pending_ob, self._episode_reward, self._episode_time = None, 0.0, time.time()
            self._terminal_state = None
        obs, rew, done, info = self.engine.env_step_host(a)
        reward, done = float(rew[0]), bool(done[0])
        self._episode_reward += reward
        out = OrderedDict()
        ob = self._ob(obs[0])
        if self.dense_cfg is not None:  # the step's reward terms (_compute_reward's info, furniture_sawyer_dense.py:574-586)
            from .dense import INFO_KEYS

            row = self.engine.get("dense_info")[0]
            out.update((k, float(v)) for k, v in zip(INFO_KEYS, row))
        elif self._step_info:  # _compute_reward's terms (furniture.py:535-540), as the step kernel wrote them
            from .engine import REWARD_INFO_KEYS

            out.update((k, float(v)) for k, v in zip(REWARD_INFO_KEYS, self.engine.reward_info()[0]))
        if self._step_info and self.engine.scene.narms == 2:
            out["ac"] = a[0].copy()  # FurnitureBaxterEnv._step (furniture_baxter.py:75)
        if done:
            unstable = int(info[0][2])
            out["episode_success"] = int(info[0][1])
            out["episode_reward"] = self._episode_reward
            out["episode_length"] = int(info[0][3])
            out["episode_time"] = time.time() - self._episode_time
            out["episode_unstable"] = -float(self.cfg.unstable_penalty_coef) if unstable else 0
            out["episode_num_connected"] = int(info[0][0])
            if self._step_info:  # the record the step kernel kept (float32 sum of the episode's rewards, plus the penalty)
                rec = self.engine.episode_info()[0]
                out["episode_reward"], out["episode_unstable"] = float(rec[0]), float(rec[1])
                if out["episode_success"]:
                    q, v = self.engine.terminal_state()
                    out["episode_success_state"] = {"qpos": q[0].astype(np.float64), "qvel": v[0].astype(np.float64)}
            self._pending_ob = ob
            if self._terminal:  # the row and the state the step kernel kept before its auto-reset
                ob = self._ob(self.engine.terminal_obs()[0])
                q, v = self.engine.terminal_state()
                self._terminal_state = {"qpos": q[0].astype(np.float64), "qvel": v[0].astype(np.float64)}
        return ob, reward, done, out

    # ---- pass-throughs of FurnitureGym (furniture_gym.py:35-50)
    def set_max_episode_steps(self, max_episode_steps):
        self._max_episode_steps = int(max_episode_steps)
        self.engine.set_max_episode_steps(self._max_episode_steps)

    def set_subtask(self, subtask, num_connects=None):
        """furniture.py:204-207: from the next reset on, episodes start with the first `subtask` recipe steps connected"""
        self.engine.set_subtask(int(subtask), num_connects)
        self._pending_ob = None  # an episode the device started on its own still has the old subtask: the next reset() resets again

    def num_subtask(self):
        return int(self.engine.num_subtask()[0])

    def set_sim_options(self, control_freq=None, no_collision=None):
        """config/furniture.py's control_freq (mj_steps of the next steps, furniture.py:2855, :2878) and no_collision (the agent's collisions
        off at once, furniture.py:1962-1965); None leaves an option as it is"""
        self.engine.set_sim_options(control_freq, no_collision)

    def set_init_qpos(self, init_qpos):
        """furniture.py:315-316 (FurnitureGym, furniture_gym.py:43): from the next reset on, episodes start from this get_env_state dict, or
        from random placement for None"""
        self.engine.set_init_qpos(init_qpos)
        self._pending_ob = None  # an episode the device started on its own still has the old start: the next reset() resets again

    def load_init_states(self, states):
        """--load_init_states (furniture.py:127-130): before each reset, keep the start with probability 0.2, else pick one from `states`"""
        self.engine.load_init_states(states)
        self._pending_ob = None

    def get_env_state(self):
        if self._terminal_state is not None:
            return {k: v.copy() for k, v in self._terminal_state.items()}
        q, v = self.engine.get_state()
        return {"qpos": q[0].astype(np.float64), "qvel": v[0].astype(np.float64)}

    def set_env_state(self, state):
        self._terminal_state = None
        self.engine.set_state(np.asarray(state["qpos"])[None], np.asarray(state["qvel"])[None])
        self.engine.set("ctrl", np.zeros((1, self.model.nu), np.float32))
        self.engine.forward()

    def render(self, mode="human"):
        raise NotImplementedError("rendering is outside the accelerated path")

    def close(self):
        self.engine.close()


def register_gym_envs():
    """Registers the accelerated counterpart of the reference's gym ids (furniture/env/__init__.py:19-114) when gym or
    gymnasium is importable: `gym.make("IKEASawyer-v0")` then builds a FurnitureGymB200 with the reference's kwargs
    (furniture_name="swivel_chair_0700").  Returns the ids registered (empty without gym)."""
    try:
        from gym.envs.registration import register
    except Exception:
        try:
            from gymnasium.envs.registration import register
        except Exception:
            return []
    specs = {"IKEASawyerDense-v0": {"id": "IKEASawyerDense-v0", "name": "FurnitureSawyerDenseRewardEnv", "unity": False},
             "furniture-sawyer-densereward-v0": {"id": "IKEASawyerDense-v0", "name": "FurnitureSawyerDenseRewardEnv", "unity": False},
             "IKEASawyer-v0": {"id": "IKEASawyer-v0", "name": "FurnitureSawyerEnv", "furniture_name": "swivel_chair_0700", "background": "Industrial", "port": 1050},
             "IKEABaxter-v0": {"id": "IKEABaxter-v0", "name": "FurnitureBaxterEnv", "furniture_id": 1, "background": "Interior", "port": 1050}}
    done = []
    try:  # the Cursor agent is host logic over the simulator surface (furniture_b200/cursor_env.py)
        register(id="IKEACursor-v0", entry_point="furniture_b200.cursor_env:FurnitureCursorEnvB200",
                 kwargs={"id": "IKEACursor-v0", "name": "FurnitureCursorEnv", "furniture_id": 0, "background": "Lab", "port": 1050})
        done.append("IKEACursor-v0")
    except Exception:
        pass
    for env_id, kwargs in specs.items():
        try:
            register(id=env_id, entry_point="furniture_b200.gym_api:FurnitureGymB200", kwargs=kwargs)
            done.append(env_id)
        except Exception:  # already registered (e.g. by the reference package itself)
            pass
    return done
