"""Batched gym/VecEnv-shaped surface over the engine (torch tensors in, torch tensors out).

Mirrors the reference's call surface for the accelerated path:
  make_vec_env(env_id, num_env, config)   furniture/env/base.py:55-80          -> BatchedFurnitureEnv
  VecEnv.reset() / step(actions)          furniture/util/vec_env.py:53-162, subproc_vec_env.py:100-113 (auto-reset on done)
  obs dict {"object_ob", "robot_ob"}      furniture.py:1344-1387, furniture_sawyer.py:103-155 (OrderedDict order kept)
  get_env_state / set_env_state           furniture.py:1781-1803
Observations live in one contiguous (N, obs_dim) float32 CUDA tensor written by the step kernel; the dict entries are
views of it.  ShardedFurnitureEnv adds the multi-GPU form: env shards are independent (one process per GPU), the only
collective is one NCCL all_gather of the packed [obs | reward | done] tensor per step (SURVEY.md 8e), optionally widened by every
env's info, dense_info and terminal observation.
"""
from __future__ import annotations

import os
import time
from collections import OrderedDict

import numpy as np

from . import mjcf
from .dense import DENSE_DEFAULTS, DENSE_ENV_DEFAULTS, INFO_KEYS as DENSE_INFO_KEYS, dense_config
from .engine import EPISODE_INFO_KEYS, INFO_DIM, OBS_DEFAULTS, REWARD_INFO_KEYS, TASK_OPTIONS, Engine, default_config, packed_columns

RESET_DEFAULTS = dict(fix_init=False, fix_init_parts=None, reset_robot_after_attach=False, assembled=False)  # config/furniture.py:116-127, :169-174, :307-312
SIM_DEFAULTS = dict(control_freq=10, no_collision=False)  # config/furniture.py:71-73, :304-306
INFO_KEYS = ("num_connected", "episode_success", "episode_unstable", "episode_length", "ncon", "solver_iters")
# env id or class name (env/__init__.py:19-114) -> (agent, whether it is FurnitureSawyerDenseRewardEnv, env/__init__.py:103-114)
ENV_IDS = {"IKEASawyer-v0": ("Sawyer", False), "FurnitureSawyerEnv": ("Sawyer", False), "IKEABaxter-v0": ("Baxter", False),
           "FurnitureBaxterEnv": ("Baxter", False), "IKEASawyerDense-v0": ("Sawyer", True), "furniture-sawyer-densereward-v0": ("Sawyer", True),
           "FurnitureSawyerDenseRewardEnv": ("Sawyer", True)}
NEW_CONTROLLERS = ("position", "position_orientation", "joint_impedance", "joint_torque", "joint_velocity")  # furniture.py:41-47
# furniture_id -> name: the reference numbers the sorted objects/*.xml (furniture/env/models/__init__.py:11-19)
FURNITURE_NAMES = (
    "bed_dalselv_0270 bench_bjoderna_0208 bench_bjursta_0210 block bookcase_agerum_0006 bookcase_besta_0165 bookcase_besta_0170 bookcase_besta_0172 "
    "bookcase_billy_0190 bookcase_billy_0191 bookcase_expedit_0373 bookcase_expedit_0374 bookcase_expedit_0376 bookcase_expedit_0385 bookcase_flaerke_0403 "
    "bookcase_grevback_0484 bookcase_hensvik_0565 box_ivar_0666 box_lekman_0858 cabinet_akurum_0011 cabinet_akurum_0014 cabinet_akurum_0019 cabinet_akurum_0021 "
    "cabinet_bjorken_0203 cabinet_lillagen_0933 chair_agam_0005 chair_agne_0007 chair_agne_0010 chair_balser_0115 chair_bernhard_0146 chair_bertil_0148 "
    "chair_ingolf_0650 chair_ivar_0668 desk_fredrik_0430 desk_hannes_0529 desk_mikael_1064 shelf_ivar_0678 shelf_liden_0922 shelf_lillagen_0927 swivel_chair_0700 "
    "table_benno_0141 table_billsta_round_0189 table_bjorkudden_0206 table_bjorkudden_0207 table_dalom_0267 table_dockstra_0279 table_expedit_0387 table_hemnes_0539 "
    "table_hemnes_0541 table_jokkmokk_0694 table_klubbo_0740 table_klubbo_0743 table_lack_0825 table_liden_0919 table_liden_0920 table_liden_0921 table_torsby_1549 "
    "three_blocks three_blocks_peg toy_table toy_table_flip tvunit_0406 tvunit_lack_0829 tvunit_lack_0830").split()


def device_view(ptr, shape, device):
    """a float32 torch tensor over `shape` contiguous floats of device memory at `ptr` that the engine owns (no copy; valid while the
    engine lives)"""
    import torch

    class _Buf:
        __cuda_array_interface__ = dict(shape=tuple(int(n) for n in shape), typestr="<f4", data=(int(ptr), False), version=2, strides=None)

    return torch.as_tensor(_Buf(), device=device)


def prefix_length(preassembled):
    """`preassembled` of config/furniture.py:158 -> how many recipe steps it names.  The accelerated path starts an episode after the first k
    steps of the recipe, which is what set_subtask produces (furniture.py:204-207) and what the dense reward assumes
    (furniture_sawyer_dense.py:128-139): any other list is refused."""
    p = [int(x) for x in (preassembled if preassembled is not None else ())]
    if p != list(range(len(p))):
        raise ValueError("preassembled must be a prefix [0, 1, ..., k-1] of the assembly recipe, got %r" % (list(preassembled),))
    return len(p)


def split_config(config):
    """Reference-style config (argparse Namespace or dict, config/furniture.py) -> (furniture name, FeConfig overrides, ignored keys).
    `furniture_name` wins over `furniture_id` as in furniture.py:157-161; keys the accelerated path has no use for (port, background,
    camera and rendering options, the speeds where no control type reads them ...) are returned so that callers can report them instead of
    failing on them.  `preassembled` (checked to be a recipe prefix), `num_connects`, `load_init_states`, `load_demo` and the observation flags
    `robot_ob`, `object_ob`, `object_ob_all`, `subtask_ob`, the reset options `fix_init`, `fix_init_parts`, `reset_robot_after_attach`, `assembled` and
    `control_freq`, `no_collision` travel with the overrides when they are set (the flags when they differ from their defaults): they are
    keywords of build_engine."""
    from .engine import FeConfig

    cfg = dict(vars(config)) if hasattr(config, "__dict__") and not isinstance(config, dict) else dict(config or {})
    if cfg.get("control_type", "impedance") not in ("impedance", "ik", "ik_quaternion") + NEW_CONTROLLERS:
        raise NotImplementedError("control_type %r is not built ('torque' drives nine actuators with eight numbers in the reference)" % cfg["control_type"])
    for k in ("unity", "visual_ob", "depth_ob", "segmentation_ob", "record_demo", "record_vid"):
        if cfg.get(k):
            raise NotImplementedError("%s=True needs the renderer, which is outside the accelerated path" % k)
    name = cfg.get("furniture_name")
    if name is None and cfg.get("furniture_id") is not None:
        name = FURNITURE_NAMES[int(cfg["furniture_id"])]
    fields = {f[0] for f in FeConfig._fields_} - {"struct_bytes"}
    over = {k: v for k, v in cfg.items() if k in fields and v is not None}
    ignored = sorted(k for k in cfg if k not in over and k not in ("furniture_name", "furniture_id", "control_type", "preassembled", "num_connects",
                                                                   "load_init_states", "load_demo") + tuple(OBS_DEFAULTS) + tuple(RESET_DEFAULTS)
                     + tuple(SIM_DEFAULTS))
    if "ik" in control_options(cfg):  # the speeds reach the IK or the controller
        ignored = [k for k in ignored if k not in ("move_speed", "rotate_speed")]
    if prefix_length(cfg.get("preassembled")):
        over["preassembled"] = list(cfg["preassembled"])
    if cfg.get("num_connects") is not None:
        over["num_connects"] = int(cfg["num_connects"])
    for k in ("load_init_states", "load_demo"):  # paths of pickles (furniture.py:121-130), read by the env constructors
        if cfg.get(k):
            over[k] = cfg[k]
    for k, default in OBS_DEFAULTS.items():  # furniture.py:103-107; a flag at its default changes nothing and is not passed on
        if cfg.get(k) is not None and bool(cfg[k]) != default:
            over[k] = bool(cfg[k])
    for k in RESET_DEFAULTS:  # config/furniture.py:116-127, :169-174, :307-312; False, None and the empty set are the defaults
        if cfg.get(k):
            over[k] = cfg[k] if k == "fix_init_parts" else bool(cfg[k])
    if cfg.get("control_freq") is not None and cfg["control_freq"] != SIM_DEFAULTS["control_freq"]:  # furniture.py:84, :2855, :2878
        over["control_freq"] = cfg["control_freq"]
    if cfg.get("no_collision"):  # furniture.py:1962-1965
        over["no_collision"] = bool(cfg["no_collision"])
    return name or "table_lack_0825", over, ignored


def control_options(config):
    """control_type and, for "ik", the speeds of config/furniture.py:84-89 -> keywords of BatchedFurnitureEnv"""
    cfg = dict(vars(config)) if hasattr(config, "__dict__") and not isinstance(config, dict) else dict(config or {})
    ct = cfg.get("control_type") or "impedance"
    out = dict(control_type=ct)
    if ct in ("ik", "ik_quaternion"):
        out["ik"] = {k: cfg[k] for k in ("move_speed", "rotate_speed") if cfg.get(k) is not None}
    elif ct in NEW_CONTROLLERS and cfg.get("move_speed") is not None:
        out["ik"] = {"move_speed": cfg["move_speed"]}  # _do_controller_step scales action[:3] with it as well (furniture.py:3069-3071)
    return out


def split_dense_config(config):
    """Config of a dense-reward env id (config/furniture_sawyer_dense.py) -> (furniture name, FeConfig overrides, dense coefficient
    overrides, ignored keys).  What that file changes in the base env (150 steps, table_lack_0825, auto_align off, the tight
    alignment thresholds) is the default here too; explicit keys of `config` win."""
    cfg = dict(vars(config)) if hasattr(config, "__dict__") and not isinstance(config, dict) else dict(config or {})
    merged = dict(DENSE_ENV_DEFAULTS)
    merged.update({k: v for k, v in cfg.items() if v is not None})
    name, over, ignored = split_config({k: v for k, v in merged.items() if k != "reset_robot_after_attach"})
    dense = {k: merged[k] for k in DENSE_DEFAULTS if k in merged}  # a list gives one value per env (Engine.set_dense_options)
    if "ctrl_penalty_coef" in over:
        dense["ctrl_penalty_coef"] = over["ctrl_penalty_coef"]
        if np.ndim(over["ctrl_penalty_coef"]) > 0:  # per env it is the phase machine's only: FeConfig keeps the default
            del over["ctrl_penalty_coef"]
    return name, over, dense, [k for k in ignored if k not in DENSE_DEFAULTS]


def apply_init_config(env, load_init_states=None, load_demo=None):
    """the constructor half of furniture.py:121-130 for an env with set_init_qpos / load_init_states: `load_demo` sets every env's start to
    the first state of that demo, `load_init_states` gives every env the list to pick from (as every VecEnv worker loads the same file).
    Each is a path, read with demo.load_init_states, or the list of states itself."""
    from .demo import load_init_states as read

    states = lambda x: read(x) if isinstance(x, (str, bytes, os.PathLike)) else list(x)
    if load_demo:
        env.set_init_qpos(states(load_demo)[0])
    if load_init_states:
        env.load_init_states(states(load_init_states))


def env_options(config, dense_reward=False):
    """Reference-style config of the sparse env, or of the dense-reward env -> (furniture name, keywords of build_engine, ignored keys)"""
    if dense_reward:
        furniture, over, dense, ignored = split_dense_config(config)
        over["dense"] = dense
    else:
        furniture, over, ignored = split_config(config)
    return furniture, dict(over, **control_options(config)), ignored


def build_engine(agent, furniture_name, num_envs, device=0, lib_path=None, dense=None, control_type="impedance", ik=None, preassembled=None,
                 num_connects=None, load_init_states=None, load_demo=None, robot_ob=True, object_ob=True, object_ob_all=True, subtask_ob=False,
                 fix_init=False, fix_init_parts=None, reset_robot_after_attach=None, control_freq=None, no_collision=False, assembled=False,
                 **cfg_overrides):
    """The Engine of `num_envs` envs of `agent` + `furniture_name` that both env surfaces run; `lib_path` as for Engine.  The keywords:
        `dense`: None for the sparse reward of FurnitureEnv; a dict of coefficient overrides (possibly empty) for the phase-based
        reward of FurnitureSawyerDenseRewardEnv, computed inside the step kernel (furniture_b200/dense.py).  A sequence gives one value per
        env (see Engine.set_dense_options; phase_ob is one per handle), the handle-wide config keeping the default.
        `control_type`: "impedance" (joint velocities, dof 9), "ik" (move 3, rotate 3, gripper, connect: dof 8) or "ik_quaternion" (the
        rotation as a quaternion relative to the hand: dof 9); the inverse kinematics and its three closed-loop repeats run inside the
        step kernel (furniture_b200/ik.py); or one of the NEW_CONTROLLERS ("position", "position_orientation", "joint_impedance",
        "joint_torque", "joint_velocity": the command of the controller, gripper, connect), which switch the scene to the torque-actuated
        robot and evaluate the controller before every mj_step inside the step kernel (furniture_b200/controllers.py); `ik`: overrides of ik.IK_DEFAULTS
        (move_speed, rotate_speed, action_repeat ...).
        `preassembled`, `num_connects`: config/furniture.py:81, :158 -- the recipe prefix [0, ..., k-1] every env starts its episodes
        from and the connections that end one; set_subtask changes them per env later.
        `load_init_states`, `load_demo`: config/furniture.py's paths (furniture.py:121-130), or the states themselves: every env picks its
        starts from the list of `load_init_states` (see load_init_states), and every env starts from the first state of the demo `load_demo`.
        `robot_ob`, `object_ob`, `object_ob_all`, `subtask_ob`: the observation flags of config/furniture.py (furniture.py:103-107, :215-252,
        :1344-1387).  object_ob_all=False keeps in object_ob only the two parts of each env's current subtask (14 numbers, zeros when none is
        left); subtask_ob=True adds their part ids + 1 (float32).  Each env's pair follows its connections and resets inside the kernels.
        `fix_init`, `fix_init_parts`, `reset_robot_after_attach`: config/furniture.py:116-127, :169-174 (see set_reset_options).  A dense env
        takes reset_robot_after_attach from `dense`, whose phase machine follows it (None: off, or the dense reward's).
        `assembled`: config/furniture.py:307-312, every episode starts from the welded furniture (see set_reset_options).
        `control_freq`, `no_collision`: config/furniture.py's (see set_sim_options), a value for every env or one per env.  control_freq sets
        the mj_steps of an env step (None: FeConfig.nsub, 50 = 10 Hz); it cannot be given together with an `nsub` override.
        The task options of config/furniture.py (TASK_OPTIONS: the alignment thresholds, auto_align, the placement noise, the reward
        coefficients, max_episode_steps): a scalar overrides FeConfig; a sequence gives one value per env (see set_task_options), the
        FeConfig field keeping its default.
    The other keywords override FeConfig fields (default_config).  The engine records `control_type` and `resize_factor`."""
    if control_freq is not None and "nsub" in cfg_overrides:
        raise ValueError("control_freq and nsub both set the mj_steps of an env step: give one of them")
    per_env = {k: cfg_overrides.pop(k) for k in list(cfg_overrides) if k in TASK_OPTIONS and np.ndim(cfg_overrides[k]) > 0}
    cfg = default_config(**cfg_overrides)
    # furn_size_rand (config/furniture.py:196-201): the reference draws one size factor per env process while loading the model.
    # A handle shares one model: the batch takes env 0's factor (the first draw of RandomState(seed)); every env's generator
    # still spends its draws like the reference's.  Different sizes side by side = several handles (MixedFurnitureEnv).
    resize_factor = None
    if cfg.furn_size_rand != 0:
        r = float(cfg.furn_size_rand)
        resize_factor = 1 + float(np.random.RandomState(int(cfg.seed)).uniform(-r, r, 1)[0])
    if control_type in NEW_CONTROLLERS:
        if agent != "Sawyer":
            raise NotImplementedError("the torque controllers are built for the Sawyer env")
        agent = "SawyerTorque"  # robots/sawyer/robot_torque.xml (furniture.py:1893-1899)
    elif control_type in ("ik", "ik_quaternion"):
        if agent not in ("Sawyer", "Baxter"):
            raise NotImplementedError("control_type='%s' is built for the Sawyer and Baxter envs" % control_type)
    elif control_type != "impedance":
        raise NotImplementedError("control_type %r is not built" % control_type)
    model = mjcf.load_scene(agent, furniture_name, resize_factor=resize_factor)
    ik_cfg = ctl_cfg = None
    if control_type in ("ik", "ik_quaternion"):
        from .ik import ik_config

        ik_cfg = ik_config(model, **dict(ik or {}, quaternion_mode=int(control_type == "ik_quaternion")))
    elif control_type in NEW_CONTROLLERS:
        from .controllers import ctl_config

        ctl_cfg = ctl_config(control_type, model=model, move_speed=(ik or {}).get("move_speed", 0.1))
    obs_flags = dict(robot_ob=bool(robot_ob), object_ob=bool(object_ob), object_ob_all=bool(object_ob_all), subtask_ob=bool(subtask_ob))
    dense_per_env = {k: v for k, v in (dense or {}).items() if np.ndim(v) > 0}
    dense_cfg = dense_config(**{k: v for k, v in dense.items() if k not in dense_per_env}) if dense is not None else None
    engine = Engine(model, num_envs, device=device, config=cfg, lib_path=lib_path, dense=dense_cfg,
                    ik=ik_cfg, controller=ctl_cfg, obs_layout=obs_flags, fix_init=fix_init, fix_init_parts=fix_init_parts,
                    reset_robot_after_attach=reset_robot_after_attach, assembled=assembled)
    engine.control_type, engine.resize_factor = control_type, resize_factor
    if control_freq is not None or np.any(no_collision):
        engine.set_sim_options(control_freq=control_freq, no_collision=no_collision if np.any(no_collision) else None)
    if per_env:
        engine.set_task_options(**per_env)
    if dense_per_env:  # a reset_robot_after_attach among them sets the arm's flag of each env too
        engine.set_dense_options(**dense_per_env)
    if prefix_length(preassembled) or num_connects is not None:
        engine.set_subtask(prefix_length(preassembled), num_connects)
    apply_init_config(engine, load_init_states, load_demo)
    return engine


class BatchedFurnitureEnv:
    def __init__(self, agent="Sawyer", furniture_name="table_lack_0825", num_envs=1, device=0, **options):
        """`num_envs` envs on CUDA device `device`; `options` are the keywords of build_engine (reward, control type, starts, observation
        flags, reset options, FeConfig overrides)."""
        import torch

        if not torch.cuda.is_available():
            raise RuntimeError("furniture_b200 needs a CUDA device (no CPU fallback)")
        self.torch = torch
        self.device = torch.device("cuda", device)
        torch.cuda.set_device(self.device)
        torch.zeros(1, device=self.device)  # make sure the primary context exists before the library binds to it
        self.engine = e = build_engine(agent, furniture_name, num_envs, device=device, **options)
        self.model, self.cfg, self.dense_cfg, self.ik_cfg, self.ctl_cfg = e.model, e.cfg, e.dense, e.ik, e.controller
        self.control_type, self.resize_factor, self.obs_flags = e.control_type, e.resize_factor, e.obs_flags
        self.num_envs, self.obs_dim, self.act_dim, self.dof, self.n_objects = num_envs, e.obs_dim, e.act_dim, e.act_dim, e.scene.npart
        cols, widths = e.obs_columns()
        self.object_ob_dim, self.subtask_ob_dim, self.robot_ob_dim, self.phase_ob_dim = (widths[k] for k in ("object_ob", "subtask_ob", "robot_ob", "phase_ob"))
        self._cols = OrderedDict((k, c if isinstance(c, slice) else torch.tensor(c, dtype=torch.long, device=self.device)) for k, c in cols.items())
        self._obs = torch.empty((num_envs, self.obs_dim), dtype=torch.float32, device=self.device)
        self._rew = torch.empty(num_envs, dtype=torch.float32, device=self.device)
        self._done = torch.empty(num_envs, dtype=torch.uint8, device=self.device)
        self._info = torch.empty((num_envs, INFO_DIM), dtype=torch.int32, device=self.device)
        self._act = torch.empty((num_envs, self.act_dim), dtype=torch.float32, device=self.device)
        # the engine's terminal buffers, which the step kernel writes for every env whose step ends an episode (the layout is fixed by now)
        tob, tq, tv = e.terminal_dev_ptrs()
        self._term_obs = device_view(tob, (num_envs, self.obs_dim), self.device)
        self._term_qpos = device_view(tq, (num_envs, self.model.nq), self.device)
        self._term_qvel = device_view(tv, (num_envs, self.model.nv), self.device)
        # the step's info dict (furniture.py:451-541), written by the step kernel: reward terms (sparse handles only) and episode records
        ri, ei = e.step_info_dev_ptrs()
        self._reward_info = device_view(ri, (num_envs, len(REWARD_INFO_KEYS)), self.device) if ri else None
        self._episode_info = device_view(ei, (num_envs, len(EPISODE_INFO_KEYS)), self.device)
        self.narms = int(e.scene.narms)
        self._last = None  # (done, info, actions) of the last step, tensors or host arrays, for step_infos
        self._episode_start = np.full(num_envs, time.time())  # host clock of each env's last reset seen by reset() / step_infos()

    def set_init_qpos(self, states):
        """FurnitureEnv.set_init_qpos (furniture.py:315-316), per env: one get_env_state dict or None for all envs, or a list of num_envs of
        them.  An env with a state starts its episodes from it, from its next reset on (auto-resets included), until an unstable step or a
        pick of load_init_states replaces it; None goes back to random placement."""
        self.engine.set_init_qpos(states)

    def load_init_states(self, states, envs=None):
        """--load_init_states (furniture.py:127-130, :1433-1434): before each reset, an env in `envs` (default: all) keeps its start with
        probability 0.2 and otherwise starts from a state drawn uniformly from `states` (a list of get_env_state dicts, e.g.
        demo.load_init_states(path)).  The draw runs inside the reset kernel on the env's own generator."""
        self.engine.load_init_states(states, envs)

    def set_init_states(self, states):
        """the raw bank of recorded starts that the per-env fields init_state / init_pick index (Engine.set_init_states)"""
        self.engine.set_init_states(states)

    def set_reset_options(self, fix_init=None, fix_init_parts=None, reset_robot_after_attach=None, envs=None, assembled=None):
        """per env (`envs`, default: all; None leaves an option as it is): fix_init keeps the furniture's start the same in every episode (the
        XML's init poses where it lists them, else the env's first random placement; no placement draw), fix_init_parts (a set or list of part
        names, or a comma string) does so for those parts only and places the others around them, reset_robot_after_attach sends the arm back
        to its start pose, with fresh noise, after every connection (furniture.py:916-924, :1389-1404, :1519-1532), assembled starts every
        episode from the welded furniture at the model's qpos0 (furniture.py:1501-1532)"""
        self.engine.set_reset_options(fix_init, fix_init_parts, reset_robot_after_attach, envs, assembled=assembled)

    def set_sim_options(self, control_freq=None, no_collision=None, envs=None):
        """per env (`envs`, default: all; a scalar or one value per env of `envs`; None leaves an option as it is): control_freq sets the
        mj_steps of the env's next steps to int((1 / control_freq) / timestep) (furniture.py:2855, :2878), no_collision switches every
        collision of the agent off at once (furniture.py:1962-1965), or back on with the model's masks.  Envs at different frequencies
        step together in one launch."""
        self.engine.set_sim_options(control_freq, no_collision, envs)

    def set_task_options(self, envs=None, **values):
        """per env (`envs`, default: all; a scalar or one value per env of `envs`): the alignment thresholds, auto_align, the placement
        noise, the reward coefficients and max_episode_steps of config/furniture.py by their key names (Engine.set_task_options), so that
        one batch can run a curriculum over them"""
        self.engine.set_task_options(envs, **values)

    def set_dense_options(self, envs=None, **values):
        """per env (`envs`, default: all; a scalar or one value per env of `envs`): the dense reward's coefficients, thresholds, diff_rew,
        early_termination and reset_robot_after_attach by the names of config/furniture_sawyer_dense.py (Engine.set_dense_options), so that
        one batch can run a reward sweep or a threshold curriculum"""
        self.engine.set_dense_options(envs, **values)

    def set_subtask(self, subtask, num_connects=None):
        """FurnitureEnv.set_subtask (furniture.py:204-207) with a scalar or an (N,) array each, so that the envs of one batch can train different
        legs of the assembly: env i's next reset (an auto-reset included) connects the first subtask[i] steps of the recipe inside the reset
        kernel, and its episodes then succeed after num_connects[i] more connections (None: once every part is connected)."""
        self.engine.set_subtask(subtask, num_connects)

    def num_subtask(self):
        """FurnitureEnv.num_subtask (furniture.py:209-213) per env, an (N,) array"""
        return self.engine.num_subtask()

    # spaces, in the reference's terms (furniture.py:215-252, :293-310)
    @property
    def observation_space(self):
        """key -> shape, in the order of the obs dict: object_ob (7 n_objects, or 14), subtask_ob (2), robot_ob, phase_ob (8, furniture_sawyer_dense.py:100-109)"""
        widths = dict(object_ob=self.object_ob_dim, subtask_ob=self.subtask_ob_dim, robot_ob=self.robot_ob_dim, phase_ob=self.phase_ob_dim)
        return OrderedDict((k, (widths[k],)) for k in self._cols)

    @property
    def action_space(self):
        return OrderedDict(default=(self.act_dim,))

    def _obs_dict(self, obs):
        d = OrderedDict()
        for k, c in self._cols.items():  # views of the row, but for the two-arm robot_ob without its joint columns
            if isinstance(c, slice):
                d[k] = obs[:, c]
            else:
                d[k] = obs.index_select(1, c) if hasattr(obs, "index_select") else obs[:, c.cpu().numpy()]
        return d

    def dense_infos(self):
        """per env, the dense reward's view of the last step (a host copy): phase, subtask, phase_bonus, the penalty terms ..."""
        if self.dense_cfg is None:
            raise RuntimeError("this env runs the sparse reward")
        rows = self.engine.get("dense_info")
        return tuple({k: float(r[j]) for j, k in enumerate(DENSE_INFO_KEYS)} for r in rows)

    def _stream(self):
        return self.torch.cuda.current_stream(self.device).cuda_stream

    def reset(self, mask=None):
        m = 0
        if mask is not None:
            mask = mask.to(device=self.device, dtype=self.torch.uint8).contiguous()
            m = mask.data_ptr()
        self.engine.env_reset(mask_dev=m, obs_dev=self._obs.data_ptr(), stream=self._stream())
        self._episode_start[mask.bool().cpu().numpy() if mask is not None else slice(None)] = time.time()
        return self._obs_dict(self._obs)

    def step(self, actions):
        """actions: (N, dof) float tensor (CUDA or CPU) in [-1, 1]; returns (obs dict, rewards, dones, info tensor)."""
        t = self.torch
        if isinstance(actions, dict):
            actions = actions["default"]
        a = t.as_tensor(actions)
        if a.device != self.device or a.dtype != t.float32 or not a.is_contiguous():
            self._act.copy_(a, non_blocking=True)
            a = self._act
        assert a.shape == (self.num_envs, self.act_dim), tuple(a.shape)
        self.engine.env_step_dev(a.data_ptr(), self._obs.data_ptr(), self._rew.data_ptr(), self._done.data_ptr(), self._info.data_ptr(), stream=self._stream())
        self._last = (self._done, self._info, a.clone() if self.narms == 2 else None)  # FurnitureBaxterEnv's info["ac"]
        return self._obs_dict(self._obs), self._rew, self._done, self._info

    def step_host(self, actions_np):
        """numpy in / numpy out through fe_env_step_host (pinned staging, copies inside the call)."""
        obs, rew, done, info = self.engine.env_step_host(actions_np)
        self._last = (done, info, np.array(actions_np, np.float32) if self.narms == 2 else None)
        return self._obs_dict(obs), rew, done.astype(bool), info

    def terminal_observation(self):
        """the observation FurnitureEnv.step returns with done (furniture.py:364-385), which step() cannot return because the env is already
        reset into its next episode: an obs dict with step()'s keys and columns, views of the device buffer the step kernel writes before the
        auto-reset (the two-arm IK / controller robot_ob is gathered, as in step()).  Row i is valid where the last step's done[i] is 1; after an
        unstable step it is the observation of the reset inside _do_simulation's except branch (furniture.py:2889-2897), as the reference's."""
        return self._obs_dict(self._term_obs)

    def terminal_state(self):
        """{"qpos" (N, nq), "qvel" (N, nv)}: what get_env_state would have returned at the end of each episode that the last step finished,
        views of the device buffers, valid where that step's done is 1"""
        return {"qpos": self._term_qpos, "qvel": self._term_qvel}

    def infos(self):
        info = self._info.cpu().numpy()
        return tuple({k: int(row[j]) for j, k in enumerate(INFO_KEYS)} for row in info)

    def reward_terms(self):
        """_compute_reward's info of the last step (furniture.py:535-540): {success_reward, touch_reward, pick_reward, ctrl_penalty}, each an
        (N,) float32 view of the device row the step kernel writes.  Where the step was not unstable, ((success_reward + touch_reward) +
        pick_reward) + ctrl_penalty is the step's reward, bit for bit; an unstable step's reward adds episode_unstable.  The dense env
        never runs that reward: its terms are dense_infos(), and this raises."""
        if self._reward_info is None:
            raise RuntimeError("this env runs the dense reward: its reward terms are dense_infos()")
        return OrderedDict((k, self._reward_info[:, j]) for j, k in enumerate(REWARD_INFO_KEYS))

    def episode_record(self):
        """_after_step's episode_reward and episode_unstable (furniture.py:469-476) of the episode the last step ended: (N,) float32 views of
        the device rows the step kernel writes before its auto-reset, valid where that step's done is 1 (the other rows are left as they
        were; rows no step has written are NaN).  episode_reward is the float32 sum of the episode's rewards before the penalty, plus the
        penalty; after an unstable step the episode is that step alone, as in the reference (furniture.py:2889-2897, :355-356)."""
        return OrderedDict((k, self._episode_info[:, j]) for j, k in enumerate(EPISODE_INFO_KEYS))

    def step_infos(self):
        """the tuple of N info dicts that the reference's SubprocVecEnv.step_wait returns for the last step (subproc_vec_env.py:100-113),
        with the keys of FurnitureEnv.step in its order (furniture.py:451-541, furniture_baxter.py:66-79): the sparse reward's four terms
        (the dense env: its dense_info keys), "ac" on the two-arm env, and at done the six episode_* keys, with episode_success_state (the
        terminal state, get_env_state's dict) on success.  episode_time is the host clock since the env's last reset that reset() or this
        method saw; every other value is the step kernel's.  One host round trip."""
        if self._last is None:
            raise RuntimeError("step_infos() describes the last step: call step() first")
        host = lambda x: x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)
        done, info, act = host(self._last[0]).astype(bool), host(self._last[1]), self._last[2]
        terms = self.engine.get("dense_info") if self._reward_info is None else host(self._reward_info)
        keys = DENSE_INFO_KEYS if self._reward_info is None else REWARD_INFO_KEYS
        now = time.time()
        ep = host(self._episode_info) if done.any() else None
        success_state = None
        if done.any() and info[done, 1].any():
            success_state = {k: host(v) for k, v in self.terminal_state().items()}
        act = host(act) if act is not None else None
        out = []
        for i in range(self.num_envs):
            d = OrderedDict((k, float(terms[i, j])) for j, k in enumerate(keys))
            if act is not None:
                d["ac"] = act[i].copy()
            if done[i]:
                d["episode_success"] = int(info[i, 1])
                d["episode_reward"] = float(ep[i, 0])
                d["episode_length"] = int(info[i, 3])
                d["episode_time"] = now - float(self._episode_start[i])
                d["episode_unstable"] = float(ep[i, 1])
                d["episode_num_connected"] = int(info[i, 0])
                if info[i, 1]:
                    d["episode_success_state"] = {k: v[i].astype(np.float64) for k, v in success_state.items()}
                self._episode_start[i] = now
            out.append(d)
        return tuple(out)

    def get_env_state(self):
        q, v = self.engine.get_state()
        return {"qpos": q, "qvel": v}

    def set_env_state(self, state):
        self.engine.set_state(state["qpos"], state["qvel"])
        self.engine.set("ctrl", np.zeros((self.num_envs, self.model.nu), np.float32))
        self.engine.forward(stream=self._stream())

    def close(self):
        self.engine.close()


def make_vec_env(env_id="IKEASawyer-v0", num_env=1, config=None, device=0):
    """make_vec_env(env_id, num_env, config) of furniture/env/base.py:55-80: `config` may be the reference's argparse
    Namespace (config/furniture.py) or a dict; options outside the accelerated path are ignored (listed in `.ignored_config`)."""
    if env_id not in ENV_IDS:
        raise ValueError("unknown env id %s (this build accelerates %s)" % (env_id, sorted(ENV_IDS)))
    agent, dense_reward = ENV_IDS[env_id]
    furniture, options, ignored = env_options(config, dense_reward)
    env = BatchedFurnitureEnv(agent, furniture, num_env, device=device, **options)
    env.ignored_config = ignored
    return env


class MixedFurnitureEnv:
    """A batch over several furniture models at once (BASELINE.json config 5; the reference reaches other furniture through
    `furniture_name` / `furniture_id`, config/furniture.py:43-55, one model per env process).  Envs are bucketed by
    furniture (SURVEY.md 8e: "bucket by furniture id first"): one engine handle per model, each with its own instance of the
    kernels (its own slice-layout table, see csrc/fe_host.cpp) and its own CUDA stream, so the buckets of a step run
    concurrently and fill the SMs together; the caller's stream waits for all of them at the end of the call.
    nq / nv / obs_dim differ per bucket; `object_ob` is returned zero-padded to the widest model, `robot_ob` is common.  With
    object_ob_all=False (a keyword passed on to every bucket, like the other observation flags) `object_ob` holds the two parts of each
    env's current subtask: 14 numbers whatever the model, so nothing is padded; `subtask_ob` (subtask_ob=True) is gathered like the rest.

      env = MixedFurnitureEnv(["table_lack_0825", "chair_ingolf_0650"], envs_per_model=64)
      obs = env.reset(); obs, rew, done, info = env.step(actions)          # actions: (num_envs, dof)
    """

    def __init__(self, furniture_names, envs_per_model, agent="Sawyer", device=0, object_ob_dim=None, pad_to=None, **cfg_overrides):
        import torch

        self.torch = torch
        self.names = list(furniture_names)
        counts = [envs_per_model] * len(self.names) if isinstance(envs_per_model, int) else list(envs_per_model)
        assert len(counts) == len(self.names)
        seed = cfg_overrides.pop("seed", 123)
        if cfg_overrides.get("fix_init_parts"):
            raise ValueError("fix_init_parts names the parts of one furniture model; set it per bucket with set_reset_options")
        self.buckets, self.offsets, off = [], [], 0
        for name, n in zip(self.names, counts):
            self.buckets.append(BatchedFurnitureEnv(agent, name, n, device=device, seed=seed + off, **cfg_overrides))
            self.offsets.append(off)
            off += n
        self.real_envs = off           # envs that exist; rows beyond them (up to pad_to) are padding for equal-sized shards
        off = max(off, pad_to or 0)
        self.num_envs = off
        b0 = self.buckets[0]
        self.device, self.act_dim, self.dof, self.robot_ob_dim = b0.device, b0.act_dim, b0.act_dim, b0.robot_ob_dim
        assert all(b.act_dim == self.act_dim and b.robot_ob_dim == self.robot_ob_dim for b in self.buckets)
        # object_ob is zero-padded to the widest model of this batch, or to `object_ob_dim` (the widest of a sharded batch, so
        # that every rank's rows have the same width); without object_ob_all it is 14 wide everywhere
        space = b0.observation_space
        self.object_ob_dim = max([b.object_ob_dim for b in self.buckets] + [object_ob_dim or 0]) if b0.obs_flags["object_ob"] else 0
        widths = OrderedDict((k, self.object_ob_dim if k == "object_ob" else space[k][0]) for k in space)
        self.obs_dim = sum(widths.values())
        self._obs = torch.zeros((off, self.obs_dim), dtype=torch.float32, device=self.device)  # [object_ob (padded) | subtask_ob | robot_ob]
        self._views, o = OrderedDict(), 0
        for k, w in widths.items():
            self._views[k], o = self._obs[:, o : o + w], o + w
        self._rew = torch.empty(off, dtype=torch.float32, device=self.device)
        self._done = torch.empty(off, dtype=torch.uint8, device=self.device)
        self._info = torch.empty((off, INFO_DIM), dtype=torch.int32, device=self.device)
        self._act = torch.empty((off, self.act_dim), dtype=torch.float32, device=self.device)
        self._streams = [torch.cuda.Stream(device=self.device) for _ in self.buckets]
        self._term_obs = torch.zeros_like(self._obs)  # terminal_observation's rows, laid out like _obs
        self.dense_cfg = b0.dense_cfg  # every bucket is built with the same reward
        self._term_views, o = OrderedDict(), 0
        for k, w in widths.items():
            self._term_views[k], o = self._term_obs[:, o : o + w], o + w

    def set_sim_options(self, control_freq=None, no_collision=None, envs=None):
        """BatchedFurnitureEnv.set_sim_options with `envs` as global indices of this batch (default: all); each value is a scalar or one
        per env of `envs`"""
        self._per_bucket(envs, dict(control_freq=control_freq, no_collision=no_collision), lambda b, idx, v: b.set_sim_options(envs=idx, **v))

    def set_task_options(self, envs=None, **values):
        """BatchedFurnitureEnv.set_task_options with `envs` as global indices of this batch (default: all); each value is a scalar or one
        per env of `envs`"""
        self._per_bucket(envs, values, lambda b, idx, v: b.set_task_options(idx, **v))

    def set_dense_options(self, envs=None, **values):
        """BatchedFurnitureEnv.set_dense_options with `envs` as global indices of this batch (default: all); each value is a scalar or one
        per env of `envs`"""
        self._per_bucket(envs, values, lambda b, idx, v: b.set_dense_options(idx, **v))

    def _per_bucket(self, envs, values, set_options):
        """set_options(bucket, its envs, their values) for every bucket that holds some of `envs` (global indices, default: all), each of
        `values` a scalar or one per env of `envs` (None: left out)"""
        idx = np.arange(self.real_envs) if envs is None else np.asarray(envs, dtype=np.int64).ravel()
        if idx.size and (idx.min() < 0 or idx.max() >= self.real_envs):
            raise IndexError("envs must lie in [0, %d), got %s" % (self.real_envs, idx.tolist()))
        per = {k: np.broadcast_to(np.asarray(v), idx.shape) for k, v in values.items() if v is not None}
        for b, off in zip(self.buckets, self.offsets):
            sel = (idx >= off) & (idx < off + b.num_envs)
            if sel.any():
                set_options(b, idx[sel] - off, {k: v[sel] for k, v in per.items()})

    def _obs_dict(self, obs):
        d, o = OrderedDict(), 0
        for k, v in self._views.items():
            d[k], o = obs[:, o : o + v.shape[1]], o + v.shape[1]
        return d

    def algorithmic_bytes_per_step(self, nsub=50):
        """SURVEY.md 8d: sum over the buckets of envs x (nsub x 4 (2 nq + 5 nv + nu) + 4 (obs + act) + 8)"""
        return sum(b.num_envs * (nsub * 4 * (2 * b.model.nq + 5 * b.model.nv + b.model.nu) + 4 * (b.obs_dim + b.act_dim) + 8) for b in self.buckets)

    def _fan_out(self, fn):
        """run fn(bucket, offset) for every bucket on the bucket's own stream, ordered after the caller's stream; join at the end"""
        t = self.torch
        cur = t.cuda.current_stream(self.device)
        for b, off, s in zip(self.buckets, self.offsets, self._streams):
            s.wait_stream(cur)
            with t.cuda.stream(s):
                fn(b, off)
        for s in self._streams:
            cur.wait_stream(s)

    def bucket_of(self, env_index):
        """(furniture name, index inside its bucket) of a global env index"""
        for name, off, b in zip(self.names, self.offsets, self.buckets):
            if off <= env_index < off + b.num_envs:
                return name, env_index - off
        raise IndexError(env_index)

    def _collect(self, b, off, od):
        sl = slice(off, off + b.num_envs)
        for k, v in od.items():
            self._views[k][sl, : v.shape[1]].copy_(v)
        return sl

    def reset(self):
        self._fan_out(lambda b, off: self._collect(b, off, b.reset()))
        return self._obs_dict(self._obs)

    def step(self, actions):
        t = self.torch
        if isinstance(actions, dict):
            actions = actions["default"]
        a = t.as_tensor(actions)
        if a.device != self.device or a.dtype != t.float32 or not a.is_contiguous():
            self._act.copy_(a, non_blocking=True)
            a = self._act
        assert a.shape == (self.num_envs, self.act_dim), tuple(a.shape)
        def one(b, off):
            od, rew, done, info = b.step(a[off : off + b.num_envs])
            sl = self._collect(b, off, od)
            self._rew[sl].copy_(rew); self._done[sl].copy_(done); self._info[sl].copy_(info)

        self._fan_out(one)
        return self._obs_dict(self._obs), self._rew, self._done, self._info

    def terminal_observation(self):
        """BatchedFurnitureEnv.terminal_observation of every bucket, gathered in global env order with step()'s layout (object_ob zero-padded to
        the batch's width, or 14 wide without object_ob_all); row i is valid where the last step's done[i] is 1"""
        for b, off in zip(self.buckets, self.offsets):
            for k, v in b.terminal_observation().items():
                self._term_views[k][off : off + b.num_envs, : v.shape[1]].copy_(v)
        return self._obs_dict(self._term_obs)

    def dense_infos(self):
        """(num_envs, 12) float32 tensor of every bucket's dense_info rows after the last step, in global env order and the order of
        dense.INFO_KEYS; padding rows are zeros (a host round trip per bucket)"""
        if self.dense_cfg is None:
            raise RuntimeError("this env runs the sparse reward")
        rows = self.torch.zeros((self.num_envs, len(DENSE_INFO_KEYS)), dtype=self.torch.float32, device=self.device)
        for b, off in zip(self.buckets, self.offsets):
            rows[off : off + b.num_envs] = self.torch.from_numpy(b.engine.get("dense_info"))
        return rows

    def _gather_rows(self, rows_of, width):
        """(num_envs, width) float32 tensor of every bucket's rows_of(bucket) in global env order; padding rows are NaN"""
        rows = self.torch.full((self.num_envs, width), float("nan"), dtype=self.torch.float32, device=self.device)
        for b, off in zip(self.buckets, self.offsets):
            rows[off : off + b.num_envs] = rows_of(b)
        return rows

    def reward_terms(self):
        """BatchedFurnitureEnv.reward_terms of every bucket in global env order: {success_reward, touch_reward, pick_reward, ctrl_penalty},
        each a (num_envs,) float32 tensor (padding rows NaN)"""
        if self.dense_cfg is not None:
            raise RuntimeError("this env runs the dense reward: its reward terms are dense_infos()")
        rows = self._gather_rows(lambda b: b._reward_info, len(REWARD_INFO_KEYS))
        return OrderedDict((k, rows[:, j]) for j, k in enumerate(REWARD_INFO_KEYS))

    def episode_record(self):
        """BatchedFurnitureEnv.episode_record of every bucket in global env order: {episode_reward, episode_unstable}, each a (num_envs,)
        float32 tensor, valid where the last step's done is 1 (padding rows NaN)"""
        rows = self._gather_rows(lambda b: b._episode_info, len(EPISODE_INFO_KEYS))
        return OrderedDict((k, rows[:, j]) for j, k in enumerate(EPISODE_INFO_KEYS))

    def step_infos(self):
        """BatchedFurnitureEnv.step_infos of every bucket in global env order, num_envs dicts; padding rows are empty dicts"""
        out = []
        for b in self.buckets:
            out.extend(b.step_infos())
        return tuple(out) + ({},) * (self.num_envs - self.real_envs)

    def terminal_state(self):
        """BatchedFurnitureEnv.terminal_state of every bucket, in bucket order (bucket i holds the envs from offsets[i] on): the models' nq and nv
        differ, so the states are not stacked"""
        return [b.terminal_state() for b in self.buckets]

    def close(self):
        for b in self.buckets:
            b.close()


def model_costs():
    """measured GPU time per env-step per env (microseconds) of every compiled Sawyer scene: compiled/cost.json, written by
    tools/calibrate_models.py on an H100; {} when absent"""
    import json
    import os

    p = os.path.join(os.path.dirname(os.path.abspath(__file__)), "compiled", "cost.json")
    if not os.path.exists(p):
        return {}
    return {k: float(v["us_per_env_step"]) for k, v in json.load(open(p)).items()}


def shard_furniture(names, envs_per_model, world, nv=None, envs_per_rank=None, cost_per_env=None, chunk=None):
    """Whole furniture buckets per GPU for a mixed batch (SURVEY.md 8e: "bucket by furniture id first so each GPU gets
    whole buckets"): longest-processing-time greedy on the cost of each bucket = envs x cost per env, the cost per env being
    the measured step time of the model (`cost_per_env`, e.g. model_costs(): the spread between furniture models is 40x and
    follows contact count and overflow, not nv) or, without measurements, nv^3 (SURVEY.md 8e).  Returns, per rank, the list
    of (name, envs) it owns; every rank computes the same answer.  With `envs_per_rank` the env counts are re-dealt inside
    each rank so that every rank holds exactly that many envs (its models share them evenly); without it ranks may own
    different numbers of envs and the caller pads the shards to the largest."""
    counts = [envs_per_model] * len(names) if isinstance(envs_per_model, int) else list(envs_per_model)
    if cost_per_env is not None and all(n in cost_per_env for n in names):
        per_env = [float(cost_per_env[n]) for n in names]
    else:
        if nv is None:
            nv = [mjcf.load_scene("Sawyer", n).nv for n in names]
        per_env = [float(v) ** 3 for v in nv]
    # with `chunk`, a bucket larger than that is dealt in pieces of at most `chunk` envs: a model whose envs cost 40x the others'
    # (SURVEY.md 8e asks for whole buckets; one such bucket alone outweighs a GPU's fair share) is spread over several ranks;
    # the pieces of one model that land on the same rank are merged back into one bucket
    items = []
    for i, (nm, c) in enumerate(zip(names, counts)):
        step = c if not chunk else chunk
        for k in range(0, c, step):
            items.append((i, min(step, c - k)))
    order = sorted(range(len(items)), key=lambda j: (-items[j][1] * per_env[items[j][0]], names[items[j][0]], j))
    load, got = [0.0] * world, [dict() for _ in range(world)]
    for j in order:
        i, c = items[j]
        r = min(range(world), key=lambda k: (load[k], k))
        load[r] += c * per_env[i]
        got[r][i] = got[r].get(i, 0) + c
    owned = [[(names[i], c) for i, c in g.items()] for g in got]  # in the order the buckets were dealt (heaviest first)
    if envs_per_rank is not None:
        for r in range(world):
            k = len(owned[r])
            assert 0 < k <= envs_per_rank, "rank %d owns %d models for %d envs" % (r, k, envs_per_rank)
            owned[r] = [(nm, envs_per_rank // k + (1 if j < envs_per_rank % k else 0)) for j, (nm, _) in enumerate(owned[r])]
    return owned


class ShardedFurnitureEnv:
    """One process per GPU (torch.distributed, backend nccl). Each rank steps its own contiguous env shard; after the
    step one all_gather makes the packed [obs | reward | done] of every shard visible on every rank.

    `gather_info` widens the message by each env's info row (and, on a dense-reward shard, its dense_info row), so that step returns the
    info of every env and dense_infos() the dense rows of every env; `gather_terminal` widens it by the terminal observation, which
    terminal_observation() returns for every env; `gather_step_info` widens it by the reward terms and the episode record, which
    reward_terms() and episode_record() return for every env.  The step kernel writes the wider rows itself (Engine.set_packed_layout,
    Engine.set_packed_step_info); a shard without that kernel (MixedFurnitureEnv, a stand-in) has the same columns filled from its own
    step, terminal_observation(), dense_infos(), reward_terms() and episode_record()."""

    def __init__(self, envs_per_gpu, agent="Sawyer", furniture_name="table_lack_0825", env=None, gather_info=False, gather_terminal=False,
                 gather_step_info=False, **cfg_overrides):
        import torch
        import torch.distributed as dist

        self.torch, self.dist = torch, dist
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        local = int(__import__("os").environ.get("LOCAL_RANK", self.rank))
        cfg_overrides.setdefault("seed", self.shard_seed(123, self.rank, envs_per_gpu))
        # `env` lets the host logic be exercised with a stand-in shard (tests/test_sharded_gloo.py)
        self.env = env if env is not None else BatchedFurnitureEnv(agent, furniture_name, envs_per_gpu, device=local, **cfg_overrides)
        self.envs_per_gpu = envs_per_gpu
        self.num_envs = envs_per_gpu * self.world
        self.gather_info, self.gather_terminal = bool(gather_info), bool(gather_terminal)
        layout = dict(info=self.gather_info, dense_info=self.gather_info and getattr(self.env, "dense_cfg", None) is not None,
                      terminal_obs=self.gather_terminal)
        self.gather_step_info = bool(gather_step_info)
        self._cols = packed_columns(self.env.obs_dim, step_info=self.gather_step_info, **layout)
        self._kernel = hasattr(self.env, "_stream")  # a BatchedFurnitureEnv: its step kernel writes the rows
        if self._kernel:
            self.env.engine.set_packed_layout(**layout)
            self.env.engine.set_packed_step_info(self.gather_step_info)
        self.pack_dim = next(reversed(self._cols.values())).stop
        self._pack = torch.empty((envs_per_gpu, self.pack_dim), dtype=torch.float32, device=self.env.device)
        self._all = torch.empty((self.num_envs, self.pack_dim), dtype=torch.float32, device=self.env.device)
        self.timing, self._events = False, []

    @staticmethod
    def shard_seed(seed, rank, envs_per_gpu):
        """env e of rank r is seeded seed + r * envs_per_gpu + e: the reference's seed + rank per env (env/base.py:77)"""
        return seed + rank * envs_per_gpu

    def _gather(self):
        self.dist.all_gather_into_tensor(self._all, self._pack)
        return self._all

    def reset(self):
        self.env.reset()
        p = self._pack  # resets are rare: packed on the host side of the stream (the step kernel writes its own rows)
        p[:, : self.env.obs_dim] = self.env._obs
        p[:, self.env.obs_dim :] = 0  # reward, done and the info, dense_info and terminal columns
        allp = self._gather()
        return self.env._obs_dict(allp[:, : self.env.obs_dim])

    def _pack_on_host(self, a):
        """the rows of a shard without the packed step kernel, filled from its own outputs into the same columns"""
        env, c, p = self.env, self._cols, self._pack
        od_, rew, done, info = env.step(a)
        p[:, c["obs"]] = env._obs
        p[:, c["reward"]] = rew.reshape(-1, 1)
        p[:, c["done"]] = done.float().reshape(-1, 1)
        if "info" in c:
            p[:, c["info"]].view(self.torch.int32).copy_(info)  # bit patterns, as the kernel writes them
        if "dense_info" in c:
            p[:, c["dense_info"]] = env.dense_infos()
        if "terminal_obs" in c:
            p[:, c["terminal_obs"]] = self.torch.cat(list(env.terminal_observation().values()), 1)
        if "reward_info" in c:  # the terms (NaN on a dense shard, as the kernel writes them); the episode record where done, as in episode_info
            t = self.torch
            dense = getattr(env, "dense_cfg", None) is not None
            p[:, c["reward_info"]] = float("nan") if dense else t.stack(list(env.reward_terms().values()), 1)
            d = t.as_tensor(done, device=p.device).bool().reshape(-1, 1)
            p[:, c["episode_info"]] = t.where(d, t.stack(list(env.episode_record().values()), 1).to(p.device), p[:, c["episode_info"]])
        return info

    def step(self, local_actions):
        """One env step of the local shard, then the single collective of the data path.  The step kernel writes
        the packed rows into the registered send buffer itself (fe_env_step_packed); with `timing` set, CUDA events
        separate the kernel from the time spent in the all-gather (which includes waiting for the slowest rank).
        Returns the gathered obs dict, rewards and dones, and the info of every env under gather_info (an int32 view of the message),
        else this shard's own info."""
        env, t = self.env, self.torch
        a = t.as_tensor(local_actions["default"] if isinstance(local_actions, dict) else local_actions)
        if a.device != env.device or a.dtype != t.float32 or not a.is_contiguous():
            env._act.copy_(a, non_blocking=True)
            a = env._act
        assert a.shape == (env.num_envs, env.act_dim), tuple(a.shape)
        if self.timing:
            ev = [t.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record()
        if self._kernel:
            env.engine.env_step_packed(a.data_ptr(), self._pack.data_ptr(), env._info.data_ptr(), stream=env._stream())
            info = env._info
        else:  # MixedFurnitureEnv, or the stand-in shard of the gloo tests
            info = self._pack_on_host(a)
        if self.timing:
            ev[1].record()
        allp = self._gather()
        if self.timing:
            ev[2].record()
            self._events.append(ev)
        c = self._cols
        if "info" in c:
            info = allp[:, c["info"]].view(t.int32)
        return env._obs_dict(allp[:, c["obs"]]), allp[:, c["reward"].start], allp[:, c["done"].start] > 0.5, info

    def terminal_observation(self):
        """the terminal observation of every env (gather_terminal=True): an obs dict with step()'s keys, views of the last gathered message;
        row i is valid where the last gathered done[i] is 1"""
        if "terminal_obs" not in self._cols:
            raise ValueError("terminal_observation() needs ShardedFurnitureEnv(..., gather_terminal=True)")
        return self.env._obs_dict(self._all[:, self._cols["terminal_obs"]])

    def dense_infos(self):
        """(num_envs, 12) float32 rows of the dense reward's dense_info of every env after the last gathered step (gather_info=True on a
        dense-reward shard), in the order of dense.INFO_KEYS; views of the message"""
        if "dense_info" not in self._cols:
            raise ValueError("dense_infos() needs ShardedFurnitureEnv(..., gather_info=True) on a shard that runs the dense reward")
        return self._all[:, self._cols["dense_info"]]

    def reward_terms(self):
        """{success_reward, touch_reward, pick_reward, ctrl_penalty} of every env after the last gathered step (gather_step_info=True), each a
        (num_envs,) view of the message; NaN on a dense-reward shard, which has no such terms"""
        if "reward_info" not in self._cols:
            raise ValueError("reward_terms() needs ShardedFurnitureEnv(..., gather_step_info=True)")
        return OrderedDict((k, self._all[:, self._cols["reward_info"].start + j]) for j, k in enumerate(REWARD_INFO_KEYS))

    def episode_record(self):
        """{episode_reward, episode_unstable} of every env (gather_step_info=True), each a (num_envs,) view of the last gathered message;
        valid where its done is 1"""
        if "episode_info" not in self._cols:
            raise ValueError("episode_record() needs ShardedFurnitureEnv(..., gather_step_info=True)")
        return OrderedDict((k, self._all[:, self._cols["episode_info"].start + j]) for j, k in enumerate(EPISODE_INFO_KEYS))

    def local_slice(self, gathered):
        """rows of this rank's own shard in a gathered (num_envs, ...) tensor"""
        return gathered[self.rank * self.envs_per_gpu : (self.rank + 1) * self.envs_per_gpu]

    def pop_timing(self):
        """(kernel_ms, gather_ms) lists of the steps since the last call (needs timing=True; synchronises)"""
        self.torch.cuda.synchronize()
        k = [e[0].elapsed_time(e[1]) for e in self._events]
        g = [e[1].elapsed_time(e[2]) for e in self._events]
        self._events = []
        return k, g
