"""Batched gym/VecEnv-shaped surface over the engine (torch tensors in, torch tensors out).

Mirrors the reference's call surface for the accelerated path:
  make_vec_env(env_id, num_env, config)   furniture/env/base.py:55-80          -> BatchedFurnitureEnv
  VecEnv.reset() / step(actions)          furniture/util/vec_env.py:53-162, subproc_vec_env.py:100-113 (auto-reset on done)
  obs dict {"object_ob", "robot_ob"}      furniture.py:1344-1387, furniture_sawyer.py:103-155 (OrderedDict order kept)
  get_env_state / set_env_state           furniture.py:1781-1803
Observations live in one contiguous (N, obs_dim) float32 CUDA tensor written by the step kernel; the dict entries are
views of it.  ShardedFurnitureEnv adds the multi-GPU form: env shards are independent (one process per GPU), the only
collective is one NCCL all_gather of the packed [obs | reward | done] tensor per step (SURVEY.md 8e).
"""
from __future__ import annotations

from collections import OrderedDict

import numpy as np

from . import mjcf
from .dense import DENSE_DEFAULTS, DENSE_ENV_DEFAULTS, INFO_KEYS as DENSE_INFO_KEYS, dense_config
from .engine import INFO_DIM, Engine, default_config

INFO_KEYS = ("num_connected", "episode_success", "episode_unstable", "episode_length", "ncon", "solver_iters")
ENV_IDS = {"IKEASawyer-v0": "Sawyer", "FurnitureSawyerEnv": "Sawyer", "IKEABaxter-v0": "Baxter", "FurnitureBaxterEnv": "Baxter",
           "IKEASawyerDense-v0": "Sawyer", "furniture-sawyer-densereward-v0": "Sawyer", "FurnitureSawyerDenseRewardEnv": "Sawyer"}
NEW_CONTROLLERS = ("position", "position_orientation", "joint_impedance", "joint_torque", "joint_velocity")  # furniture.py:41-47
DENSE_IDS = {"IKEASawyerDense-v0", "furniture-sawyer-densereward-v0", "FurnitureSawyerDenseRewardEnv"}  # env/__init__.py:103-114
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


def split_config(config):
    """Reference-style config (argparse Namespace or dict, config/furniture.py) -> (furniture name, FeConfig overrides, ignored keys).
    `furniture_name` wins over `furniture_id` as in furniture.py:157-161; keys the accelerated path has no use for (port, background,
    camera and rendering options ...) are returned so that callers can report them instead of failing on them."""
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
    renamed = {"furn_xyz_rand": "furn_xyz_rand", "furn_rot_rand": "furn_rot_rand", "agent_xyz_rand": "agent_xyz_rand", "alignment_pos_dist": "alignment_pos_dist"}
    over = {renamed.get(k, k): v for k, v in cfg.items() if renamed.get(k, k) in fields and v is not None}
    ignored = sorted(k for k in cfg if k not in over and k not in ("furniture_name", "furniture_id", "control_type"))
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
    name, over, ignored = split_config(merged)
    dense = {k: merged[k] for k in DENSE_DEFAULTS if k in merged}
    if "ctrl_penalty_coef" in over:
        dense["ctrl_penalty_coef"] = over["ctrl_penalty_coef"]
    return name, over, dense, [k for k in ignored if k not in DENSE_DEFAULTS]


class BatchedFurnitureEnv:
    def __init__(self, agent="Sawyer", furniture_name="table_lack_0825", num_envs=1, device=0, dense=None, control_type="impedance", ik=None,
                 **cfg_overrides):
        """`dense`: None for the sparse reward of FurnitureEnv; a dict of coefficient overrides (possibly empty) for the phase-based
        reward of FurnitureSawyerDenseRewardEnv, computed inside the step kernel (furniture_b200/dense.py).
        `control_type`: "impedance" (joint velocities, dof 9), "ik" (move 3, rotate 3, gripper, connect: dof 8) or "ik_quaternion" (the
        rotation as a quaternion relative to the hand: dof 9); the inverse kinematics and its three closed-loop repeats run inside the
        step kernel (furniture_b200/ik.py); or one of the NEW_CONTROLLERS ("position", "position_orientation", "joint_impedance",
        "joint_torque", "joint_velocity": the command of the controller, gripper, connect), which switch the scene to the torque-actuated
        robot and evaluate the controller before every mj_step inside the step kernel (furniture_b200/controllers.py); `ik`: overrides of ik.IK_DEFAULTS
        (move_speed, rotate_speed, action_repeat ...)."""
        import torch

        if not torch.cuda.is_available():
            raise RuntimeError("furniture_b200 needs a CUDA device (no CPU fallback)")
        self.torch = torch
        self.device = torch.device("cuda", device)
        torch.cuda.set_device(self.device)
        torch.zeros(1, device=self.device)  # make sure the primary context exists before the library binds to it
        self.cfg = default_config(**cfg_overrides)
        # furn_size_rand (config/furniture.py:196-201): the reference draws one size factor per env process while loading the model.
        # A handle shares one model: the batch takes env 0's factor (the first draw of RandomState(seed)); every env's generator
        # still spends its draws like the reference's.  Different sizes side by side = several handles (MixedFurnitureEnv).
        self.resize_factor = None
        if self.cfg.furn_size_rand != 0:
            r = float(self.cfg.furn_size_rand)
            self.resize_factor = 1 + float(np.random.RandomState(int(self.cfg.seed)).uniform(-r, r, 1)[0])
        if control_type in NEW_CONTROLLERS:
            if agent != "Sawyer":
                raise NotImplementedError("the torque controllers are built for the Sawyer env")
            agent = "SawyerTorque"  # robots/sawyer/robot_torque.xml (furniture.py:1893-1899)
        self.model = mjcf.load_scene(agent, furniture_name, resize_factor=self.resize_factor)
        self.dense_cfg = dense_config(**dense) if dense is not None else None
        self.control_type = control_type
        self.ik_cfg = None
        if control_type in ("ik", "ik_quaternion"):
            if agent not in ("Sawyer", "Baxter"):
                raise NotImplementedError("control_type='%s' is built for the Sawyer and Baxter envs" % control_type)
            from .ik import ik_config

            self.ik_cfg = ik_config(self.model, **dict(ik or {}, quaternion_mode=int(control_type == "ik_quaternion")))
        self.ctl_cfg = None
        if control_type in NEW_CONTROLLERS:
            from .controllers import ctl_config

            self.ctl_cfg = ctl_config(control_type, model=self.model, move_speed=(ik or {}).get("move_speed", 0.1))
        elif control_type not in ("impedance", "ik", "ik_quaternion"):
            raise NotImplementedError("control_type %r is not built" % control_type)
        self.engine = Engine(self.model, num_envs, device=device, config=self.cfg, dense=self.dense_cfg, ik=self.ik_cfg, controller=self.ctl_cfg)
        self.num_envs = num_envs
        self.obs_dim, self.act_dim = self.engine.obs_dim, self.engine.act_dim
        self.n_objects = self.engine.scene.npart
        self.object_ob_dim = 7 * self.n_objects
        self.robot_ob_dim = self.engine.scene.robot_ob_dim
        # control_type="ik": robot_ob is gripper_qpos, eef_pos, eef_quat, eef_velp, eef_velr only -- no joint positions / velocities
        # (furniture_sawyer.py:110-125); the device row always holds all of it, the 15 numbers are its tail
        self._robot_skip = 0 if control_type == "impedance" else 14
        self._narms = max(1, int(self.engine.scene.narms))
        self.robot_ob_dim -= self._robot_skip * self._narms
        self._robot_cols = None
        if self._robot_skip and self._narms > 1:  # two arms: the 15-number tail of each arm's block (furniture_baxter.py:137-160)
            per = self.engine.scene.robot_ob_dim // self._narms
            cols = [self.object_ob_dim + a * per + k for a in range(self._narms) for k in range(self._robot_skip, per)]
            self._robot_cols = torch.tensor(cols, dtype=torch.long, device=self.device)
        self.phase_ob_dim = 8 if self.engine.scene.phase_ob else 0
        self.dof = self.act_dim
        self._obs = torch.empty((num_envs, self.obs_dim), dtype=torch.float32, device=self.device)
        self._rew = torch.empty(num_envs, dtype=torch.float32, device=self.device)
        self._done = torch.empty(num_envs, dtype=torch.uint8, device=self.device)
        self._info = torch.empty((num_envs, INFO_DIM), dtype=torch.int32, device=self.device)
        self._act = torch.empty((num_envs, self.act_dim), dtype=torch.float32, device=self.device)

    # spaces, in the reference's terms (furniture.py:215-252, :293-310)
    @property
    def observation_space(self):
        sp = OrderedDict(object_ob=(self.object_ob_dim,), robot_ob=(self.robot_ob_dim,))
        if self.phase_ob_dim:
            sp["phase_ob"] = (8,)  # furniture_sawyer_dense.py:100-109
        return sp

    @property
    def action_space(self):
        return OrderedDict(default=(self.act_dim,))

    def _obs_dict(self, obs):
        a, b = self.object_ob_dim, self.object_ob_dim + self._robot_skip * self._narms + self.robot_ob_dim
        if self._robot_cols is not None:
            cols = self._robot_cols if hasattr(obs, "index_select") else self._robot_cols.cpu().numpy()
            d = OrderedDict(object_ob=obs[:, :a], robot_ob=obs.index_select(1, cols) if hasattr(obs, "index_select") else obs[:, cols])
        else:
            d = OrderedDict(object_ob=obs[:, :a], robot_ob=obs[:, a + self._robot_skip : b])
        if self.phase_ob_dim:
            d["phase_ob"] = obs[:, b:]
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
        return self._obs_dict(self._obs), self._rew, self._done, self._info

    def step_host(self, actions_np):
        """numpy in / numpy out through fe_env_step_host (pinned staging, copies inside the call)."""
        obs, rew, done, info = self.engine.env_step_host(actions_np)
        return self._obs_dict(obs), rew, done.astype(bool), info

    def infos(self):
        info = self._info.cpu().numpy()
        return tuple({k: int(row[j]) for j, k in enumerate(INFO_KEYS)} for row in info)

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
    agent = ENV_IDS.get(env_id)
    if agent is None:
        raise ValueError("unknown env id %s (this build accelerates %s)" % (env_id, sorted(ENV_IDS)))
    ctl = control_options(config)
    if env_id in DENSE_IDS:
        furniture, over, dense, ignored = split_dense_config(config)
        env = BatchedFurnitureEnv(agent, furniture, num_env, device=device, dense=dense, **ctl, **over)
    else:
        furniture, over, ignored = split_config(config)
        env = BatchedFurnitureEnv(agent, furniture, num_env, device=device, **ctl, **over)
    ignored = [k for k in ignored if k not in ("move_speed", "rotate_speed")] if "ik" in ctl else ignored
    env.ignored_config = ignored
    return env


class MixedFurnitureEnv:
    """A batch over several furniture models at once (BASELINE.json config 5; the reference reaches other furniture through
    `furniture_name` / `furniture_id`, config/furniture.py:43-55, one model per env process).  Envs are bucketed by
    furniture (SURVEY.md 8e: "bucket by furniture id first"): one engine handle per model, each with its own instance of the
    kernels (its own slice-layout table, see csrc/fe_host.cpp) and its own CUDA stream, so the buckets of a step run
    concurrently and fill the SMs together; the caller's stream waits for all of them at the end of the call.
    nq / nv / obs_dim differ per bucket; `object_ob` is returned zero-padded to the widest model, `robot_ob` is common.

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
        # that every rank's rows have the same width)
        self.object_ob_dim = max([b.object_ob_dim for b in self.buckets] + [object_ob_dim or 0])
        self.obs_dim = self.object_ob_dim + self.robot_ob_dim
        self._obs = torch.zeros((off, self.obs_dim), dtype=torch.float32, device=self.device)  # [object_ob (padded) | robot_ob]
        self._object_ob, self._robot_ob = self._obs[:, : self.object_ob_dim], self._obs[:, self.object_ob_dim :]
        self._rew = torch.empty(off, dtype=torch.float32, device=self.device)
        self._done = torch.empty(off, dtype=torch.uint8, device=self.device)
        self._info = torch.empty((off, INFO_DIM), dtype=torch.int32, device=self.device)
        self._act = torch.empty((off, self.act_dim), dtype=torch.float32, device=self.device)
        self._streams = [torch.cuda.Stream(device=self.device) for _ in self.buckets]

    def _obs_dict(self, obs):
        return OrderedDict(object_ob=obs[:, : self.object_ob_dim], robot_ob=obs[:, self.object_ob_dim :])

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
        self._object_ob[sl, : b.object_ob_dim].copy_(od["object_ob"])
        self._robot_ob[sl].copy_(od["robot_ob"])
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
    step one all_gather makes the packed [obs | reward | done] of every shard visible on every rank."""

    def __init__(self, envs_per_gpu, agent="Sawyer", furniture_name="table_lack_0825", env=None, **cfg_overrides):
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
        self.pack_dim = self.env.obs_dim + 2
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
        p[:, self.env.obs_dim :] = 0
        allp = self._gather()
        return self.env._obs_dict(allp[:, : self.env.obs_dim])

    def step(self, local_actions):
        """One env step of the local shard, then the single collective of the data path.  The step kernel writes
        [obs | reward | done] rows into the registered send buffer itself (fe_env_step_packed); with `timing` set, CUDA events
        separate the kernel from the time spent in the all-gather (which includes waiting for the slowest rank)."""
        env, t = self.env, self.torch
        a = t.as_tensor(local_actions["default"] if isinstance(local_actions, dict) else local_actions)
        if a.device != env.device or a.dtype != t.float32 or not a.is_contiguous():
            env._act.copy_(a, non_blocking=True)
            a = env._act
        assert a.shape == (env.num_envs, env.act_dim), tuple(a.shape)
        if self.timing:
            ev = [t.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record()
        if hasattr(env, "_stream"):
            env.engine.env_step_packed(a.data_ptr(), self._pack.data_ptr(), env._info.data_ptr(), stream=env._stream())
            info = env._info
        else:  # stand-in shard of the gloo tests
            od_, rew, done, info = env.step(a)
            self._pack[:, : env.obs_dim] = env._obs
            self._pack[:, env.obs_dim] = rew
            self._pack[:, env.obs_dim + 1] = done.float()
        if self.timing:
            ev[1].record()
        allp = self._gather()
        if self.timing:
            ev[2].record()
            self._events.append(ev)
        od = env.obs_dim
        return env._obs_dict(allp[:, :od]), allp[:, od], allp[:, od + 1] > 0.5, info

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
