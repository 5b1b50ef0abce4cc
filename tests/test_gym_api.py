"""Single-env gym surface (FurnitureGym, furniture_gym.py:11-80) over the engine, on the lane-emulated build (the torque controllers on the CUDA build too): observation dict
layout, reward / done as Python scalars, the reference's episode keys in `info` at episode end, and one reset's worth of numpy
draws per episode (the env equals the oracle env seeded the same way across an episode boundary)."""
import numpy as np
import pytest

from furniture_b200.gym_api import FurnitureGymB200
from oracle.ref_env import Cfg, OracleFurnitureEnv
from parity_util import build_emu


def test_gym_surface_follows_the_reference_env_across_an_episode_boundary():
    seed = 41
    env = FurnitureGymB200(name="FurnitureSawyerEnv", furniture_name="table_lack_0825", lib_path=build_emu(), seed=seed, max_episode_steps=3, nsub=10)
    cfg = Cfg()
    cfg.seed, cfg.max_episode_steps = seed, 3
    ref = OracleFurnitureEnv(env.model, cfg)
    ref.nsub = 10
    ob = env.reset()
    rob = ref.reset()
    assert list(ob.keys()) == ["object_ob", "robot_ob"] and ob["object_ob"].shape == (35,) and ob["robot_ob"].shape == (29,)
    assert np.abs(np.concatenate(list(ob.values())) - rob).max() < 2e-4
    rng = np.random.RandomState(3)
    for ep in range(2):
        for k in range(3):
            a = rng.uniform(-1, 1, env.dof)
            a[-1] = -1
            ob, rew, done, info = env.step({"default": a})
            rob, r, d, inf = ref.step(a)
            assert isinstance(rew, float) and isinstance(done, bool) and done == d and abs(rew - r) < 1e-5
            if not done:
                assert info == {} and np.abs(np.concatenate(list(ob.values())) - rob).max() < 2e-4
        assert done and info["episode_length"] == 3 and info["episode_success"] == 0 and info["episode_unstable"] == 0
        assert set(info) == {"episode_success", "episode_reward", "episode_length", "episode_time", "episode_unstable", "episode_num_connected"}
        ob = env.reset()  # hands back the episode the device has already started: no second reset, no extra draws
        rob = ref.reset()
        assert np.abs(np.concatenate(list(ob.values())) - rob).max() < 2e-4, ep
    st = env.get_env_state()
    assert st["qpos"].shape == (env.model.nq,) and st["qvel"].shape == (env.model.nv,)
    env.close()


def test_reference_style_config_and_episode_length_passthrough():
    """the reference hands its envs an argparse Namespace with dozens of keys (config/furniture.py) and a furniture_id; keys of the
    renderer are ignored (and listed), physics keys map onto fe_config; set_max_episode_steps passes through (furniture_gym.py:35-37)"""
    import argparse

    from furniture_b200.env import FURNITURE_NAMES, split_config

    assert len(FURNITURE_NAMES) == 64 and FURNITURE_NAMES[52] == "table_lack_0825" and FURNITURE_NAMES[39] == "swivel_chair_0700"  # SURVEY.md 8d ids
    ns = argparse.Namespace(furniture_id=52, furniture_name=None, port=1050, background="Lab", unity=False, control_type="impedance",
                            max_episode_steps=7, furn_xyz_rand=0.01, seed=5, robot_ob=True, object_ob=True, visual_ob=False)
    name, over, ignored = split_config(ns)
    assert name == "table_lack_0825" and over == {"max_episode_steps": 7, "furn_xyz_rand": 0.01, "seed": 5}
    assert "port" in ignored and "background" in ignored
    env = FurnitureGymB200(name="FurnitureSawyerEnv", lib_path=build_emu(), id="IKEASawyer-v0", nsub=2, **vars(ns))
    assert env.cfg.max_episode_steps == 7 and env._max_episode_steps == 7
    env.set_max_episode_steps(2)
    env.reset()
    a = np.zeros(env.dof); a[-1] = -1
    _, _, done, _ = env.step(a)
    assert not done
    _, _, done, info = env.step(a)
    assert done and info["episode_length"] == 2
    # stepping on without reset(): the stale first observation is dropped, the next episode counts from 1
    _, _, done, info = env.step(a)
    assert not done and env._pending_ob is None
    _, _, done, info = env.step(a)
    assert done and info["episode_length"] == 2
    env.close()
    import pytest

    with pytest.raises(NotImplementedError):
        split_config({"control_type": "torque"})  # eight numbers for nine actuators in the reference; not built


def test_demo_files_have_the_reference_recorder_format(tmp_path):
    """BatchDemoRecorder writes what furniture/util/demo_recorder.py:58-87 writes: same keys, len(obs) = len(actions) + 1, the
    connect action appended to every low-level action; load_init_states reads the states back"""
    import pickle

    import numpy as np

    from furniture_b200.demo import BatchDemoRecorder, load_init_states
    from furniture_b200.engine import Engine, default_config
    from furniture_b200 import mjcf
    from collections import OrderedDict

    class Shard:  # minimal batched env over the lane-emulated engine
        def __init__(self, n):
            self.model = mjcf.load_scene("Sawyer", "table_lack_0825")
            self.engine = Engine(self.model, n, config=default_config(nsub=2), lib_path=build_emu())
            self.num_envs = n
        def _od(self, o): return OrderedDict(object_ob=o[:, :35], robot_ob=o[:, 35:])
        def reset(self): self.engine.env_reset(); return self._od(self.engine.get("obs"))
        def step(self, a): o, r, d, i = self.engine.env_step_host(a); return self._od(o), r, d, i
        def get_env_state(self): q, v = self.engine.get_state(); return {"qpos": q, "qvel": v}

    env = Shard(2)
    rec = BatchDemoRecorder(env, demo_dir=str(tmp_path), metadata={"furniture": "table_lack_0825"})
    rec.add_reset(env.reset())
    rng = np.random.RandomState(0)
    for k in range(3):
        a = rng.uniform(-1, 1, (2, 9)).astype(np.float32)
        od, rew, done, info = env.step(a)
        rec.add_step(a, od, rew)
    paths = rec.save("Sawyer_table_lack_0825_")
    assert [p[-8:] for p in paths] == ["0000.pkl", "0001.pkl"]
    demo = pickle.load(open(paths[1], "rb"))
    assert set(demo) == {"states", "obs", "actions", "rewards", "low_level_obs", "low_level_actions", "connect_actions", "metadata"}
    assert len(demo["obs"]) == 4 and len(demo["actions"]) == 3 and len(demo["states"]) == 4 and demo["low_level_actions"][0].shape == (9,)
    assert list(demo["obs"][0].keys()) == ["object_ob", "robot_ob"] and demo["states"][0]["qpos"].shape == (44,)
    states = load_init_states(paths[0])
    assert len(states) == 4 and states[3]["qvel"].shape == (39,)


def test_dense_reward_env_id_through_the_gym_surface():
    """gym.make("IKEASawyerDense-v0") of the reference builds FurnitureGym(name="FurnitureSawyerDenseRewardEnv", unity=False)
    (env/__init__.py:103-114); the same kwargs here: config/furniture_sawyer_dense.py's defaults, the phase one-hot on request, the
    reward terms in info, and an episode of 150 steps at most."""
    from furniture_b200.env import split_dense_config

    name, over, dense, ignored = split_dense_config(dict(phase_bonus=1000.0, early_termination=True, port=1050))
    assert name == "table_lack_0825" and over["max_episode_steps"] == 150 and over["auto_align"] is False and over["alignment_pos_dist"] == 0.02
    assert dense == dict(phase_bonus=1000.0, early_termination=True) and ignored == ["port"]
    env = FurnitureGymB200(name="FurnitureSawyerDenseRewardEnv", id="IKEASawyerDense-v0", unity=False, lib_path=build_emu(), nsub=2, phase_ob=True,
                           max_episode_steps=3)
    assert list(env.observation_space) == ["object_ob", "robot_ob", "phase_ob"] if isinstance(env.observation_space, dict) else True
    ob = env.reset()
    assert ob["phase_ob"].tolist() == [0, 1, 0, 0, 0, 0, 0, 0]  # first leg of table_lack: straight to move_eef_above_leg
    a = np.zeros(env.dof)
    a[-2] = -1.0
    total = 0.0
    for t in range(3):
        ob, r, done, info = env.step(a)
        total += r
        assert info["phase"] == 1 and info["subtask"] == 0 and info["gripper_penalty"] == 1.0 and info["ctrl_penalty"] == 0.0
        assert done == (t == 2)
    assert info["episode_length"] == 3 and abs(info["episode_reward"] - total) < 1e-6 and info["episode_success"] == 0
    # no recipe, no dense reward: the library says so
    import pytest

    with pytest.raises(RuntimeError, match="recipe"):
        FurnitureGymB200(name="FurnitureSawyerDenseRewardEnv", furniture_name="swivel_chair_0700", lib_path=build_emu())


def test_ik_control_type_through_the_gym_surface():
    """control_type="ik" is the reference's default (config/furniture.py:57): dof 8 = move 3 + rotate 3 + gripper + connect
    (furniture_sawyer.py:60-61); move_speed / rotate_speed come from the config"""
    from furniture_b200.env import control_options, split_config

    assert control_options(dict(control_type="ik", move_speed=0.05, rotate_speed=10.0)) == dict(control_type="ik", ik=dict(move_speed=0.05, rotate_speed=10.0))
    assert control_options(None) == dict(control_type="impedance")
    split_config(dict(control_type="ik"))  # accepted
    import pytest

    split_config(dict(control_type="position_orientation"))  # the five NEW_CONTROLLERS are accepted as well
    env = FurnitureGymB200(name="FurnitureSawyerEnv", lib_path=build_emu(), control_type="ik", move_speed=0.05, nsub=5, max_episode_steps=2)
    assert env.dof == 8 and abs(env.ik_cfg.move_speed - 0.05) < 1e-9 and env.ik_cfg.action_repeat == 3
    ob = env.reset()
    full = env.engine.get("obs")[0]
    assert ob["robot_ob"].shape == (15,) and np.allclose(ob["robot_ob"], full[35 + 14 : 64])  # gripper_qpos, eef pos / quat / velp / velr (furniture_sawyer.py:43-48)
    a = np.zeros(8)
    a[0], a[-2], a[-1] = 1.0, -1.0, -1.0
    ob, r, done, info = env.step(a)
    assert abs(r + 1e-3 * 3) < 1e-7 and not done  # ctrl penalty on the policy's 8 numbers
    ob, r, done, info = env.step(a)
    assert done and info["episode_length"] == 2
    bx = FurnitureGymB200(name="FurnitureBaxterEnv", furniture_name="chair_ingolf_0650", lib_path=build_emu(), control_type="ik", nsub=3)
    assert bx.dof == 15 and bx.ik_cfg.narms == 2  # (move, rotate) x 2, two grippers, connect (furniture_baxter.py:56-57)
    ob = bx.reset()
    full = bx.engine.get("obs")[0]
    n = bx.object_ob_dim
    assert ob["robot_ob"].shape == (30,) and np.allclose(ob["robot_ob"][:15], full[n + 14 : n + 29]) and np.allclose(ob["robot_ob"][15:], full[n + 29 + 14 : n + 58])
    ob, r, done, info = bx.step(np.zeros(15))
    assert np.isfinite(ob["robot_ob"]).all() and r == 0.0
    bq = FurnitureGymB200(name="FurnitureBaxterEnv", furniture_name="chair_ingolf_0650", lib_path=build_emu(), control_type="ik_quaternion", nsub=3)
    assert bq.dof == 17  # (move 3, quaternion 4) x 2, two grippers, connect
    with pytest.raises(NotImplementedError):
        FurnitureGymB200(name="FurnitureBaxterEnv", furniture_name="chair_ingolf_0650", lib_path=build_emu(), control_type="position")


def test_torque_controllers_through_the_gym_surface():
    """control_type in NEW_CONTROLLERS (furniture.py:41-47): the scene switches to the torque-actuated Sawyer, the action is the controller's
    command + gripper + connect, robot_ob the 15-number proprioception of every non-impedance control type (furniture_sawyer.py:110-155)"""
    _torque_controllers_through_the_gym_surface(False)


@pytest.mark.gpu
def test_torque_controllers_through_the_gym_surface_cuda():
    """the same on the CUDA build"""
    _torque_controllers_through_the_gym_surface(True)


def _torque_controllers_through_the_gym_surface(gpu):
    lib = dict(device=0) if gpu else dict(lib_path=build_emu())
    for ct, dof in (("position_orientation", 8), ("position", 5), ("joint_impedance", 9), ("joint_velocity", 9), ("joint_torque", 9)):
        env = FurnitureGymB200(name="FurnitureSawyerEnv", control_type=ct, nsub=3, max_episode_steps=2, move_speed=0.05, **lib)
        assert env.dof == dof and env.model.meta["agent"] == "SawyerTorque" and abs(env.ctl_cfg.move_speed - 0.05) < 1e-12
        ob = env.reset()
        assert ob["robot_ob"].shape == (15,)
        a = np.zeros(dof)
        a[-1] = -1.0
        ob, r, done, info = env.step(a)
        assert np.isfinite(ob["robot_ob"]).all() and abs(r + 1e-3) < 1e-7 and not done
        ob, r, done, info = env.step(a)
        assert done and info["episode_length"] == 2
        env.close()
