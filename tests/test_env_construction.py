"""Both env surfaces construct their engine through env.build_engine: FurnitureGymB200 from a reference-style config and the keywords that
make_vec_env hands BatchedFurnitureEnv give the same engine (config, scene and controller bytes, every writable field), on the lane-emulated
build and, with -m gpu, on the device."""
import numpy as np
import pytest

from furniture_b200 import mjcf
from furniture_b200.engine import Engine, default_config
from furniture_b200.env import build_engine
from furniture_b200.gym_api import FurnitureGymB200
from parity_util import build_emu

LACK = "table_lack_0825"
DENSE_ENV = dict(max_episode_steps=150, auto_align=False, alignment_pos_dist=0.02, alignment_rot_dist_up=0.99, alignment_rot_dist_forward=0.99,
                 alignment_project_dist=0.0)  # config/furniture_sawyer_dense.py
# id: (FurnitureGymB200 keywords, (agent, furniture, keywords of BatchedFurnitureEnv), dof, obs dict key -> width)
CASES = {
    "impedance": (dict(name="FurnitureSawyerEnv", port=1050), ("Sawyer", LACK, {}), 9, dict(object_ob=35, robot_ob=29)),
    "ik": (dict(name="IKEASawyer-v0", control_type="ik", move_speed=0.05, rotate_speed=10.0),
           ("Sawyer", LACK, dict(control_type="ik", ik=dict(move_speed=0.05, rotate_speed=10.0))), 8, dict(object_ob=35, robot_ob=15)),
    "ik_quaternion": (dict(name="FurnitureSawyerEnv", control_type="ik_quaternion"), ("Sawyer", LACK, dict(control_type="ik_quaternion", ik={})), 9,
                      dict(object_ob=35, robot_ob=15)),
    "position_orientation": (dict(name="Sawyer", control_type="position_orientation", move_speed=0.05),
                             ("Sawyer", LACK, dict(control_type="position_orientation", ik=dict(move_speed=0.05))), 8, dict(object_ob=35, robot_ob=15)),
    "baxter_ik": (dict(name="FurnitureBaxterEnv", furniture_name="chair_ingolf_0650", control_type="ik"),
                  ("Baxter", "chair_ingolf_0650", dict(control_type="ik", ik={})), 15, dict(object_ob=35, robot_ob=30)),
    "dense": (dict(name="FurnitureSawyerDenseRewardEnv", id="IKEASawyerDense-v0", unity=False, phase_ob=True, phase_bonus=1000.0),
              ("Sawyer", LACK, dict(dense=dict(phase_ob=True, phase_bonus=1000.0), **DENSE_ENV)), 9, dict(object_ob=35, robot_ob=29, phase_ob=8)),
    "obs_flags": (dict(name="FurnitureSawyerEnv", object_ob_all=False, subtask_ob=True), ("Sawyer", LACK, dict(object_ob_all=False, subtask_ob=True)), 9,
                  dict(object_ob=14, subtask_ob=2, robot_ob=29)),
    "no_robot_ob": (dict(name="FurnitureSawyerEnv", robot_ob=False, control_type="ik"), ("Sawyer", LACK, dict(robot_ob=False, control_type="ik", ik={})),
                    8, dict(object_ob=35)),
    "reset_options": (dict(name="FurnitureSawyerEnv", fix_init=True, fix_init_parts="1_part1", reset_robot_after_attach=True),
                      ("Sawyer", LACK, dict(fix_init=True, fix_init_parts="1_part1", reset_robot_after_attach=True)), 9, dict(object_ob=35, robot_ob=29)),
    "preassembled": (dict(name="FurnitureSawyerEnv", preassembled=[0, 1], num_connects=1), ("Sawyer", LACK, dict(preassembled=[0, 1], num_connects=1)),
                     9, dict(object_ob=35, robot_ob=29)),
    "load_demo": (dict(name="FurnitureSawyerEnv", load_demo="DEMO", load_init_states="INIT", seed=3),
                  ("Sawyer", LACK, dict(load_demo="DEMO", load_init_states="INIT", seed=3)), 9, dict(object_ob=35, robot_ob=29)),
}
WRITABLE = ("qpos", "qvel", "qacc_warmstart", "ctrl", "qfrc_applied", "gravcomp", "eq_data", "static_pos", "geom_contype", "geom_conaffinity", "eq_active",
            "flags", "order", "group", "site_connected", "num_connected", "prev_num_connected", "touched", "picked", "episode_length", "mt_state", "mt_pos",
            "preassembled", "num_connects", "init_state", "init_pick", "init_mt_state", "init_mt_pos", "fix_init", "fix_init_parts", "fix_have", "fix_pose",
            "reset_robot_after_attach")


@pytest.fixture(scope="module")
def starts(sawyer_model, tmp_path_factory):
    """a demo file and an init-states pickle: the paths that stand for DEMO and INIT"""
    from test_init_states import _write_files

    demo, init, _, _ = _write_files(sawyer_model, tmp_path_factory.mktemp("starts"))
    return {"DEMO": str(demo), "INIT": str(init)}


def _case(case, starts):
    gym_kw, (agent, furniture, kw), dof, widths = CASES[case]
    sub = lambda d: {k: starts.get(v, v) if isinstance(v, str) else v for k, v in d.items()}
    return sub(gym_kw), agent, furniture, sub(kw), dof, widths


def _dump(eng):
    """the engine's configuration bytes and every writable field, as built"""
    out = {k: None if getattr(eng, k) is None else bytes(getattr(eng, k)) for k in ("cfg", "scene", "ik", "controller", "dense")}
    out.update((f, eng.get(f).tobytes()) for f in WRITABLE)
    out.update((f, eng.get(f).tobytes()) for f, on in (("ik_state", eng.ik), ("ctl_state", eng.controller), ("dense_state", eng.dense)) if on is not None)
    q, v, npick = eng.init_states()
    out["init_states"] = (q.tobytes(), v.tobytes(), npick)
    out["agent"] = eng.model.meta.get("agent")
    return out


def _check_surface(env, dof, widths):
    assert env.dof == dof and env.engine.act_dim == dof
    assert list(env._cols) == list(widths)
    assert (env.object_ob_dim, env.subtask_ob_dim, env.robot_ob_dim, env.phase_ob_dim) == tuple(widths.get(k, 0) for k in ("object_ob", "subtask_ob", "robot_ob", "phase_ob"))


@pytest.mark.parametrize("case", list(CASES))
def test_builder_and_gym_build_the_same_engine(case, starts):
    gym_kw, agent, furniture, kw, dof, widths = _case(case, starts)
    lib = build_emu()
    gym = FurnitureGymB200(lib_path=lib, nsub=2, **gym_kw)
    eng = build_engine(agent, furniture, 1, lib_path=lib, nsub=2, **kw)
    assert _dump(eng) == _dump(gym.engine)
    _check_surface(gym, dof, widths)
    assert gym.model is gym.engine.model and gym.cfg is gym.engine.cfg and gym.control_type == eng.control_type == kw.get("control_type", "impedance")
    assert {k: len(c) for k, c in gym._cols.items()} == widths
    eng.close()
    gym.close()


def test_furn_size_rand_reaches_load_scene_from_both_surfaces(monkeypatch):
    """furn_size_rand (config/furniture.py:196-201): both surfaces load the scene at the first draw of RandomState(seed)"""
    seen, load = [], mjcf.load_scene

    def record(agent, furniture, resize_factor=None):
        seen.append(resize_factor)
        return load(agent, furniture)  # the unit-size scene: no asset tree needed

    monkeypatch.setattr(mjcf, "load_scene", record)
    FurnitureGymB200(name="FurnitureSawyerEnv", lib_path=build_emu(), furn_size_rand=0.1, seed=77).close()
    eng = build_engine("Sawyer", LACK, 1, lib_path=build_emu(), furn_size_rand=0.1, seed=77)
    r = float(np.float32(0.1))  # FeConfig.furn_size_rand is a float
    want = 1 + np.random.RandomState(77).uniform(-r, r, 1)[0]
    assert seen == [want, want] and eng.resize_factor == want
    eng.close()
    seen.clear()
    build_engine("Sawyer", LACK, 1, lib_path=build_emu()).close()
    assert seen == [None]


def test_load_init_states_on_a_model_whose_xml_lists_some_parts():
    partial = mjcf.load_scene("Sawyer", LACK)
    partial.meta = dict(partial.meta, xml_initpos_parts=["0_part0", "1_part1"])
    eng = Engine(partial, 2, config=default_config(), lib_path=build_emu())
    q, v = eng.get_state()
    eng.load_init_states([{"qpos": q[0], "qvel": v[0]}])
    assert list(eng.get("init_pick")[:, 0]) == [1, 1] and eng.init_states()[2] == 1
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_batched_env_builds_the_gym_engine(case, starts):
    from furniture_b200.env import BatchedFurnitureEnv

    gym_kw, agent, furniture, kw, dof, widths = _case(case, starts)
    env = BatchedFurnitureEnv(agent, furniture, 1, nsub=2, **kw)
    gym = FurnitureGymB200(nsub=2, **gym_kw)
    assert _dump(env.engine) == _dump(gym.engine)
    _check_surface(env, dof, widths)
    assert env.observation_space == {k: (w,) for k, w in widths.items()} and list(env.observation_space) == list(widths)
    e = env.engine
    assert all(a is b for a, b in zip((env.model, env.cfg, env.dense_cfg, env.ik_cfg, env.ctl_cfg), (e.model, e.cfg, e.dense, e.ik, e.controller)))
    assert env.obs_flags == e.obs_flags and env.control_type == kw.get("control_type", "impedance") and env.resize_factor is None
    assert (env.num_envs, env.obs_dim, env.act_dim, env.n_objects) == (1, e.obs_dim, dof, e.scene.npart)
    assert {k: v.shape[1] for k, v in env._obs_dict(env._obs).items()} == widths  # views and gathers of the obs buffer
    env.close()
    gym.close()
