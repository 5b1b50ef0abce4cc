"""The per-env option fields as the C-ABI describes them and the one write path of the engine: fe_field_dtype for every registered field,
the env indices and value shapes every setter accepts, and one value per env for the boolean reset options (lane-emulated build; the
mixed batch on the GPU)."""
import os
import re

import numpy as np
import pytest

from furniture_b200 import mjcf
from furniture_b200.env import build_engine
from parity_util import build_emu
from test_reset_options import LEGS, _engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# how Python read these fields when it typed them by name, before fe_field_dtype
INT32_FIELDS = ("order geom_contype geom_conaffinity eq_active touch flags ncon niter stats con_geom con_state group site_connected num_connected "
                "prev_num_connected touched picked episode_length done mt_pos preassembled num_connects init_state init_pick init_mt_pos "
                "subtask_part fix_init fix_init_parts fix_have reset_robot_after_attach substeps no_collision assembled auto_align max_episode_steps").split()
FIELD_DTYPES = dict({f: "<i4" for f in INT32_FIELDS}, mt_state="<u4", init_mt_state="<u4", fix_pose="<f8", alignment="<f8", ik_state="|u1",
                    ctl_state="|u1", dense_state="|u1", qpos="<f4", qvel="<f4", dense_info="<f4", reward_coef="<f4", terminal_obs="<f4")


@pytest.fixture(scope="module")
def lack():
    return mjcf.load_scene("Sawyer", "table_lack_0825")


def test_field_dtype_matches_every_registered_field():
    """fe_field_dtype: for every field the C-ABI registers (in handles with the IK, a torque controller and the dense reward, which add
    fields), a typestr whose size is the field's element size and whose dtype is what Engine.get returns; the fields Python used to type by
    name keep their types; an unknown name gives NULL and an error message"""
    src = open(os.path.join(ROOT, "furniture_b200", "csrc", "fe_api.inl")).read()
    registered = set(re.findall(r'ALLOC\([^;]*?"(\w+)"', src)) | set(re.findall(r'add_field\(h, "(\w+)"', src))
    assert {"qpos", "fix_pose", "ik_state", "dense_info", "terminal_obs"} <= registered
    engines = [build_engine("Sawyer", "table_lack_0825", 2, lib_path=build_emu(), dense={}, control_type="ik"),
               build_engine("Sawyer", "table_lack_0825", 2, lib_path=build_emu(), control_type="joint_impedance")]
    seen = set()
    for eng in engines:
        for name in sorted(registered):
            if eng.L.fe_field_dtype(eng.h, name.encode()) is None:
                assert name in ("ik_state", "ctl_state", "dense_state", "dense_info") and b"unknown field" in eng.L.fe_last_error(eng.h)
                continue
            t = eng.L.fe_field_dtype(eng.h, name.encode()).decode()
            dim, elem = eng.field_info(name)
            x = eng.get(name)
            assert np.dtype(t).itemsize == elem and x.dtype == np.dtype(t) and x.shape == (2, dim), (name, t, elem, x.dtype)
            assert FIELD_DTYPES.get(name, t) == t, (name, t)
            seen.add(name)
        assert eng.L.fe_field_dtype(eng.h, b"no_such_field") is None and b"unknown field no_such_field" in eng.L.fe_last_error(eng.h)
        eng.close()
    assert seen == registered


def test_every_setter_refuses_envs_outside_the_handle(lack):
    """a negative index or one past the last env is an IndexError from each of the three setters, and nothing is written"""
    eng = _engine(lack, 2, False)
    before = {f: eng.get(f) for f in ("fix_init", "assembled", "substeps", "no_collision", "reward_coef")}
    for envs in ([-1], [2], [0, 5]):
        with pytest.raises(IndexError):
            eng.set_reset_options(fix_init=True, envs=envs)
        with pytest.raises(IndexError):
            eng.set_reset_options(assembled=True, envs=envs)
        with pytest.raises(IndexError):
            eng.set_sim_options(control_freq=20, no_collision=True, envs=envs)
        with pytest.raises(IndexError):
            eng.set_task_options(envs=envs, touch_reward=1.0)
    assert all(np.array_equal(eng.get(f), v) for f, v in before.items())


def test_boolean_options_take_one_value_per_env(lack):
    """fix_init, reset_robot_after_attach and assembled take a scalar or one value per env of `envs`, like the sim and task options; a
    sequence of another length is a ValueError and writes nothing"""
    eng = _engine(lack, 3, False)
    eng.set_reset_options(fix_init=[True, False, True], reset_robot_after_attach=[False, True, True], assembled=[False, True, False])
    assert [eng.get(f)[:, 0].tolist() for f in ("fix_init", "reset_robot_after_attach", "assembled")] == [[1, 0, 1], [0, 1, 1], [0, 1, 0]]
    eng.set_reset_options(fix_init=[False, True], assembled=[True, False], envs=[2, 0], fix_init_parts=list(LEGS))
    mask = eng.part_mask(LEGS)
    assert [eng.get(f)[:, 0].tolist() for f in ("fix_init", "assembled", "fix_init_parts")] == [[1, 0, 0], [0, 1, 1], [mask, 0, mask]]
    before = [eng.get(f) for f in ("fix_init", "reset_robot_after_attach")]
    with pytest.raises(ValueError):
        eng.set_reset_options(fix_init=True, reset_robot_after_attach=[True, False])
    assert all(np.array_equal(eng.get(f), b) for f, b in zip(("fix_init", "reset_robot_after_attach"), before))


@pytest.mark.gpu
def test_mixed_setters_refuse_envs_outside_the_batch():
    """both setters of a mixed batch refuse a negative global index and one past its envs with IndexError, instead of matching no bucket"""
    from furniture_b200.env import MixedFurnitureEnv

    mix = MixedFurnitureEnv(["table_lack_0825", "chair_ingolf_0650"], 2)
    for envs in ([-1], [4], [7], [1, 4]):
        with pytest.raises(IndexError):
            mix.set_sim_options(control_freq=20, envs=envs)
        with pytest.raises(IndexError):
            mix.set_task_options(envs=envs, max_episode_steps=5)
    assert [b.engine.get("substeps")[:, 0].tolist() for b in mix.buckets] == [[50, 50], [50, 50]]
    assert [b.engine.get("max_episode_steps")[:, 0].tolist() for b in mix.buckets] == [[2000, 2000], [2000, 2000]]
    mix.close()
