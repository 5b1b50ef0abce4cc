"""The drop-in boundary: furniture_b200/libfurniture_b200.so must load without a GPU and export every entry point that
include/furniture_b200.h declares; blob sizes must agree with the Python-side struct layouts; the error path of
fe_create must answer with a code and a message instead of crashing (no device work is attempted on the CPU box)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "furniture_b200.h")
LIB = os.path.join(ROOT, "furniture_b200", "libfurniture_b200.so")


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(fe_[a-z_0-9]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(LIB):
        pytest.fail("CUDA library not built: run `python -c 'import __graft_entry__ as g; g.build()'`")
    return C.CDLL(LIB)


def test_every_declared_entry_point_is_exported(lib):
    names = declared_functions()
    assert len(names) >= 20 and "fe_env_step" in names and "fe_create" in names
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing


def test_blob_sizes_match_the_python_layouts(lib):
    from furniture_b200.engine import FeConfig, FeScene
    from furniture_b200.engine_model import FeModel

    for fn, cls in (("fe_model_sizeof", FeModel), ("fe_scene_sizeof", FeScene), ("fe_config_sizeof", FeConfig)):
        f = getattr(lib, fn)
        f.restype = C.c_size_t
        assert f() == C.sizeof(cls), fn
    assert lib.fe_is_cuda() == 1  # the shipped library is the CUDA build, not the lane-emulated harness


def test_create_rejects_bad_blobs_with_a_message(lib):
    from furniture_b200.engine import default_config

    lib.fe_last_error.restype = C.c_char_p
    lib.fe_last_error.argtypes = [C.c_void_p]
    h = C.c_void_p()
    cfg = default_config()
    junk = (C.c_char * 64)()
    rc = lib.fe_create(junk, C.c_size_t(64), None, C.c_size_t(0), C.byref(cfg), 4, 0, C.byref(h))
    assert rc < 0 and not h.value
    assert len(lib.fe_last_error(None)) > 0


def test_engine_refuses_to_run_without_the_cuda_library(tmp_path):
    """no CPU fallback: a missing library is an error, not a silent switch to another path"""
    from furniture_b200 import mjcf
    from furniture_b200.engine import Engine

    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    with pytest.raises(RuntimeError):
        Engine(m, 2, lib_path=str(tmp_path / "nope.so"))


@pytest.mark.parametrize("gpu", [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)])
def test_get_and_set_state_round_trip(gpu):
    """fe_get_state / fe_set_state (get_env_state / set_env_state, furniture.py:1781-1803) on the lane-emulated build and on the sm_90a library:
    the state planted comes back bit for bit, and stepping from it equals stepping from the same state planted field by field"""
    import sys

    import numpy as np

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from furniture_b200 import mjcf
    from parity_util import make_engine, settled_state

    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    eng = make_engine(m, 3, gpu)
    Q = np.array([settled_state(m, i, robot_noise=0.2) for i in range(3)], np.float32)
    V = np.random.RandomState(0).normal(size=(3, m.nv)).astype(np.float32) * 0.1
    eng.set_state(Q, V)
    q, v = eng.get_state()
    assert np.array_equal(q, Q) and np.array_equal(v, V)
    eng.forward(); eng.step(5)
    other = make_engine(m, 3, gpu)
    other.set("qpos", Q); other.set("qvel", V)
    other.forward(); other.step(5)
    assert np.array_equal(eng.get_state()[0], other.get("qpos")) and np.array_equal(eng.get_state()[1], other.get("qvel"))


def test_scene_file_round_trip(tmp_path):
    """fe_scene_file_write / fe_create_from_file: a handle created from the binary scene file (what a non-Python binder uses)
    steps exactly like one created from the blobs (lane-emulated build; the CUDA library shares the code)"""
    import sys

    import numpy as np

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from furniture_b200 import mjcf
    from furniture_b200.engine import build_scene, default_config
    from furniture_b200.engine_model import EngineModel
    from parity_util import build_emu, make_engine

    L = C.CDLL(build_emu())
    L.fe_last_error.restype = C.c_char_p
    L.fe_last_error.argtypes = [C.c_void_p]
    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    em = EngineModel(m)
    sc = build_scene(m, em)
    path = str(tmp_path / "scene.feb").encode()
    assert L.fe_scene_file_write(path, C.byref(em.fm), C.c_size_t(C.sizeof(em.fm)), C.byref(sc), C.c_size_t(C.sizeof(sc))) == 0
    cfg = default_config(nsub=3, maxcon=44)
    h = C.c_void_p()
    assert L.fe_create_from_file(path, C.byref(cfg), 2, 0, C.byref(h)) == 0, L.fe_last_error(None)
    assert L.fe_env_reset(h, None, None, None) == 0
    a = np.random.RandomState(0).uniform(-1, 1, (2, 9)).astype(np.float32)
    obs = np.empty((2, 64), np.float32)
    assert L.fe_env_step_host(h, a.ctypes.data_as(C.c_void_p), obs.ctypes.data_as(C.c_void_p), None, None, None) == 0
    eng = make_engine(m, 2, False, nsub=3, maxcon=44)
    eng.env_reset()
    obs2 = eng.env_step_host(a)[0]
    assert np.array_equal(obs, obs2)
    L.fe_destroy(h)
    bad = tmp_path / "bad.feb"
    bad.write_bytes(b"nope" * 100)
    assert L.fe_create_from_file(str(bad).encode(), C.byref(cfg), 2, 0, C.byref(h)) < 0 and b"scene file" in L.fe_last_error(None)
