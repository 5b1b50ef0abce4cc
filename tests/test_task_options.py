"""The task options of config/furniture.py per env, inside the kernels: the alignment thresholds and auto_align (:95-100, :203-226), the
placement noise (:177-194), the reward coefficients (:291-295) and max_episode_steps (:163-168).

The CPU env's sparse reward and episode end are pinned to the reference's own _compute_reward / _ctrl_penalty / _after_step by
tests/golden/task_options.npz (tools/make_golden_task_options.py).  The device, lane-emulated ([emu]) and on the GPU ([cuda]), is held to
CPU envs built with each env's values at the bars of tests/test_sim_options.py, and a handle whose envs mix values is held bit for bit to
handles that take one value for all their envs through FeConfig.
"""
import ctypes as C
import os

import numpy as np
import pytest

from assembled_oracle import AssembledDenseEnv, AssembledIKEnv, AssembledInitStateEnv
from furniture_b200 import mjcf
from furniture_b200.engine import TASK_OPTIONS, default_config
from furniture_b200.env import build_engine
from oracle.ref_env import DenseCfg, OracleFurnitureEnv
from parity_util import build_emu
from test_assembled import _assert_reset_equal
from test_env_parity import _grasp_and_align_state, _sync_oracle_from_engine
from test_reset_options import _assert_parts_close, _cfg, _engine, _same_generator

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
COEF_KEYS = ("success_reward", "touch_reward", "pick_reward", "ctrl_penalty_coef", "unstable_penalty_coef")
# two envs' values, every one off its default; the second env's episode ends at its third step
VALUES = [dict(alignment_pos_dist=0.15, alignment_rot_dist_up=0.85, alignment_rot_dist_forward=0.8, alignment_project_dist=0.2, auto_align=False,
               furn_xyz_rand=0.05, furn_rot_rand=6.0, agent_xyz_rand=0.01, success_reward=50.0, touch_reward=3.0, pick_reward=7.0,
               ctrl_penalty_coef=0.02, unstable_penalty_coef=30.0, max_episode_steps=5),
          dict(alignment_pos_dist=0.05, alignment_rot_dist_up=0.95, alignment_rot_dist_forward=0.97, alignment_project_dist=0.1, auto_align=True,
               furn_xyz_rand=0.0, furn_rot_rand=0.0, agent_xyz_rand=0.0, success_reward=7.0, touch_reward=1.0, pick_reward=2.5,
               ctrl_penalty_coef=0.5, unstable_penalty_coef=1000.0, max_episode_steps=3)]


@pytest.fixture(scope="module")
def lack():
    return mjcf.load_scene("Sawyer", "table_lack_0825")


def _dense_values(v):
    """a dense handle takes only unstable_penalty_coef among the coefficients"""
    return {k: x for k, x in v.items() if k not in COEF_KEYS[:4]}


# ------------------------------------------------------------------ the CPU env against the reference's own code
def test_oracle_sparse_reward_and_episode_end_equal_the_reference(lack):
    """every golden step (four coefficient sets x episode lengths 2, 3, 5, 2000; scripted finger / floor contacts, connections and failed
    steps): the CPU env's reward, done and episode length equal the reference's"""
    g = np.load(os.path.join(HERE, "golden", "task_options.npz"))
    e = OracleFurnitureEnv(lack)
    assert e.npart == g["bits"].shape[1]

    def new_episode():
        e.touched, e.picked = [False] * e.npart, [False] * e.npart
        e.num_connected = e.prev_num_connected = e.episode_len = 0

    e.reset, e.obs, e.connected_body1 = new_episode, lambda: np.zeros(1), None
    case = -1
    for k in range(len(g["reward"])):
        if g["case"][k] != case:
            case = g["case"][k]
            e.cfg = _cfg(**dict(zip(COEF_KEYS, g["coefs"][g["coef"][k]].tolist())), max_episode_steps=int(g["length"][k]))
            new_episode()
        fail, bits = bool(g["fail"][k]), [int(b) for b in g["bits"][k]]
        e._simulate = lambda raw, fail=fail: (fail, fail)
        e.touch_bits = lambda bits=bits: bits
        if not fail:
            e.num_connected = int(g["num_connected"][k])
        _, r, d, info = e.step(g["ac"][k])
        assert r == pytest.approx(g["reward"][k], rel=1e-12, abs=1e-12) and d == bool(g["done"][k]), (k, r, g["reward"][k], d)
        assert info["episode_length"] == g["episode_length"][k], k
        if d:
            new_episode()
    assert g["fail"].any() and (g["num_connected"] == e.npart - 1).any() and len(set(g["coef"].tolist())) == 4


# ------------------------------------------------------------------ the device against CPU envs built with each env's values
def _oracle(m, kind, values):
    if kind == "dense":
        return AssembledDenseEnv(m, _cfg(DenseCfg, **values), {})
    if kind == "ik":
        return AssembledIKEnv(m, _cfg(**values))
    return AssembledInitStateEnv(m, _cfg(**values))


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("kind", ["sparse", "dense", "ik", "baxter"])
def test_env_values_match_cpu_envs(lack, gpu, kind):
    """two envs, each with its own non-default values: the reset equals a CPU env built with them as its config (generator exactly, poses at
    the reset bar), then 3 random steps at the obs / reward bars.  Env 1's episode ends at step 3; its auto-reset draws as the CPU env's
    next reset does."""
    from test_dense_reward import _adopt_device_anchors, _dense_state
    from test_obs_layout import _sync_ik

    m = mjcf.load_scene("Baxter", "table_lack_0825") if kind == "baxter" else lack
    values = [_dense_values(v) for v in VALUES] if kind == "dense" else VALUES
    eng = _engine(m, 2, gpu, dense=kind == "dense", ik=kind == "ik")
    for i, v in enumerate(values):
        eng.set_task_options(envs=[i], **v)
    eng.env_reset()
    envs = []
    for i, v in enumerate(values):
        e = _oracle(m, kind, v)
        e.rng = np.random.RandomState(123 + i)
        e.reset()
        _assert_reset_equal(eng, i, e, (kind, i))
        _sync_oracle_from_engine(e, eng, i)
        e.sim.qfrc_bias[: e.nr] = eng.get("qfrc_bias")[i]
        if kind == "dense":
            e.dense.begin_episode()
            _adopt_device_anchors(e.dense, _dense_state(eng, i))
        if kind == "ik":
            _sync_ik(e, eng, i)
        envs.append(e)
    rng = np.random.RandomState(5)
    for k in range(3):
        a = rng.uniform(-1, 1, (2, eng.act_dim)).astype(np.float32)
        a[:, -1] = -0.5
        obs, rew, done, info = eng.env_step_host(a)
        for i, e in enumerate(envs):
            ob, r, d, _ = e.step(a[i].astype(np.float64))
            assert bool(done[i]) == d == (k == 2 and i == 1), (k, i)
            assert abs(rew[i] - r) < (2e-2 + 1e-5 * abs(r) if kind == "dense" else 1e-5), (k, i, rew[i], r)
            if d:  # the device has reset the env inside the step: compare its reset with the CPU env's next one
                e.reset()
                assert _same_generator(eng, i, e), (k, i)
                _assert_parts_close(eng, i, e, (kind, k))
            else:
                assert np.abs(obs[i] - ob).max() < 2e-4, (k, i, np.abs(obs[i] - ob).max())


@pytest.mark.parametrize("gpu", BACKENDS)
def test_alignment_threshold_decides_the_connection(lack, gpu):
    """a grasped leg with its connector 0.15 below the table's: the env at alignment_pos_dist 0.2 connects, its neighbour at 0.1 does not,
    each as the CPU env with that threshold"""
    env0 = OracleFurnitureEnv(lack)
    env0.reset()
    q = _grasp_and_align_state(lack, env0)
    ta = env0.part_qadr[4]
    q[ta + 2] += 0.15
    eng = _engine(lack, 2, gpu, cfg=dict(nsub=1))
    eng.set_task_options(alignment_pos_dist=[0.2, 0.1])
    eng.env_reset()
    eng.set("qpos", q); eng.set("qvel", np.zeros(lack.nv)); eng.set("qacc_warmstart", np.zeros(lack.nv))
    eng.forward()
    a = np.zeros((2, eng.act_dim), np.float32)
    a[:, -2] = 1.0
    a[:, -1] = 1.0
    obs, rew, done, info = eng.env_step_host(a)
    assert info[:, 0].tolist() == [1, 0]
    for i, pd in enumerate((0.2, 0.1)):
        e = OracleFurnitureEnv(lack, _cfg(alignment_pos_dist=pd))
        e.reset()
        e.nsub = 1
        e.sim.qpos[:] = q; e.sim.qvel[:] = 0; e.sim.qacc_warmstart[:] = 0; e.sim.ctrl[:] = 0
        e.sim.forward()
        ob, r, d, inf = e.step(a[i].astype(np.float64))
        assert inf["num_connected"] == info[i][0] and list(e.sim.eq_active) == list(eng.get("eq_active")[i]), i
        assert abs(rew[i] - r) < 1e-3, (i, rew[i], r)
        assert np.abs(eng.get("qpos")[i] - e.sim.qpos).max() < 2e-3, i


# ------------------------------------------------------------------ one handle, mixed values
def _rollout(eng, steps=5, seed=7):
    """reset + `steps` random env steps; every output and the state after each call"""
    eng.env_reset()
    out = [eng.get("obs"), eng.get("qpos"), eng.get("mt_state"), eng.get("mt_pos")]
    rng = np.random.RandomState(seed)
    for _ in range(steps):
        out += list(eng.env_step_host(rng.uniform(-1, 1, (eng.N, eng.act_dim)).astype(np.float32)))
        out += [eng.get("qpos"), eng.get("qvel"), eng.get("eq_active"), eng.get("group"), eng.get("mt_state"), eng.get("mt_pos"),
                eng.get("episode_length")]
    return out


def _handle(gpu, n, control_type, **kw):
    return build_engine("Sawyer", "table_lack_0825", n, control_type=control_type, **({} if gpu else dict(lib_path=build_emu())), **kw)


PROFILES = [dict(VALUES[0], max_episode_steps=2), dict(VALUES[1], max_episode_steps=3), dict(max_episode_steps=5)]


@pytest.mark.parametrize("gpu,control_type", [pytest.param(g, c, id="%s-%s" % ("cuda" if g else "emu", c), marks=[pytest.mark.gpu] if g else [])
                                                for g in (False, True) for c in ("impedance", "ik")])
def test_per_env_values_equal_handles_with_fe_config(gpu, control_type):
    """envs cycling through three value sets (max_episode_steps 2 / 3 / 5 side by side, so auto-resets fall in different steps) in one handle,
    given as build_engine sequences, equal bit for bit the same envs of handles built with the values as FeConfig overrides, over reset + 5
    steps.  On the GPU 64 envs share blocks across the sets."""
    n = 64 if gpu else 3
    which = np.arange(n) % 3
    seqs = {k: [PROFILES[j].get(k, getattr(default_config(), k)) for j in which] for k in TASK_OPTIONS}
    seqs["auto_align"] = [bool(x) for x in seqs["auto_align"]]
    mixed = _rollout(_handle(gpu, n, control_type, **seqs))
    for j, prof in enumerate(PROFILES):
        ref = _rollout(_handle(gpu, n, control_type, **prof))
        for i in np.flatnonzero(which == j):
            for x, y in zip(mixed, ref):
                assert np.array_equal(np.asarray(x)[i], np.asarray(y)[i]), (control_type, j, i)


@pytest.mark.parametrize("gpu", BACKENDS)
def test_defaults_change_nothing(lack, gpu):
    """the default values written, or the setter never called: reset + 5 steps bit-identical to an untouched handle"""
    n = 32 if gpu else 2
    defaults = {k: getattr(default_config(), k) for k in TASK_OPTIONS}
    plain = _rollout(_engine(lack, n, gpu, cfg=dict(max_episode_steps=3)))
    written = _engine(lack, n, gpu, cfg=dict(max_episode_steps=3))
    written.set_task_options(**dict(defaults, max_episode_steps=3))
    seq = _handle(gpu, n, "impedance", **{k: [v] * n for k, v in dict(defaults, max_episode_steps=3).items()})
    for eng in (written, seq):
        for x, y in zip(plain, _rollout(eng)):
            assert x.dtype == y.dtype and np.array_equal(x, y)


def test_set_max_episode_steps_applies_to_every_env(lack):
    eng = _engine(lack, 3, False)
    eng.set_task_options(max_episode_steps=[2, 3, 4])
    eng.set_max_episode_steps(1)
    assert eng.get("max_episode_steps")[:, 0].tolist() == [1, 1, 1] and eng.cfg.max_episode_steps == 1
    eng.env_reset()
    _, _, done, info = eng.env_step_host(np.zeros((3, eng.act_dim), np.float32))
    assert done.tolist() == [1, 1, 1] and (info[:, 2] == 0).all()


# ------------------------------------------------------------------ refusals and surfaces
def test_refusals(lack):
    from furniture_b200.engine import Engine

    eng = _engine(lack, 2, False)
    for bad in (dict(alignment_pos_dist=np.nan), dict(furn_xyz_rand=np.inf), dict(touch_reward=np.nan), dict(max_episode_steps=0),
                dict(auto_align=2)):
        with pytest.raises(RuntimeError):
            eng.set_task_options(**bad)
    with pytest.raises(ValueError):
        eng.set_task_options(touch_reward=[1.0, 2.0, 3.0])  # two envs
    with pytest.raises(ValueError):
        eng.set_task_options(envs=[0], touch_reward=[1.0, 2.0])
    with pytest.raises(IndexError):
        eng.set_task_options(envs=[2], touch_reward=1.0)
    with pytest.raises(IndexError):
        eng.set_task_options(envs=[-1], touch_reward=1.0)
    with pytest.raises(ValueError):
        eng.set_task_options(discrete_grip=0)  # changes what an action means: handle-wide
    with pytest.raises(RuntimeError):
        eng.set("reward_coef", np.full((2, 5), np.nan, np.float32))
    with pytest.raises(ValueError):
        _handle(False, 2, "impedance", max_episode_steps=[3, 4, 5])
    before = [eng.get(f) for f in ("alignment", "auto_align", "placement_rand", "reward_coef", "max_episode_steps")]
    assert [b.tolist() for b in before] == [[[0.1, 0.9, 0.9, 0.3]] * 2, [[1]] * 2, [np.float32([0.02, 3, 0.001]).tolist()] * 2,
                                            [np.float32([100, 10, 100, 1e-3, 100]).tolist()] * 2, [[2000]] * 2]
    dense = _engine(lack, 2, False, dense=True)
    for k in COEF_KEYS[:4]:
        with pytest.raises(RuntimeError):
            dense.set_task_options(envs=[1], **{k: 0.5})
    dense.set_task_options(envs=[1], unstable_penalty_coef=5.0, alignment_pos_dist=0.05)
    assert dense.get("reward_coef")[:, 4].tolist() == [100.0, 5.0] and dense.get("alignment")[:, 0].tolist() == [0.02, 0.05]
    cursor = Engine(mjcf.load_scene("Cursor", "toy_table"), 1, lib_path=build_emu())
    with pytest.raises(ValueError):
        cursor.set_task_options(success_reward=1.0)
    with pytest.raises(ValueError):
        build_engine("Cursor", "toy_table", 1, lib_path=build_emu(), success_reward=[1.0])


def test_build_engine_sequences_and_scalars():
    """a scalar goes into FeConfig as before; a sequence leaves FeConfig at the default and sets each env's field"""
    eng = _handle(False, 3, "impedance", furn_xyz_rand=0.04, touch_reward=[1.0, 2.0, 3.0], max_episode_steps=[4, 5, 6], auto_align=[True, False, True],
                  alignment_project_dist=[0.1, 0.2, 0.3])
    assert eng.cfg.furn_xyz_rand == np.float32(0.04) and eng.cfg.touch_reward == 10.0 and eng.cfg.max_episode_steps == 2000
    assert eng.get("placement_rand")[:, 0].tolist() == [np.float32(0.04)] * 3
    assert eng.get("reward_coef")[:, 1].tolist() == [1.0, 2.0, 3.0] and eng.get("max_episode_steps")[:, 0].tolist() == [4, 5, 6]
    assert eng.get("auto_align")[:, 0].tolist() == [1, 0, 1] and eng.get("alignment")[:, 3].tolist() == [0.1, 0.2, 0.3]
    eng.set_task_options(envs=[2, 0], pick_reward=[9.0, 8.0], agent_xyz_rand=0.5)
    assert eng.get("reward_coef")[:, 2].tolist() == [8.0, 100.0, 9.0] and eng.get("placement_rand")[:, 2].tolist() == [0.5, np.float32(0.001), 0.5]


def test_scene_file_handle_takes_the_fields(lack):
    """a handle created by fe_create_from_file starts from its fe_config's values and takes the fields through fe_set_field"""
    L = C.CDLL(build_emu())
    L.fe_last_error.restype = C.c_char_p
    L.fe_last_error.argtypes = [C.c_void_p]
    cfg = default_config(maxcon=44, touch_reward=4.0, max_episode_steps=7, alignment_rot_dist_up=0.8)
    h = C.c_void_p()
    path = os.path.join(ROOT, "furniture_b200", "compiled", "Sawyer_table_lack_0825.feb").encode()
    assert L.fe_create_from_file(path, C.byref(cfg), 2, 0, C.byref(h)) == 0, L.fe_last_error(None)

    def get(name, dt, dim):
        x = np.empty((2, dim), dt)
        assert L.fe_get_field(h, name, x.ctypes.data_as(C.c_void_p), C.c_size_t(x.nbytes)) == 0, L.fe_last_error(h)
        return x

    def put(name, x):
        return L.fe_set_field(h, name, x.ctypes.data_as(C.c_void_p), C.c_size_t(x.nbytes))

    assert get(b"reward_coef", np.float32, 5)[:, 1].tolist() == [4.0, 4.0] and get(b"max_episode_steps", np.int32, 1)[:, 0].tolist() == [7, 7]
    assert get(b"alignment", np.float64, 4)[:, 1].tolist() == [0.8, 0.8]
    assert put(b"max_episode_steps", np.array([[1], [3]], np.int32)) == 0
    assert put(b"max_episode_steps", np.array([[1], [0]], np.int32)) != 0 and put(b"auto_align", np.array([[0], [2]], np.int32)) != 0
    assert L.fe_env_reset(h, None, None, None) == 0
    act = np.zeros((2, L.fe_action_dim(h)), np.float32)
    obs, rew = np.empty((2, L.fe_obs_dim(h)), np.float32), np.empty(2, np.float32)
    done, info = np.empty(2, np.uint8), np.empty((2, L.fe_info_dim(h)), np.int32)
    assert L.fe_env_step_host(h, *(x.ctypes.data_as(C.c_void_p) for x in (act, obs, rew, done, info))) == 0
    assert done.tolist() == [1, 0]
    assert L.fe_set_max_episode_steps(h, 2) == 0 and get(b"max_episode_steps", np.int32, 1)[:, 0].tolist() == [2, 2]
    L.fe_destroy(h)


@pytest.mark.gpu
def test_batched_and_mixed_envs_pass_through():
    from furniture_b200.env import BatchedFurnitureEnv, MixedFurnitureEnv

    env = BatchedFurnitureEnv("Sawyer", "table_lack_0825", 2, max_episode_steps=[3, 4])
    env.set_task_options(envs=[1], touch_reward=2.0)
    assert env.engine.get("max_episode_steps")[:, 0].tolist() == [3, 4] and env.engine.get("reward_coef")[:, 1].tolist() == [10.0, 2.0]
    env.close()
    mix = MixedFurnitureEnv(["table_lack_0825", "chair_ingolf_0650"], 2)
    mix.set_task_options(envs=[1, 2], max_episode_steps=[5, 6], furn_rot_rand=1.5)
    assert [b.engine.get("max_episode_steps")[:, 0].tolist() for b in mix.buckets] == [[2000, 5], [6, 2000]]
    assert [b.engine.get("placement_rand")[:, 1].tolist() for b in mix.buckets] == [[3.0, 1.5], [1.5, 3.0]]
    with pytest.raises(IndexError):
        mix.set_task_options(envs=[4], max_episode_steps=5)
    mix.close()
