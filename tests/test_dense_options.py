"""The dense reward's coefficients, thresholds, diff_rew, early_termination and reset_robot_after_attach per env, inside the kernels
(config/furniture_sawyer_dense.py:23-70).

tests/golden/dense_options.npz is the reference's own _compute_reward on the scripted world of tools/make_golden_dense.py with one
coefficient set per episode (tools/make_golden_dense_options.py); the numpy oracle and the device machine (fe_dense_eval) reproduce it.
The device env steps, lane-emulated ([emu]) and on the GPU ([cuda]), are held to CPU dense envs built with each env's config, and a handle
whose envs mix configs is held bit for bit to handles that take one config for all their envs.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest

from furniture_b200 import mjcf
from furniture_b200.dense import _COEFS, DENSE_DEFAULTS, PER_ENV_KEYS, FeDenseConfig, dense_config
from furniture_b200.env import build_engine, env_options
from oracle import dense_oracle as D
from oracle.ref_env import DenseCfg, OracleDenseEnv
from parity_util import build_emu
from reset_options_oracle import ResetOptionsDenseEnv
from test_dense_reward import DENSE_BASE, PREV_KEYS, GoldenWorld, _adopt_device_anchors, _assert_same_machine, _dense_state, _device_inputs, _packed_recipe
from test_reset_options import _cfg, _same_generator

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FLAGS = ("diff_rew", "early_termination", "phase_ob", "reset_robot_after_attach")
# four configs side by side: the defaults, plain rewards, early termination at tight thresholds, reset_robot_after_attach with other coefficients
CONFIGS = [dict(), dict(diff_rew=False),
           dict(early_termination=True, eef_rot_threshold=0.99, move_pos_threshold=0.01, move_rot_threshold=0.99, lift_xy_pos_threshold=0.01),
           dict(reset_robot_after_attach=True, phase_bonus=1234.0, ctrl_penalty_coef=0.05, gripper_penalty_coef=3.0, move_eef_pos_dist_coef=42.0,
                drop_penalty_coef=7.0, aligned_bonus_coef=2.5)]


@pytest.fixture(scope="module")
def golden():
    g = np.load(os.path.join(HERE, "golden", "dense_options.npz"))
    return {k: g[k] for k in g.files}


@pytest.fixture(scope="module")
def lack():
    return mjcf.load_scene("Sawyer", "table_lack_0825")


def _episode_cfg(g, ep):
    cfg = {k: float(v) for k, v in zip(g["coef_names"], g["ep_coefs"][ep])}
    cfg.update({k: bool(g["ep_" + k][ep]) for k in FLAGS})
    return cfg


def _handle(gpu, n, **kw):
    return build_engine("Sawyer", "table_lack_0825", n, **dict(DENSE_BASE, **kw, **({} if gpu else dict(lib_path=build_emu()))))


# ------------------------------------------------------------------ the fixture: oracle and device machine against the reference
def test_fixture_moves_every_coefficient(golden):
    assert list(golden["coef_names"]) == list(_COEFS)
    defaults = np.array([DENSE_DEFAULTS[k] for k in _COEFS])
    assert np.all(golden["ep_coefs"] != defaults[None, :])
    for k in FLAGS:
        assert 0 < golden["ep_" + k].mean() < 1, k
    assert len(set(golden["phase"].tolist())) == 8 and golden["success"].sum() >= 5


def test_oracle_reproduces_the_reference_per_coefficient_set(golden):
    g = golden
    recipes = [json.loads(str(r)) for r in g["recipe_json"]]
    for t in range(len(g["reward"])):
        ep = int(g["episode"][t])
        if g["is_reset"][t]:
            world = GoldenWorld(g, recipes[int(g["ep_recipe"][ep])])
            world.t = t
            orc = D.DenseOracle(world, recipes[int(g["ep_recipe"][ep])], _episode_cfg(g, ep))
            orc.begin_episode()
        else:
            world.t = t
            r, done, info = orc.step(g["ac"][t], bool(g["connected"][t]))
            assert done == bool(g["done"][t]) and orc.success == bool(g["success"][t]), t
            ref = g["reward"][t]
            assert (np.isnan(ref) and np.isnan(r)) or abs(r - ref) <= 1e-11 * max(1.0, abs(ref)), (t, r, ref)
        assert orc.phase == int(g["phase"][t]) and orc.subtask == int(g["subtask"][t]), t


def _check_device_per_coefficient_set(eng, g):
    recipes = [json.loads(str(r)) for r in g["recipe_json"]]
    spos, smat, ppos, touch = _device_inputs(g, recipes)
    starts = np.flatnonzero(g["is_reset"])
    ends = np.append(starts[1:], len(g["reward"]))
    for ep, (a, b) in enumerate(zip(starts, ends)):
        recipe = recipes[int(g["ep_recipe"][ep])]
        dc = dense_config(**_episode_cfg(g, ep))
        rew, done, info = eng.dense_eval(dc, _packed_recipe(recipe), [0.02, 0.99, 0.99, 0.0], len(recipe["recipe"]), [a], [b - a], spos, smat, ppos, touch,
                                         g["is_reset"], g["connected"], g["ac"])
        sl = slice(a, b)
        assert np.array_equal(info[sl, 0].astype(int), g["phase"][sl]) and np.array_equal(info[sl, 1].astype(int), g["subtask"][sl]), ep
        assert np.array_equal(done[sl] & 1, g["done"][sl].astype(np.uint8)) and np.array_equal((done[sl] >> 1) & 1, g["success"][sl].astype(np.uint8)), ep
        ref = g["reward"][sl]
        assert np.array_equal(np.isnan(ref), np.isnan(rew[sl])), ep
        ok = ~np.isnan(ref)
        assert np.all(np.abs(rew[sl][ok] - ref[ok]) <= 1e-11 * np.maximum(1.0, np.abs(ref[ok]))), ep


@pytest.mark.parametrize("gpu", BACKENDS)
def test_device_machine_reproduces_the_reference_per_coefficient_set(golden, gpu):
    from parity_util import make_engine

    _check_device_per_coefficient_set(make_engine(mjcf.load_scene("None", "table_lack_0825"), 1, gpu), golden)


# ------------------------------------------------------------------ one handle with mixed configs against uniform handles
def _rollout(eng, steps=6, seed=3):
    """reset + `steps` random env steps: every output, the dense info and state, and the terminal rows after each call"""
    eng.env_reset()
    out = [eng.get("obs"), eng.get("dense_state"), eng.get("qpos")]
    rng = np.random.RandomState(seed)
    for _ in range(steps):
        a = rng.uniform(-1, 1, (eng.N, eng.act_dim)).astype(np.float32)
        obs, rew, done, info = eng.env_step_host(a)
        out += [obs, rew, done, info, eng.get("dense_info"), eng.get("dense_state"), eng.get("qpos"), eng.get("reset_robot_after_attach")]
        out += [np.where(done[:, None] != 0, x, 0) for x in (eng.get("terminal_obs"), eng.get("terminal_qpos"), eng.get("terminal_qvel"))]
    return out


@pytest.mark.parametrize("gpu,control_type", [pytest.param(g, c, id="%s-%s" % ("cuda" if g else "emu", c), marks=[pytest.mark.gpu] if g else [])
                                                for g in (False, True) for c in ("impedance", "ik")])
def test_mixed_configs_equal_uniform_handles(gpu, control_type):
    """envs cycling through the four CONFIGS in one handle, given as build_engine sequences, equal bit for bit the same envs of handles
    built with one config each, over reset + 6 steps at max_episode_steps 3 (two auto-resets).  On the GPU 64 envs share blocks."""
    n = 64 if gpu else 4
    which = np.arange(n) % 4
    keys = sorted({k for c in CONFIGS for k in c})
    seqs = {k: [CONFIGS[j].get(k, DENSE_DEFAULTS[k]) for j in which] for k in keys}
    mixed = _rollout(_handle(gpu, n, control_type=control_type, max_episode_steps=3, dense=seqs))
    assert mixed[-4][:, 0].tolist() == [int(j == 3) for j in which]  # the arm's flag follows each env's row
    for j, c in enumerate(CONFIGS):
        ref = _rollout(_handle(gpu, n, control_type=control_type, max_episode_steps=3, dense=c))
        for i in np.flatnonzero(which == j):
            for k, (x, y) in enumerate(zip(mixed, ref)):
                assert np.array_equal(np.asarray(x)[i], np.asarray(y)[i]), (control_type, j, i, k)


@pytest.mark.parametrize("gpu", BACKENDS)
def test_defaults_written_change_nothing(gpu):
    n = 32 if gpu else 2
    plain = _rollout(_handle(gpu, n, max_episode_steps=3, dense={}))
    written = _handle(gpu, n, max_episode_steps=3, dense={})
    written.set_dense_options(**{k: DENSE_DEFAULTS[k] for k in PER_ENV_KEYS})
    for x, y in zip(plain, _rollout(written)):
        assert x.dtype == y.dtype and np.array_equal(x, y)


@pytest.mark.parametrize("gpu", BACKENDS)
def test_diff_rew_switched_mid_episode_waits_for_the_reset(gpu):
    """diff_rew turned off after the first step: the rewards stay those of an untouched twin until the episode ends (its terminal step
    included), then they are those of a handle built with diff_rew off"""
    n = 8 if gpu else 2
    hs = [_handle(gpu, n, max_episode_steps=3, dense=d) for d in ({}, {}, dict(diff_rew=False))]
    rews = [[] for _ in hs]
    for h in hs:
        h.env_reset()
    rng = np.random.RandomState(9)
    for k in range(6):
        a = rng.uniform(-1, 1, (n, hs[0].act_dim)).astype(np.float32)
        if k == 1:
            hs[0].set_dense_options(diff_rew=False)
        for h, r in zip(hs, rews):
            r.append(h.env_step_host(a)[1])
    switched, twin, off = (np.array(r) for r in rews)
    assert np.array_equal(switched[:3], twin[:3]) and np.array_equal(switched[3:], off[3:])
    assert not np.array_equal(twin[3:], off[3:])


# ------------------------------------------------------------------ the device env against CPU dense envs built with each env's config
@pytest.mark.parametrize("gpu", BACKENDS)
def test_env_configs_match_cpu_envs(lack, gpu):
    """reset + 3 steps of a handle whose envs hold the four CONFIGS: each env's obs, reward, done and machine state equal a CPU dense env built
    with its config"""
    n = 4
    keys = sorted({k for c in CONFIGS for k in c})
    eng = _handle(gpu, n, dense={k: [c.get(k, DENSE_DEFAULTS[k]) for c in CONFIGS] for k in keys})
    eng.env_reset()
    from test_env_parity import _sync_oracle_from_engine

    envs = []
    for i, c in enumerate(CONFIGS):
        cfg = DenseCfg()
        cfg.seed = 123 + i
        if "ctrl_penalty_coef" in c:
            cfg.ctrl_penalty_coef = c["ctrl_penalty_coef"]
        e = OracleDenseEnv(lack, cfg, c)
        e.reset()
        _sync_oracle_from_engine(e, eng, i)
        e.sim.qfrc_bias[: e.nr] = eng.get("qfrc_bias")[i]
        e.dense.begin_episode()
        _assert_same_machine(_dense_state(eng, i), e.dense, ("reset", i), tol=5e-4)
        _adopt_device_anchors(e.dense, _dense_state(eng, i))
        envs.append(e)
    rng = np.random.RandomState(11)
    for k in range(3):
        a = rng.uniform(-1, 1, (n, eng.act_dim)).astype(np.float32)
        a[:, -1] = -0.5
        obs, rew, done, info = eng.env_step_host(a)
        for i, e in enumerate(envs):
            ob, r, d, _ = e.step(a[i].astype(np.float64))
            assert np.abs(obs[i] - ob).max() < 2e-4, (k, i)
            assert abs(rew[i] - r) < 2e-2 + 1e-5 * abs(r), (k, i, rew[i], r)
            assert bool(done[i]) == d, (k, i)
            _assert_same_machine(_dense_state(eng, i), e.dense, (k, i))


@pytest.mark.parametrize("gpu", BACKENDS)
def test_connection_follows_each_envs_reset_robot_after_attach(lack, gpu):
    """the recipe's first leg attached in two envs of one handle, env 0 with reset_robot_after_attach off, env 1 with it on: only env 1's arm
    goes home, and the next subtask (whose recipe step has a grip_init_pos) starts at INIT_EEF in env 0 and at ABOVE_LEG in env 1, as in the
    CPU dense env of each config"""
    eng = _handle(gpu, 2, nsub=1, auto_align=1, dense=dict(reset_robot_after_attach=[False, True]))
    eng.env_reset()
    assert eng.get("reset_robot_after_attach")[:, 0].tolist() == [0, 1]
    envs, qs = [], []
    for i, rra in enumerate((False, True)):
        cfg = _cfg(DenseCfg, seed=123 + i)
        cfg.auto_align = True
        e = ResetOptionsDenseEnv(lack, cfg, dict(reset_robot_after_attach=rra), reset_robot_after_attach=rra)
        e.reset()
        assert _same_generator(eng, i, e)
        qs.append(_grasp_and_align(lack, e))
        envs.append(e)
    eng.set("qpos", np.stack(qs)); eng.set("qvel", np.zeros(lack.nv)); eng.set("qacc_warmstart", np.zeros(lack.nv))
    eng.forward()
    st = eng.get("dense_state").copy()
    rows = []
    for i, e in enumerate(envs):
        raw = bytearray(st[i].tobytes())
        ints, dbl = np.frombuffer(raw[:32], np.int32).copy(), np.frombuffer(raw[32:], np.float64).copy()
        o = e.dense
        ints[:7] = [o.phase, o.subtask, 0, 0, 0, 0, 0]
        dbl[0:3], dbl[3:6], dbl[6:9] = o.table_site0, o.leg0, o.lift_target
        for k, name in enumerate(PREV_KEYS):
            dbl[12 + k] = o.prev.get(name, 0.0)
        rows.append(np.frombuffer(ints.tobytes() + dbl.tobytes(), np.uint8))
    eng.set("dense_state", np.stack(rows).view(st.dtype).reshape(st.shape))
    a = np.zeros((2, eng.act_dim), np.float32)
    a[:, -2], a[:, -1] = 1.0, -1.0
    eng.env_step_host(a)  # the held legs are noticed
    for i, e in enumerate(envs):
        e.step(a[i].astype(np.float64))
    a[:, -1] = 1.0
    obs, rew, done, info = eng.env_step_host(a)
    q = eng.get("qpos")
    for i, e in enumerate(envs):
        ob, r, d, inf = e.step(a[i].astype(np.float64))
        assert inf["num_connected"] == 1 and info[i][0] == 1 and not done[i] and not d, i
        assert _same_generator(eng, i, e), i
        arm = e.arm_idx + e.grip_idx
        assert np.abs(q[i][arm] - e.sim.qpos[arm]).max() < 1e-3, i
        ds = _dense_state(eng, i)
        assert (ds["subtask"], ds["phase"]) == (e.dense.subtask, e.dense.phase) == (1, 1 if i else 0), i
        assert abs(rew[i] - r) < 0.5 + 1e-4 * abs(r), (i, rew[i], r)
    home = np.asarray(lack.meta["robot_init_qpos"])
    arm_q = [q[i][envs[i].arm_idx] for i in range(2)]
    assert np.abs(arm_q[1] - home).max() < 0.05 < np.abs(arm_q[0] - home).max()


def _grasp_and_align(m, e):
    from test_env_parity import _grasp_and_align_state

    q = _grasp_and_align_state(m, e, leg=1, leg_site="leg-table,0,90,180,270,conn_site2", table_site="table-leg,0,90,180,270,conn_site2",
                               arm_qpos=[-0.28, -0.9, 0.0, 1.86, 0.0, 0.6, 1.57])
    e.nsub = 1
    e.sim.qvel[:] = 0; e.sim.qacc_warmstart[:] = 0; e.sim.ctrl[:] = 0
    e.sim.forward()
    e.dense.begin_episode()
    return q


# ------------------------------------------------------------------ refusals and surfaces
def test_field_rules():
    eng = _handle(False, 2, dense={})
    assert eng.L.fe_field_dtype(eng.h, b"dense_config").decode() == "|V%d" % C.sizeof(FeDenseConfig)
    assert eng.field_info("dense_config") == (1, C.sizeof(FeDenseConfig)) and np.dtype(FeDenseConfig).itemsize == C.sizeof(FeDenseConfig)
    good = eng.get("dense_config")
    bad_rows = []
    for member, value in (("struct_bytes", 8), ("diff_rew", 2), ("early_termination", -1), ("reset_robot_after_attach", 3), ("phase_ob", 1),
                          ("phase_bonus", np.nan), ("move_rot_threshold", np.inf), ("aligned_bonus_coef", -np.inf)):
        x = good.copy()
        x[1:, 0].view(np.dtype(FeDenseConfig))[member] = value
        bad_rows.append((member, x))
    for member, x in bad_rows:
        with pytest.raises(RuntimeError, match="dense_config"):
            eng.set("dense_config", x)
        assert eng.get("dense_config").tobytes() == good.tobytes(), member
    x = good.copy()
    x[:, 0].view(np.dtype(FeDenseConfig))["reset_robot_after_attach"] = [1, 0]
    eng.set("dense_config", x)
    assert eng.get("reset_robot_after_attach")[:, 0].tolist() == [1, 0]
    phased = _handle(False, 1, dense=dict(phase_ob=True))
    row = phased.get("dense_config")
    row[:, 0].view(np.dtype(FeDenseConfig))["phase_ob"] = 0
    with pytest.raises(RuntimeError, match="phase_ob"):
        phased.set("dense_config", row)


def test_setter_refusals_and_reset_robot_after_attach():
    eng = _handle(False, 3, dense={})
    before = eng.get("dense_config")
    for bad in (dict(phase_ob=True), dict(no_such_coef=1.0), dict(alignment_pos_dist=0.1)):
        with pytest.raises(ValueError):
            eng.set_dense_options(**bad)
    with pytest.raises(ValueError):
        eng.set_dense_options(phase_bonus=[1.0, 2.0])
    with pytest.raises(ValueError):
        eng.set_dense_options(envs=[0, 1], phase_bonus=[[1.0, 2.0]])
    with pytest.raises(IndexError):
        eng.set_dense_options(envs=[3], phase_bonus=1.0)
    assert eng.get("dense_config").tobytes() == before.tobytes()
    sparse = build_engine("Sawyer", "table_lack_0825", 1, lib_path=build_emu())
    with pytest.raises(ValueError, match="sparse"):
        sparse.set_dense_options(phase_bonus=1.0)
    cursor = build_engine("Cursor", "toy_table", 1, lib_path=build_emu())
    with pytest.raises(ValueError, match="Cursor"):
        cursor.set_dense_options(phase_bonus=1.0)
    # the arm's flag must agree with each env's row
    eng.set_dense_options(envs=[1], reset_robot_after_attach=True)
    assert eng.get("reset_robot_after_attach")[:, 0].tolist() == [0, 1, 0]
    eng.set_reset_options(reset_robot_after_attach=[False, True, False])
    with pytest.raises(RuntimeError, match="row"):
        eng.set_reset_options(reset_robot_after_attach=True)
    with pytest.raises(RuntimeError, match="row"):
        eng.set_reset_options(envs=[1], reset_robot_after_attach=False)
    assert eng.get("reset_robot_after_attach")[:, 0].tolist() == [0, 1, 0]
    eng.set_dense_options(envs=[0, 2], align_pos_threshold=[0.3, 0.1], early_termination=True)
    rows = eng.dense_rows()
    assert rows["align_pos_threshold"].tolist() == [0.3, 0.2, 0.1] and rows["early_termination"].tolist() == [1, 0, 1]
    assert rows["reset_robot_after_attach"].tolist() == [0, 1, 0] and rows["phase_ob"].tolist() == [0, 0, 0]


def test_build_engine_sequences_and_config_lists():
    """a scalar goes into the handle-wide fe_dense_config as before, a sequence sets each env's row; the config of a dense env id passes
    list-valued keys through"""
    eng = _handle(False, 3, dense=dict(phase_bonus=100.0, move_pos_threshold=[0.01, 0.02, 0.03], diff_rew=[True, False, True],
                                       reset_robot_after_attach=[False, False, True], ctrl_penalty_coef=[0.1, 0.2, 0.3]))
    assert eng.dense.phase_bonus == 100.0 and eng.dense.move_pos_threshold == DENSE_DEFAULTS["move_pos_threshold"] and eng.dense.diff_rew == 1
    rows = eng.dense_rows()
    assert rows["phase_bonus"].tolist() == [100.0] * 3 and rows["move_pos_threshold"].tolist() == [0.01, 0.02, 0.03]
    assert rows["diff_rew"].tolist() == [1, 0, 1] and rows["ctrl_penalty_coef"].tolist() == [0.1, 0.2, 0.3]
    assert eng.get("reset_robot_after_attach")[:, 0].tolist() == [0, 0, 1]
    furniture, options, ignored = env_options(dict(align_rot_threshold=[0.7, 0.8], early_termination=[True, False], ctrl_penalty_coef=[0.01, 0.02],
                                                   reset_robot_after_attach=[True, False], phase_bonus=10.0), dense_reward=True)
    assert "ctrl_penalty_coef" not in options and "reset_robot_after_attach" not in options and not ignored
    eng = build_engine("Sawyer", furniture, 2, lib_path=build_emu(), **options)
    rows = eng.dense_rows()
    assert rows["align_rot_threshold"].tolist() == [0.7, 0.8] and rows["early_termination"].tolist() == [1, 0]
    assert rows["ctrl_penalty_coef"].tolist() == [0.01, 0.02] and rows["phase_bonus"].tolist() == [10.0, 10.0]
    assert eng.get("reset_robot_after_attach")[:, 0].tolist() == [1, 0] and eng.cfg.ctrl_penalty_coef == np.float32(1e-3)
    with pytest.raises(ValueError):
        _handle(False, 2, dense=dict(phase_bonus=[1.0, 2.0, 3.0]))


def test_scene_file_handle_takes_the_rows():
    """a handle created by fe_create_from_file takes the dense reward and its per-env rows through the C-ABI alone"""
    from furniture_b200.engine import default_config

    L = C.CDLL(build_emu())
    L.fe_last_error.restype = C.c_char_p
    L.fe_last_error.argtypes = [C.c_void_p]
    L.fe_field_dtype.restype = C.c_char_p
    L.fe_field_dtype.argtypes = [C.c_void_p, C.c_char_p]
    h = C.c_void_p()
    path = os.path.join(ROOT, "furniture_b200", "compiled", "Sawyer_table_lack_0825.feb").encode()
    assert L.fe_create_from_file(path, C.byref(default_config(**DENSE_BASE)), 2, 0, C.byref(h)) == 0, L.fe_last_error(None)
    assert L.fe_field_dtype(h, b"dense_config") is None
    dc = dense_config()
    assert L.fe_enable_dense_reward(h, C.byref(dc)) == 0, L.fe_last_error(h)
    rows = np.zeros(2, np.dtype(FeDenseConfig))
    assert L.fe_get_field(h, b"dense_config", rows.ctypes.data_as(C.c_void_p), C.c_size_t(rows.nbytes)) == 0
    assert rows.tobytes() == bytes(dc) * 2
    rows["reset_robot_after_attach"] = [0, 1]
    rows["early_termination"] = [1, 0]
    assert L.fe_set_field(h, b"dense_config", rows.ctypes.data_as(C.c_void_p), C.c_size_t(rows.nbytes)) == 0, L.fe_last_error(h)
    rra = np.zeros((2, 1), np.int32)
    assert L.fe_get_field(h, b"reset_robot_after_attach", rra.ctypes.data_as(C.c_void_p), C.c_size_t(rra.nbytes)) == 0 and rra[:, 0].tolist() == [0, 1]
    rows["diff_rew"] = [0, 5]
    assert L.fe_set_field(h, b"dense_config", rows.ctypes.data_as(C.c_void_p), C.c_size_t(rows.nbytes)) != 0 and b"0 or 1" in L.fe_last_error(h)
    assert L.fe_env_reset(h, None, None, None) == 0
    L.fe_destroy(h)


@pytest.mark.gpu
def test_batched_mixed_and_vec_envs_pass_through():
    from furniture_b200.env import BatchedFurnitureEnv, MixedFurnitureEnv, make_vec_env

    env = BatchedFurnitureEnv("Sawyer", "table_lack_0825", 2, dense=dict(phase_bonus=[1.0, 2.0]))
    env.set_dense_options(envs=[1], align_pos_threshold=0.3)
    rows = env.engine.dense_rows()
    assert rows["phase_bonus"].tolist() == [1.0, 2.0] and rows["align_pos_threshold"].tolist() == [0.2, 0.3]
    env.close()
    mix = MixedFurnitureEnv(["table_lack_0825", "toy_table"], 2, dense={})
    mix.set_dense_options(envs=[1, 2], move_pos_threshold=[0.04, 0.05], early_termination=True)
    assert [b.engine.dense_rows()["move_pos_threshold"].tolist() for b in mix.buckets] == [[0.06, 0.04], [0.05, 0.06]]
    assert [b.engine.dense_rows()["early_termination"].tolist() for b in mix.buckets] == [[0, 1], [1, 0]]
    with pytest.raises(IndexError):
        mix.set_dense_options(envs=[4], phase_bonus=1.0)
    mix.close()
    vec = make_vec_env("IKEASawyerDense-v0", 2, dict(lift_z_pos_threshold=[0.01, 0.03], reset_robot_after_attach=[False, True]))
    rows = vec.engine.dense_rows()
    assert rows["lift_z_pos_threshold"].tolist() == [0.01, 0.03] and vec.engine.get("reset_robot_after_attach")[:, 0].tolist() == [0, 1]
    vec.reset()
    vec.step(np.zeros((2, vec.act_dim), np.float32))
    vec.close()
