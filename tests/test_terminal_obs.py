"""What a finished episode leaves: the terminal observation row and qpos / qvel that every env step writes, before its auto-reset, for each
env whose step returns done (the terminal `ob` of FurnitureEnv.step, furniture.py:364-385, and get_env_state at that point).

`emu` runs the lane-emulated build on the CPU, `cuda` the sm_90a library (marked gpu)."""
import ctypes as C

import numpy as np
import pytest

from furniture_b200 import mjcf
from furniture_b200.engine import FLAG_DIVERGED, default_config
from furniture_b200.env import build_engine
from oracle.preassembled_oracle import PreassembledDenseEnv, PreassembledEnv
from oracle.ref_env import Cfg, DenseCfg, OracleFurnitureEnv
from parity_util import build_emu, make_engine, quat_err
from test_dense_reward import PREV_KEYS, _dense_engine
from test_env_parity import _sync_oracle_from_engine
from test_preassembled import _hold_leg_of_step

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]
TERMINAL = ("terminal_obs", "terminal_qpos", "terminal_qvel")


def _lib(gpu):
    return None if gpu else build_emu()


def _fill_nan(eng):
    """every row of the three terminal buffers to NaN, so that a row no step wrote shows"""
    dims = [eng.field_info(f)[0] for f in TERMINAL]
    for ptr, dim in zip(eng.terminal_dev_ptrs(), dims):
        if eng.is_cuda:
            from furniture_b200.env import device_view

            device_view(ptr, (eng.N, dim), "cuda:0").fill_(float("nan"))
            import torch

            torch.cuda.synchronize()
        else:  # the emulated build's "device" memory is host memory
            np.ctypeslib.as_array((C.c_float * (eng.N * dim)).from_address(ptr)).fill(np.nan)


def _terminal(eng):
    return [eng.get(f) for f in TERMINAL]


# ------------------------------------------------------------------ 1. time-limit ends, bit for bit
CASES = {
    "sparse": ("Sawyer", "table_lack_0825", {}),
    "dense-phase_ob": ("Sawyer", "table_lack_0825", dict(dense=dict(phase_ob=True))),
    "ik": ("Sawyer", "table_lack_0825", dict(control_type="ik")),
    "joint_velocity": ("Sawyer", "table_lack_0825", dict(control_type="joint_velocity")),
    "baxter": ("Baxter", "table_lack_0825", {}),
    "pair-subtask_ob": ("Sawyer", "table_lack_0825", dict(object_ob_all=False, subtask_ob=True)),
}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("gpu", BACKENDS)
def test_time_limit_end_keeps_the_row_and_state_the_longer_episode_has(case, gpu):
    """handle A ends env i's episode at step 3 + i % 3 (per-env max_episode_steps), handle B runs the same seed and actions with the limit at
    2000: at each env's last step A's terminal row and state are B's obs row and state, bit for bit; A returns exactly what handle C, the same
    as A but whose terminal buffers are never read, returns; rows of envs that have not finished keep the NaN they were filled with"""
    agent, furn, opts = CASES[case]
    n = 64 if gpu else 3
    limits = 3 + np.arange(n) % 3
    mk = lambda **kw: build_engine(agent, furn, n, lib_path=_lib(gpu), nsub=2, **dict(opts, **kw))
    A, B, Cc = mk(max_episode_steps=limits), mk(), mk(max_episode_steps=limits)
    for e in (A, B, Cc):
        e.env_reset()
    _fill_nan(A)
    rng = np.random.RandomState(7)
    ended = np.zeros(n, bool)
    for t in range(1, int(limits.max()) + 1):
        a = rng.uniform(-1, 1, (n, A.act_dim)).astype(np.float32)
        a[:, -1] = -1.0  # no connect request
        ra, rb, rc = A.env_step_host(a), B.env_step_host(a), Cc.env_step_host(a)
        for x, y in zip(ra, rc):
            assert np.array_equal(x, y, equal_nan=True), (case, t)
        last = limits == t
        assert (ra[2][last] == 1).all() and (ra[2][limits > t] == 0).all() and not rb[2][~ended].any(), (case, t)
        to, tq, tv = _terminal(A)
        qb, vb = B.get_state()
        assert np.array_equal(to[last], rb[0][last]) and np.array_equal(tq[last], qb[last]) and np.array_equal(tv[last], vb[last]), (case, t)
        live = limits > t
        assert np.array_equal(ra[0][live], rb[0][live]) and np.array_equal(ra[1][live], rb[1][live]), (case, t)
        assert np.isnan(to[live]).all() and np.isnan(tq[live]).all() and np.isnan(tv[live]).all(), (case, t)
        ended |= last
        assert not np.isnan(to[ended]).any()
    assert ended.all()


# ------------------------------------------------------------------ 2. success ends, against the CPU env
def _set_dense_state(eng, o):
    """the CPU env's phase machine into every env of the device handle (as test_preassembled does)"""
    st = eng.get("dense_state").copy()
    raw = bytearray(st[0].tobytes())
    ints, dbl = np.frombuffer(raw[:32], np.int32).copy(), np.frombuffer(raw[32:], np.float64).copy()
    ints[:7] = [o.phase, o.subtask, 0, 0, 0, 0, 0]
    dbl[0:3], dbl[3:6], dbl[6:9], dbl[9:12] = o.table_site0, o.leg0, o.lift_target, getattr(o, "init_eef", np.zeros(3))
    for j, name in enumerate(PREV_KEYS):
        dbl[12 + j] = o.prev.get(name, 0.0)
    row = np.frombuffer(ints.tobytes() + dbl.tobytes(), np.uint8)
    eng.set("dense_state", np.stack([row] * eng.N).view(st.dtype).reshape(st.shape))


@pytest.mark.parametrize("dense", [False, True], ids=["sparse", "dense"])
@pytest.mark.parametrize("gpu", BACKENDS)
def test_success_end_keeps_the_connected_world(gpu, dense):
    """from a k = 3 preassembled start, the grasp -> connect script on the last leg ends env 0's episode with success (the dense reward's phase
    machine ends it too): the terminal row and state are the CPU env's observation and state at that step, while the step returns the next
    episode's first row"""
    m, k = mjcf.load_scene("Sawyer", "table_lack_0825"), 3
    cfg = DenseCfg() if dense else Cfg()
    cfg.auto_align = True
    env = PreassembledDenseEnv(m, cfg) if dense else PreassembledEnv(m, cfg)
    env.set_subtask(k)
    env.reset()
    eng = _dense_engine(m, 2, gpu, nsub=1, auto_align=1) if dense else make_engine(m, 2, gpu, nsub=1, auto_align=1)
    eng.set_subtask(k)
    eng.env_reset()
    _fill_nan(eng)
    _sync_oracle_from_engine(env, eng, 0)
    q = _hold_leg_of_step(m, env, k)
    env.nsub = 1
    env.sim.qvel[:] = 0; env.sim.qacc_warmstart[:] = 0; env.sim.ctrl[:] = 0
    env.sim.forward()
    eng.set("qpos", q); eng.set("qvel", np.zeros(m.nv)); eng.set("qacc_warmstart", np.zeros(m.nv))
    eng.forward()
    if dense:
        env.dense.begin_episode()
        _set_dense_state(eng, env.dense)
    a = np.zeros((2, eng.act_dim), np.float32)
    a[:, -2], a[:, -1] = 1.0, -1.0
    obs, rew, done, info = eng.env_step_host(a)  # the grasp
    ob, r, d, inf = env.step(a[0].astype(np.float64))
    assert not done.any() and not d
    a[0, -1] = 1.0  # env 0 connects
    obs, rew, done, info = eng.env_step_host(a)
    ob, r, d, inf = env.step(a[0].astype(np.float64))
    assert d and inf["success"] == 1 and inf["num_connected"] == k + 1, "the CPU env did not finish: test state is wrong"
    assert bool(done[0]) and info[0][1] == 1 and not done[1]
    to, tq, tv = _terminal(eng)
    assert np.abs(to[0] - ob).max() < 2e-4, np.abs(to[0] - ob).max()
    assert np.abs(obs[0] - to[0]).max() > 1e-3  # the step itself returned the next episode's first row
    for p in range(env.npart):
        qa = 9 + 7 * p
        assert np.abs(tq[0, qa : qa + 3] - env.sim.qpos[qa : qa + 3]).max() < 5e-4 and quat_err(tq[0, qa + 3 : qa + 7], env.sim.qpos[qa + 3 : qa + 7]) < 5e-4, p
    assert np.abs(tq[0, :9] - env.sim.qpos[:9]).max() < 5e-4
    assert np.isnan(to[1]).all() and np.isnan(tq[1]).all() and np.isnan(tv[1]).all()


# ------------------------------------------------------------------ 3. unstable steps: the world of the reset inside the step
@pytest.mark.parametrize("gpu", BACKENDS)
def test_unstable_end_keeps_the_world_of_the_internal_reset(gpu):
    """a diverged step resets inside _do_simulation's except branch and returns that world's observation (furniture.py:2889-2897); the terminal
    row and state are the CPU env's after its second reset, and the generator has still spent three resets' draws (the auto-reset's too)"""
    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    n, seed = 2, 321
    eng = make_engine(m, n, gpu, seed=seed, nsub=2)
    eng.env_reset()
    _fill_nan(eng)
    v = eng.get("qvel").copy()
    v[1, 0] = 1e8
    eng.set("qvel", v)
    a = np.zeros((n, eng.act_dim), np.float32)
    a[:, -1] = -1
    obs, rew, done, info = eng.env_step_host(a)
    assert not done[0] and done[1] and info[1][2] == 1
    to, tq, tv = _terminal(eng)
    cfg = Cfg()
    cfg.seed = seed + 1
    e = OracleFurnitureEnv(m, cfg)
    e.reset()
    ob = e.reset()  # the reset of the except branch
    assert np.abs(tq[1] - e.sim.qpos).max() < 1e-5 and np.abs(tv[1] - e.sim.qvel).max() < 2e-4
    assert np.abs(to[1] - ob).max() < 2e-4
    e.reset()  # the auto-reset
    s = e.rng.get_state()
    assert int(eng.get("mt_pos")[1, 0]) == s[2] and np.array_equal(eng.get("mt_state")[1], s[1])
    assert np.abs(eng.get("qpos")[1] - e.sim.qpos).max() < 1e-5 and np.abs(obs[1] - e.obs()).max() < 2e-4
    assert np.isnan(to[0]).all() and np.isnan(tq[0]).all() and np.isnan(tv[0]).all()
    assert (eng.get("flags")[:, 0] & FLAG_DIVERGED == 0).all()


# ------------------------------------------------------------------ 4. the three step entry points write the same rows
@pytest.mark.parametrize("gpu", BACKENDS)
def test_packed_and_host_steps_leave_the_rows_of_fe_env_step(gpu):
    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    n = 64 if gpu else 3
    limits = 2 + np.arange(n) % 2
    engs = [make_engine(m, n, gpu, nsub=2) for _ in range(3)]
    for e in engs:
        e.set_task_options(max_episode_steps=limits)
        e.env_reset()
        _fill_nan(e)
    if gpu:
        import torch

        buf = lambda shape, dt=torch.float32: torch.zeros(shape, dtype=dt, device="cuda:0")
        ptr = lambda x: x.data_ptr()
        host = lambda x: (torch.cuda.synchronize(), x.cpu().numpy())[1]
        u8, i32 = torch.uint8, torch.int32
    else:
        buf = lambda shape, dt=np.float32: np.zeros(shape, dt)
        ptr = lambda x: x.ctypes.data
        host = lambda x: x
        u8, i32 = np.uint8, np.int32
    obs, rew, done, info = buf((n, engs[0].obs_dim)), buf(n), buf(n, u8), buf((n, 6), i32)
    packed = buf((n, engs[0].obs_dim + 2))
    rng = np.random.RandomState(3)
    for t in range(1, 4):
        a = rng.uniform(-1, 1, (n, engs[0].act_dim)).astype(np.float32)
        a[:, -1] = -1
        ad = buf(a.shape)
        if gpu:
            ad.copy_(torch.from_numpy(a))
        else:
            ad[:] = a
        engs[0].env_step_dev(ptr(ad), ptr(obs), ptr(rew), ptr(done), ptr(info))
        engs[1].env_step_packed(ptr(ad), ptr(packed))
        ho, hr, hd, hi = engs[2].env_step_host(a)
        d0, pk = host(done).astype(bool), host(packed)
        assert np.array_equal(d0, hd.astype(bool)) and np.array_equal(d0, pk[:, -1] > 0.5) and np.array_equal(d0, limits == t)
        assert np.array_equal(host(obs), ho) and np.array_equal(pk[:, :-2], ho)
        rows = [_terminal(e) for e in engs]
        for k in range(3):
            assert np.array_equal(rows[0][k], rows[1][k], equal_nan=True) and np.array_equal(rows[0][k], rows[2][k], equal_nan=True), (t, TERMINAL[k])
            assert np.isnan(rows[0][k][limits > t]).all() and not np.isnan(rows[0][k][limits <= t]).any(), (t, TERMINAL[k])


# ------------------------------------------------------------------ 5. surfaces
def test_c_abi_fields_and_what_is_refused():
    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    eng = make_engine(m, 2, False, nsub=2)
    assert eng.field_info("terminal_obs") == (eng.obs_dim, 4)
    assert eng.field_info("terminal_qpos") == (m.nq, 4) and eng.field_info("terminal_qvel") == (m.nv, 4)
    for f in TERMINAL:
        with pytest.raises(RuntimeError, match="read-only"):
            eng.set(f, np.zeros((2, eng.field_info(f)[0]), np.float32))
    assert all(p for p in eng.terminal_dev_ptrs())
    # fe_set_obs_layout gives terminal_obs the new width
    old = eng.terminal_dev_ptrs()[0]
    eng.set_obs_layout(object_ob_all=False, subtask_ob=True)
    assert eng.field_info("terminal_obs") == (eng.obs_dim, 4) == (14 + 2 + eng.scene.robot_ob_dim, 4)
    assert eng.terminal_obs().shape == (2, eng.obs_dim) and eng.terminal_dev_ptrs()[0] != old
    # a handle without a scene blob has no env step and no terminal fields
    L, em = eng.L, eng.em
    cfg = default_config(nsub=2, maxcon=eng.cfg.maxcon)
    h = C.c_void_p()
    assert L.fe_create(C.byref(em.fm), C.c_size_t(C.sizeof(em.fm)), None, C.c_size_t(0), C.byref(cfg), 2, 0, C.byref(h)) == 0
    try:
        d, e = C.c_int(), C.c_int()
        for f in TERMINAL:
            assert L.fe_field_dim(h, f.encode(), C.byref(d), C.byref(e)) == -3
        assert L.fe_field_dim(h, b"qpos", C.byref(d), C.byref(e)) == 0
        assert L.fe_terminal_obs_dev(h) is None and L.fe_terminal_qpos_dev(h) is None and L.fe_terminal_qvel_dev(h) is None
    finally:
        L.fe_destroy(h)


def _gym(gpu, **kw):
    from furniture_b200.gym_api import FurnitureGymB200

    return FurnitureGymB200(name="FurnitureSawyerEnv", furniture_name="table_lack_0825", lib_path=_lib(gpu), nsub=2, max_episode_steps=3, **kw)


@pytest.mark.parametrize("gpu", BACKENDS)
def test_gym_terminal_observation(gpu):
    """terminal_observation=True: step returns B's row with done, get_env_state B's state until reset(), and reset() returns the same first
    observation and leaves the same generator as the default mode, which is unchanged"""
    T, D = _gym(gpu, terminal_observation=True), _gym(gpu)
    B = _gym(gpu)
    B.set_max_episode_steps(2000)
    assert "terminal_observation" not in T.ignored_config
    obs = [g.reset() for g in (T, D, B)]
    for k in obs[0]:
        assert np.array_equal(obs[0][k], obs[1][k]) and np.array_equal(obs[0][k], obs[2][k])
    rng = np.random.RandomState(5)
    for t in range(3):
        a = rng.uniform(-1, 1, T.dof).astype(np.float32)
        a[-1] = -1
        (ot, rt, dt, it), (od, rd, dd, idd), (ob, rb, db, ib) = T.step(a), D.step(a), B.step(a)
        assert rt == rd == rb and dt == dd and not db and set(it) == set(idd)
        if t < 2:
            assert not dt
            continue
        assert dt and set(it) == {"episode_success", "episode_reward", "episode_length", "episode_time", "episode_unstable", "episode_num_connected"}
        for k in ot:
            assert np.array_equal(ot[k], ob[k]), k
            assert not np.array_equal(od[k], ob[k]) or k == "subtask_ob"  # the default mode returns the next episode's first row
        st, sb, sd = T.get_env_state(), B.get_env_state(), D.get_env_state()
        assert np.array_equal(st["qpos"], sb["qpos"]) and np.array_equal(st["qvel"], sb["qvel"])
        assert not np.array_equal(sd["qpos"], sb["qpos"])
    rt_, rd_ = T.reset(), D.reset()
    for k in rt_:
        assert np.array_equal(rt_[k], rd_[k]) and np.array_equal(rt_[k], od[k])
    assert np.array_equal(T.get_env_state()["qpos"], D.get_env_state()["qpos"])
    for f in ("mt_state", "mt_pos"):
        assert np.array_equal(T.engine.get(f), D.engine.get(f))
    for g in (T, D, B):
        g.close()


@pytest.mark.gpu
@pytest.mark.parametrize("control_type", ["impedance", "ik"])
def test_batched_env_terminal_observation(control_type):
    """keys and shapes of BatchedFurnitureEnv.terminal_observation (the IK robot_ob keeps its 15 numbers), views of the device buffer that hold
    the rows of the finished envs"""
    import torch

    from furniture_b200.env import BatchedFurnitureEnv

    n = 8
    env = BatchedFurnitureEnv("Sawyer", "table_lack_0825", n, control_type=control_type, nsub=2, max_episode_steps=list(2 + np.arange(n) % 2))
    obs = env.reset()
    assert list(env.terminal_observation()) == list(obs)
    for step in range(2):
        ob, rew, done, info = env.step(torch.zeros((n, env.act_dim), device=env.device))
        to, ts = env.terminal_observation(), env.terminal_state()
        for k in ob:
            assert to[k].shape == ob[k].shape and to[k].device == env.device
        if control_type == "ik":
            assert to["robot_ob"].shape == (n, 15)
        assert ts["qpos"].shape == (n, env.model.nq) and ts["qvel"].shape == (n, env.model.nv)
    d = done.bool().cpu().numpy()
    assert d.any() and not d.all()
    host = env.engine.terminal_obs()
    assert np.array_equal(to["object_ob"].cpu().numpy()[d], host[d][:, : env.object_ob_dim])
    assert np.array_equal(to["robot_ob"].cpu().numpy()[d], host[d][:, -env.robot_ob_dim :])
    q, v = env.engine.terminal_state()
    assert np.array_equal(ts["qpos"].cpu().numpy(), q) and np.array_equal(ts["qvel"].cpu().numpy(), v)
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize("object_ob_all", [True, False], ids=["padded", "pair"])
def test_mixed_env_gathers_the_terminal_rows_like_step(object_ob_all):
    import torch

    from furniture_b200.env import MixedFurnitureEnv

    names = ["table_lack_0825", "chair_ingolf_0650", "toy_table"]
    env = MixedFurnitureEnv(names, 4, nsub=2, max_episode_steps=2, object_ob_all=object_ob_all)
    env.reset()
    for _ in range(2):
        ob, rew, done, info = env.step(torch.zeros((env.num_envs, env.act_dim), device=env.device))
    assert done.bool().all()
    to = env.terminal_observation()
    assert list(to) == list(ob) and all(to[k].shape == ob[k].shape for k in ob)
    assert to["object_ob"].shape[1] == (env.object_ob_dim if object_ob_all else 14)
    for b, off in zip(env.buckets, env.offsets):
        bt = b.terminal_observation()
        for k, v in bt.items():
            assert torch.equal(to[k][off : off + b.num_envs, : v.shape[1]], v), k
            if k == "object_ob" and v.shape[1] < to[k].shape[1]:
                assert (to[k][off : off + b.num_envs, v.shape[1] :] == 0).all()
    states = env.terminal_state()
    assert len(states) == 3 and all(s["qpos"].shape == (b.num_envs, b.model.nq) for s, b in zip(states, env.buckets))
    env.close()
