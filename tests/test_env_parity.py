"""Env-level parity: the device FurnitureEnv logic (fe_env_step / fe_env_reset through the C-ABI) against the CPU
env oracle (oracle/ref_env.py, a restatement of FurnitureSawyerEnv with control_type="impedance").
`emu` runs the lane-emulated harness build on CPU, `cuda` the sm_90a library (marked gpu)."""
import json
import os

import numpy as np
import pytest

from furniture_b200 import mjcf
from oracle import assembly_oracle as A
from oracle.ref_env import Cfg, OracleFurnitureEnv
from parity_util import make_engine

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]


def _sync_oracle_from_engine(env, eng, i):
    """copy env i of the engine (state + the per-env model bits the reference mutates) into the oracle env"""
    sim, m = env.sim, env.m
    sim.qpos[:] = eng.get("qpos")[i]; sim.qvel[:] = eng.get("qvel")[i]; sim.qacc_warmstart[:] = eng.get("qacc_warmstart")[i]
    ct, ca = eng.get("geom_contype")[i], eng.get("geom_conaffinity")[i]
    for k, g in enumerate(eng.em.geom_src):
        sim.geom_contype[g] = ct[k]; sim.geom_conaffinity[g] = ca[k]
    sim.eq_active[:] = eng.get("eq_active")[i]
    sim.eq_data[:] = eng.get("eq_data")[i]
    sim.forward()


@pytest.mark.parametrize("gpu", BACKENDS)
def test_reset_settles_like_the_reference_protocol(sawyer_model, gpu):
    m = sawyer_model
    n = 8
    eng = make_engine(m, n, gpu)
    eng.env_reset()
    q, v = eng.get("qpos"), eng.get("qvel")
    assert (eng.get("flags") == 0).all()
    # parts rest on the floor (leg half-width 0.015, table half-thickness 0.02) within furn_xyz_rand of their XML slots
    z = q[:, 9 + 2 :: 7]
    assert np.allclose(z[:, :4], 0.015, atol=2e-4) and np.allclose(z[:, 4], 0.02, atol=2e-4)
    for p, name in enumerate(m.meta["part_names"]):
        init = m.meta["part_init_qpos"][name]
        assert np.abs(q[:, 9 + 7 * p : 11 + 7 * p] - init[:2]).max() < 0.02 + 5e-3
    assert np.abs(v[:, 9:]).max() < 5e-3
    # arm stays near init_qpos (it sags a little under the stale gravity compensation, as in the reference), gripper open->0
    assert np.abs(q[:, :7] - m.meta["robot_init_qpos"]).max() < 0.25
    # envs got different random placements
    assert np.abs(q[0, 9:11] - q[1, 9:11]).max() > 1e-4
    # same protocol on the CPU oracle env: same resting heights, arm sag of the same size
    env = OracleFurnitureEnv(m)
    env.reset()
    assert np.allclose(env.sim.qpos[9 + 2 :: 7][:4], 0.015, atol=2e-4)
    assert np.abs(env.sim.qpos[:7] - q[:, :7].mean(0)).max() < 0.02
    # masks restored, welds off, bookkeeping cleared
    assert np.array_equal(eng.get("geom_contype")[0], np.array([1 if (t & (1 << 30)) else c for t, c in zip(list(eng.em.fm.geom_tag)[: eng.em.fm.ngeom], list(eng.em.fm.geom_contype0)[: eng.em.fm.ngeom])]))
    assert (eng.get("eq_active") == 0).all() and (eng.get("num_connected") == 0).all()


@pytest.mark.parametrize("gpu", BACKENDS)
def test_env_step_matches_cpu_env(sawyer_model, gpu):
    """3 env steps (50 mj_steps each) with random actions: obs / reward / done of the device env equal the CPU env
    started from the same post-reset state."""
    m = sawyer_model
    n = 3
    eng = make_engine(m, n, gpu)
    eng.env_reset()
    envs = [OracleFurnitureEnv(m) for _ in range(n)]
    for i, e in enumerate(envs):
        e.reset()  # initialises bookkeeping; the state is overwritten next
        _sync_oracle_from_engine(e, eng, i)
        e.sim.qfrc_bias[: e.nr] = eng.get("qfrc_bias")[i]  # gravity compensation source = last forward of the reset
    rng = np.random.RandomState(5)
    for k in range(3):
        a = rng.uniform(-1, 1, (n, eng.act_dim)).astype(np.float32)
        a[:, -1] = -0.5
        obs, rew, done, info = eng.env_step_host(a)
        for i, e in enumerate(envs):
            ob, r, d, inf = e.step(a[i].astype(np.float64))
            assert np.abs(obs[i] - ob).max() < 2e-4, (k, i, np.abs(obs[i] - ob).max())
            assert abs(rew[i] - r) < 1e-5 and bool(done[i]) == d
            assert info[i][0] == inf["num_connected"] and info[i][3] == inf["episode_length"]


@pytest.mark.parametrize("gpu", BACKENDS)
def test_env_reset_and_step_swivel_chair(swivel_model, gpu):
    """the env path on a second furniture (3 parts, 2 welds, obs_dim 50): reset settles the parts at their resting heights
    (chair base z = 0.007, the value the reference's own demo recording shows, SURVEY.md 8c) and env steps follow the
    CPU env."""
    m = swivel_model
    n = 2
    eng = make_engine(m, n, gpu)
    eng.env_reset()
    assert (eng.get("flags") == 0).all()
    q = eng.get("qpos")
    assert np.allclose(q[:, 9 + 2], 0.007, atol=3e-4), q[:, 9 + 2]
    if not gpu:  # the reference's own MuJoCo recording has the base at rest at 0.0069975 (tests/golden/demo_facts.json)
        import json, os
        z_demo = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "demo_facts.json")))["swivel_chair_base_rest_z"]
        assert np.abs(q[:, 9 + 2] - z_demo).max() < 2e-7, (q[:, 9 + 2], z_demo)
    envs = [OracleFurnitureEnv(m) for _ in range(n)]
    for i, e in enumerate(envs):
        e.reset()
        _sync_oracle_from_engine(e, eng, i)
        e.sim.qfrc_bias[: e.nr] = eng.get("qfrc_bias")[i]
    rng = np.random.RandomState(7)
    for k in range(2):
        a = rng.uniform(-1, 1, (n, eng.act_dim)).astype(np.float32)
        a[:, -1] = -0.5
        obs, rew, done, info = eng.env_step_host(a)
        for i, e in enumerate(envs):
            ob, r, d, inf = e.step(a[i].astype(np.float64))
            assert obs.shape[1] == 50 and np.abs(obs[i] - ob).max() < 2e-4, (k, i, np.abs(obs[i] - ob).max())
            assert abs(rew[i] - r) < 1e-5 and bool(done[i]) == d


def _grasp_and_align_state(m, env, leg=0, leg_site="leg-table,0,90,180,270,conn_site1", table_site="table-leg,0,90,180,270,conn_site1", arm_qpos=None):
    """state in which leg `leg` sits between the finger tips (1 mm interpenetration on both sides) and the table top is
    placed so that its connector `table_site` coincides with the leg's `leg_site`."""
    sim = env.sim
    sim.reset()
    for p, name in enumerate(env.parts):
        sim.qpos[env.part_qadr[p] : env.part_qadr[p] + 7] = m.meta["part_init_qpos"][name]
    sim.qpos[:7] = m.meta["robot_init_qpos"] if arm_qpos is None else arm_qpos
    gl, gr = m.names["geom"].index("l_fingertip_g0"), m.names["geom"].index("r_fingertip_g0")

    def tips(g):
        sim.qpos[7], sim.qpos[8] = g, -g
        sim.stage("kinematics")
        return sim.geom_xpos[3 * gl : 3 * gl + 3].copy(), sim.geom_xpos[3 * gr : 3 * gr + 3].copy()

    lo, hi = 0.0, 0.020833
    for _ in range(50):
        mid = 0.5 * (lo + hi)
        cl, cr = tips(mid)
        if np.linalg.norm(cr - cl) > 0.036:
            hi = mid
        else:
            lo = mid
    cl, cr = tips(0.5 * (lo + hi))
    d = (cr - cl) / np.linalg.norm(cr - cl)
    zl = np.array([0, 0, -1.0]) - d * (-d[2])
    zl /= np.linalg.norm(zl)
    yl = np.cross(zl, d)
    R = np.stack([d, yl, zl], axis=1)  # leg x along the finger axis, leg z (its top) pointing down
    # a slight tilt keeps the pad / leg faces from being exactly parallel: with parallel faces the choice of box-box
    # contact points is decided by rounding, and the fp32 and fp64 pipelines would then follow different (equally valid) paths
    ty, tz = 0.011, 0.007
    Ry = np.array([[np.cos(ty), 0, np.sin(ty)], [0, 1, 0], [-np.sin(ty), 0, np.cos(ty)]])
    Rz = np.array([[np.cos(tz), -np.sin(tz), 0], [np.sin(tz), np.cos(tz), 0], [0, 0, 1]])
    R = R @ Ry @ Rz
    leg_q = np.concatenate([0.5 * (cl + cr), mjcf.mat_to_q(R)])
    s1 = m.names["site"].index(leg_site)
    s2 = m.names["site"].index(table_site)
    site1_world = leg_q[:3] + R @ m.site_pos[s1]
    table_q = np.concatenate([site1_world - R @ m.site_pos[s2], mjcf.mat_to_q(R)])
    sim.qpos[env.part_qadr[leg] : env.part_qadr[leg] + 7] = leg_q
    sim.qpos[env.part_qadr[4] : env.part_qadr[4] + 7] = table_q
    return sim.qpos.copy()


@pytest.mark.parametrize("gpu", BACKENDS)
def test_connect_path_matches_cpu_env(sawyer_model, gpu):
    """finger contact scan -> _try_connect -> _is_aligned -> _connect (masks, snap, weld, group merge, re-pin) on the
    device equals the CPU restatement: same decisions (integers exact), same poses to fp32 tolerance."""
    m = sawyer_model
    env = OracleFurnitureEnv(m)
    env.reset()
    q = _grasp_and_align_state(m, env)
    env.nsub = 1
    env.sim.qvel[:] = 0; env.sim.qacc_warmstart[:] = 0; env.sim.ctrl[:] = 0
    env.sim.forward()
    eng = make_engine(m, 2, gpu, nsub=1)
    eng.env_reset()
    eng.set("qpos", q); eng.set("qvel", np.zeros(m.nv)); eng.set("qacc_warmstart", np.zeros(m.nv))
    eng.forward()
    a = np.zeros((2, eng.act_dim), np.float32)
    a[:, -2] = 1.0
    a[0, -1] = 1.0   # env 0 asks to connect, env 1 does not
    a[1, -1] = -1.0
    obs, rew, done, info = eng.env_step_host(a)
    ob, r, d, inf = env.step(a[0].astype(np.float64))
    assert inf["num_connected"] == 1, "the CPU env did not connect: test state is wrong"
    assert info[0][0] == 1 and info[1][0] == 0
    assert abs(rew[0] - r) < 1e-3 and rew[0] > 100  # success_reward for one connection (+ touch reward)
    # integer model state: exact
    e = 0  # weld 0_part0 <-> 4_part4
    assert list(eng.get("eq_active")[0]) == list(env.sim.eq_active) and eng.get("eq_active")[0][e] == 1
    assert (eng.get("eq_active")[1] == 0).all()
    ct, ca = eng.get("geom_contype")[0], eng.get("geom_conaffinity")[0]
    for k, g in enumerate(eng.em.geom_src):
        assert ct[k] == env.sim.geom_contype[g] and ca[k] == env.sim.geom_conaffinity[g]
    grp = eng.get("group")[0]
    assert len({tuple(sorted(p for p in range(5) if _find(grp, p) == _find(grp, r_))) for r_ in range(5)}) == 4  # {0,4} merged
    assert _find(list(grp), 0) == _find(list(grp), 4)
    # welded relative pose and the resulting state: fp32 tolerance
    assert np.abs(eng.get("eq_data")[0].reshape(-1, 7)[e] - env.sim.eq_data[7 * e : 7 * e + 7]).max() < 2e-4
    assert np.abs(eng.get("qpos")[0] - env.sim.qpos).max() < 5e-4
    assert np.abs(obs[0] - ob).max() < 1e-3
    # the weld that was just activated holds: relative pose of the two parts equals the stored eq_data
    q0 = eng.get("qpos")[0]
    rel = A.rel_pose(q0[9 + 0 : 9 + 7].astype(np.float64), q0[9 + 28 : 9 + 35].astype(np.float64))
    assert np.abs(rel[:3] - eng.get("eq_data")[0].reshape(-1, 7)[e][:3]).max() < 2e-3


def _find(g, i):
    while g[i] != i:
        i = g[i]
    return i


@pytest.mark.gpu
def test_every_env_is_stepped_exactly_once_under_block_packing(sawyer_model):
    """the step kernel packs envs into blocks by the work of their previous step (heavy envs get partly empty blocks):
    whatever the packing, each env advances exactly one env-step per call and envs do not influence each other."""
    m = sawyer_model
    n = 300  # not a multiple of the block size
    eng = make_engine(m, n, True)
    eng.env_reset()
    rng = np.random.RandomState(0)
    acts = [rng.uniform(-1, 1, (n, eng.act_dim)).astype(np.float32) for _ in range(4)]
    for k, a in enumerate(acts):
        obs, rew, done, info = eng.env_step_host(a)
        assert (info[:, 3] == k + 1).all(), "episode_length must advance by one per call for every env"
    q_all = eng.get("qpos").copy()
    # envs 0..7 alone, same seed and actions: identical trajectories (the packing of the big batch was different)
    eng2 = make_engine(m, 8, True)
    eng2.env_reset()
    for a in acts:
        eng2.env_step_host(a[:8])
    assert np.array_equal(eng2.get("qpos"), q_all[:8])


@pytest.mark.gpu
@pytest.mark.parametrize("scene,n", [("table_lack_0825", 4096), ("swivel_chair_0700", 8192)])
def test_full_size_batches_through_size_independent_properties(scene, n):
    """BASELINE.json's full sizes (4096 envs of Sawyer+table_lack, 8192 of Sawyer+swivel_chair on one GPU), checked through
    properties that do not need the oracle at that size: no divergence flag, unit quaternions, parts at rest stay at rest
    under zero arm action, every env advances one step per call, and the first 8 envs are bit-identical to the same envs
    stepped in a batch of 8 (which is the size the oracle parity tests run at)."""
    m = mjcf.load_scene("Sawyer", scene)
    eng = make_engine(m, n, True)
    eng.env_reset()
    assert (eng.get("flags") == 0).all()
    q0 = eng.get("qpos")
    assert np.isfinite(q0).all()
    np_ = len(m.meta["part_names"])
    for p in range(np_):
        quat = q0[:, 9 + 7 * p + 3 : 9 + 7 * p + 7]
        assert np.abs(np.linalg.norm(quat, axis=1) - 1).max() < 1e-5
    a = np.zeros((n, eng.act_dim), np.float32)
    a[:, -2] = -1.0  # gripper open
    a[:, -1] = -1.0  # no connect
    for k in range(2):
        obs, rew, done, info = eng.env_step_host(a)
        assert (info[:, 3] == k + 1).all() and not done.any() and (info[:, 2] == 0).all()
    q1 = eng.get("qpos")
    assert (eng.get("flags") == 0).all()
    assert np.abs(q1[:, 9:] - q0[:, 9:]).max() < 2e-4, "settled parts must stay where they are"
    small = make_engine(m, 8, True)
    small.env_reset()
    assert np.array_equal(small.get("qpos"), q0[:8])
    for k in range(2):
        small.env_step_host(a[:8])
    assert np.array_equal(small.get("qpos"), q1[:8])


@pytest.mark.parametrize("gpu", BACKENDS)
def test_episode_end_and_auto_reset_follow_the_vecenv_worker(sawyer_model, gpu):
    """SubprocVecEnv's worker resets an env as soon as it reports done and returns the reset observation with the
    terminal reward (subproc_vec_env.py:16-20).  With max_episode_steps = 2 every second step ends an episode: the
    device env must report done / reward / episode_length like the CPU env, and hand back the observation of a reset
    that continues the env's numpy random stream (same placements as the oracle env seeded the same way)."""
    m = sawyer_model
    n, seed = 2, 321
    eng = make_engine(m, n, gpu, seed=seed, max_episode_steps=2, nsub=10)
    eng.env_reset()
    envs = []
    for i in range(n):
        cfg = Cfg()
        cfg.seed, cfg.max_episode_steps = seed + i, 2
        e = OracleFurnitureEnv(m, cfg)
        e.nsub = 10
        e.reset()
        envs.append(e)
    assert np.abs(eng.get("qpos") - np.array([e.sim.qpos for e in envs])).max() < 1e-5
    rng = np.random.RandomState(11)
    dones = []
    for k in range(5):
        a = rng.uniform(-1.3, 1.3, (n, eng.act_dim)).astype(np.float32)  # beyond [-1, 1]: clipped by _setup_action
        a[:, -1] = -0.5
        obs, rew, done, info = eng.env_step_host(a)
        for i, e in enumerate(envs):
            ob, r, d, inf = e.step(a[i].astype(np.float64))
            if d:
                ob = e.reset()  # the worker's auto-reset
            assert bool(done[i]) == d and abs(rew[i] - r) < 1e-5
            assert info[i][3] == inf["episode_length"]
            assert np.abs(obs[i] - ob).max() < 2e-4, (k, i, np.abs(obs[i] - ob).max())
        dones.append(done.copy())
    assert [bool(d[0]) for d in dones] == [False, True, False, True, False]


@pytest.mark.gpu
def test_long_random_rollout_stays_physical():
    """1024 envs x 40 env steps (2000 mj_steps each) of uniform random actions, the bench workload: observations stay
    finite, no part sinks through the floor or flies off, quaternions stay unit, no solver failure bit is raised, at most
    the (rare, flagged) contact-capacity bit; envs the engine reports unstable are reset and counted, not hidden."""
    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    n = 1024
    eng = make_engine(m, n, True, seed=7)
    eng.env_reset()
    rng = np.random.RandomState(0)
    unstable = 0
    for k in range(40):
        a = rng.uniform(-1, 1, (n, eng.act_dim)).astype(np.float32)
        obs, rew, done, info = eng.env_step_host(a)
        assert np.isfinite(obs).all() and np.isfinite(rew).all()
        unstable += int(info[:, 2].sum())
        assert (info[:, 3] == k + 1)[~done.astype(bool)].all()
    q = eng.get("qpos")
    parts = q[:, 9:].reshape(n, 5, 7)
    assert parts[:, :, 2].min() > -0.01 and parts[:, :, 2].max() < 1.5, (parts[:, :, 2].min(), parts[:, :, 2].max())
    assert np.abs(parts[:, :, :2]).max() < 3.0
    assert np.abs(np.linalg.norm(parts[:, :, 3:], axis=2) - 1).max() < 1e-4
    flags = eng.get("flags")[:, 0]
    assert ((flags & ~1) == 0).all(), np.unique(flags)
    assert (flags & 1).mean() < 0.01
    assert unstable <= n // 100


@pytest.mark.parametrize("gpu", BACKENDS)
def test_last_connection_ends_the_episode_with_success(sawyer_model, gpu):
    """success test of FurnitureEnv._step (furniture.py:440-445): with three of the four welds already counted, the
    connection made in this step brings num_connected to npart - 1: success reward, done, info.success, and -- as a
    VecEnv worker does -- the observation handed back is that of the reset that follows."""
    m = sawyer_model
    seed = 77
    cfg = Cfg()
    cfg.seed = seed
    env = OracleFurnitureEnv(m, cfg)
    env.reset()
    q = _grasp_and_align_state(m, env)
    env.nsub = 1
    env.sim.qvel[:] = 0; env.sim.qacc_warmstart[:] = 0; env.sim.ctrl[:] = 0
    env.sim.forward()
    env.num_connected = env.prev_num_connected = 3
    eng = make_engine(m, 1, gpu, nsub=1, seed=seed)
    eng.env_reset()
    eng.set("qpos", q); eng.set("qvel", np.zeros(m.nv)); eng.set("qacc_warmstart", np.zeros(m.nv))
    eng.set("num_connected", 3); eng.set("prev_num_connected", 3)
    eng.forward()
    a = np.zeros((1, eng.act_dim), np.float32)
    a[:, -2] = 1.0
    a[:, -1] = 1.0
    obs, rew, done, info = eng.env_step_host(a)
    ob, r, d, inf = env.step(a[0].astype(np.float64))
    assert d and inf["success"] == 1 and inf["num_connected"] == 4, "the CPU env did not finish: test state is wrong"
    assert bool(done[0]) and info[0][1] == 1 and info[0][0] == 4
    assert abs(rew[0] - r) < 1e-3 and rew[0] > cfg.success_reward
    ob = env.reset()  # the worker's auto-reset; the device env has done the same inside the step
    assert np.abs(obs[0] - ob).max() < 2e-4
    assert (eng.get("num_connected") == 0).all() and (eng.get("eq_active") == 0).all()


@pytest.mark.parametrize("gpu", BACKENDS)
def test_single_step_parity_along_a_drifting_rollout(gpu):
    """16 envs x 25 env steps of uniform random actions (the bench workload: arms flail, hit parts, pin them to the floor).
    Before every step the CPU env is re-synchronised to the device env's state, so each comparison is one env step (50
    mj_steps) from identical states, but over states no hand-made test reaches.  Found with it: the fp32 closest-point test at
    the end of MPR put the contact normal of a 0.5 mm cylinder-box penetration 40 degrees off (fixed: evaluated in float64).
    What is left is the MPR portal tolerance (normals to ~1e-3) amplified by stiff contact: a few steps in a thousand above 1e-3."""
    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    n, steps = 16, 25
    eng = make_engine(m, n, gpu, seed=1000)
    eng.env_reset()
    envs = []
    for i in range(n):
        cfg = Cfg()
        cfg.seed = 1000 + i
        e = OracleFurnitureEnv(m, cfg)
        e.reset()
        envs.append(e)
    rng = np.random.RandomState(0)
    worst, above, errs = 0.0, 0, []
    for k in range(steps):
        bias, tb, pk, nc, ln = eng.get("qfrc_bias"), eng.get("touched"), eng.get("picked"), eng.get("num_connected"), eng.get("episode_length")
        for i, e in enumerate(envs):
            _sync_oracle_from_engine(e, eng, i)
            e.sim.qfrc_bias[: e.nr] = bias[i]
            e.touched = [bool(x) for x in tb[i]]
            e.picked = [bool(x) for x in pk[i]]
            e.num_connected = e.prev_num_connected = int(nc[i, 0])
            e.episode_len = int(ln[i, 0])
        a = rng.uniform(-1, 1, (n, eng.act_dim)).astype(np.float32)
        obs, rew, done, info = eng.env_step_host(a)
        assert (eng.get("flags")[:, 0] & ~1 == 0).all()
        for i, e in enumerate(envs):
            ob, r, d, inf = e.step(a[i].astype(np.float64))
            assert bool(done[i]) == d
            if d:
                continue
            err = np.abs(obs[i] - ob).max()
            worst = max(worst, err)
            above += err > 1e-3
            errs.append(err)
            assert abs(rew[i] - r) < 1e-4
    # histogram of the per-step obs error (decades), printed with -s and kept next to the other measured artefacts
    edges = [0, 1e-6, 1e-5, 1e-4, 1e-3, 1e-2, 1e9]
    hist = np.histogram(errs, edges)[0].tolist()
    print("drifting-rollout obs error histogram (<1e-6, <1e-5, <1e-4, <1e-3, <1e-2, >=1e-2):", hist, "worst %.3g" % worst)
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    if os.path.isdir(out):
        with open(os.path.join(out, "drift_hist_%s.json" % ("cuda" if gpu else "emu")), "w") as f:
            json.dump({"edges": edges[:-1], "hist": hist, "worst": worst, "steps": len(errs)}, f)
    assert worst < 2e-2 and above <= 8, (worst, above, hist)


@pytest.mark.parametrize("gpu", BACKENDS)
def test_connect_decisions_over_perturbed_alignments(gpu):
    """48 variations of the grasp-and-align state: the table top displaced (up to a few cm) and rotated (up to 25 degrees) away from
    the aligned pose, so that some requests connect and others must not.  Every decision (num_connected, weld activation), reward and
    post-connect state of the device env equals the CPU env's (lane-emulated build and, gpu-marked, the sm_90a library)."""
    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    env0 = OracleFurnitureEnv(m)
    env0.reset()
    q0 = _grasp_and_align_state(m, env0)
    rng = np.random.RandomState(0)
    n = 48
    Q = np.tile(q0, (n, 1))
    ta = env0.part_qadr[4]
    for i in range(n):
        dp = rng.normal(size=3) * (0.03 if i % 2 else 0.008)
        ax = rng.normal(size=3)
        ax /= np.linalg.norm(ax)
        ang = np.deg2rad(rng.uniform(0, 25 if i % 3 else 6))
        Q[i, ta : ta + 3] += dp
        Q[i, ta + 3 : ta + 7] = mjcf.q_mul(np.concatenate([[np.cos(ang / 2)], ax * np.sin(ang / 2)]), Q[i, ta + 3 : ta + 7])
    eng = make_engine(m, n, gpu, nsub=1)
    eng.env_reset()
    eng.set("qpos", Q); eng.set("qvel", np.zeros(m.nv)); eng.set("qacc_warmstart", np.zeros(m.nv))
    eng.forward()
    a = np.zeros((n, eng.act_dim), np.float32)
    a[:, -2] = 1.0
    a[:, -1] = 1.0
    obs, rew, done, info = eng.env_step_host(a)
    qe, ea = eng.get("qpos"), eng.get("eq_active")
    connected = 0
    for i in range(n):
        e = OracleFurnitureEnv(m)
        e.reset()
        e.nsub = 1
        e.sim.qpos[:] = Q[i]; e.sim.qvel[:] = 0; e.sim.qacc_warmstart[:] = 0; e.sim.ctrl[:] = 0
        e.sim.forward()
        ob, r, d, inf = e.step(a[i].astype(np.float64))
        assert inf["num_connected"] == info[i][0] and list(e.sim.eq_active) == list(ea[i]), i
        assert abs(rew[i] - r) < 1e-3, i
        if inf["num_connected"]:
            assert np.abs(qe[i] - e.sim.qpos).max() < 2e-3, i
        connected += inf["num_connected"]
    assert 10 <= connected <= n - 5  # both outcomes are exercised
