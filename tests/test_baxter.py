"""FurnitureBaxterEnv (BASELINE.json config 4: Baxter + chair_ingolf_0650; furniture/env/furniture_baxter.py): two arms, 17
actions, 58 + 35 observations, per-arm finger scans, armature / margin / capsule / <exclude> in the model.  The device env is
compared with the CPU env oracle (oracle/ref_env.py) from the same seeds: `emu` = lane-emulated build, `cuda` = the sm_90a library."""
import numpy as np
import pytest

from furniture_b200 import mjcf
from oracle.ref_env import Cfg, OracleFurnitureEnv
from parity_util import make_engine

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]


def test_baxter_scene_dimensions():
    m = mjcf.load_scene("Baxter", "chair_ingolf_0650")
    # SURVEY.md A.1: nq 54, nv 49, nu 18 (14 velocity servos + 2 x 2 gripper position servos), 12 welds
    assert (m.nq, m.nv, m.nu, m.neq) == (54, 49, 18, 12)
    assert len(m.meta["robot_joints"]) == 14 and len(m.meta["gripper_joints"]) == 4
    assert m.dof_armature[:19].max() == 0.01 and m.geom_margin.max() == 0.001  # robots/baxter/robot.xml
    assert (m.geom_type == mjcf.GEOM_CAPSULE).sum() == 1  # pedestal_2_collision
    assert len(m.exclude) == 8


@pytest.mark.parametrize("gpu", BACKENDS)
def test_baxter_reset_and_steps_match_the_cpu_env(gpu):
    m = mjcf.load_scene("Baxter", "chair_ingolf_0650")
    n, seed = 2, 500
    eng = make_engine(m, n, gpu, seed=seed)
    assert (eng.obs_dim, eng.act_dim) == (58 + 35, 17)  # furniture_baxter.py:36-42, :52-58
    eng.env_reset()
    assert (eng.get("flags") == 0).all()
    envs = []
    for i in range(n):
        cfg = Cfg()
        cfg.seed = seed + i
        e = OracleFurnitureEnv(m, cfg)
        ob = e.reset()
        envs.append(e)
        assert np.abs(eng.get("qpos")[i] - e.sim.qpos).max() < 2e-5  # same draws, same 300 settle steps
        assert np.abs(eng.get("obs")[i] - ob).max() < 2e-5
    # the generator consumed 14 noise draws per robot-pose call (furniture.py:1766): same stream position as numpy's
    assert eng.get("mt_pos")[0, 0] == envs[0].rng.get_state()[2] and np.array_equal(eng.get("mt_state")[0], envs[0].rng.get_state()[1])
    rng = np.random.RandomState(1)
    for k in range(3):
        a = rng.uniform(-1, 1, (n, eng.act_dim)).astype(np.float32)
        a[:, -1] = -1
        obs, rew, done, info = eng.env_step_host(a)
        for i, e in enumerate(envs):
            ob, r, d, inf = e.step(a[i].astype(np.float64))
            assert np.abs(obs[i] - ob).max() < 2e-4, (k, i, np.abs(obs[i] - ob).max())
            assert abs(rew[i] - r) < 1e-5 and bool(done[i]) == d and info[i][3] == inf["episode_length"]
    # the head joint gets no gravity compensation and no reset pose; the arms hold their pose under theirs
    assert np.abs(eng.get("qfrc_applied")[:, 0]).max() == 0
    eng.close()


def _left_grasp_state(m, env):
    """a table leg between the finger tips of Baxter's LEFT gripper (1 mm interpenetration on both pads)"""
    sim = env.sim
    sim.reset()
    for p, name in enumerate(env.parts):
        sim.qpos[env.part_qadr[p] : env.part_qadr[p] + 7] = m.meta["part_init_qpos"][name]
    sim.qpos[env.arm_idx] = m.meta["robot_init_qpos"]
    sim.qpos[env.grip_idx] = m.meta["gripper_init_qpos"]
    gl, gr = m.names["geom"].index("l_g_l_fingertip_g0"), m.names["geom"].index("l_g_r_fingertip_g0")

    def tips(g):
        sim.qpos[env.grip_idx[2]], sim.qpos[env.grip_idx[3]] = g, -g
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
    R = np.stack([d, np.cross(zl, d), zl], axis=1)
    ty, tz = 0.011, 0.007  # slight tilt: pad and leg faces not exactly parallel (box-box point choice stays well conditioned)
    Ry = np.array([[np.cos(ty), 0, np.sin(ty)], [0, 1, 0], [-np.sin(ty), 0, np.cos(ty)]])
    Rz = np.array([[np.cos(tz), -np.sin(tz), 0], [np.sin(tz), np.cos(tz), 0], [0, 0, 1]])
    sim.qpos[env.part_qadr[0] : env.part_qadr[0] + 7] = np.concatenate([0.5 * (cl + cr), mjcf.mat_to_q(R @ Ry @ Rz)])
    return sim.qpos.copy()


@pytest.mark.parametrize("gpu", BACKENDS)
def test_second_arm_finger_scan_gives_the_touch_and_pick_reward(gpu):
    """a leg held by the LEFT gripper only: the per-arm scan of furniture.py:492-523 / :1290-1322 finds both fingers of arm 1 on
    the part (touch bits 8 | 16), the first arm touches nothing: touch + pick reward once, identical on device and CPU env"""
    m = mjcf.load_scene("Baxter", "table_lack_0825")
    env = OracleFurnitureEnv(m)
    env.reset()
    q = _left_grasp_state(m, env)
    env.nsub = 1
    env.sim.qvel[:] = 0; env.sim.qacc_warmstart[:] = 0; env.sim.ctrl[:] = 0
    env.sim.forward()
    eng = make_engine(m, 1, gpu, nsub=1)
    eng.env_reset()
    eng.set("qpos", q); eng.set("qvel", np.zeros(m.nv)); eng.set("qacc_warmstart", np.zeros(m.nv))
    eng.forward()
    a = np.zeros((1, eng.act_dim), np.float32)
    a[0, 15] = -1.0  # close the left gripper
    a[0, -1] = 1.0   # connect request: the scan runs for both arms, nothing is aligned
    obs, rew, done, info = eng.env_step_host(a)
    ob, r, d, inf = env.step(a[0].astype(np.float64))
    bits = env.touch_bits()
    assert bits[0] & 24 == 24 and bits[0] & 3 == 0, bits
    assert eng.get("touch")[0][0] & 24 == 24 and eng.get("touch")[0][0] & 3 == 0
    assert r > 100 and abs(rew[0] - r) < 1e-4  # touch 10 + pick 100 - control penalty
    assert info[0][0] == 0 and np.abs(obs[0] - ob).max() < 2e-4
    obs, rew, done, info = eng.env_step_host(a)
    ob, r, d, inf = env.step(a[0].astype(np.float64))
    assert r < 1 and abs(rew[0] - r) < 1e-4  # rewarded once per part
    eng.close()
