"""control_type="ik" (SURVEY 8 f4): what _do_ik_step does around the solver is pinned to the reference's own code
(tests/golden/ik_pre.npz, tools/make_golden_ik.py); the solver itself (damped least squares on the arm's chain, in place of the
pybullet call) is checked for reaching its target and device-against-oracle."""
import os

import numpy as np
import pytest

from furniture_b200 import ik as IK
from furniture_b200 import mjcf
from furniture_b200.engine import FLAG_DIVERGED
from oracle import ik_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(scope="module")
def sawyer():
    return mjcf.load_scene("Sawyer", "table_lack_0825")


def test_ik_step_preamble_equals_the_reference_code():
    g = np.load(os.path.join(HERE, "golden", "ik_pre.npz"))
    p = dict(IK.IK_DEFAULTS)
    assert set(g["n_sim"]) == {p["action_repeat"]} and set(g["n_closed_loop"]) == {p["action_repeat"] - 1}
    for i in range(len(g["action"])):
        hq = O.mat2quat(g["hand_R"][i].reshape(3, 3))
        d_pos, rot, s_new, grip = O.ik_pre(g["action"][i], g["hand_pos"][i], hq, g["s_in"][i], p)
        assert np.array_equal(d_pos, g["dpos"][i]), i
        assert np.allclose(s_new, g["s_out"][i], rtol=0, atol=1e-15), i
        assert np.abs(rot - g["rotation"][i].reshape(3, 3)).max() < 2e-6, i  # float32 quaternion products; the hand quaternion's sign is free
        assert grip == g["low_grip"][i]


def test_ik_quaternion_preamble_equals_the_reference_code():
    g = np.load(os.path.join(HERE, "golden", "ik_pre.npz"))
    p = dict(IK.IK_DEFAULTS)
    assert set(g["q_n_sim"]) == {3} and set(g["q_n_closed_loop"]) == {2}
    for i in range(len(g["q_action"])):
        hq = O.mat2quat(g["q_hand_R"][i].reshape(3, 3))
        d_pos, rot, grip = O.ik_pre_quaternion(g["q_action"][i], g["q_hand_pos"][i], hq, p)
        assert np.array_equal(d_pos, g["q_dpos"][i]) and grip == g["q_low_grip"][i], i
        assert np.abs(rot - g["q_rotation"][i].reshape(3, 3)).max() < 2e-6, i


def test_baxter_ik_preamble_equals_the_reference_code():
    """the two-arm branch of _do_ik_step (furniture.py:2933-2970): each arm like the one-arm case, both gripper actions passed through"""
    g = np.load(os.path.join(HERE, "golden", "ik_pre.npz"))
    p = dict(IK.IK_DEFAULTS)
    for i in range(len(g["b_action"])):
        a = g["b_action"][i]
        for arm in range(2):
            hq = O.mat2quat(g["b_hand_R"][i][arm].reshape(3, 3))
            arm_action = np.concatenate([a[6 * arm : 6 * arm + 6], [a[12 + arm], a[14]]])
            d_pos, rot, s_new, grip = O.ik_pre(arm_action, g["b_hand_pos"][i][arm], hq, g["b_s_in"][i][arm], p)
            assert np.array_equal(d_pos, g["b_dpos"][i][arm]), (i, arm)
            assert np.allclose(s_new, g["b_s_out"][i][arm], rtol=0, atol=1e-15) and np.abs(rot - g["b_rotation"][i][arm].reshape(3, 3)).max() < 2e-6, (i, arm)
            assert grip == g["b_low_grips"][i][arm]


def test_baxter_ik_quaternion_preamble_equals_the_reference_code():
    g = np.load(os.path.join(HERE, "golden", "ik_pre.npz"))
    p = dict(IK.IK_DEFAULTS)
    for i in range(len(g["bq_action"])):
        a = g["bq_action"][i]
        for arm in range(2):
            hq = O.mat2quat(g["bq_hand_R"][i][arm].reshape(3, 3))
            arm_action = np.concatenate([a[7 * arm : 7 * arm + 7], [a[14 + arm], a[16]]])
            d_pos, rot, grip = O.ik_pre_quaternion(arm_action, g["bq_hand_pos"][i][arm], hq, p)
            assert np.array_equal(d_pos, g["bq_dpos"][i][arm]) and grip == g["bq_low_grips"][i][arm], (i, arm)
            assert np.abs(rot - g["bq_rotation"][i][arm].reshape(3, 3)).max() < 2e-6, (i, arm)


def test_chain_and_solver_reach_the_commanded_hand_pose(sawyer):
    m = sawyer
    p = IK.ik_params(m)
    q = np.array(m.meta["robot_init_qpos"], dtype=float)
    full = np.array(m.qpos0, dtype=float)
    full[p["chain"]["qadr"]] = q
    kin = mjcf.kinematics_np(m, full)
    hb = m.names["body"].index("right_hand")
    hp, hq, _, _ = O.chain_fk(p["chain"], q)
    assert np.abs(hp - kin["xpos"][hb]).max() < 1e-12 and np.abs(hq - kin["xquat"][hb]).max() < 1e-12  # the chain is the model's arm
    rng = np.random.RandomState(0)
    for _ in range(20):
        tp = hp + rng.uniform(-0.06, 0.06, 3)
        tq = mjcf.q_norm(mjcf.q_mul(mjcf.q_axis_angle(rng.normal(size=3), rng.uniform(0, 0.3)), hq))
        qs, it = O.solve_ik(p, q, tp, tq)
        a, b, _, _ = O.chain_fk(p["chain"], qs)
        assert it < p["max_iters"] - 1 and np.linalg.norm(a - tp) < p["tol_pos"] and np.linalg.norm(O.rot_error(tq, b)) < p["tol_rot"]
        assert (qs >= np.array(p["lower"]) - 1e-12).all() and (qs <= np.array(p["upper"]) + 1e-12).all()


# ------------------------------------------------------------------ the IK env: device step against the CPU env
def _ik_engine(m, n, gpu, quaternion_mode=0, **cfg):
    from furniture_b200.engine import Engine, default_config
    from parity_util import build_emu

    c = default_config(**cfg)
    ikc = IK.ik_config(m, quaternion_mode=quaternion_mode)
    return Engine(m, n, device=0, config=c, ik=ikc) if gpu else Engine(m, n, config=c, lib_path=build_emu(), ik=ikc)


def _ik_state(eng, i):
    raw = eng.get("ik_state")[i].tobytes()
    f = np.frombuffer(raw[: 44 * 4], np.float32)  # s[2][4], target_pos[2][3], q_cmd[14], low[16], then iters[2]
    it = np.frombuffer(raw[44 * 4 : 46 * 4], np.int32)
    return dict(s=f[0:4], target_pos=f[8:11], q_cmd=f[14:21], low=np.concatenate([f[28:35], f[35:36]]), iters=int(it[0]),
                s2=f[4:8], target_pos2=f[11:14], q_cmd2=f[21:28], low_all=f[28:44], iters2=int(it[1]))


QUAT_BACKENDS = BACKENDS + [pytest.param("emu-quaternion", id="emu-ik_quaternion")]  # the quaternion variant: lane-emulated build only


@pytest.mark.parametrize("gpu", QUAT_BACKENDS)
def test_ik_env_steps_match_the_cpu_env(sawyer, gpu):
    """reset + 3 env steps with control_type="ik" (8-number actions, three closed-loop repeats of 50 mj_steps): targets, joint command,
    low-level action, observation, reward of the device equal the CPU env (oracle physics + the float64 copy of the solver)"""
    from oracle.ref_env import OracleIKEnv
    from test_env_parity import _sync_oracle_from_engine

    m = sawyer
    n = 2
    quat = gpu == "emu-quaternion"
    gpu = False if quat else gpu
    eng = _ik_engine(m, n, gpu, quaternion_mode=int(quat))
    dof = 9 if quat else 8
    assert eng.act_dim == dof
    eng.env_reset()
    envs = [OracleIKEnv(m, quaternion_mode=int(quat)) for _ in range(n)]
    lpos, lquat = eng.get("link_xpos"), eng.get("link_xquat")
    for i, e in enumerate(envs):
        e.reset()
        _sync_oracle_from_engine(e, eng, i)
        e.sim.qfrc_bias[: e.nr] = eng.get("qfrc_bias")[i]
        # the targets start from the hand pose of the reset's last forward pass (what sim.data holds in the reference): hand it to the oracle
        hl = eng.scene.hand_link[0]
        ikc = eng.ik
        R = mjcf.q_to_mat(lquat[i][4 * hl : 4 * hl + 4].astype(np.float64))
        hp = lpos[i][3 * hl : 3 * hl + 3].astype(np.float64) + R @ np.array(ikc.hand_pos[:])
        hq = mjcf.q_norm(mjcf.q_mul(lquat[i][4 * hl : 4 * hl + 4].astype(np.float64), np.array(ikc.hand_quat[:], dtype=np.float64)))
        e.ik.sync(hp, hq)
        e._hand0 = (hp, hq)
    rng = np.random.RandomState(3)
    for k in range(3):
        a = rng.uniform(-1, 1, (n, dof)).astype(np.float32)
        a[:, -1] = -0.5
        if quat:  # a small rotation relative to the hand, (w, x, y, z)
            v = rng.normal(size=(n, 3)) * 0.05
            a[:, 3], a[:, 4:7] = 1.0, v
            a[:, 3:7] /= np.linalg.norm(a[:, 3:7], axis=1, keepdims=True)
        if k == 0:  # first step: the oracle's sim.data would be one integration newer than the device's stored kinematics; show it the same hand pose
            for e in envs:
                e._hand = lambda arm=0, hp_hq=e._hand0: hp_hq
        obs, rew, done, info = eng.env_step_host(a)
        for i, e in enumerate(envs):
            ob, r, d, inf = e.step(a[i].astype(np.float64))
            if k == 0:
                del e._hand
            st = _ik_state(eng, i)
            assert np.abs(st["target_pos"] - e.ik.target_pos).max() < 2e-6, (k, i)
            assert quat or min(np.abs(st["s"] - e.ik.s).max(), np.abs(st["s"] + e.ik.s).max()) < 1e-5, (k, i)
            assert np.abs(st["q_cmd"] - e.ik.q_cmd).max() < 2e-4, (k, i, st["q_cmd"], e.ik.q_cmd)
            assert np.abs(st["low"] - e.low_action).max() < 2e-3, (k, i, st["low"], e.low_action)
            assert np.abs(obs[i] - ob).max() < 1e-3, (k, i, np.abs(obs[i] - ob).max())
            assert abs(rew[i] - r) < 1e-5 and bool(done[i]) == d and info[i][3] == inf["episode_length"] == k + 1


@pytest.mark.parametrize("gpu", BACKENDS)
def test_ik_control_moves_the_hand_where_the_actions_say(sawyer, gpu):
    """four steps of "move" along one action axis, then four of zero action: the hand follows the accumulated target (0.3 x move_speed per
    step along the swapped axes of furniture.py:2912-2913) and keeps its orientation"""
    m = sawyer
    eng = _ik_engine(m, 1, gpu)
    eng.env_reset()
    hl = eng.scene.hand_link[0]

    def hand():
        lp, lq = eng.get("link_xpos")[0], eng.get("link_xquat")[0]
        R = mjcf.q_to_mat(lq[4 * hl : 4 * hl + 4].astype(np.float64))
        return lp[3 * hl : 3 * hl + 3] + R @ np.array(eng.ik.hand_pos[:]), mjcf.q_mul(lq[4 * hl : 4 * hl + 4].astype(np.float64), np.array(eng.ik.hand_quat[:], dtype=np.float64))

    p0, q0 = hand()
    a = np.zeros((1, 8), np.float32)
    a[0, 1], a[0, 6], a[0, 7] = 1.0, -1.0, -1.0  # action[1] -> -x after the swap
    for _ in range(4):
        eng.env_step_host(a)
    a[0, 1] = 0.0
    for _ in range(4):
        eng.env_step_host(a)
    p1, q1 = hand()
    Rb = mjcf.q_to_mat(np.array(eng.ik.base_quat[:], dtype=np.float64))  # the displacement is added to the target in the robot's base frame
    want = p0 + Rb @ np.array([-4 * 0.1 * 0.3, 0.0, 0.0])
    assert np.linalg.norm(p1 - want) < 0.012, (p1 - p0, want - p0)
    assert abs(abs(np.dot(mjcf.q_norm(q0), mjcf.q_norm(q1))) - 1) < 2e-3
    st = _ik_state(eng, 0)
    assert st["iters"] <= 3 and np.abs(st["low"][:7]).max() < 0.2  # at rest on the target: the solve is immediate, the velocities small


def test_enable_ik_and_dense_refuse_what_they_cannot_serve(sawyer):
    """the C-ABI answers with a code and a message: IK on a two-arm scene, the dense reward on a furniture without a recipe, a config
    struct of the wrong size"""
    import ctypes as C

    from furniture_b200.dense import dense_config
    from furniture_b200.engine import Engine, default_config
    from parity_util import build_emu

    ikc = IK.ik_config(sawyer)
    baxter = mjcf.load_scene("Baxter", "chair_ingolf_0650")
    with pytest.raises(RuntimeError, match="as many arms"):
        Engine(baxter, 1, config=default_config(), lib_path=build_emu(), ik=ikc)  # a one-arm IK config on the two-arm scene
    with pytest.raises(RuntimeError, match="recipe"):
        Engine(mjcf.load_scene("Sawyer", "swivel_chair_0700"), 1, config=default_config(), lib_path=build_emu(), dense=dense_config())
    eng = Engine(sawyer, 1, config=default_config(), lib_path=build_emu())
    bad = IK.ik_config(sawyer)
    bad.struct_bytes = 12
    assert eng.L.fe_enable_ik(eng.h, C.byref(bad)) < 0 and b"size mismatch" in eng.L.fe_last_error(eng.h)
    assert eng.L.fe_action_dim(eng.h) == 9  # still the impedance handle
    assert eng.L.fe_enable_ik(eng.h, C.byref(ikc)) == 0 and eng.L.fe_action_dim(eng.h) == 8


def test_dense_reward_under_ik_control_matches_the_cpu_env(sawyer):
    """IKEASawyerDense-v0 with the reference's default control type: the phase machine reads the policy's 8-number action (gripper = ac[-2],
    connect = ac[-1], control penalty on ac[:-2]) while the arm is driven by the IK's joint velocities -- device vs CPU env, emulated build"""
    from furniture_b200.dense import dense_config
    from furniture_b200.engine import Engine, default_config
    from oracle.ref_env import DenseCfg, OracleDenseIKEnv
    from parity_util import build_emu
    from test_dense_reward import DENSE_BASE, _adopt_device_anchors, _assert_same_machine, _dense_state
    from test_env_parity import _sync_oracle_from_engine

    m = sawyer
    eng = Engine(m, 1, config=default_config(**DENSE_BASE), lib_path=build_emu(), dense=dense_config(), ik=IK.ik_config(m))
    eng.env_reset()
    e = OracleDenseIKEnv(m, DenseCfg())
    e.reset()
    _sync_oracle_from_engine(e, eng, 0)
    e.sim.qfrc_bias[: e.nr] = eng.get("qfrc_bias")[0]
    hl = eng.scene.hand_link[0]
    lp, lq = eng.get("link_xpos")[0], eng.get("link_xquat")[0]
    R = mjcf.q_to_mat(lq[4 * hl : 4 * hl + 4].astype(np.float64))
    hand0 = (lp[3 * hl : 3 * hl + 3].astype(np.float64) + R @ np.array(eng.ik.hand_pos[:]),
             mjcf.q_norm(mjcf.q_mul(lq[4 * hl : 4 * hl + 4].astype(np.float64), np.array(eng.ik.hand_quat[:], dtype=np.float64))))
    e.ik.sync(*hand0)
    e.dense.begin_episode()
    _adopt_device_anchors(e.dense, _dense_state(eng, 0))
    rng = np.random.RandomState(4)
    for k in range(2):
        a = rng.uniform(-1, 1, (1, 8)).astype(np.float32)
        a[0, -1] = -0.5
        if k == 0:
            e._hand = lambda arm=0: hand0
        obs, rew, done, info = eng.env_step_host(a)
        ob, r, d, inf = e.step(a[0].astype(np.float64))
        if k == 0:
            del e._hand
        assert abs(rew[0] - r) < 5e-2 + 1e-5 * abs(r), (k, rew[0], r)
        assert abs(eng.get("dense_info")[0][3] - e.dense_info["ctrl_penalty"]) < 1e-6  # -coef * |ac[:-2]| over six numbers
        _assert_same_machine(_dense_state(eng, 0), e.dense, k, tol=5e-4)
        assert np.abs(obs[0] - ob).max() < 1e-3 and bool(done[0]) == d


def test_unstable_ik_step_resets_mid_step_and_once_more_at_the_end(sawyer):
    """a _do_simulation that blows up inside _do_ik_step resets the env on the spot and the remaining repeats run on the new episode
    (furniture.py:2889-2897 inside the loop of :2977-2995); the step then ends the episode with the unstable penalty and the VecEnv worker
    resets again: three resets' worth of random draws in all, like the impedance path"""
    from oracle.ref_env import Cfg, OracleFurnitureEnv

    m, seed = sawyer, 99
    eng = _ik_engine(m, 2, False, seed=seed, nsub=2)
    eng.env_reset()
    v = eng.get("qvel").copy()
    v[1, 0] = 1e8
    eng.set("qvel", v)
    a = np.zeros((2, 8), np.float32)
    a[:, -1] = -1
    obs, rew, done, info = eng.env_step_host(a)
    assert not done[0] and done[1] and info[1][2] == 1 and info[0][2] == 0 and rew[1] < -50
    ln, pos, st = eng.get("episode_length")[:, 0], eng.get("mt_pos")[:, 0], eng.get("mt_state")
    assert ln[0] == 1 and ln[1] == 0
    for i, nreset in ((0, 1), (1, 3)):
        cfg = Cfg()
        cfg.seed = seed + i
        e = OracleFurnitureEnv(m, cfg)
        for _ in range(nreset):
            e.place()
            for _ in range(101):
                e.rng.uniform(-cfg.agent_xyz_rand, cfg.agent_xyz_rand, e.narm)
        s = e.rng.get_state()
        assert s[2] == pos[i] and np.array_equal(s[1], st[i]), i
    assert np.isfinite(obs).all() and (eng.get("flags")[:, 0] & FLAG_DIVERGED == 0).all()
    obs, rew, done, info = eng.env_step_host(a)
    assert info[1][3] == 1 and info[0][3] == 2 and not done.any()
    assert np.isfinite(eng.get("ik_state")[1].view(np.float32)[:44]).all()  # the new episode's targets were re-synchronised from a sane pose


@pytest.mark.parametrize("quat", [0, 1], ids=["ik", "ik_quaternion"])
def test_baxter_ik_env_steps_match_the_cpu_env(quat):
    """control_type="ik" / "ik_quaternion" on the two-arm env (15 / 17-number actions: move / rotate per arm, two grippers, connect): both
    arms' targets, joint commands and low-level actions, observation and reward of the device equal the CPU env -- emulated build"""
    from furniture_b200.engine import Engine, default_config
    from oracle.ref_env import OracleIKEnv
    from parity_util import build_emu
    from test_env_parity import _sync_oracle_from_engine

    m = mjcf.load_scene("Baxter", "chair_ingolf_0650")
    ikc = IK.ik_config(m, quaternion_mode=quat)
    assert ikc.narms == 2 and abs(ikc.kp - 2.0) < 1e-9 and abs(ikc.user_sensitivity - 1.0) < 1e-9 and abs(ikc.damping - 0.7) < 1e-7
    eng = Engine(m, 1, config=default_config(), lib_path=build_emu(), ik=ikc)
    dof = 17 if quat else 15
    assert eng.act_dim == dof
    eng.env_reset()
    e = OracleIKEnv(m, quaternion_mode=quat)
    e.reset()
    _sync_oracle_from_engine(e, eng, 0)
    e.sim.qfrc_bias[: e.nr] = eng.get("qfrc_bias")[0]
    lpos, lquat = eng.get("link_xpos")[0], eng.get("link_xquat")[0]
    hands = []
    for arm in range(2):
        hl = eng.scene.hand_link[arm]
        R = mjcf.q_to_mat(lquat[4 * hl : 4 * hl + 4].astype(np.float64))
        hp = lpos[3 * hl : 3 * hl + 3].astype(np.float64) + R @ np.array(ikc.arm[arm].hand_pos[:])
        hq = mjcf.q_norm(mjcf.q_mul(lquat[4 * hl : 4 * hl + 4].astype(np.float64), np.array(ikc.arm[arm].hand_quat[:], dtype=np.float64)))
        e.iks[arm].sync(hp, hq)
        hands.append((hp, hq))
    rng = np.random.RandomState(6)
    for k in range(2):
        a = rng.uniform(-1, 1, (1, dof)).astype(np.float32)
        a[0, -1] = -0.5
        if quat:
            for off in (3, 10):
                a[0, off], a[0, off + 1 : off + 4] = 1.0, rng.normal(size=3) * 0.05
                a[0, off : off + 4] /= np.linalg.norm(a[0, off : off + 4])
        if k == 0:
            e._hand = lambda arm=0: hands[arm]
        obs, rew, done, info = eng.env_step_host(a)
        ob, r, d, inf = e.step(a[0].astype(np.float64))
        if k == 0:
            del e._hand
        st = _ik_state(eng, 0)
        for arm, (tp, qc) in enumerate(((st["target_pos"], st["q_cmd"]), (st["target_pos2"], st["q_cmd2"]))):
            assert np.abs(tp - e.iks[arm].target_pos).max() < 2e-6 and np.abs(qc - e.iks[arm].q_cmd).max() < 3e-4, (k, arm, qc, e.iks[arm].q_cmd)
        assert np.abs(st["low_all"] - e.low_action).max() < 2e-3, (k, st["low_all"], e.low_action)
        assert np.abs(obs[0] - ob).max() < 1e-3 and abs(rew[0] - r) < 1e-5 and bool(done[0]) == d
