"""fix_init, fix_init_parts and reset_robot_after_attach (config/furniture.py:116-127, :169-174) inside the reset and step kernels, per env.

The oracle's placement (tests/reset_options_oracle.py) is pinned to the reference's own _reset / _place_objects / UniformRandomSampler by
tests/golden/reset_options.npz (tools/make_golden_reset_options.py); the device, lane-emulated ([emu]) and on the GPU ([cuda]), is held to
the oracle: placements and generator states exactly, poses at the reset bar of tests/test_preassembled.py.
"""
import os

import numpy as np
import pytest

from furniture_b200 import mjcf
from furniture_b200.engine import Engine, default_config
from oracle.ref_env import Cfg, DenseCfg
from parity_util import build_emu
from reset_options_oracle import ResetOptionsDenseEnv, ResetOptionsEnv, ResetOptionsIKEnv
from test_env_parity import _grasp_and_align_state

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]
HERE = os.path.dirname(os.path.abspath(__file__))
LEGS = ("1_part1", "3_part3")


@pytest.fixture(scope="module")
def lack():
    return mjcf.load_scene("Sawyer", "table_lack_0825")


@pytest.fixture(scope="module")
def klubbo():
    return mjcf.load_scene("Sawyer", "table_klubbo_0740")


def _engine(m, n, gpu, dense=False, ik=False, cfg=None, **opts):
    from furniture_b200.dense import dense_config
    from furniture_b200.ik import ik_config
    from test_dense_reward import DENSE_BASE

    kw = dict(config=default_config(**dict(DENSE_BASE if dense else {}, **(cfg or {}))), ik=ik_config(m) if ik else None, **opts)
    if dense:
        kw["dense"] = dense_config(**(dense if isinstance(dense, dict) else {}))
    return Engine(m, n, device=0, **kw) if gpu else Engine(m, n, lib_path=build_emu(), **kw)


def _cfg(base=Cfg, seed=123, **kw):
    c = base()
    c.seed = seed
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def _same_generator(eng, i, e):
    st = e.rng.get_state()
    return np.array_equal(eng.get("mt_state")[i], st[1]) and int(eng.get("mt_pos")[i, 0]) == st[2]


def _quat_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return min(np.abs(a - b).max(), np.abs(a + b).max())


def _assert_parts_close(eng, i, e, tag):
    q = eng.get("qpos")[i]
    for p in range(e.npart):
        a = e.part_qadr[p]
        assert np.abs(q[a : a + 3] - e.sim.qpos[a : a + 3]).max() < 5e-4 and _quat_err(q[a + 3 : a + 7], e.sim.qpos[a + 3 : a + 7]) < 5e-4, (tag, i, p)


# ------------------------------------------------------------------ the oracle against the reference's own code
@pytest.fixture(scope="module")
def golden():
    g = np.load(os.path.join(HERE, "golden", "reset_options.npz"))
    return {k: g[k] for k in g.files}


def _words(s0, s1):
    """32-bit words a RandomState consumed between states s0 and s1"""
    rs = np.random.RandomState()
    rs.set_state(s0)
    n = 0
    while not (rs.get_state()[2] == s1[2] and np.array_equal(rs.get_state()[1], s1[1])):
        rs.bytes(4)
        n += 1
    return n


def test_oracle_placements_equal_the_reference(golden):
    """every golden case (fix_init x fix_init_parts none / one / two legs, table_lack_0825 with XML poses and table_klubbo_0740 without, a
    furn_xyz_rand wide enough that tries are rejected against the fixed parts), four consecutive resets: the planted poses bit for bit, the
    tries, the draws each reset consumes and init_pos after it"""
    g = golden
    models = {}
    for c in range(len(g["case_furniture"])):
        furn = str(g["case_furniture"][c])
        m = models.setdefault(furn, mjcf.load_scene("Sawyer", furn))
        e = ResetOptionsEnv(m, _cfg(furn_xyz_rand=float(g["case_xyz"][c])), fix_init=bool(g["case_fix_init"][c]), fix_init_parts=str(g["case_parts"][c]))
        for r in range(g["pos"].shape[1]):
            s0 = e.rng.get_state()
            placed = e.place()
            assert _words(s0, e.rng.get_state()) == int(g["draws"][c, r]) and sum(e.tries) == int(g["tries"][c, r]), (c, r)
            assert ";".join(e.rejected) == str(g["rejected"][c, r]), (c, r, e.rejected, g["rejected"][c, r])
            for k, (p, q) in enumerate(placed):
                assert np.array_equal(p, g["pos"][c, r, k]) and np.array_equal(q, g["quat"][c, r, k]), (c, r, k)
                assert np.array_equal(np.concatenate([e.init_pos[e.parts[k]], e.init_quat[e.parts[k]]]), g["init_pos"][c, r, k]), (c, r, k)
    assert (g["draws"] == 0).any()  # fix_init starts drew nothing
    # some try is rejected by a fixed part that comes later in XML order than the part being placed
    order = mjcf.load_scene("Sawyer", "table_lack_0825").meta["part_names"]
    later = [rj for c in range(len(g["case_parts"])) for rr in g["rejected"][c] for rj in str(rr).split(";") if rj
             and rj.split("<")[1] in str(g["case_parts"][c]).split(",") and order.index(rj.split("<")[1]) > order.index(rj.split("<")[0])]
    assert later, "no rejection against a later fixed part"


def test_oracle_connect_tail_equals_the_reference(golden, lack):
    """_connect with reset_robot_after_attach, the reference's own code: after the weld and _get_next_subtask, one _initialize_robot_pos (and
    sync_state for ik) taking 7 doubles; the arm and gripper qpos it writes equal the oracle's _init_robot from the same generator; a reset
    that preassembles 2 recipe steps calls it once per connection, before the 101 robot poses after random placement, and from a recorded
    start only for the connections"""
    g = golden
    for c in range(len(g["connect_case"])):
        case, ctl, calls = str(g["connect_case"][c]), str(g["connect_control"][c]), str(g["connect_calls"][c]).split(";")
        if case == "policy":
            assert calls == ["connect", "activate_weld", "get_next_subtask", "initialize_robot_pos"] + (["sync_state"] if ctl == "ik" else [])
            assert int(g["connect_words"][c]) == 14
            e = ResetOptionsEnv(lack, _cfg(), reset_robot_after_attach=True)
            e._init_robot()
            arm = e.arm_idx + e.grip_idx
            assert np.array_equal(e.sim.qpos[arm], g["connect_qpos"][c]), (e.sim.qpos[arm], g["connect_qpos"][c])
        else:
            pre = calls[: calls.index("initialize_robot_pos", calls.index("connect", 1)) + 1]
            assert pre == ["connect", "activate_weld", "get_next_subtask", "initialize_robot_pos"] * 2, calls
            robot_poses = calls.count("initialize_robot_pos") - 2
            assert robot_poses == (101 if case == "preassembly_random" else 0)
            assert int(g["connect_words"][c]) == 14 * (2 + robot_poses)


# ------------------------------------------------------------------ fix_init / fix_init_parts on the device
def _fix_pose(eng, i):
    return eng.get("fix_pose")[i].reshape(-1, 7)


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("furn", ["table_lack_0825", "table_klubbo_0740"])
def test_fix_init_keeps_each_envs_placement(gpu, furn):
    """fix_init on two envs: each env's placement stays its own bit for bit through resets and an auto-reset; on table_lack it is the XML
    pose from the first reset on and the sampler draws nothing; poses after the first reset and the generator after three are the CPU env's"""
    m = mjcf.load_scene("Sawyer", furn)
    eng = _engine(m, 2, gpu, cfg=dict(max_episode_steps=1), fix_init=True)
    envs = [ResetOptionsEnv(m, _cfg(seed=123 + i), fix_init=True) for i in range(2)]
    xml = mjcf.xml_init_poses(m.meta)
    eng.env_reset()
    first = [_fix_pose(eng, i) for i in range(2)]
    for i, e in enumerate(envs):
        e.reset()
        if xml is not None:  # the settled poses at the reset bar on the model the parity tests use
            _assert_parts_close(eng, i, e, "first reset")
        want = np.array([np.concatenate([e.init_pos[n], e.init_quat[n]]) for n in e.parts])
        assert np.abs(first[i] - want).max() < 1e-6, i
    if xml is not None:
        assert all(np.array_equal(f, np.array([xml[n] for n in m.meta["part_names"]])) for f in first)
    else:
        assert not np.array_equal(first[0], first[1])  # each env keeps the placement its own first reset drew
    eng.env_reset()
    eng.env_step_host(np.zeros((2, eng.act_dim), np.float32))  # a one-step episode: the auto-reset inside the step kernel
    assert (eng.get("episode_length") == 0).all()
    for i, e in enumerate(envs):
        e.reset(); e.reset()
        assert np.array_equal(_fix_pose(eng, i), first[i]) and _same_generator(eng, i, e), i
    assert (eng.get("fix_have") == 1).all()


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("furn,xyz,parts", [("table_lack_0825", 0.02, LEGS), ("table_klubbo_0740", 0.02, LEGS), ("table_lack_0825", 0.3, LEGS),
                                            ("table_lack_0825", 0.3, ("4_part4",))])
def test_fix_init_parts_reset_equals_the_cpu_env(gpu, furn, xyz, parts):
    """fix_init_parts: three resets against the CPU env, part poses at the reset bar, the remembered placement, and the generator exactly.
    With the table top fixed at furn_xyz_rand 0.3, tries of a leg that comes before it in XML order are rejected against it"""
    m = mjcf.load_scene("Sawyer", furn)
    eng = _engine(m, 1, gpu, cfg=dict(furn_xyz_rand=xyz), fix_init_parts=set(parts))
    e = ResetOptionsEnv(m, _cfg(furn_xyz_rand=xyz), fix_init_parts=",".join(parts))
    assert int(eng.get("fix_init_parts")[0, 0]) == sum(1 << m.meta["part_names"].index(n) for n in parts)
    rejected = []
    for r in range(3):
        eng.env_reset()
        e.reset()
        rejected += e.rejected
        assert _same_generator(eng, 0, e), r
        want = np.array([np.concatenate([e.init_pos[n], e.init_quat[n]]) for n in e.parts])
        assert np.abs(_fix_pose(eng, 0) - want).max() < 1e-6, r
        if xyz == 0.02 and furn == "table_lack_0825":  # the settled poses at the reset bar on the model the parity tests use
            _assert_parts_close(eng, 0, e, r)
    if parts == ("4_part4",):
        assert any(rj.endswith("<4_part4") for rj in rejected), rejected


@pytest.mark.parametrize("gpu", BACKENDS)
def test_options_per_env_equal_handles_of_their_own(lack, gpu):
    """one handle with fix_init on env 0, nothing on env 1 and fix_init_parts on env 2: after three resets every env's state and generator
    equal those of a one-env handle seeded as that env, bit for bit"""
    opts = [dict(fix_init=True), dict(), dict(fix_init_parts=list(LEGS))]
    eng = _engine(lack, 3, gpu)
    for i, o in enumerate(opts):
        eng.set_reset_options(envs=[i], **o)
    for _ in range(3):
        eng.env_reset()
    for i, o in enumerate(opts):
        own = _engine(lack, 1, gpu, cfg=dict(seed=123 + i), **o)
        for _ in range(3):
            own.env_reset()
        for f in ("qpos", "qvel", "obs", "mt_state", "mt_pos", "fix_pose"):
            assert np.array_equal(eng.get(f)[i], own.get(f)[0]), (i, f)


# ------------------------------------------------------------------ reset_robot_after_attach
def _connect_setup(m, gpu, kind, num_connects=None):
    """the CPU env and a one-env handle, both with reset_robot_after_attach, a leg held aligned with the table (test_env_parity's scripted grasp)"""
    if kind == "ik":
        e = ResetOptionsIKEnv(m, _cfg(), reset_robot_after_attach=True)
        eng = _engine(m, 1, gpu, ik=True, cfg=dict(nsub=1), reset_robot_after_attach=True)
    else:
        e = ResetOptionsEnv(m, _cfg(), reset_robot_after_attach=True)
        eng = _engine(m, 1, gpu, cfg=dict(nsub=1), reset_robot_after_attach=True)
    if num_connects is not None:
        e.set_subtask(0, num_connects)
        eng.set_subtask(0, num_connects)
    e.reset()
    eng.env_reset()
    assert _same_generator(eng, 0, e)
    q = _grasp_and_align_state(m, e)
    e.nsub = 1
    e.sim.qvel[:] = 0; e.sim.qacc_warmstart[:] = 0; e.sim.ctrl[:] = 0
    e.sim.forward()
    eng.set("qpos", q); eng.set("qvel", np.zeros(m.nv)); eng.set("qacc_warmstart", np.zeros(m.nv))
    eng.forward()
    return e, eng


@pytest.mark.parametrize("gpu", BACKENDS)
def test_connection_sends_the_arm_home(lack, gpu):
    """grasp -> connect: after the connecting step the arm is back at its start pose with fresh noise, as in the CPU env, and both generators
    took the same 7 draws; 3 more steps at the obs bar"""
    m = lack
    e, eng = _connect_setup(m, gpu, "sparse")
    st0 = e.rng.get_state()
    a = np.zeros((1, eng.act_dim), np.float32)
    a[:, -2], a[:, -1] = 1.0, 1.0
    obs, rew, done, info = eng.env_step_host(a)
    ob, r, d, inf = e.step(a[0].astype(np.float64))
    assert inf["num_connected"] == 1 and info[0][0] == 1 and not done[0]
    assert _words(st0, e.rng.get_state()) == 14 and _same_generator(eng, 0, e)  # one _initialize_robot_pos: 7 doubles
    arm = e.arm_idx + e.grip_idx
    home = np.concatenate([m.meta["robot_init_qpos"], m.meta["gripper_init_qpos"]])
    assert np.abs(eng.get("qpos")[0][arm] - e.sim.qpos[arm]).max() < 1e-3 and np.abs(e.sim.qpos[arm] - home).max() < 5e-2
    assert np.abs(obs[0] - ob).max() < 1e-3
    a[:, -1] = -1.0
    for k in range(3):
        obs, *_ = eng.env_step_host(a)
        ob, *_ = e.step(a[0].astype(np.float64))
        assert np.abs(obs[0] - ob).max() < 2e-3, k


@pytest.mark.parametrize("gpu", BACKENDS)
def test_dense_connection_sends_the_arm_home(lack, gpu):
    """the dense env with reset_robot_after_attach attaches the recipe's first leg (test_obs_layout's scripted dense connect): after the
    connecting step the arm qpos, the generator, the phase, the subtask and the reward are the CPU dense env's, then 3 more steps at the obs
    bar -- the one existing behaviour this option changes: the phase machine starting at ABOVE_LEG now finds the arm at home"""
    from test_dense_reward import PREV_KEYS, _dense_state

    m = lack
    cfg = _cfg(DenseCfg)
    cfg.auto_align = True
    e = ResetOptionsDenseEnv(m, cfg, dict(reset_robot_after_attach=True), reset_robot_after_attach=True)
    e.reset()
    eng = _engine(m, 1, gpu, dense=dict(reset_robot_after_attach=True), cfg=dict(nsub=1, auto_align=1))
    eng.env_reset()
    assert int(eng.get("reset_robot_after_attach")[0, 0]) == 1 and _same_generator(eng, 0, e)
    q = _grasp_and_align_state(m, e, leg=1, leg_site="leg-table,0,90,180,270,conn_site2", table_site="table-leg,0,90,180,270,conn_site2",
                               arm_qpos=[-0.28, -0.9, 0.0, 1.86, 0.0, 0.6, 1.57])
    e.nsub = 1
    e.sim.qvel[:] = 0; e.sim.qacc_warmstart[:] = 0; e.sim.ctrl[:] = 0
    e.sim.forward()
    e.dense.begin_episode()
    eng.set("qpos", q); eng.set("qvel", np.zeros(m.nv)); eng.set("qacc_warmstart", np.zeros(m.nv))
    eng.forward()
    st = eng.get("dense_state").copy()
    raw = bytearray(st[0].tobytes())
    ints, dbl = np.frombuffer(raw[:32], np.int32).copy(), np.frombuffer(raw[32:], np.float64).copy()
    o = e.dense
    ints[:7] = [o.phase, o.subtask, 0, 0, 0, 0, 0]
    dbl[0:3], dbl[3:6], dbl[6:9] = o.table_site0, o.leg0, o.lift_target
    for k, name in enumerate(PREV_KEYS):
        dbl[12 + k] = o.prev.get(name, 0.0)
    eng.set("dense_state", np.frombuffer(ints.tobytes() + dbl.tobytes(), np.uint8)[None].view(st.dtype).reshape(st.shape))
    a = np.zeros((1, eng.act_dim), np.float32)
    a[:, -2], a[:, -1] = 1.0, -1.0
    eng.env_step_host(a)  # the held leg is noticed
    e.step(a[0].astype(np.float64))
    st0 = e.rng.get_state()
    a[:, -1] = 1.0
    obs, rew, done, info = eng.env_step_host(a)
    ob, r, d, inf = e.step(a[0].astype(np.float64))
    assert inf["num_connected"] == 1 and info[0][0] == 1 and not done[0] and not d
    assert _words(st0, e.rng.get_state()) == 14 and _same_generator(eng, 0, e)
    arm = e.arm_idx + e.grip_idx
    assert np.abs(eng.get("qpos")[0][arm] - e.sim.qpos[arm]).max() < 1e-3
    ds = _dense_state(eng, 0)
    assert (ds["subtask"], ds["phase"]) == (e.dense.subtask, e.dense.phase) and e.dense.subtask == 1
    assert abs(float(rew[0]) - r) < 1e-2 * max(1.0, abs(r)), (rew[0], r)
    assert np.abs(obs[0] - ob).max() < 1e-3
    a[:, -1] = -1.0
    for k in range(3):
        obs, rew, done, info = eng.env_step_host(a)
        ob, r, d, inf = e.step(a[0].astype(np.float64))
        ds = _dense_state(eng, 0)
        assert (ds["subtask"], ds["phase"]) == (e.dense.subtask, e.dense.phase), k
        assert np.abs(obs[0] - ob).max() < 2e-3 and abs(float(rew[0]) - r) < 1e-2 * max(1.0, abs(r)), (k, np.abs(obs[0] - ob).max(), rew[0], r)


@pytest.mark.parametrize("gpu", BACKENDS)
def test_ik_connection_against_the_cpu_env(lack, gpu):
    """control_type="ik" with reset_robot_after_attach, grasp -> connect against the CPU IK env: arm qpos and generator after the connecting
    step; on the next command the position target is re-seeded (sync_state) and the orientation target kept, as the CPU env's; 3 steps at the
    obs bar"""
    from test_ik import _ik_state

    m = lack
    e, eng = _connect_setup(m, gpu, "ik")
    eng.set("episode_length", 0)  # both controllers start from the scripted scene: the next command seeds s and the target, like _ik_sync
    e._ik_sync()
    a = np.zeros((1, eng.act_dim), np.float32)
    a[:, -2], a[:, -1] = 1.0, 1.0
    st0 = e.rng.get_state()
    obs, rew, done, info = eng.env_step_host(a)
    ob, r, d, inf = e.step(a[0].astype(np.float64))
    assert inf["num_connected"] == 1 and info[0][0] == 1
    assert _words(st0, e.rng.get_state()) == 14 and _same_generator(eng, 0, e)
    arm = e.arm_idx + e.grip_idx
    assert np.abs(eng.get("qpos")[0][arm] - e.sim.qpos[arm]).max() < 1e-3
    s_before = _ik_state(eng, 0)["s"].copy()
    a[:, -1] = -1.0
    for k in range(3):
        obs, *_ = eng.env_step_host(a)
        ob, *_ = e.step(a[0].astype(np.float64))
        st = _ik_state(eng, 0)
        if k == 0:
            assert np.array_equal(st["s"], s_before) and np.abs(st["s"] - e.ik.s).max() < 1e-5
        assert np.abs(st["target_pos"] - e.ik.target_pos).max() < 1e-4, (k, st["target_pos"], e.ik.target_pos)
        assert np.abs(obs[0] - ob).max() < 2e-3, (k, np.abs(obs[0] - ob).max())


@pytest.mark.parametrize("gpu", BACKENDS)
def test_ik_connection_reseeds_the_position_target_only(lack, gpu):
    """control_type="ik": the command after the connection takes the hand pose of the re-pin step as its position target (sync_state), and
    the accumulated orientation target is left as it was"""
    from test_ik import _ik_state

    m = lack
    e, eng = _connect_setup(m, gpu, "ik")
    a = np.zeros((1, eng.act_dim), np.float32)
    a[:, -2] = 1.0
    eng.env_step_host(a)  # a step of the episode, so that the next command is not the episode's first
    s_before = _ik_state(eng, 0)["s"].copy()
    a[:, -1] = 1.0
    obs, rew, done, info = eng.env_step_host(a)
    assert info[0][0] == 1 and int(eng.get("episode_length")[0, 0]) == 2
    ikc = eng.ik
    hl = eng.scene.hand_link[0]
    lpos, lquat = eng.get("link_xpos")[0].astype(np.float64), eng.get("link_xquat")[0].astype(np.float64)
    hp = lpos[3 * hl : 3 * hl + 3] + mjcf.q_to_mat(lquat[4 * hl : 4 * hl + 4]) @ np.array(ikc.hand_pos[:])
    Rb = mjcf.q_to_mat(np.array(ikc.base_quat[:], np.float64))
    hb = Rb.T @ (hp - np.array(ikc.base_pos[:]))
    a[:, -1] = -1.0
    eng.env_step_host(a)  # zero move, zero rotation: target = the re-seeded hand pose, s unchanged
    st = _ik_state(eng, 0)
    assert np.abs(st["target_pos"] - hb).max() < 1e-4, (st["target_pos"], hb)
    assert np.array_equal(st["s"], s_before)


@pytest.mark.parametrize("gpu", BACKENDS)
def test_episode_ending_connection_draws_before_the_auto_reset(lack, gpu):
    """a connection that ends the episode (num_connects = 1): the arm reset's 7 draws come before the auto-reset's, as in the CPU env"""
    e, eng = _connect_setup(lack, gpu, "sparse", num_connects=1)
    a = np.zeros((1, eng.act_dim), np.float32)
    a[:, -2], a[:, -1] = 1.0, 1.0
    obs, rew, done, info = eng.env_step_host(a)
    ob, r, d, inf = e.step(a[0].astype(np.float64))
    assert d and done[0] and info[0][1] == 1
    e.reset()  # the VecEnv worker's reset after done
    assert _same_generator(eng, 0, e)
    # the order: the reset's robot poses took the noise that follows the arm reset's 7 draws, so the new episode's arm is the CPU env's
    arm = e.arm_idx + e.grip_idx
    assert np.abs(eng.get("qpos")[0][arm] - e.sim.qpos[arm]).max() < 5e-5, np.abs(eng.get("qpos")[0][arm] - e.sim.qpos[arm]).max()


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("branch", ["random", "init_state"])
def test_preassembly_sends_the_arm_home(lack, gpu, branch):
    """preassembled = 2 with reset_robot_after_attach, after random placement and from a recorded start: every preassembly connection takes
    its 7 draws; the reset equals the CPU env's, generator exactly"""
    from reset_options_oracle import ResetOptionsInitStateEnv

    m = lack
    eng = _engine(m, 1, gpu, reset_robot_after_attach=True)
    e = ResetOptionsInitStateEnv(m, _cfg(), reset_robot_after_attach=True)
    if branch == "init_state":
        from test_init_states import _mid_assembly_state

        st = _mid_assembly_state(m)
        eng.set_init_qpos(st)
        e.set_init_qpos(st)
    eng.set_subtask(2)
    e.set_subtask(2)
    eng.env_reset()
    s0 = e.rng.get_state()
    e.reset()
    assert _words(s0, e.rng.get_state()) == (2 * 14 if branch == "init_state" else 2 * 14 + 30 + 101 * 14)
    assert _same_generator(eng, 0, e)
    _assert_parts_close(eng, 0, e, branch)
    arm = e.arm_idx + e.grip_idx  # the arm after the reset: the noise of the draws in the CPU env's order
    assert np.abs(eng.get("qpos")[0][arm] - e.sim.qpos[arm]).max() < 5e-5, np.abs(eng.get("qpos")[0][arm] - e.sim.qpos[arm]).max()


# ------------------------------------------------------------------ defaults, host surface, refusals
@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("ik", [False, True], ids=["sparse", "ik"])
def test_default_options_change_nothing(lack, gpu, ik):
    """an untouched handle and one whose options are all set to their defaults, its remembered placement cleared: reset + 5 steps bit-identical"""
    from test_obs_layout import _run

    plain = _engine(lack, 2, gpu, ik=ik)
    explicit = _engine(lack, 2, gpu, ik=ik, fix_init=False, fix_init_parts=set(), reset_robot_after_attach=False)
    explicit.set_reset_options(fix_init=False, fix_init_parts="", reset_robot_after_attach=False)
    explicit.set("fix_have", 0)
    for x, y in zip(_run(plain), _run(explicit)):
        assert x.dtype == y.dtype and np.array_equal(x, y)


def test_refusals_and_config_keys(lack):
    """the C-ABI refuses flags outside {0, 1}, mask bits at or beyond npart, non-finite poses, and a reset_robot_after_attach that disagrees
    with the dense reward's; unknown part names are a ValueError; split_config consumes the three keys, and leaves them out at their defaults"""
    from furniture_b200.env import split_config, split_dense_config

    eng = _engine(lack, 2, False)
    for name, bad in (("fix_init", 2), ("reset_robot_after_attach", -1), ("fix_have", 3), ("fix_init_parts", 1 << 5), ("fix_init_parts", -1)):
        with pytest.raises(RuntimeError):
            eng.set(name, bad)
    pose = eng.get("fix_pose")
    pose[1, 3] = np.nan
    with pytest.raises(RuntimeError):
        eng.set("fix_pose", pose)
    pose = eng.get("fix_pose")
    pose[0, 3:7] = 0.0
    with pytest.raises(RuntimeError):
        eng.set("fix_pose", pose)
    fresh = _engine(mjcf.load_scene("Sawyer", "table_klubbo_0740"), 1, False)  # no XML poses: nothing remembered yet
    with pytest.raises(RuntimeError):
        fresh.set("fix_have", 1)
    with pytest.raises(ValueError):
        eng.set_reset_options(fix_init_parts={"1_part1", "no_such_part"})
    eng.set("fix_init_parts", (1 << 5) - 1)
    partial = mjcf.load_scene("Sawyer", "table_lack_0825")  # a model whose XML lists only some parts: fix_init is undefined, nothing is seeded
    partial.meta = dict(partial.meta, xml_initpos_parts=["0_part0", "1_part1"])
    with pytest.raises(ValueError):
        _engine(partial, 1, False, fix_init=True)
    with pytest.raises(ValueError):
        _engine(partial, 1, False, fix_init_parts=["2_part2"])
    some = _engine(partial, 1, False, fix_init_parts=["1_part1"])
    assert int(some.get("fix_have")[0, 0]) == 0
    dense = _engine(lack, 1, False, dense=True)
    with pytest.raises(RuntimeError):
        dense.set("reset_robot_after_attach", 1)
    with pytest.raises(ValueError):
        _engine(lack, 1, False, dense=True, reset_robot_after_attach=True)
    on = _engine(lack, 1, False, dense=dict(reset_robot_after_attach=True))
    assert int(on.get("reset_robot_after_attach")[0, 0]) == 1
    _, over, ignored = split_config(dict(fix_init=True, fix_init_parts="1_part1,3_part3", reset_robot_after_attach=True, port=1))
    assert over == dict(fix_init=True, fix_init_parts="1_part1,3_part3", reset_robot_after_attach=True) and ignored == ["port"]
    _, over, ignored = split_config(dict(fix_init=False, fix_init_parts=None, reset_robot_after_attach=False))
    assert over == {} and ignored == []
    _, over, dense_over, ignored = split_dense_config(dict(reset_robot_after_attach=True))
    assert "reset_robot_after_attach" not in over and dense_over["reset_robot_after_attach"] is True and ignored == []


@pytest.mark.gpu
def test_make_vec_env_gym_and_the_mixed_batch(lack):
    """the config keys through make_vec_env and the gym env, every bucket of a mixed batch, and its refusal of part names"""
    from furniture_b200.env import MixedFurnitureEnv, make_vec_env
    from furniture_b200.gym_api import FurnitureGymB200

    env = make_vec_env("IKEASawyer-v0", 2, dict(fix_init=True, fix_init_parts="1_part1", reset_robot_after_attach=True, port=1))
    eg = env.engine
    assert env.ignored_config == ["port"] and (eg.get("fix_init") == 1).all() and (eg.get("reset_robot_after_attach") == 1).all()
    assert (eg.get("fix_init_parts") == 2).all()
    env.reset()
    env.close()
    g = FurnitureGymB200("IKEASawyer-v0", fix_init=True, reset_robot_after_attach=True)
    assert int(g.engine.get("fix_init")[0, 0]) == 1 and int(g.engine.get("reset_robot_after_attach")[0, 0]) == 1
    mixed = MixedFurnitureEnv(["table_lack_0825", "table_klubbo_0740"], 2, fix_init=True, reset_robot_after_attach=True)
    assert all((b.engine.get("fix_init") == 1).all() and (b.engine.get("reset_robot_after_attach") == 1).all() for b in mixed.buckets)
    mixed.close()
    with pytest.raises(ValueError):
        MixedFurnitureEnv(["table_lack_0825", "table_klubbo_0740"], 2, fix_init_parts={"1_part1"})
