"""Parity of the engine kernels against the CPU oracle (oracle/fe_oracle.c) on the same seeded inputs.

Each test runs twice: `emu` = the lane-emulated harness build of the kernel source (CPU, keeps the kernel logic covered
when no GPU is present) and `cuda` = the real sm_90a library through the C-ABI (marked gpu).  Tolerances are fp32-vs-fp64
and written next to each assertion.  Reference path being replaced: MjSim.forward()/step(), furniture.py:2877-2879."""
import os

import numpy as np
import pytest

from furniture_b200 import mjcf
from oracle.oracle import OracleSim
from parity_util import have_gpu, make_engine, oracle_link_poses, quat_err, settled_state, to_z

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]
G = os.path.join(os.path.dirname(__file__), "golden")


def _pose_arm_over_parts(model, sim_q, rng):
    """random arm poses that often bring links / fingers into contact with parts and floor"""
    q = sim_q.copy()
    q[:7] = model.meta["robot_init_qpos"] + rng.uniform(-0.8, 0.8, 7)
    q[7:9] = rng.uniform([-0.0115, -0.020833], [0.020833, 0.0115])
    return q


@pytest.mark.parametrize("gpu", BACKENDS)
def test_forward_stages_match_oracle(sawyer_model, gpu):
    m = sawyer_model
    n = 16
    eng = make_engine(m, n, gpu)
    em = eng.em
    rng = np.random.RandomState(7)
    Q, V, U = [], [], []
    for i in range(n):
        q = settled_state(m, i, robot_noise=0.3, dz=rng.uniform(-0.003, 0.01))
        if i % 2:
            q = _pose_arm_over_parts(m, q, rng)
        Q.append(q); V.append(rng.normal(size=m.nv) * 0.3); U.append(rng.uniform(-1.5, 1.5, m.nu))
    eng.set("qpos", np.array(Q)); eng.set("qvel", np.array(V)); eng.set("ctrl", np.array(U))
    eng.forward()
    lp, lq = eng.get("link_xpos"), eng.get("link_xquat")
    bias, Mr, fs, as_, x = eng.get("qfrc_bias"), eng.get("dbg_Mr"), eng.get("dbg_fs"), eng.get("dbg_as"), eng.get("dbg_x")
    fc, linert = eng.get("dbg_fc"), eng.get("dbg_linert")
    ncon, flags = eng.get("ncon")[:, 0], eng.get("flags")[:, 0]
    cdist, cpos, cframe = eng.get("con_dist"), eng.get("con_pos"), eng.get("con_frame")
    sim = OracleSim(m)
    total_con = 0
    for i in range(n):
        sim.qpos[:] = Q[i]; sim.qvel[:] = V[i]; sim.ctrl[:] = U[i]
        sim.qacc_warmstart[:] = 0
        sim.forward()
        xp, xq, xm = oracle_link_poses(sim, em)
        assert np.abs(lp[i].reshape(-1, 3) - xp).max() < 1e-6                      # positions, metres
        assert max(quat_err(a, b) for a, b in zip(lq[i].reshape(-1, 4), xq)) < 1e-6
        M = sim.qM.reshape(m.nv, m.nv)[:9, :9]
        assert np.abs(Mr[i].reshape(9, 9) - M).max() < 1e-5 * np.abs(M).max()       # CRBA
        assert np.abs(bias[i] - sim.qfrc_bias[:9]).max() < 1e-4 * max(1, np.abs(sim.qfrc_bias[:9]).max())  # RNE
        assert np.abs(fs[i][:9] - sim.qfrc_smooth[:9]).max() < 1e-4 * max(1, np.abs(sim.qfrc_smooth[:9]).max())
        zs = to_z(m, em, xm, sim.qacc_smooth)
        assert np.abs(as_[i] - zs).max() < 2e-4 * max(1, np.abs(zs).max())
        assert flags[i] == 0
        # contacts: same set in the same order (pair-list order), geometry to fp32 accuracy
        oc = sim.contacts()
        assert ncon[i] == len(oc), (i, ncon[i], len(oc))
        total_con += len(oc)
        any_mpr = False
        for c, o in enumerate(oc):
            # analytic pairs agree to fp32 round-off; MPR pairs (cylinder vs sphere/cylinder/box) stop at the portal
            # tolerance 1e-6 of the Minkowski difference, which bounds depth to ~1e-5 and the normal to ~1e-3
            mpr = 5 in (m.geom_type[o.geom1], m.geom_type[o.geom2]) and 0 not in (m.geom_type[o.geom1], m.geom_type[o.geom2])
            any_mpr |= bool(mpr)
            assert abs(cdist[i][c] - o.dist) < (1e-4 if mpr else 2e-6), (i, c, cdist[i][c], o.dist)
            assert np.abs(cpos[i].reshape(-1, 3)[c] - np.array(list(o.pos))).max() < (2e-3 if mpr else 5e-6)
            fe_, fo_ = cframe[i].reshape(-1, 9)[c], np.array(list(o.frame))
            if mpr:  # portal refinement: the direction is only defined up to the portal found (true of MuJoCo/libccd too)
                assert fe_[:3] @ fo_[:3] > 0.9
            else:
                assert np.abs(fe_ - fo_).max() < 2e-4
        # constrained acceleration (Newton solver, elliptic cones): relative to its scale.  Cases with an MPR contact
        # are compared through the engine's own optimality residual instead: the fp32 and fp64 portals give normals
        # that differ by ~1e-2 and a deep random interpenetration amplifies that into a different (equally valid) qacc.
        zo = to_z(m, em, xm, sim.qacc)
        if not any_mpr:
            assert np.abs(x[i] - zo).max() < 2e-3 * max(1.0, np.abs(zo).max()), (i, np.abs(x[i] - zo).max(), np.abs(zo).max())
        Mx = np.zeros(m.nv)
        Mx[:9] = Mr[i].reshape(9, 9).astype(np.float64) @ x[i][:9]
        for p in range(em.npart):
            I = linert[i].reshape(-1, 10)[9 + p].astype(np.float64)
            mass, h, Io = I[0], I[1:4], np.array([[I[4], I[7], I[8]], [I[7], I[5], I[9]], [I[8], I[9], I[6]]])
            w_, v_ = x[i][9 + 6 * p : 12 + 6 * p].astype(np.float64), x[i][12 + 6 * p : 15 + 6 * p].astype(np.float64)
            Mx[9 + 6 * p : 12 + 6 * p] = Io @ w_ + np.cross(h, v_)
            Mx[12 + 6 * p : 15 + 6 * p] = mass * v_ - np.cross(h, w_)
        res = Mx - fs[i] - fc[i]
        assert np.abs(res).max() < 2e-4 * max(1.0, np.abs(fs[i]).max(), np.abs(fc[i]).max()), (i, np.abs(res).max())
    assert total_con > 100  # the cases do exercise contact


@pytest.mark.parametrize("gpu", BACKENDS)
def test_trajectory_matches_oracle(sawyer_model, gpu):
    """200 mj_steps from rest with two random control bursts: fp32 engine stays within 2e-5 of the fp64 oracle
    (per-step parity; long contact-rich horizons diverge chaotically and are not compared)."""
    m = sawyer_model
    eng = make_engine(m, 4, gpu)
    sims = [OracleSim(m) for _ in range(4)]
    rng = np.random.RandomState(3)
    Q = np.array([settled_state(m, i, robot_noise=0.0) for i in range(4)])
    eng.set("qpos", Q)
    for i, s in enumerate(sims):
        s.qpos[:] = Q[i]; s.forward()
    eng.forward()
    for burst in range(4):
        U = rng.uniform(-1, 1, (4, m.nu)) * m.actuator_ctrlrange[:, 1]
        eng.set("ctrl", U)
        eng.set("qfrc_applied", eng.get("qfrc_bias"))  # gravity compensation refresh, furniture.py:3372-3377
        for i, s in enumerate(sims):
            s.ctrl[:] = U[i]; s.qfrc_applied[:9] = s.qfrc_bias[:9]
            s.step(50)
        eng.step(50)
        qe, ve = eng.get("qpos"), eng.get("qvel")
        for i, s in enumerate(sims):
            assert np.abs(qe[i] - s.qpos).max() < 2e-5, (burst, i, np.abs(qe[i] - s.qpos).max())
            assert np.abs(ve[i] - s.qvel).max() < 2e-4, (burst, i, np.abs(ve[i] - s.qvel).max())
    assert (eng.get("flags") == 0).all()


@pytest.mark.parametrize("gpu", BACKENDS)
def test_trajectory_matches_oracle_swivel_chair(swivel_model, gpu):
    """second furniture (cylinder parts: the MPR pairs): parts dropped from 3 mm settle on the floor while the arm moves
    under constant controls; 150 mj_steps stay within 5e-6 of the oracle."""
    m = swivel_model
    eng = make_engine(m, 2, gpu)
    sims = [OracleSim(m) for _ in range(2)]
    rng = np.random.RandomState(1)
    for i, s in enumerate(sims):
        q = settled_state(m, i, robot_noise=0.0, dz=0.003)
        c = rng.uniform(-0.3, 0.3, m.nu)
        s.qpos[:] = q; s.qvel[:] = 0; s.ctrl[:] = c
        s.forward()
        if i == 0:
            Q, U = [q], [c]
        else:
            Q.append(q); U.append(c)
    eng.set("qpos", np.array(Q)); eng.set("qvel", np.zeros((2, m.nv))); eng.set("ctrl", np.array(U))
    eng.forward()
    for _ in range(3):
        for s in sims:
            s.step(50)
        eng.step(50)
        qe, ve = eng.get("qpos"), eng.get("qvel")
        for i, s in enumerate(sims):
            assert int(eng.get("ncon")[i][0]) == s.ncon
            assert np.abs(qe[i] - s.qpos).max() < 5e-6, np.abs(qe[i] - s.qpos).max()
            assert np.abs(ve[i] - s.qvel).max() < 1e-4, np.abs(ve[i] - s.qvel).max()
    assert (eng.get("flags") == 0).all()


@pytest.mark.parametrize("gpu", BACKENDS)
def test_joint_limit_rows_match_oracle(sawyer_model, gpu):
    """gripper fingers pushed past their stops (the everyday case: the robot block then has joint-limit rows only and is
    solved by the dedicated per-lane Newton): constrained robot acceleration equals the oracle's."""
    m = sawyer_model
    eng = make_engine(m, 4, gpu)
    sim = OracleSim(m)
    qs, vs, cs, ref = [], [], [], []
    for seed in range(4):
        q = settled_state(m, seed, dz=0.01)
        rng = np.random.RandomState(seed)
        q[7] = 0.0210 + 0.0002 * seed   # range (-0.0115, 0.020833)
        q[8] = -0.0211                  # range (-0.020833, 0.0115)
        v = rng.normal(size=m.nv) * 0.3
        c = rng.uniform(-1, 1, m.nu)
        sim.qpos[:] = q; sim.qvel[:] = v; sim.ctrl[:] = c; sim.qacc_warmstart[:] = 0
        sim.forward()
        qs.append(q); vs.append(v); cs.append(c); ref.append(sim.qacc[:9].copy())
    eng.set("qpos", np.array(qs)); eng.set("qvel", np.array(vs)); eng.set("ctrl", np.array(cs)); eng.set("qacc_warmstart", np.zeros((4, m.nv)))
    eng.forward()
    x = eng.get("dbg_x")
    st = eng.get("stats")
    for e in range(4):
        assert st[e][2] == 1  # the robot block did need a constraint solve
        assert np.abs(x[e][:9] - ref[e]).max() < 2e-5 * max(1.0, np.abs(ref[e]).max()), (e, np.abs(x[e][:9] - ref[e]).max())


@pytest.mark.parametrize("gpu", BACKENDS)
def test_grasped_part_coupled_solve_matches_oracle(sawyer_model, gpu):
    """a leg pinched between the finger pads couples the robot block to a free part (the coupled component of nA = 15 dofs,
    solved by fe_solve_comp<16>; the parts left on the floor go to the grouped solver): constrained accelerations and a short
    trajectory follow the oracle.  tests/test_solver_branches.py covers the other branches of fe_solve."""
    from oracle.ref_env import OracleFurnitureEnv
    from test_env_parity import _grasp_and_align_state

    m = sawyer_model
    env = OracleFurnitureEnv(m)
    env.reset()
    q = _grasp_and_align_state(m, env)
    qs = settled_state(m, 0, dz=0.0)
    q2 = qs.copy()
    q2[:9] = q[:9]       # robot pose of the grasp
    q2[9:16] = q[9:16]   # leg 0 between the pads; the other parts rest on the floor
    eng = make_engine(m, 2, gpu)
    em = eng.em
    sim = OracleSim(m)
    v = np.random.RandomState(3).normal(size=m.nv) * 0.05
    sim.qpos[:] = q2; sim.qvel[:] = v; sim.qacc_warmstart[:] = 0
    sim.forward()
    eng.set("qpos", q2); eng.set("qvel", v); eng.set("qacc_warmstart", np.zeros(m.nv))
    eng.forward()
    assert eng.get("stats")[0][1] == 1  # the coupled scope was taken
    assert int(eng.get("ncon")[0][0]) == sim.ncon
    _, _, xm = oracle_link_poses(sim, em)
    zs = to_z(m, em, xm, sim.qacc)
    x = eng.get("dbg_x")[0]
    # stiff pinch (|qacc| ~ 5e2): 5e-5 relative on the coupled dofs
    assert np.abs(x - zs).max() < 5e-5 * np.abs(zs).max(), np.abs(x - zs).max()
    for _ in range(5):
        sim.step()
        eng.step(1)
    assert np.abs(eng.get("qpos")[0] - sim.qpos).max() < 5e-6
    assert np.abs(eng.get("qvel")[0] - sim.qvel).max() < 2e-3  # |qvel| ~ 1 after the pinch relaxes


@pytest.mark.parametrize("gpu", BACKENDS)
def test_weld_constraint_matches_oracle(gpu):
    from oracle.assembly_oracle import rel_pose

    m = mjcf.load_scene("None", "table_lack_0825")
    eng = make_engine(m, 1, gpu)
    sim = OracleSim(m)
    q = m.qpos0.copy()
    for k, name in enumerate(m.meta["part_names"]):
        q[7 * k : 7 * k + 7] = m.meta["part_init_qpos"][name]
        q[7 * k + 2] += 0.3
    v = np.zeros(m.nv)
    v[0:6] = [0.3, -0.2, 0.0, 1.0, 2.0, -1.5]
    e = 0
    i1 = m.names["jnt"].index(m.names["body"][m.eq_obj1id[e]]); i2 = m.names["jnt"].index(m.names["body"][m.eq_obj2id[e]])
    rel = rel_pose(q[7 * i1 : 7 * i1 + 7], q[7 * i2 : 7 * i2 + 7])
    rel[:3] += [0.002, -0.001, 0.003]  # start with a violated weld so that the position rows are active
    eqd = m.eq_data.copy(); eqd[e] = rel
    act = np.zeros(m.neq, np.int32); act[e] = 1
    sim.qpos[:] = q; sim.qvel[:] = v; sim.eq_data[:] = eqd.ravel(); sim.eq_active[:] = act
    eng.set("qpos", q); eng.set("qvel", v); eng.set("eq_data", eqd.ravel()); eng.set("eq_active", act)
    for k in range(10):
        sim.step(10); eng.step(10)
        assert np.abs(eng.get("qpos")[0] - sim.qpos).max() < 5e-5
        assert np.abs(eng.get("qvel")[0] - sim.qvel).max() < 5e-3 * max(1, np.abs(sim.qvel).max())


@pytest.mark.parametrize("gpu", BACKENDS)
def test_is_aligned_bit_exact_vs_reference_goldens(sawyer_model, gpu):
    """Device _is_aligned on the golden site poses produced by the reference's own Python (furniture.py:1057-1153):
    decisions identical on every case, target quaternion bit-identical (see the note on the no-angle branch)."""
    z = np.load(os.path.join(G, "is_aligned.npz"))
    eng = make_engine(sawyer_model, 1, gpu)
    stride = 1 if gpu else 1
    sl = slice(0, None, stride)
    al, tq = eng.is_aligned(z["p1"][sl], z["m1"][sl], z["p2"][sl], z["m2"][sl], z["angles"][sl], z["nangles"][sl], z["thr"][sl])
    assert np.array_equal(al, z["aligned"][sl])
    assert np.array_equal(np.isnan(tq[:, 0]), ~z["tq_set"][sl])
    # sites with an allowed-angle list (every connector in the shipped furniture): bit-identical target quaternion.
    # The no-angle branch evaluates `cos ** 2` through libm pow(), which is 1 ulp off the exact square for some inputs
    # (transform_utils.py:752); there the quaternion may differ in the last bit -- the decision does not depend on it.
    withang = z["tq_set"][sl] & (z["nangles"][sl] > 0)
    noang = z["tq_set"][sl] & (z["nangles"][sl] == 0)
    assert withang.sum() > 2000 and noang.sum() > 500
    assert np.array_equal(tq[withang], z["tq"][sl][withang])
    assert np.abs(tq[noang] - z["tq"][sl][noang]).max() < 5e-16


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("furn,key,ncon", [("swivel_chair_0700", "cursor7_rest_state", 14), ("block", "baxter0_rest_state", 8)])
def test_state_recorded_from_mujoco_is_an_equilibrium_of_the_engine(furn, key, ncon, gpu):
    """the rest states MuJoCo itself left in the reference's demo recordings (tests/golden/demo_facts.json, see
    test_oracle_physics.py) planted in the fp32 engine: after 2000 mj_steps nothing has moved (5e-6 m, 5e-6 in the quaternion)"""
    from test_oracle_physics import _planted_rest_state

    m = mjcf.load_scene("Sawyer", furn)
    q, facts = _planted_rest_state(m, key)
    eng = make_engine(m, 2, gpu)
    eng.set("qpos", q)
    eng.forward()
    eng.set("qfrc_applied", eng.get("qfrc_bias"))
    eng.step(2000)
    qe = eng.get("qpos")
    assert (eng.get("flags") == 0).all()
    if not gpu:
        assert (eng.get("ncon")[:, 0] == ncon).all()
    for n in m.meta["part_names"]:
        qa = m.jnt_qposadr[m.names["jnt"].index(n)]
        assert np.abs(qe[:, qa : qa + 3] - np.array(facts[n][:3])).max() < 5e-6, n
        assert np.abs(qe[:, qa + 3 : qa + 7] - np.array(facts[n][3:])).max() < 5e-6, n
