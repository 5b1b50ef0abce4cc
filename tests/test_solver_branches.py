"""Every branch of the constraint-solver dispatch (fe_solve, fe_engine.h) against the fp64 oracle, at the stage level.

fe_solve splits the constraint set of one mj_step into pieces and sends each to its own solver:
  grouped        fe_solve_parts_grouped: free parts that touch only the static world, 4-lane units (2 units for a part with
                 5-8 contacts, another pass once the 8 units are used)
  robot limits   fe_solve_robot_limits: the robot block when its only rows are joint limits
  comp<16|24|32> fe_solve_comp: the coupled component (robot with contacts, parts touching the robot or each other, welded
                 parts) when it has nA <= 32 dofs and ncc <= 32 contacts; the template is picked by nA
  coop           fe_solve_coop beyond that, over all dofs: the register Newton direction fe_newton_regs when the robot block
                 and the coupled parts have <= 32 dofs and no part has more than 8 static contacts, else the shared-memory
                 fe_chol / fe_chol_solve
`classify` restates that rule on the oracle's contact list, so that every state says which branch it is meant to reach and
the coverage table below is asserted, not assumed.

The states are seeded random piles of parts dropped with the oracle next to the arm, sampled every 20 mj_steps so that qvel
and qacc_warmstart are realistic.  Each state is run through the engine's forward() and one mj_step and compared with the
oracle: flags, the ordered contact list, the constrained acceleration (states without an MPR contact), the engine's own
optimality residual, and qpos / qvel after the step.

`emu` = the lane-emulated build of the kernel source (CPU); `cuda` = the sm_90a library (marked gpu)."""
import functools

import numpy as np
import pytest

from furniture_b200 import mjcf
from furniture_b200.engine import FLAG_CONTACT_FULL, auto_maxcon
from furniture_b200.engine_model import EngineModel
from oracle.assembly_oracle import rel_pose
from oracle.oracle import OracleSim
from parity_util import make_engine, oracle_link_poses, settled_state, to_z

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]
GEOM_CYLINDER, GEOM_MESH = 5, 7
NEAR = 1e-5  # fp32 and fp64 may disagree on whether a contact this close to its activation distance exists


# ---------------------------------------------------------------- the dispatch rule of fe_solve, restated
def classify(m, em, contacts, eq_active):
    """fe_solve's decision for one constraint set.  Contact kind as in fe_assemble: 0 a free part against the static world,
    1 robot only, 2 robot against a part, 3 part against part."""
    nrl, npart, nr = em.nrlink, em.npart, em.nrlink
    link = lambda g: em.weld_link(int(m.geom_bodyid[g]))
    kinds, owner = [], []
    for c in contacts:
        A, B = link(c.geom1), link(c.geom2)
        pa, pb = A >= nrl, B >= nrl
        kinds.append(0 if (pa and B < 0) or (pb and A < 0) else 3 if (pa and pb) else 2 if (pa or pb) else 1)
        owner.append(max(A, B) - nrl)
    robot_in = any(k in (1, 2) for k in kinds)
    nstat = [0] * npart
    touch = [False] * npart  # part in a kind 2 / 3 contact
    for c, k in zip(contacts, kinds):
        for g in (c.geom1, c.geom2):
            p = link(g) - nrl
            if p < 0:
                continue
            if k == 0:
                nstat[p] += 1
            else:
                touch[p] = True
    welded = [False] * npart
    for e in range(m.neq):
        if eq_active[e]:
            for b in (m.eq_obj1id[e], m.eq_obj2id[e]):
                p = em.weld_link(int(b)) - nrl
                if p >= 0:
                    welded[p] = True
    cpl = [touch[p] or welded[p] or nstat[p] > 8 for p in range(npart)]
    nA = (nr if robot_in else 0) + 6 * sum(cpl)
    ncc = sum(1 for k, p in zip(kinds, owner) if k != 0 or cpl[p])
    info = dict(nA=nA, ncc=ncc, ncpl=sum(cpl), nstat=nstat, robot_in=robot_in, weld=any(welded), ncon=len(contacts))
    if not any(cpl) and not robot_in:
        units, passes, p0 = [], 0, 0
        while p0 < npart:  # fe_solve_parts_grouped's packing: 8 units of 4 lanes per pass, a wide part on an aligned pair
            nu, p = 0, p0
            while p < npart:
                need = 2 if nstat[p] > 4 else 1
                nu += need == 2 and nu & 1
                if nu + need > 8:
                    break
                nu += need
                p += 1
            passes, p0 = passes + 1, p
        return dict(info, branch="grouped", passes=passes)
    if nA <= 32 and ncc <= 32:
        return dict(info, branch="comp%d" % (16 if nA <= 16 else 24 if nA <= 24 else 32))
    # fe_solve_coop: its register active set is the robot block plus the coupled parts; a part with more than 8 static
    # contacts also sends the direction to the Cholesky path
    nreg = nr + 6 * sum(cpl)
    regs = nreg <= 32 and max(nstat, default=0) <= 8
    return dict(info, branch="coop_regs" if regs else "coop_chol")


# ---------------------------------------------------------------- seeded pile states from the oracle
def _near_activation(m, em, probe, q, eqa, eqd, oc):
    """a contact of a free part whose distance is within NEAR of its activation distance, on either side.  (The arm at its
    start pose keeps one pair of its own, right_l0 against the base, 3e-7 outside contact whatever its joint angles; the
    existing parity tests show that fp32 and fp64 agree it is not a contact.)"""
    on_part = lambda c: max(em.weld_link(int(m.geom_bodyid[c.geom1])), em.weld_link(int(m.geom_bodyid[c.geom2]))) >= em.nrlink
    if any(abs(c.dist - c.margin) < NEAR for c in oc if on_part(c)):
        return True
    probe.qpos[:] = q; probe.eq_active[:] = eqa; probe.eq_data[:] = eqd
    probe.stage("kinematics"); probe.stage("collision")
    return sum(map(on_part, probe.contacts())) != sum(map(on_part, oc))


def _mpr(m, contacts):
    """a contact that the narrow phase finds with MPR: a cylinder against anything but a plane, or a mesh"""
    types = [(m.geom_type[c.geom1], m.geom_type[c.geom2]) for c in contacts]
    return any(GEOM_CYLINDER in t and 0 not in t or GEOM_MESH in t for t in types)


@functools.lru_cache(maxsize=None)
def pile_states(name, npile, seed, weld_every=0, spread=0.05, away=0.0):
    """States of `npile` seeded piles of Sawyer + `name`: the parts dropped with random orientations over a square of half-width
    `spread` next to the arm (at its start pose +- 0.3 rad; `away` moves the square along y), sampled every 20 mj_steps.
    With weld_every = k, every k-th pile runs with one weld active (eq_data = the relative pose of its bodies at the drop).  States with a contact within NEAR
    of its activation distance are dropped."""
    m = mjcf.load_scene("Sawyer", name)
    em = EngineModel(m)
    sim, probe = OracleSim(m), OracleSim(m)
    probe.set_model("geom_margin", np.asarray(m.a["geom_margin"], np.float64) + NEAR)
    rng = np.random.RandomState(seed)
    parts = m.meta["part_names"]
    out = []
    for t in range(npile):
        q = settled_state(m, seed * 1000 + t, robot_noise=0.3, dz=0.0)
        cx, cy = rng.uniform(-0.1, 0.1, 2) + [0.0, away]
        for k, p in enumerate(parts):
            qa = m.jnt_qposadr[m.names["jnt"].index(p)]
            q[qa : qa + 3] = [cx + rng.uniform(-spread, spread), cy + rng.uniform(-spread, spread), 0.05 + 0.06 * k]
            u = rng.normal(size=4)
            q[qa + 3 : qa + 7] = u / np.linalg.norm(u)
        eqa = np.zeros(m.neq, np.int32)
        eqd = np.asarray(m.eq_data, np.float64).reshape(m.neq, -1).copy()
        if weld_every and t % weld_every == 0 and m.neq:
            e = rng.randint(m.neq)
            b1, b2 = m.names["body"][m.eq_obj1id[e]], m.names["body"][m.eq_obj2id[e]]
            i1, i2 = (m.jnt_qposadr[m.names["jnt"].index(b)] for b in (b1, b2))
            eqd[e, :7] = rel_pose(q[i1 : i1 + 7], q[i2 : i2 + 7])
            eqa[e] = 1
        sim.reset()
        sim.qpos[:] = q; sim.qvel[:] = 0; sim.qacc_warmstart[:] = 0; sim.eq_active[:] = eqa; sim.eq_data[:] = eqd.ravel()
        for s in range(400):
            sim.step()
            if s % 20 != 19:
                continue
            q_, v_, w_ = sim.qpos.copy(), sim.qvel.copy(), sim.qacc_warmstart.copy()
            sim.forward()  # the contacts of this state (after step() they are those of the state before it)
            oc = sim.contacts()
            if _near_activation(m, em, probe, q_, eqa, eqd.ravel(), oc):
                continue
            out.append(dict(qpos=q_, qvel=v_, warm=w_, eq_active=eqa.copy(), eq_data=eqd.ravel().copy(), mpr=_mpr(m, oc), nl=sim.solver_info()["nl"],
                            **classify(m, em, oc, eqa)))
    return m, em, out


# ---------------------------------------------------------------- the coverage table
# sources of states: (model, piles, seed, weld_every, spread, away)
SOURCES = {
    "lack": ("table_lack_0825", 60, 0, 0, 0.05, 0.0),
    "lack_weld": ("table_lack_0825", 20, 1, 2, 0.05, 0.0),
    "lack_away": ("table_lack_0825", 30, 2, 0, 0.05, 0.4),
    "ingolf": ("chair_ingolf_0650", 20, 0, 0, 0.05, 0.0),
    "ingolf2": ("chair_ingolf_0650", 30, 4, 0, 0.05, 0.0),
    "ingolf_away": ("chair_ingolf_0650", 30, 2, 0, 0.05, 0.4),
    "peg": ("three_blocks_peg", 20, 0, 0, 0.05, 0.0),
    "liden_spread": ("table_liden_0921", 4, 0, 0, 0.7, 0.0),  # 12 parts on the floor: more than the 8 units of one pass
}
# row: (source, predicate, states without an MPR contact it needs)
ROWS = {
    "grouped: all parts <= 4 contacts": ("lack", lambda s: s["branch"] == "grouped" and 0 < max(s["nstat"]) <= 4, 3),
    # exactly 5 contacts: the smallest part that needs the second unit
    "grouped: a part with 5-8 contacts": ("peg", lambda s: s["branch"] == "grouped" and 5 in s["nstat"], 3),
    "grouped: two passes": ("liden_spread", lambda s: s["branch"] == "grouped" and s["passes"] >= 2, 3),
    "robot limits only": ("limits", lambda s: s["branch"] == "grouped" and s["nl"] > 0, 3),
    "comp16: nA 9 (robot only)": ("lack", lambda s: s["branch"] == "comp16" and s["nA"] == 9, 3),
    "comp16: nA 12 (parts only)": ("lack", lambda s: s["branch"] == "comp16" and s["nA"] == 12, 3),
    "comp16: nA 15 (robot + 1 part)": ("lack_away", lambda s: s["branch"] == "comp16" and s["nA"] == 15, 3),
    "comp24: nA 18": ("ingolf", lambda s: s["branch"] == "comp24" and s["nA"] == 18, 3),
    "comp24: nA 21": ("lack", lambda s: s["branch"] == "comp24" and s["nA"] == 21, 3),
    "comp24: nA 24 (four parts, no robot)": ("lack_away", lambda s: s["branch"] == "comp24" and s["nA"] == 24 and not s["robot_in"], 3),
    "comp32: nA 27": ("lack", lambda s: s["branch"] == "comp32" and s["nA"] == 27, 3),
    # five coupled parts and no robot with at most 32 contacts: the seeded search finds one such state
    "comp32: nA 30": ("lack_away", lambda s: s["branch"] == "comp32" and s["nA"] == 30, 1),
    "comp32: weld with contacts": ("lack_weld", lambda s: s["branch"] == "comp32" and s["weld"] and s["ncc"] > 0, 3),
    "contact edge: ncc 32 in comp": ("ingolf", lambda s: s["branch"].startswith("comp") and s["ncc"] == 32, 3),
    "contact edge: ncc 33 in coop": ("ingolf_away", lambda s: s["branch"].startswith("coop") and s["ncc"] == 33, 3),
    "coop, register direction": ("ingolf", lambda s: s["branch"] == "coop_regs" and s["nA"] <= 32 and s["ncc"] > 32, 3),
    "coop, Cholesky: nA 33": ("lack", lambda s: s["branch"] == "coop_chol" and s["nA"] == 33, 3),
    "coop, Cholesky: nA 39": ("lack_weld", lambda s: s["branch"] == "coop_chol" and s["nA"] == 39, 3),
    "coop, Cholesky: part with > 8 static contacts": ("ingolf+ingolf2", lambda s: s["branch"] == "coop_chol" and max(s["nstat"]) > 8, 3),
    # the robot block with more than 32 contacts of its own and no coupled part: the free parts are independent blocks of
    # the cooperative solve
    "coop, robot block only": ("floor", lambda s: s["branch"] == "coop_regs" and s["ncpl"] == 0 and s["ncc"] > 32, 3),
}


@functools.lru_cache(maxsize=None)
def limit_states():
    """grouped states of the pile source with both fingers pushed past their stops (range (-0.0115, 0.020833) and
    (-0.020833, 0.0115)): the robot block's only rows are then joint limits"""
    m, em, states = pile_states(*SOURCES["lack"])
    sim = OracleSim(m)
    out = []
    for s in states:
        if s["branch"] != "grouped":
            continue
        q = s["qpos"].copy()
        q[7], q[8] = 0.0212, -0.0211
        sim.qpos[:] = q; sim.qvel[:] = s["qvel"]; sim.qacc_warmstart[:] = s["warm"]
        sim.forward()
        oc = sim.contacts()
        out.append(dict(s, qpos=q, nl=sim.solver_info()["nl"], **classify(m, em, oc, s["eq_active"])))
    return m, em, out


# Sawyer joint angles (7 arm joints, 2 fingers) that press the gripper, wrist and forearm into the floor: 33 contacts, every
# one against the floor and at most 5 cm deep.  Found by a seeded random search over the joint ranges; only forward() and one
# mj_step are run from them, so they need not be reachable.
FLOOR_POSES = [
    [1.0938, -3.7266, -3.5843, 1.1069, -2.5768, 1.134, 1.8143, 0.0024, -0.0089],
    [-1.118, 0.8512, -3.4275, 0.3658, 0.1351, -2.4323, -1.5418, 0.0088, 0.0087],
]


@functools.lru_cache(maxsize=None)
def floor_states():
    """grouped states of the pile source in which every part rests on the floor, with the arm set to each of FLOOR_POSES"""
    m, em, states = pile_states(*SOURCES["lack"])
    sim, probe = OracleSim(m), OracleSim(m)
    probe.set_model("geom_margin", np.asarray(m.a["geom_margin"], np.float64) + NEAR)
    out = []
    for s in states:
        if s["branch"] != "grouped" or min(s["nstat"]) == 0:
            continue
        for arm in FLOOR_POSES:
            q = s["qpos"].copy()
            q[: len(arm)] = arm
            sim.qpos[:] = q; sim.qvel[:] = s["qvel"]; sim.qacc_warmstart[:] = s["warm"]; sim.eq_active[:] = s["eq_active"]; sim.eq_data[:] = s["eq_data"]
            sim.forward()
            oc = sim.contacts()
            if _near_activation(m, em, probe, q, s["eq_active"], s["eq_data"], oc):
                continue
            out.append(dict(s, qpos=q, mpr=_mpr(m, oc), nl=sim.solver_info()["nl"], **classify(m, em, oc, s["eq_active"])))
    return m, em, out


def source(names):
    """the states of one source, or of several joined by '+' (same model)"""
    built = {"limits": limit_states, "floor": floor_states}
    got = [built[n]() if n in built else pile_states(*SOURCES[n]) for n in names.split("+")]
    return got[0][0], got[0][1], [s for g in got for s in g[2]]


def coverage():
    """{row: (model, em, [states])}: the first states of the row without an MPR contact and the first with one"""
    out = {}
    for row, (src, pred, need) in ROWS.items():
        m, em, states = source(src)
        hit = [s for s in states if pred(s)]
        out[row] = (m, em, [s for s in hit if not s["mpr"]][: max(need, 3)] + [s for s in hit if s["mpr"]][:1])
    return out


def test_every_dispatch_branch_is_reached():
    """the seeded states still reach every row of the table (a change to the generator or to the oracle that loses a branch
    fails here, not silently in the parity test)"""
    cov = coverage()
    clean = {row: sum(not s["mpr"] for s in st) for row, (_, _, st) in cov.items()}
    missing = {row: n for row, n in clean.items() if n < ROWS[row][2]}
    assert not missing, missing





def _check_forward(m, em, eng, states, tag):
    """forward() of every state against the oracle: flags, the ordered contact pairs, the constrained acceleration and the
    engine's own optimality residual"""
    n = len(states)
    eng.set("qpos", np.array([s["qpos"] for s in states])); eng.set("qvel", np.array([s["qvel"] for s in states]))
    eng.set("qacc_warmstart", np.array([s["warm"] for s in states]))
    eng.set("eq_active", np.array([s["eq_active"] for s in states])); eng.set("eq_data", np.array([s["eq_data"] for s in states]))
    eng.forward()
    ncon, flags, cg = eng.get("ncon")[:, 0], eng.get("flags")[:, 0], eng.get("con_geom")
    x, fs, fc, Mr, linert = eng.get("dbg_x"), eng.get("dbg_fs"), eng.get("dbg_fc"), eng.get("dbg_Mr"), eng.get("dbg_linert")
    nr = em.nrlink
    sims = []
    for i, s in enumerate(states):
        sim = OracleSim(m)
        sim.qpos[:] = s["qpos"]; sim.qvel[:] = s["qvel"]; sim.qacc_warmstart[:] = s["warm"]
        sim.eq_active[:] = s["eq_active"]; sim.eq_data[:] = s["eq_data"]
        sim.forward()
        sims.append(sim)
        oc = sim.contacts()
        where = (tag, i, s["branch"], s["nA"], s["ncc"])
        assert flags[i] == 0, where
        assert ncon[i] == len(oc), (where, ncon[i], len(oc))
        pairs_e = [tuple(sorted((int(em.geom_src[g & 255]), int(em.geom_src[g >> 8])))) for g in cg[i][: ncon[i]]]
        assert pairs_e == [tuple(sorted((c.geom1, c.geom2))) for c in oc], where
        _, _, xm = oracle_link_poses(sim, em)
        zo = to_z(m, em, xm, sim.qacc)
        if not s["mpr"]:  # MPR contacts: fp32 and fp64 portals differ in the normal (see test_forward_stages_match_oracle)
            assert np.abs(x[i] - zo).max() < 2e-3 * max(1.0, np.abs(zo).max()), (where, np.abs(x[i] - zo).max(), np.abs(zo).max())
        Mx = np.zeros(m.nv)
        Mx[:nr] = Mr[i].reshape(nr, nr).astype(np.float64) @ x[i][:nr]
        for p in range(em.npart):
            I = linert[i].reshape(-1, 10)[nr + p].astype(np.float64)
            mass, h, Io = I[0], I[1:4], np.array([[I[4], I[7], I[8]], [I[7], I[5], I[9]], [I[8], I[9], I[6]]])
            w_, v_ = x[i][nr + 6 * p : nr + 6 * p + 3].astype(np.float64), x[i][nr + 6 * p + 3 : nr + 6 * p + 6].astype(np.float64)
            Mx[nr + 6 * p : nr + 6 * p + 3] = Io @ w_ + np.cross(h, v_)
            Mx[nr + 6 * p + 3 : nr + 6 * p + 6] = mass * v_ - np.cross(h, w_)
        res = Mx - fs[i] - fc[i]
        assert np.abs(res).max() < 2e-4 * max(1.0, np.abs(fs[i]).max(), np.abs(fc[i]).max()), (where, np.abs(res).max())
    return sims


@pytest.mark.parametrize("gpu", BACKENDS)
def test_every_dispatch_branch_matches_oracle(gpu):
    """every row of the coverage table: forward() against the oracle, then one mj_step (qpos to 5e-6, qvel to 2e-3, the bars of
    test_grasped_part_coupled_solve_matches_oracle)"""
    by_model = {}
    for row, (m, em, states) in coverage().items():
        by_model.setdefault(m.meta["furniture_name"] if "furniture_name" in m.meta else id(m), (m, em, []))[2].extend((row, s) for s in states)
    for m, em, rs in by_model.values():
        states = [s for _, s in rs]
        # room for every contact: the arm pressed into the floor next to resting parts has more than the scene's default
        eng = make_engine(m, len(states), gpu, maxcon=max(auto_maxcon(em), max(s["ncon"] for s in states)))
        sims = _check_forward(m, em, eng, states, rs[0][0])
        eng.step(1)
        qe, ve = eng.get("qpos"), eng.get("qvel")
        for i, sim in enumerate(sims):
            sim.step()
            assert (eng.get("flags")[i] == 0).all(), rs[i][0]
            assert np.abs(qe[i] - sim.qpos).max() < 5e-6, (rs[i][0], i, np.abs(qe[i] - sim.qpos).max())
            assert np.abs(ve[i] - sim.qvel).max() < 2e-3 * max(1.0, np.abs(sim.qvel).max()), (rs[i][0], i, np.abs(ve[i] - sim.qvel).max())
        eng.close()


def broad_phase_candidates(m, sim):
    """pairs of the compiled pair list that pass fe_collide's broad phase (contype / conaffinity, bounding spheres, plane
    half-space), from the oracle's geom poses"""
    a = m.a
    ct, ca = np.asarray(a["geom_contype"]), np.asarray(a["geom_conaffinity"])
    rb, mg, gt = np.asarray(a["geom_rbound"]), np.asarray(a["geom_margin"]), np.asarray(a["geom_type"])
    gp, gm = sim.geom_xpos.reshape(-1, 3), sim.geom_xmat.reshape(-1, 3, 3)
    n = 0
    for g1, g2 in np.asarray(a["collision_pairs"]).reshape(-1, 2):
        if not ((ct[g1] & ca[g2]) or (ct[g2] & ca[g1])):
            continue
        t, mm = gp[g2] - gp[g1], max(mg[g1], mg[g2])
        n += bool(t @ gm[g1][:, 2] <= rb[g2] + mm) if gt[g1] == 0 else bool(t @ t <= (rb[g1] + rb[g2] + mm) ** 2)
    return n


@pytest.mark.parametrize("gpu", BACKENDS)
def test_contact_capacity_edges(gpu):
    """maxcon equal to the oracle's contact count: no flag and full parity; one less: FLAG_CONTACT_FULL, ncon == maxcon, and the
    contacts kept are the oracle's first maxcon in order"""
    m, em, states = pile_states(*SOURCES["lack"])
    s = next(s for s in states if s["branch"] == "comp24" and not s["mpr"])
    k = s["ncon"]
    _check_forward(m, em, make_engine(m, 1, gpu, maxcon=k), [s], "maxcon = ncon")
    eng = make_engine(m, 1, gpu, maxcon=k - 1)
    eng.set("qpos", s["qpos"][None]); eng.set("qvel", s["qvel"][None]); eng.set("qacc_warmstart", s["warm"][None])
    eng.forward()
    sim = OracleSim(m)
    sim.qpos[:] = s["qpos"]; sim.qvel[:] = s["qvel"]; sim.forward()
    oc = sim.contacts()
    assert eng.get("flags")[0][0] & FLAG_CONTACT_FULL and eng.get("ncon")[0][0] == k - 1
    kept = [tuple(sorted((int(em.geom_src[g & 255]), int(em.geom_src[g >> 8])))) for g in eng.get("con_geom")[0][: k - 1]]
    assert kept == [tuple(sorted((c.geom1, c.geom2))) for c in oc[: k - 1]]


@pytest.mark.parametrize("gpu", BACKENDS)
def test_broad_phase_keeps_every_candidate(gpu):
    """more than 96 broad-phase candidates (piles of chair_ingolf_0650, whose seat has 17 geoms; bookcase_grevback_0484 at its
    start state has 190): the contact set equals the oracle's and no flag is raised"""
    m, em, states = pile_states(*SOURCES["ingolf"])
    sim = OracleSim(m)
    many = []
    for s in states:
        sim.qpos[:] = s["qpos"]; sim.eq_active[:] = s["eq_active"]
        sim.stage("kinematics")
        if broad_phase_candidates(m, sim) > 96:
            many.append(s)
    assert len(many) >= 3
    _check_forward(m, em, make_engine(m, len(many[:8]), gpu, maxcon=128), many[:8], "ingolf > 96 candidates")
    m = mjcf.load_scene("Sawyer", "bookcase_grevback_0484")
    em = EngineModel(m)
    sim = OracleSim(m)
    q = settled_state(m, 0, robot_noise=0.0, dz=0.0)
    sim.qpos[:] = q; sim.forward()
    assert broad_phase_candidates(m, sim) > 96
    eng = make_engine(m, 1, gpu, maxcon=255)
    eng.set("qpos", q[None])
    eng.forward()
    assert eng.get("flags")[0][0] == 0
    oc = sim.contacts()
    assert eng.get("ncon")[0][0] == len(oc)
    got = [tuple(sorted((int(em.geom_src[g & 255]), int(em.geom_src[g >> 8])))) for g in eng.get("con_geom")[0][: len(oc)]]
    assert got == [tuple(sorted((c.geom1, c.geom2))) for c in oc]
