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
from parity_util import arm_qadr, joint_qadr, make_engine, oracle_link_poses, settled_state, to_z

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]
GEOM_CAPSULE, GEOM_CYLINDER, GEOM_MESH = 3, 5, 7
NEAR = 1e-5  # fp32 and fp64 may disagree on whether a contact this close to its activation distance exists


# ---------------------------------------------------------------- the dispatch rule of fe_solve, restated
def classify(m, em, contacts, eq_active):
    """fe_solve's decision for one constraint set.  Contact kind as in fe_assemble: 0 a free part against the static world,
    1 robot only, 2 robot against a part, 3 part against part; `kinds` per contact, `cpl` per part (in the coupled component)."""
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
    info = dict(nA=nA, ncc=ncc, ncpl=sum(cpl), nstat=nstat, robot_in=robot_in, weld=any(welded), ncon=len(contacts), kinds=kinds, cpl=cpl)
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
# where the piles fall (x, y): under the gripper of each arm at its start pose (Baxter's hands are at x = -0.27 / +0.23,
# y = -0.18, 0.4 m above the floor)
AGENT_PILE_CENTRES = {"Baxter": [(-0.27, -0.18), (0.23, -0.18)]}


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
    """a contact that the narrow phase finds with MPR: a cylinder or a capsule against anything but a plane, or a mesh"""
    types = [(m.geom_type[c.geom1], m.geom_type[c.geom2]) for c in contacts]
    return any((GEOM_CYLINDER in t or GEOM_CAPSULE in t) and 0 not in t or GEOM_MESH in t for t in types)


@functools.lru_cache(maxsize=None)
def pile_states(name, npile, seed, weld_every=0, spread=0.05, away=0.0, agent="Sawyer"):
    """States of `npile` seeded piles of `agent` + `name`: the parts dropped with random orientations over a square of
    half-width `spread` next to the arm (at its start pose +- 0.3 rad; `away` moves the square along y), sampled every 20
    mj_steps.  Sawyer's square is centred on the origin, under its gripper; Baxter's alternates between the points under its
    right and left grippers (AGENT_PILE_CENTRES).  With weld_every = k, every k-th pile runs with one weld active (eq_data =
    the relative pose of its bodies at the drop).  States with a contact within NEAR of its activation distance are dropped."""
    m = mjcf.load_scene(agent, name)
    em = EngineModel(m)
    sim, probe = OracleSim(m), OracleSim(m)
    probe.set_model("geom_margin", np.asarray(m.a["geom_margin"], np.float64) + NEAR)
    rng = np.random.RandomState(seed)
    parts = m.meta["part_names"]
    centres = AGENT_PILE_CENTRES.get(agent, [(0.0, 0.0)])
    out = []
    for t in range(npile):
        q = settled_state(m, seed * 1000 + t, robot_noise=0.3, dz=0.0)
        cx, cy = rng.uniform(-0.1, 0.1, 2) + [0.0, away] + centres[t % len(centres)]
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
# sources of states: (model, piles, seed, weld_every, spread, away[, agent]) -- Sawyer unless an agent is named
SOURCES = {
    "lack": ("table_lack_0825", 60, 0, 0, 0.05, 0.0),
    "lack_weld": ("table_lack_0825", 20, 1, 2, 0.05, 0.0),
    "lack_away": ("table_lack_0825", 30, 2, 0, 0.05, 0.4),
    "ingolf": ("chair_ingolf_0650", 20, 0, 0, 0.05, 0.0),
    "ingolf2": ("chair_ingolf_0650", 30, 4, 0, 0.05, 0.0),
    "ingolf_away": ("chair_ingolf_0650", 30, 2, 0, 0.05, 0.4),
    "peg": ("three_blocks_peg", 20, 0, 0, 0.05, 0.0),
    "liden_spread": ("table_liden_0921", 4, 0, 0, 0.7, 0.0),  # 12 parts on the floor: more than the 8 units of one pass
    # Baxter: 19 robot dofs (head pan, two 7-joint arms, two 2-finger grippers), a branched tree, armature on 15 dofs and a
    # 1 mm contact margin on 25 geoms
    "bx_ingolf": ("chair_ingolf_0650", 30, 0, 0, 0.05, 0.0, "Baxter"),
    "bx_lack": ("table_lack_0825", 30, 0, 0, 0.05, 0.0, "Baxter"),
    # no robot (nr = 0): the parts alone
    "none_lack": ("table_lack_0825", 40, 0, 0, 0.05, 0.0, "None"),
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
    # Baxter's 19-dof robot block: fe_robot_solve_regs<24> (lanes 19-23 padding) in the smooth acceleration, the limit
    # solve and the implicit damping; in the components it straddles the 16-lane boundary of the register factorisations
    "Baxter grouped": ("bx_ingolf", lambda s: s["branch"] == "grouped", 3),
    "Baxter robot limits only": ("bx_limits", lambda s: s["branch"] == "grouped" and s["nl"] >= 6, 3),
    "Baxter comp24: nA 19 (robot only)": ("bx_ingolf", lambda s: s["branch"] == "comp24" and s["nA"] == 19, 3),
    "Baxter comp32: nA 25 (robot + 1 part)": ("bx_lack", lambda s: s["branch"] == "comp32" and s["nA"] == 25, 3),
    "Baxter comp32: nA 31 (robot + 2 parts, one lane padding)": ("bx_ingolf", lambda s: s["branch"] == "comp32" and s["nA"] == 31, 3),
    "Baxter contact edge: ncc 32 in comp": ("bx_ingolf", lambda s: s["branch"].startswith("comp") and s["ncc"] == 32, 3),
    "Baxter contact edge: ncc 33 in coop": ("bx_ingolf", lambda s: s["branch"].startswith("coop") and s["ncc"] == 33, 3),
    # the piles of the chair reach it without planted arm poses: the robot and two parts (19 + 12 dofs) with > 32 contacts
    "Baxter coop, register direction": ("bx_ingolf", lambda s: s["branch"] == "coop_regs" and s["robot_in"] and s["ncpl"] <= 2 and s["ncc"] > 32, 3),
    "Baxter coop, Cholesky: nA 37": ("bx_ingolf", lambda s: s["branch"] == "coop_chol" and s["nA"] == 37, 3),
    # no robot: the nr = 0 skips of fe_kin_smooth, fe_integrate and fe_solve_robot_limits.  The cooperative solver is out of
    # reach here: five coupled parts are 30 dofs, and the piles of the five boxes never have more than 26 coupled contacts
    "no robot: grouped": ("none_lack", lambda s: s["branch"] == "grouped", 3),
    "no robot: comp16 nA 12": ("none_lack", lambda s: s["branch"] == "comp16" and s["nA"] == 12, 3),
    "no robot: comp24 nA 18": ("none_lack", lambda s: s["branch"] == "comp24" and s["nA"] == 18, 3),
    "no robot: comp24 nA 24": ("none_lack", lambda s: s["branch"] == "comp24" and s["nA"] == 24, 3),
    "no robot: comp32 nA 30": ("none_lack", lambda s: s["branch"] == "comp32" and s["nA"] == 30, 3),
}


# arm joints that limit_states pushes past their upper stop, one per arm (Sawyer's arm stays where the pile left it)
LIMIT_ARM_JOINTS = {"Baxter": ["right_w1", "left_w1"]}


@functools.lru_cache(maxsize=None)
def limit_states(src="lack"):
    """grouped states of the pile source `src` with every finger pushed past its stop (range (-0.0115, 0.020833) and
    (-0.020833, 0.0115)) and the joints of LIMIT_ARM_JOINTS 0.01 rad past their upper stop: the robot block's only rows are
    then joint limits"""
    m, em, states = pile_states(*SOURCES[src])
    sim, probe = OracleSim(m), OracleSim(m)
    probe.set_model("geom_margin", np.asarray(m.a["geom_margin"], np.float64) + NEAR)
    _, grip = arm_qadr(m)
    stops = LIMIT_ARM_JOINTS.get(m.meta["agent"], [])
    arm = joint_qadr(m, stops)
    upper = np.array([m.a["jnt_range"][m.names["jnt"].index(j)][1] for j in stops])
    out = []
    for s in states:
        if s["branch"] != "grouped":
            continue
        q = s["qpos"].copy()
        q[grip] = [0.0212, -0.0211] * (len(grip) // 2)
        q[arm] = upper + 0.01
        sim.qpos[:] = q; sim.qvel[:] = s["qvel"]; sim.qacc_warmstart[:] = s["warm"]
        sim.forward()
        oc = sim.contacts()
        if len(stops) and _near_activation(m, em, probe, q, s["eq_active"], s["eq_data"], oc):
            continue  # the moved wrists may bring a new pair to its activation distance
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
    built = {"limits": limit_states, "floor": floor_states, "bx_limits": functools.partial(limit_states, "bx_ingolf")}
    got = [built[n]() if n in built else pile_states(*SOURCES[n]) for n in names.split("+")]
    scene = lambda mm: (mm.meta["agent"], mm.meta["furniture"])
    assert all(scene(g[0]) == scene(got[0][0]) for g in got), names  # every state runs on the first source's model
    return got[0][0], got[0][1], [s for g in got for s in g[2]]


# rows whose first MPR state needs a looser bar than the default (residual 2e-4, qpos after one step 5e-6), with the worst case
# measured.  Both states are MPR contacts of a Baxter arm cylinder (1 mm margin, so the shapes are inflated by 0.5 mm each)
# against a box of the chair.  The MPR normal there is ill-conditioned: the same MPR, run in fp64 and in fp32 on the same fp64
# geom poses, ends on portals 1.05 degrees apart, and without the inflation the fp64 normal itself moves by 4.2 degrees; the
# engine's is 1.9 degrees from the oracle's.  A different but equally valid normal gives a different constrained acceleration.
ROW_BARS = {
    # the robot + two chair parts, 33 contacts: a light part spins up at 5.1e3 rad/s^2, so M x is a difference of terms ~1e3.
    # Residual 2.4e-4 (emu) / 8.4e-5 (cuda, H100); its x agrees with the oracle to 1.2e-6.
    "Baxter contact edge: ncc 33 in coop": dict(res_bar=5e-4),
    "Baxter coop, register direction": dict(res_bar=5e-4),
    # the left wrist cylinder 0.73 mm into a chair part: qacc differs by 58 on |qacc| 388; after one mj_step qpos by 7.8e-5
    # (emu) / 7.7e-5 (cuda, H100) and qvel by 2.5e-3 (emu) / 2.5e-3 (cuda) of its scale
    "Baxter coop, Cholesky: nA 37": dict(qpos_bar=2e-4, qvel_bar=5e-3),
}


def coverage():
    """{row: (model, em, [states])}: the first states of the row without an MPR contact and the first with one"""
    out = {}
    for row, (src, pred, need) in ROWS.items():
        m, em, states = source(src)
        hit = [s for s in states if pred(s)]
        picked = [s for s in hit if not s["mpr"]][: max(need, 3)] + [s for s in hit if s["mpr"]][:1]
        out[row] = (m, em, [dict(s, mpr_bars=ROW_BARS[row]) if s["mpr"] else s for s in picked] if row in ROW_BARS else picked)
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
        assert np.abs(res).max() < s.get("mpr_bars", {}).get("res_bar", 2e-4) * max(1.0, np.abs(fs[i]).max(), np.abs(fc[i]).max()), (where, np.abs(res).max())
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
            assert np.abs(qe[i] - sim.qpos).max() < states[i].get("mpr_bars", {}).get("qpos_bar", 5e-6), (rs[i][0], i, np.abs(qe[i] - sim.qpos).max())
            assert np.abs(ve[i] - sim.qvel).max() < states[i].get("mpr_bars", {}).get("qvel_bar", 2e-3) * max(1.0, np.abs(sim.qvel).max()), (rs[i][0], i, np.abs(ve[i] - sim.qvel).max())
        eng.close()


# ---------------------------------------------------------------- planted pairs: the margin band and the capsule
def _support(m, sim, g, u):
    """point of geom g (sphere, box, cylinder or capsule) furthest along the world direction u, from the oracle's geom pose"""
    c, R = sim.geom_xpos.reshape(-1, 3)[g], sim.geom_xmat.reshape(-1, 3, 3)[g]
    sz, t, l = np.asarray(m.a["geom_size"], np.float64).reshape(-1, 3)[g], m.geom_type[g], R.T @ u
    if t == 2:
        p = l / np.linalg.norm(l) * sz[0]
    elif t == 6:
        p = np.where(l >= 0, sz, -sz)
    elif t == 5:  # perpendicular to the axis: the middle of the side line
        n = np.hypot(l[0], l[1])
        p = np.array([l[0] / n * sz[0], l[1] / n * sz[0], 0.0 if abs(l[2]) < 1e-9 else sz[1] if l[2] >= 0 else -sz[1]])
    else:
        assert t == 3
        p = l / np.linalg.norm(l) * sz[0] + [0, 0, sz[1] if l[2] >= 0 else -sz[1]]
    return c + R @ p


def plant(m, part, geom, other, u, sep, quat):
    """qpos (robot at its start pose, the other parts at their init poses) with `part` turned to `quat` and moved so that its geom
    `geom`'s extreme point along u lies `sep` before `other`'s extreme point along -u: two convex shapes whose extreme points
    face each other across a gap sep along u are exactly sep apart (sep < 0: pressed that far into each other along u)"""
    q = settled_state(m, 0, robot_noise=0.0, dz=0.0)
    qa = m.jnt_qposadr[m.names["jnt"].index(part)]
    q[qa + 3 : qa + 7] = quat
    sim = OracleSim(m)
    sim.qpos[:] = q
    sim.stage("kinematics")
    g, o = m.names["geom"].index(geom), m.names["geom"].index(other)
    if u is None:  # +z made perpendicular to the axis of `other`
        a = sim.geom_xmat.reshape(-1, 3, 3)[o][:, 2]
        u = np.array([0.0, 0.0, 1.0]) - a[2] * a
    u = np.asarray(u, np.float64) / np.linalg.norm(u)
    q[qa : qa + 3] += _support(m, sim, o, -u) - sep * u - _support(m, sim, g, u)
    return q


def _qmul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return [w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2,
            w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2]


_c, _s = np.cos(np.pi / 8), np.sin(np.pi / 8)
R90X, R90Y = [np.sqrt(0.5), np.sqrt(0.5), 0, 0], [np.sqrt(0.5), 0, np.sqrt(0.5), 0]  # the leg's long axis along -y / along x
LEG_X_EDGE = _qmul([_c, _s, 0, 0], R90Y)  # along x, turned 45 degrees about it: a long edge faces +-y and +-z
LEG_Y_EDGE = _qmul([_c, 0, _s, 0], R90X)  # along y, turned 45 degrees about it: a long edge faces +-x and +-z
LEG = ("0_part0", "noviz_collision_0_part0_0")  # a 3 x 3 x 26 cm box leg of table_lack_0825
# (other geom, approach direction u (None: up, perpendicular to the other geom's axis), leg orientation).  Every pair meets at a point on a smooth part of both surfaces, so that
# the contact normal is well defined (on an edge of the Minkowski difference MPR may end on any normal of its cone).  Baxter's
# geoms with a 1 mm margin: a head sphere above the leg's long face (sphere-box, analytic) and the right lower forearm cylinder
# (axis along x) above a long edge of the leg crossing it (MPR on shapes inflated by 0.5 mm each); then the pedestal capsule
# (axis vertical, 1 mm margin) side-on against a long edge of the leg, from -y and from -x.  (A box edge pressed onto the
# capsule's dome is not used: there the fp32 and fp64 MPR normals differ by ~1 degree, which moves qvel by 4e-2 after one
# step on the CUDA build.)
MARGIN_TARGETS = [("collision_head_link_1_geom_2_collision", [0, 0, 1], R90Y), ("right_lower_forearm_collision", None, LEG_Y_EDGE)]
CAPSULE_POSES = [([0, 1, 0], LEG_X_EDGE), ([1, 0, 0], LEG_Y_EDGE)]


def _planted_states(cases):
    m = mjcf.load_scene("Baxter", "table_lack_0825")
    em = EngineModel(m)
    probe = OracleSim(m)
    probe.set_model("geom_margin", np.asarray(m.a["geom_margin"], np.float64) + NEAR)
    out = []
    for other, u, quat, sep in cases:
        q = plant(m, *LEG, other, u, sep, quat)
        sim = OracleSim(m)
        sim.qpos[:] = q
        sim.forward()
        oc = sim.contacts()
        eqa, eqd = np.zeros(m.neq, np.int32), np.asarray(m.eq_data, np.float64).ravel()
        assert not _near_activation(m, em, probe, q, eqa, eqd, oc), (other, sep)  # NEAR away from every activation distance
        g, o = m.names["geom"].index(LEG[1]), m.names["geom"].index(other)
        pair = [c for c in oc if {c.geom1, c.geom2} == {g, o}]
        out.append(dict(qpos=q, qvel=np.zeros(m.nv), warm=np.zeros(m.nv), eq_active=eqa, eq_data=eqd, mpr=_mpr(m, pair), case=(other, sep),
                        pair=(g, o), pair_dist=[c.dist for c in pair], **classify(m, em, oc, eqa)))
    return m, em, out


def _check_planted(m, em, states, gpu):
    """forward() and one mj_step against the oracle (_check_forward and the bars of the dispatch table), and the contact
    geometry at the bars of test_forward_stages_match_oracle: dist 2e-6, pos 5e-6, frame 2e-4 for analytic pairs; dist 1e-4,
    pos 2e-3, normal dot > 0.9 for MPR pairs"""
    eng = make_engine(m, len(states), gpu, maxcon=max(auto_maxcon(em), max(s["ncon"] for s in states)))
    sims = _check_forward(m, em, eng, states, "planted")
    cd, cp, cf, cg = eng.get("con_dist"), eng.get("con_pos"), eng.get("con_frame"), eng.get("con_geom")
    for i, (s, sim) in enumerate(zip(states, sims)):
        for c, o in enumerate(sim.contacts()):
            assert {int(em.geom_src[cg[i][c] & 255]), int(em.geom_src[cg[i][c] >> 8])} == {o.geom1, o.geom2}
            mpr = _mpr(m, [o])
            assert abs(cd[i][c] - o.dist) < (1e-4 if mpr else 2e-6), (s["case"], c, cd[i][c], o.dist)
            assert np.abs(cp[i].reshape(-1, 3)[c] - np.array(list(o.pos))).max() < (2e-3 if mpr else 5e-6), s["case"]
            fe_, fo_ = cf[i].reshape(-1, 9)[c], np.array(list(o.frame))
            assert (fe_[:3] @ fo_[:3] > 0.9) if mpr else (np.abs(fe_ - fo_).max() < 2e-4), s["case"]
    eng.step(1)
    qe, ve = eng.get("qpos"), eng.get("qvel")
    for i, sim in enumerate(sims):
        sim.step()
        assert (eng.get("flags")[i] == 0).all(), states[i]["case"]
        assert np.abs(qe[i] - sim.qpos).max() < 5e-6, (states[i]["case"], np.abs(qe[i] - sim.qpos).max())
        assert np.abs(ve[i] - sim.qvel).max() < 2e-3 * max(1.0, np.abs(sim.qvel).max()), (states[i]["case"], np.abs(ve[i] - sim.qvel).max())
    eng.close()


@pytest.mark.parametrize("gpu", BACKENDS)
def test_margin_band_matches_oracle(gpu):
    """a box leg planted under a Baxter geom with a 1 mm margin: at +0.5 mm the pair is a contact with dist > 0 (its row acts on
    dist - margin), at +1.5 mm it is none, at -0.5 mm it is a contact with dist < 0"""
    cases = [(o, u, qt, sep) for o, u, qt in MARGIN_TARGETS for sep in (5e-4, 1.5e-3, -5e-4)]
    m, em, states = _planted_states(cases)
    for s in states:
        sep = s["case"][1]
        if sep > 1e-3:
            assert s["pair_dist"] == [], s["case"]
        else:
            # analytic pairs find the planted distance; MPR on the inflated shapes overestimates the depth (0.17 mm found at
            # +0.5 mm: the portal stops 1e-6 short on a 0.5 mm rounded edge) but keeps its sign
            ok = (lambda d: d * sep > 0) if s["mpr"] else (lambda d: abs(d - sep) < 1e-5)
            assert len(s["pair_dist"]) >= 1 and all(map(ok, s["pair_dist"])), (s["case"], s["pair_dist"])
    assert sum(s["mpr"] for s in states) == 2  # the wrist cylinder's two contacts (+0.5 and -0.5 mm) are MPR pairs
    _check_planted(m, em, states, gpu)


@pytest.mark.parametrize("gpu", BACKENDS)
def test_capsule_pedestal_matches_oracle(gpu):
    """the box leg against Baxter's pedestal capsule (1 mm margin) side-on in two orientations, 2 mm and 0.2 mm deep and 0.5 mm
    out (inside the margin): MPR with the capsule support, one contact each"""
    cases = [("pedestal_2_collision", u, qt, sep) for u, qt in CAPSULE_POSES for sep in (-2e-3, -2e-4, 5e-4)]
    m, em, states = _planted_states(cases)
    for s in states:
        assert len(s["pair_dist"]) == 1 and s["mpr"], s["case"]
        assert s["pair_dist"][0] * s["case"][1] > 0, (s["case"], s["pair_dist"])
    _check_planted(m, em, states, gpu)


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
