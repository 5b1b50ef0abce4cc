"""The constraint stage (fe_assemble and the four solvers fe_solve dispatches to) against the fp64 oracle, row by row.

The other parity suites check what goes into this stage (the contact list) and what comes out of it (qacc, one mj_step), at
bars scaled to the largest value of the state.  Here every row the engine assembles is compared with the oracle's row of the
same constraint, each against its own magnitude:
  contacts     aref of the normal and both tangent rows, D of the normal and the friction rows, mu and friction, the solved
               force as a world-frame vector (frame^T f: the two sides' tangent conventions cannot matter) and the cone zone
  welds        the six aref and D of every active weld, and its force
  limits       side, aref, D and force of every joint past its stop (joint -> dof through jnt_dofadr)
  per dof      the constrained acceleration dbg_x and the net constraint force dbg_fc, in solver coordinates, each robot dof
               against its own magnitude and each part's 6-block against its own norm (never against the state's maximum)

Two modes per state:
  own          the oracle's forward pass as it is (states without an MPR contact: the fp32 and fp64 portals may end on
               different normals, see test_solver_branches.ROW_BARS)
  injected     the oracle's kinematics, smooth and collision stages, then its contacts' dist, pos and full frame overwritten
               with the engine's fp32 ones before make_constraint and solve: narrow-phase error is taken out, so MPR, mesh,
               capsule and margin states get the same bars as the rest

`emu` = the lane-emulated build of the kernel source (CPU); `cuda` = the sm_90a library (marked gpu)."""
import copy
import functools

import numpy as np
import pytest

from furniture_b200 import mjcf
from furniture_b200.engine import auto_maxcon
from furniture_b200.engine_model import EngineModel
from oracle.assembly_oracle import rel_pose
from oracle.oracle import OracleSim
from parity_util import make_engine, oracle_link_poses, settled_state, to_z
from test_engine_parity import ARM_SCENES, _pose_arm_over_parts
from test_solver_branches import CAPSULE_POSES, LEG, MARGIN_TARGETS, _mpr, _planted_states, classify, coverage, pile_states, plant

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]
EQ, LIM, CON = 0, 1, 2  # efc_type of the oracle's rows (OM_EFC_*)
GEOM_CAPSULE, GEOM_MESH = 3, 7

# ---------------------------------------------------------------- bars (worst cases measured: DESIGN §5, row a4)
# every error is |engine - oracle| / max(|oracle|, floor), the floor in the quantity's own unit
AREF_FLOOR = 1e-1   # m/s^2 (rad/s^2 for rotational weld rows), under the size of an aref's two terms
FORCE_FLOOR = 1e-2  # N (N m for weld torques), per contact / weld / limit / dof
ACC_FLOOR = 1.0     # m/s^2, rad/s^2, per robot dof and per part 6-block
BARS = {  # at most 4x the worst case measured on either build (emulated / CUDA on an H100 SXM; DESIGN §5)
    "con_aref": 8e-3, "con_D": 2e-3, "con_mu": 3e-7, "con_force": 4e-2,
    "con_fric": 6e-8,  # the fp32 rounding of the geoms' friction (measured 0 on both builds)
    "weld_aref": 2.5e-2, "weld_D": 6e-4, "weld_force": 5e-3,
    "lim_aref": 1.7e-3, "lim_D": 4.8e-4, "lim_force": 2.3e-3,
    "qacc": 9e-3, "fc": 3.4e-2,
}
ZONE_BAND = 1e-4  # a contact whose oracle zone test is within 1e-4 (relative) of a boundary may fall either side in fp32: skipped


# ---------------------------------------------------------------- the two sides
def run_engine(m, em, states, gpu, maxcon=None):
    """forward() of every state on one engine; the dumped rows as numpy arrays"""
    maxcon = maxcon or max(auto_maxcon(em), max(s.get("ncon", 0) for s in states))
    eng = make_engine(m, len(states), gpu, maxcon=maxcon)
    for k in ("qpos", "qvel", "eq_active", "eq_data"):
        eng.set(k, np.array([s[k] for s in states]))
    eng.set("qacc_warmstart", np.array([s["warm"] for s in states]))
    if "ctrl" in states[0]:
        eng.set("ctrl", np.array([s["ctrl"] for s in states]))
    if states[0].get("no_contacts"):
        eng.set("geom_contype", 0); eng.set("geom_conaffinity", 0)
    eng.forward()
    names = ("ncon", "flags", "niter", "con_geom", "con_dist", "con_pos", "con_frame", "con_aref", "con_D", "con_force", "con_state", "con_mu",
             "con_friction", "weld_aref", "weld_D", "weld_force", "limit_sign", "limit_aref", "limit_D", "limit_force", "dbg_x", "dbg_fc", "dbg_fs")
    got = {k: eng.get(k) for k in names}
    return eng, got


def oracle_model(m, s):
    """the model the oracle runs a state on: every contact mask zero for a state without contacts"""
    if not s.get("no_contacts"):
        return m
    m2 = copy.copy(m)
    m2.a = dict(m.a, geom_contype=np.zeros(m.ngeom, np.int32), geom_conaffinity=np.zeros(m.ngeom, np.int32))
    return m2


def oracle_sim(m, s):
    sim = OracleSim(oracle_model(m, s))
    sim.qpos[:] = s["qpos"]; sim.qvel[:] = s["qvel"]; sim.qacc_warmstart[:] = s["warm"]
    sim.eq_active[:] = s["eq_active"]; sim.eq_data[:] = s["eq_data"]
    if "ctrl" in s:
        sim.ctrl[:] = s["ctrl"]
    return sim


def engine_pairs(em, got, i):
    n = int(got["ncon"][i][0])
    return [tuple(sorted((int(em.geom_src[g & 255]), int(em.geom_src[g >> 8])))) for g in got["con_geom"][i][:n]]


def oracle_forward(m, em, s, got, i, inject):
    """the oracle's forward pass of state i; with `inject`, on the engine's contacts (dist, pos, frame)"""
    sim = oracle_sim(m, s)
    if not inject:
        sim.forward()
        assert engine_pairs(em, got, i) == [tuple(sorted((c.geom1, c.geom2))) for c in sim.contacts()]
        return sim
    for st in ("kinematics", "smooth", "collision"):
        sim.stage(st)
    oc = sim.contacts()  # views into the oracle's contact buffer
    assert engine_pairs(em, got, i) == [tuple(sorted((c.geom1, c.geom2))) for c in oc]
    cd, cp, cf = got["con_dist"][i], got["con_pos"][i].reshape(-1, 3), got["con_frame"][i].reshape(-1, 9)
    for c, o in enumerate(oc):
        o.dist = float(cd[c])
        for k in range(3):
            o.pos[k] = float(cp[c][k])
        for k in range(9):
            o.frame[k] = float(cf[c][k])
    sim.stage("make_constraint"); sim.stage("solve")
    return sim


# ---------------------------------------------------------------- the comparison
def _impedance_branch(pos, si):
    """fe_impedance's branch for a row at distance |pos - margin|: 0 x <= mid, 1 mid < x < 1, 2 x >= 1 (x = dist / width)"""
    x = abs(pos) / si[2]
    return 2 if x >= 1 else (0 if x <= si[3] else 1)


def _zone(j, mu, f1, f2):
    """fe_cone_t's zone of jar rows j (0 above the cone, 1 below its dual, 2 on the cone) and the relative distance to the
    nearer zone boundary"""
    N, U1, U2 = j[0] * mu, j[1] * f1, j[2] * f2
    T = np.hypot(U1, U2)
    top, bot = N - mu * T, mu * N + T
    zone = 0 if (N >= mu * T or (T <= 0 and N >= 0)) else (1 if (mu * N + T <= 0 or (T <= 0 and N < 0)) else 2)
    return zone, min(abs(top), abs(bot)) / max(abs(N) + mu * T, 1e-30)


class Record:
    """worst error per category, and what the case set reached"""

    def __init__(self):
        self.worst, self.reached, self.skips, self.contacts = {}, set(), 0, 0

    def err(self, cat, e, where):
        e = float(np.max(e)) if np.size(e) else 0.0
        if e > self.worst.get(cat, (0.0, None))[0]:
            self.worst[cat] = (e, where)
        assert e < BARS[cat], (cat, e, where)


def _rel(a, b, floor):
    return np.abs(np.asarray(a, np.float64) - b) / np.maximum(np.abs(b), floor)


def solver_of(s, kind, coupled):
    """which solver fe_solve hands a contact (kind as in fe_assemble, coupled: its part is in the coupled component) or, with
    kind None, the robot's limit rows"""
    b = s["branch"]
    if b.startswith("coop"):
        return "coop"
    if b == "grouped":
        return "grouped" if kind is not None else "limits"
    if kind is None:
        return "comp" if s["robot_in"] else "limits"
    return "comp" if kind != 0 or coupled else "grouped"


def compare(m, em, s, got, i, sim, rec, where):
    """every row of state i against the oracle's (sim after its forward pass)"""
    nv, nr, nrl = m.nv, em.nrlink, em.nrlink
    etype, eid = sim.efc_type, sim.efc_id
    aref, D, R, force = sim.efc_aref, sim.efc_D, sim.efc_R, sim.efc_force
    J = sim.efc_J.reshape(-1, nv)
    jar = J @ sim.qacc - aref
    # the scale of each aref: the size of its two terms, b |J qvel| + k imp |pos - margin| (they may cancel)
    kbip = sim.efc_KBIP.reshape(-1, 4)
    aref_sc = np.maximum(kbip[:, 1] * np.abs(sim.efc_vel) + kbip[:, 0] * kbip[:, 2] * np.abs(sim.efc_pos - sim.efc_margin), AREF_FLOOR)
    # ---- contacts
    oc = sim.contacts()
    link = lambda g: em.weld_link(int(m.geom_bodyid[g]))
    info = classify(m, em, oc, s["eq_active"])  # fe_solve's dispatch: each contact's kind, each part's coupling
    sr = np.asarray(m.a["geom_solref"], np.float64).reshape(-1, 2)[:, 0]
    ea, eD, ef = got["con_aref"][i].reshape(-1, 3), got["con_D"][i].reshape(-1, 2), got["con_force"][i].reshape(-1, 3)
    emu_, efr, est, eF = got["con_mu"][i], got["con_friction"][i], got["con_state"][i], got["con_frame"][i].reshape(-1, 9)
    for c, o in enumerate(oc):
        a = o.efc_address
        if a < 0:
            continue
        assert etype[a] == CON and o.dim == 3, where
        rec.contacts += 1
        w = (where, "contact", c, (o.geom1, o.geom2))
        Fo, Fe = np.array(list(o.frame)).reshape(3, 3), eF[c].reshape(3, 3).astype(np.float64)
        # aref: normal row, and the tangent rows projected onto the oracle's tangents
        at = Fo[1:] @ (Fe[1:].T @ ea[c][1:])
        rec.err("con_aref", np.abs(np.r_[ea[c][0], at] - aref[a : a + 3]) / aref_sc[a : a + 3], w)
        assert R[a + 2] == R[a + 1], w  # fe_assemble keeps one D for both friction rows
        rec.err("con_D", _rel(eD[c], D[a : a + 2], 0.0), w)
        rec.err("con_mu", _rel(emu_[c], o.mu, 0.0), w)
        rec.err("con_fric", _rel(efr[c], o.friction[0], 0.0), w)
        fw_o, fw_e = Fo.T @ force[a : a + 3], Fe.T @ ef[c]
        rec.err("con_force", np.linalg.norm(fw_e - fw_o) / max(np.linalg.norm(fw_o), FORCE_FLOOR), w)
        zone, gap = _zone(jar[a : a + 3], o.mu, o.friction[0], o.friction[1])
        if gap < ZONE_BAND:
            rec.skips += 1
        else:
            assert est[c] == zone, (w, est[c], zone, gap)
        owner = max(link(o.geom1), link(o.geom2)) - nrl
        if "branch" in s:
            rec.reached.add(("zone", solver_of(s, info["kinds"][c], owner >= 0 and info["cpl"][owner]), zone))
        # fe_assemble's solref: the average of two positive time constants (reached when they differ), clamped to 2 timestep
        t1, t2 = sr[o.geom1], sr[o.geom2]
        if t1 > 0 and t2 > 0 and t1 != t2:
            rec.reached.add(("solref", "mix"))
        if 0 < (0.5 * (t1 + t2) if t1 > 0 and t2 > 0 else min(t1, t2)) < 2 * m.a["opt_timestep"]:
            rec.reached.add(("solref", "refsafe"))
        rec.reached.add(("imp", "contact", _impedance_branch(sim.efc_pos[a] - sim.efc_margin[a], o.solimp)))
        types = {m.geom_type[o.geom1], m.geom_type[o.geom2]}
        if _mpr(m, [o]):
            rec.reached.add(("mpr", s.get("inject", False)))
        if GEOM_MESH in types:
            rec.reached.add(("mesh", s.get("inject", False)))
        if GEOM_CAPSULE in types:
            rec.reached.add(("capsule", s.get("inject", False)))
    # ---- welds: 6 rows per active weld, in weld order
    rows = np.flatnonzero(etype == EQ)
    assert len(rows) == 6 * int(np.sum(s["eq_active"])), where
    wa, wD, wf = got["weld_aref"][i], got["weld_D"][i], got["weld_force"][i]
    for r in rows:
        e, k = int(eid[r]), int(r - rows[0]) % 6
        w = (where, "weld", e, k)
        rec.err("weld_aref", abs(wa[6 * e + k] - aref[r]) / aref_sc[r], w)
        rec.err("weld_D", _rel(wD[6 * e + k], D[r], 0.0), w)
        if s.get("weld_forces", True):
            rec.err("weld_force", _rel(wf[6 * e + k], force[r], FORCE_FLOOR), w)
        if e >= 32:
            rec.reached.add(("weld", ">=32"))
    # ---- joint limits: one row per joint past a stop
    rows = np.flatnonzero(etype == LIM)
    ls, la, lD, lf = got["limit_sign"][i], got["limit_aref"][i], got["limit_D"][i], got["limit_force"][i]
    seen = set()
    for r in rows:
        d = int(m.a["jnt_dofadr"][int(eid[r])])
        seen.add(d)
        w = (where, "limit", d)
        assert ls[d] == J[r, d], (w, ls[d], J[r, d])
        rec.err("lim_aref", abs(la[d] - aref[r]) / aref_sc[r], w)
        rec.err("lim_D", _rel(lD[d], D[r], 0.0), w)
        rec.err("lim_force", _rel(lf[d], force[r], FORCE_FLOOR), w)
        jnt = int(eid[r])
        si = np.asarray(m.a["jnt_solimp"], np.float64).reshape(-1, 5)[jnt]
        rec.reached.add(("imp", "limit", _impedance_branch(sim.efc_pos[r], si)))
        if "branch" in s:
            rec.reached.add(("limit", solver_of(s, None, False)))
    assert all(ls[d] == 0 for d in range(nr) if d not in seen), where
    # ---- per dof: acceleration and net constraint force, in solver coordinates
    _, _, xm = oracle_link_poses(sim, em)
    for cat, e_, o_, floor in (("qacc", got["dbg_x"][i], to_z(m, em, xm, sim.qacc), ACC_FLOOR),
                               ("fc", got["dbg_fc"][i], to_z(m, em, xm, sim.qfrc_constraint), FORCE_FLOOR)):
        sc = np.maximum(np.abs(o_), floor)
        for p in range(em.npart):
            sc[nr + 6 * p : nr + 6 * p + 6] = max(np.linalg.norm(o_[nr + 6 * p : nr + 6 * p + 6]), floor)
        rec.err(cat, np.abs(e_ - o_) / sc, (where, cat, int(np.argmax(np.abs(e_ - o_) / sc))))


def check_states(m, em, states, gpu, tag, modes=("own", "injected"), maxcon=None):
    """forward() of the states on the engine, every row against the oracle in each mode; the Record"""
    rec = Record()
    eng, got = run_engine(m, em, states, gpu, maxcon)
    for i, s in enumerate(states):
        assert got["flags"][i][0] == 0, (tag, i)
        for mode in modes:
            if mode == "own" and s.get("mpr"):
                continue
            inj = mode == "injected"
            sim = oracle_forward(m, em, s, got, i, inj)
            compare(m, em, dict(s, inject=inj), got, i, sim, rec, (tag, i, mode, s.get("row", "")))
    eng.close()
    return rec


# ---------------------------------------------------------------- case sets
def solver_branch_states():
    """every row of test_solver_branches.coverage(), grouped by model: [(m, em, [state])]"""
    by = {}
    for row, (m, em, states) in coverage().items():
        key = (m.meta["agent"], m.meta["furniture"])
        by.setdefault(key, (m, em, []))[2].extend(dict(s, row=row) for s in states)
    return list(by.values())


def forward_stage_states(agent, furn):
    """the states of test_forward_stages_match_oracle (same seeds): parts near their init poses, arms often over them"""
    m = mjcf.load_scene(agent, furn)
    em = EngineModel(m)
    rng = np.random.RandomState(7)
    out = []
    for i in range(16):
        q = settled_state(m, i, robot_noise=0.3, dz=rng.uniform(-0.003, 0.01))
        if i % 2:
            q = _pose_arm_over_parts(m, q, rng)
        v = rng.normal(size=m.nv) * 0.3
        u = rng.uniform(-1.5, 1.5, m.nu)
        if agent == "SawyerTorque":
            u *= m.actuator_ctrlrange[:, 1]
        sim = OracleSim(m)
        sim.qpos[:] = q; sim.forward()
        out.append(dict(qpos=q, qvel=v, warm=np.zeros(m.nv), ctrl=u, eq_active=np.zeros(m.neq, np.int32),
                        eq_data=np.asarray(m.eq_data, np.float64).ravel(), mpr=_mpr(m, sim.contacts()), ncon=sim.ncon))
    return m, em, out


# fe_impedance's three branches (solimp width 1 mm, midpoint 0.5): a box corner, a cylinder against a box, and joints past
# their stops, each 0.3, 0.7 and 1.5 mm deep
DEPTHS = (3e-4, 7e-4, 1.5e-3)


def impedance_states():
    """Baxter + table_lack_0825 (the same scene as the planted margin and capsule states): the leg's corner planted into the
    floor (analytic) and under Baxter's right lower forearm cylinder (MPR), and every limited hinge and slide of the robot past
    one of its stops"""
    m = mjcf.load_scene("Baxter", "table_lack_0825")
    em = EngineModel(m)
    s2 = np.sqrt(0.5)
    corner = [np.cos(0.3), np.sin(0.3) * s2, np.sin(0.3) * s2, 0.0]  # tilted about (1, 1, 0): one corner lowest
    cases = [("floor", [0, 0, 1], corner, -d) for d in DEPTHS] + [("right_lower_forearm_collision", None, MARGIN_TARGETS[1][2], -d) for d in DEPTHS]
    out = []
    floor = next(n for n in m.names["geom"] if m.geom_type[m.names["geom"].index(n)] == 0)
    lim = [m.names["jnt"][j] for j in range(m.a["jnt_type"].__len__()) if m.a["jnt_limited"][j] and m.a["jnt_type"][j] in (2, 3)]
    for other, u, quat, sep in cases:
        other = floor if other == "floor" else other
        if other == floor:  # the leg's lowest corner `sep` into the floor plane, far from the robot
            q = settled_state(m, 0, robot_noise=0.0, dz=0.0)
            qa = m.jnt_qposadr[m.names["jnt"].index(LEG[0])]
            q[qa + 3 : qa + 7] = quat
            sim = OracleSim(m)
            sim.qpos[:] = q; sim.stage("kinematics")
            g = m.names["geom"].index(LEG[1])
            c, R = sim.geom_xpos.reshape(-1, 3)[g], sim.geom_xmat.reshape(-1, 3, 3)[g]
            sz = np.asarray(m.a["geom_size"], np.float64).reshape(-1, 3)[g]
            low = min((c + R @ (sz * np.array(sg)))[2] for sg in np.ndindex(2, 2, 2) for sg in [np.array(sg) * 2 - 1])
            q[qa + 2] += sep - low
        else:
            q = plant(m, *LEG, other, u, sep, quat)
        out.append(q)
    # joints past their stops: every limited joint of the robot by the same depths, lower and upper stops in turn
    rng = np.random.RandomState(3)
    base = settled_state(m, 0, robot_noise=0.0, dz=0.0)
    for k, d in enumerate(DEPTHS):
        q = base.copy()
        for n in lim:
            j = m.names["jnt"].index(n)
            lo, hi = m.a["jnt_range"][j]
            q[m.jnt_qposadr[j]] = (lo - d) if (j + k) % 2 else (hi + d)
        out.append(q)
    states = []
    for q in out:
        sim = OracleSim(m)
        sim.qpos[:] = q; sim.forward()
        states.append(dict(qpos=q, qvel=rng.normal(size=m.nv) * 0.05, warm=np.zeros(m.nv), eq_active=np.zeros(m.neq, np.int32),
                           eq_data=np.asarray(m.eq_data, np.float64).ravel(), mpr=_mpr(m, sim.contacts()), ncon=sim.ncon))
    return m, em, states


def planted_states():
    """the planted pairs of test_margin_band_matches_oracle and test_capsule_pedestal_matches_oracle"""
    cases = [(o, u, qt, sep) for o, u, qt in MARGIN_TARGETS for sep in (5e-4, 1.5e-3, -5e-4)]
    cases += [("pedestal_2_collision", u, qt, sep) for u, qt in CAPSULE_POSES for sep in (-2e-3, -2e-4, 5e-4)]
    return _planted_states(cases)


def mesh_states():
    """the first states with a mesh contact of two seeded piles of chair_bertil_0148 (10 mesh-hull geoms)"""
    m, em, states = pile_states("chair_bertil_0148", 2, 0)
    sim = OracleSim(m)
    out = []
    for s in states:
        sim.qpos[:] = s["qpos"]; sim.forward()
        if any(GEOM_MESH in (m.geom_type[c.geom1], m.geom_type[c.geom2]) for c in sim.contacts()):
            out.append(s)
    return m, em, out[:6]


WELD_MODELS = [("Sawyer", "bookcase_billy_0191"), ("Sawyer", "bookcase_expedit_0376"), ("Baxter", "chair_ingolf_0650"), ("Sawyer", "table_lack_0825")]


def _spanning_tree(m, em):
    """welds of one spanning tree of the weld graph, the highest indices first (so billy_0191's tree has welds >= 32)"""
    root = list(range(em.nlink + 1))

    def find(x):
        while root[x] != x:
            root[x] = root[root[x]]
            x = root[x]
        return x

    on = []
    for e in reversed(range(m.neq)):
        a, b = find(em.weld_link(int(m.eq_obj1id[e])) + 1), find(em.weld_link(int(m.eq_obj2id[e])) + 1)
        if a != b:
            root[a] = b
            on.append(e)
    return sorted(on)


@functools.lru_cache(maxsize=None)
def weld_states(agent, furn):
    """the parts at their start poses lifted 0.5 m clear of the floor, every contact mask zero (welds are the only rows), each
    weld's eq_data the parts' relative pose perturbed by up to 2 mm / 0.02 rad, random qvel.  Two states with every weld on
    (over-constrained: individual weld forces not compared), two with one spanning tree of the weld graph on"""
    m = mjcf.load_scene(agent, furn)
    em = EngineModel(m)
    rng = np.random.RandomState(11)
    tree = _spanning_tree(m, em)
    out = []
    for t in range(4):
        q = settled_state(m, t, robot_noise=0.1, dz=0.5)
        eqd = np.asarray(m.eq_data, np.float64).reshape(m.neq, -1).copy()
        for e in range(m.neq):
            b1, b2 = m.names["body"][m.eq_obj1id[e]], m.names["body"][m.eq_obj2id[e]]
            i1, i2 = (m.jnt_qposadr[m.names["jnt"].index(b)] for b in (b1, b2))
            eqd[e, :7] = rel_pose(q[i1 : i1 + 7], q[i2 : i2 + 7])
            eqd[e, :3] += rng.uniform(-2e-3, 2e-3, 3)
            h = rng.uniform(-0.01, 0.01, 3)  # half-angles: up to 0.02 rad about each axis
            dq = np.r_[np.sqrt(1 - h @ h), h]
            w1, x1, y1, z1 = eqd[e, 3:7]
            w2, x2, y2, z2 = dq
            eqd[e, 3:7] = [w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                           w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2]
        eqa = np.ones(m.neq, np.int32)
        if t >= 2:
            eqa[:] = 0
            eqa[tree] = 1
        out.append(dict(qpos=q, qvel=rng.normal(size=m.nv) * 0.1, warm=np.zeros(m.nv), eq_active=eqa, eq_data=eqd.ravel(), mpr=False,
                        no_contacts=True, weld_forces=t >= 2, ncon=0))
    return m, em, out, tree


# ---------------------------------------------------------------- tests
def _merge(recs):
    rec = Record()
    for r in recs:
        for k, v in r.worst.items():
            if v[0] >= rec.worst.get(k, (0.0,))[0]:
                rec.worst[k] = v
        rec.reached |= r.reached; rec.skips += r.skips; rec.contacts += r.contacts
    return rec


@functools.lru_cache(maxsize=None)
def branch_rows(gpu):
    return _merge(check_states(m, em, states, gpu, m.meta["agent"] + "/" + m.meta["furniture"]) for m, em, states in solver_branch_states())


@functools.lru_cache(maxsize=None)
def forward_rows(agent, furn, gpu):
    m, em, states = forward_stage_states(agent, furn)
    return check_states(m, em, states, gpu, agent)


@functools.lru_cache(maxsize=None)
def planted_rows(gpu):
    m, em, states = planted_states()
    r1 = check_states(m, em, states, gpu, "planted")
    m, em, states = impedance_states()
    r2 = check_states(m, em, states, gpu, "impedance")
    m, em, states = mesh_states()
    assert len(states) >= 3
    return _merge([r1, r2, check_states(m, em, states, gpu, "mesh")])


@functools.lru_cache(maxsize=None)
def weld_rows(agent, furn, gpu):
    m, em, states, _ = weld_states(agent, furn)
    return check_states(m, em, states, gpu, furn, modes=("own",))


@pytest.mark.parametrize("gpu", BACKENDS)
def test_rows_of_every_solver_branch(gpu):
    """every row of the solver-branch coverage table, in both modes: the forces of all four solvers"""
    rec = branch_rows(gpu)
    assert rec.skips <= 0.01 * rec.contacts, (rec.skips, rec.contacts)


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("agent,furn", ARM_SCENES)
def test_rows_of_forward_stage_states(agent, furn, gpu):
    """the states of test_forward_stages_match_oracle (with their controls)"""
    rec = forward_rows(agent, furn, gpu)
    assert rec.skips <= 0.01 * rec.contacts, (rec.skips, rec.contacts)


@pytest.mark.parametrize("gpu", BACKENDS)
def test_rows_of_planted_pairs(gpu):
    """the margin-band and capsule states, the three branches of fe_impedance for contacts (a box corner on the floor,
    analytic; the box under a cylinder, MPR) and for joint limits, and mesh-hull contacts"""
    rec = planted_rows(gpu)
    assert rec.skips <= 0.01 * rec.contacts, (rec.skips, rec.contacts)


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("agent,furn", WELD_MODELS)
def test_rows_of_welds(agent, furn, gpu):
    """every weld of the model on (the lane-strided weld loops' second pass: billy_0191 has 37), and one spanning tree of the
    weld graph on; the constraint set is welds only on both sides.  Then one mj_step of every state.

    Both sides integrate mj_Euler's (M + h D) a = qfrc_smooth + qfrc_constraint, not the solved qacc.  With every weld on, the
    weld forces reach 8e3 N and net to 3-30 N per part, so the fp32 J^T f carries a cancellation error of up to 5e-3 N (6e-7
    of the forces, within the dbg_fc bar), and a part whose smallest principal inertia is 5e-7 kg m^2 (h D = 2e-7 beside it)
    turns that into 0.33 rad/s in one step.  The step is therefore held to what its own constraint force explains: the
    velocity change minus h (M + h D)^-1 (fc_engine - fc_oracle + fs_engine - fs_oracle), from the same state's forward pass,
    per dof.  The spanning-tree states, where the forces are well-posed, are also held to the plain bars."""
    m, em, states, tree = weld_states(agent, furn)
    weld_rows(agent, furn, gpu)
    eng, got = run_engine(m, em, states, gpu)
    eng.step(1)
    qe, ve = eng.get("qpos"), eng.get("qvel")
    h, nr = float(m.a["opt_timestep"]), em.nrlink
    for i, s in enumerate(states):
        sim = oracle_sim(m, s)
        sim.forward()
        _, _, xm = oracle_link_poses(sim, em)

        def to_qvel(z):  # solver coordinates [torque world; force] -> MuJoCo's dof order (force; torque in the body frame)
            q = np.array(z, np.float64)
            for p in range(em.npart):
                R, da = xm[nr + p].reshape(3, 3), nr + 6 * p
                q[da : da + 3], q[da + 3 : da + 6] = z[da + 3 : da + 6], R.T @ z[da : da + 3]
            return q

        dfc = got["dbg_fc"][i] - to_z(m, em, xm, sim.qfrc_constraint)
        dfs = got["dbg_fs"][i] - to_z(m, em, xm, sim.qfrc_smooth)
        A = sim.qM.reshape(m.nv, m.nv) + h * np.diag(np.asarray(m.a["dof_damping"], np.float64))
        explained = h * np.linalg.solve(A, to_qvel(dfc + dfs))
        sim.step()
        assert (eng.get("flags")[i] == 0).all(), (furn, i)
        gap = ve[i] - sim.qvel
        # what the step adds beyond its force error: worst 2.2e-6 (emu) / 2.9e-6 (cuda) m/s on gaps up to 0.56 rad/s
        assert np.abs(gap - explained).max() < 8e-6, (furn, i, np.abs(gap - explained).max(), np.abs(gap).max())
        # qpos: within h times the largest velocity gap (a quaternion moves by at most h/2 of it), plus 5e-6
        qbar = 5e-6 + h * np.abs(gap).max()
        assert np.abs(qe[i] - sim.qpos).max() < qbar, (furn, i, np.abs(qe[i] - sim.qpos).max(), qbar)
        if s["weld_forces"]:
            assert np.abs(qe[i] - sim.qpos).max() < 5e-6, (furn, i, np.abs(qe[i] - sim.qpos).max())  # worst 7.5e-7 (emu)
            # each qvel against its own magnitude, floor 1e-2 m/s (rad/s): worst 2.4e-3 (emu)
            assert (np.abs(gap) / np.maximum(np.abs(sim.qvel), 1e-2)).max() < 1e-2, (furn, i)
    eng.close()


def test_every_row_category_is_reached():
    """the case sets reach, on the emulated build: all three cone zones under the grouped, coupled-component and cooperative
    solvers; joint-limit rows under the robot-limits, component and cooperative solvers; all three branches of fe_impedance for
    contacts and for limits; an active weld with index >= 32; MPR, mesh and capsule contacts with the engine's contacts
    injected; a contact whose solref is the average of two different time constants, and one clamped to 2 timestep
    (refsafe: two part geoms of table_lack_0825 with 1 ms each)"""
    rec = _merge([branch_rows(False), planted_rows(False)] + [forward_rows(a, f, False) for a, f in (p.values for p in ARM_SCENES)]
                 + [weld_rows(a, f, False) for a, f in WELD_MODELS])
    want = {("zone", sv, z) for sv in ("grouped", "comp", "coop") for z in range(3)}
    want |= {("limit", sv) for sv in ("limits", "comp", "coop")}
    want |= {("imp", kind, b) for kind in ("contact", "limit") for b in range(3)}
    want |= {("weld", ">=32"), ("mpr", True), ("mesh", True), ("capsule", True), ("solref", "mix"), ("solref", "refsafe")}
    assert not want - rec.reached, sorted(want - rec.reached)
