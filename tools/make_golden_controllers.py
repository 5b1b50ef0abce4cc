"""Golden vectors for the five torque controllers of furniture/env/controllers/arm_controller.py (NEW_CONTROLLERS, furniture.py:41-47), made
by running the REFERENCE'S OWN classes, unmodified, with the parameters of controllers/controller_config.hjson (the way
FurnitureEnv._load_controller builds them, furniture.py:1664-1701).  Runs only in the build container.

What runs from the reference: Controller.update_model / update_mass_matrix / transform_action / linear_interpolate /
calculate_orientation_error, and action_to_torques of JointTorqueController, JointVelocityController, JointImpedanceController,
PositionOrientationController, PositionController (+ update_model_opspace, set_goal_position / set_goal_orientation).
The simulator is a stand-in that shows, per mj_step, a hand pose and velocity, joint positions / velocities, the hand Jacobian and the
joint-space inertia (smooth random sequences; physical consistency is irrelevant to the arithmetic being pinned).  mujoco_py is absent:
`mujoco_py.cymj._mj_fullM` is replaced by a function that hands the controller the stand-in's dense inertia matrix.
Layout of the file: for controller c, arrays c/<name> with one row per mj_step; `policy_step` marks the first mj_step of an env step and
`reset` the first of an episode.

A second file, controllers_edges.npz (same layout, its own random stream), holds what the first never reaches:
  * the singular-value cut of update_model_opspace (:784-793): every record's Jx M^-1 Jx^T and Jr M^-1 Jr^T have eigenvalues drawn from
    EIGS, on both sides of 0.00025 and at least 10 % away from it (the 6x6 J M^-1 J^T stays invertible for scipy.linalg.inv)
  * the end of the 2000-step goal ramp: an episode of RAMP_EP records with a policy step at 0 and another at RAMP_SECOND, after the hold
  * Controller.reset() on a controller that lives on (FurnitureEnv._reset between episodes): `renew` marks the records where a new
    controller is built, `reset` those where an episode starts; reset without renew is ctl.reset() on the existing object.
"""
import os
import sys
import types
import zipfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden_assembly import import_reference, rand_rot, small_rot  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
NV, NSUB = 9, 50
JIDX = list(range(7))
EIGS = (1e-6, 1.5e-4, 2.2e-4, 2.8e-4, 4e-4, 1e-2)  # around the singular-value cut 0.00025
RAMP_EP, RAMP_SECOND, NSUB_EDGE = 2020, 2005, 10
FIELDS = ("reset", "policy_step", "action", "pos", "R", "velp", "velr", "q", "qvel", "Jx", "Jr", "M", "torques")


def savez(path, **arrays):
    """np.savez_compressed with a fixed date on every entry, so that a rerun writes the same bytes"""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED, allowZip64=True) as z:
        for k, v in arrays.items():
            zi = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            zi.compress_type = zipfile.ZIP_DEFLATED
            with z.open(zi, "w", force_zip64=True) as f:
                np.lib.format.write_array(f, np.asanyarray(v), allow_pickle=False)


class FakeSim:
    def __init__(self, rng):
        self.rng = rng
        self.model = types.SimpleNamespace(opt=types.SimpleNamespace(timestep=0.002), body_name2id=lambda name: 3)
        A = rng.normal(size=(NV, NV)) * 0.2
        self.M0 = A @ A.T + np.diag(rng.uniform(0.5, 3.0, NV))
        self.pos = rng.uniform(-0.3, 0.3, 3) + [0, 0, 0.4]
        self.R = rand_rot(rng)
        self.q = rng.uniform(-1, 1, NV)
        self.qv = rng.normal(size=NV) * 0.3
        self.J0 = rng.normal(size=(6, NV)) * 0.4
        self.t = 0
        self.data = types.SimpleNamespace(get_body_jacp=lambda name: self.J[:3].ravel().copy(), get_body_jacr=lambda name: self.J[3:].ravel().copy())
        self.advance()

    def advance(self):
        rng, t = self.rng, self.t
        self.pos = self.pos + rng.normal(size=3) * 0.001
        self.R = small_rot(rng, 0.3) @ self.R
        self.q = self.q + self.qv * 0.002
        self.qv = 0.98 * self.qv + rng.normal(size=NV) * 0.05
        if t % 97 == 96:
            self.qv[:7] *= 12.0  # now and then fast enough to pass the 7 rad/s norm test of the joint impedance controller
        self.J = self.J0 + 0.05 * np.sin(0.01 * t + np.arange(6 * NV).reshape(6, NV))
        self.M = self.M0 + 0.05 * np.cos(0.007 * t) * np.eye(NV)
        velp, velr = rng.normal(size=3) * 0.05, rng.normal(size=3) * 0.2
        d = self.data
        d.body_xpos = {3: self.pos.copy()}
        d.body_xmat = {3: self.R.ravel().copy()}
        d.body_xvelp = {3: velp}
        d.body_xvelr = {3: velr}
        d.qpos, d.qvel, d.qM = self.q.copy(), self.qv.copy(), self.M.copy()
        self.t += 1


class EdgeSim(FakeSim):
    """FakeSim whose arm Jacobian puts the eigenvalues of Jx M^-1 Jx^T and Jr M^-1 Jr^T at EIGS: with M = L L^T, J = U diag(sqrt(s)) W^T L^T
    gives J M^-1 J^T = U diag(s) U^T; W (7 x 6, orthonormal columns) splits into the columns of Jx and of Jr, so the 6x6 J M^-1 J^T is
    block-diagonal with the same eigenvalues.  `frozen`: advance() keeps the readings (the hold of a long episode, which compresses)"""

    frozen = False

    def advance(self):
        if self.frozen:
            return
        super().advance()
        rng = self.rng
        L = np.linalg.cholesky(self.M[np.ix_(JIDX, JIDX)])
        W = np.linalg.qr(rng.normal(size=(7, 6)))[0]
        J = self.J.copy()
        for part in range(2):
            s = rng.choice(EIGS, 3, replace=False)
            J[3 * part : 3 * part + 3, JIDX] = rand_rot(rng) @ np.diag(np.sqrt(s)) @ W[:, 3 * part : 3 * part + 3].T @ L.T
        self.J = J


def edge_records(classes, params):
    """controllers_edges.npz: per controller, [new controller: a ramp-end episode, then two episodes after ctl.reset()], [new controller:
    one more episode]"""
    rng = np.random.RandomState(20261017)
    out = {}
    for name, cls in classes.items():
        rec = {k: [] for k in FIELDS + ("renew",)}

        def run(ctl, sim, steps, renew):
            """steps: the records of each env step of one episode; the sim is frozen after the first NSUB_EDGE records of each"""
            for j, count in enumerate(steps):
                a = rng.uniform(-1.3, 1.3, size=ctl.control_dim)
                for i in range(count):
                    sim.frozen = i >= NSUB_EDGE
                    ctl.update_model(sim, id_name="right_hand", joint_index=JIDX)
                    d = sim.data
                    rec["reset"].append(j == 0 and i == 0); rec["renew"].append(renew and j == 0 and i == 0); rec["policy_step"].append(i == 0)
                    rec["action"].append(np.concatenate([a, np.zeros(6 - len(a))]) if len(a) < 7 else a[:7])
                    rec["pos"].append(d.body_xpos[3].copy()); rec["R"].append(d.body_xmat[3].copy()); rec["velp"].append(d.body_xvelp[3].copy())
                    rec["velr"].append(d.body_xvelr[3].copy()); rec["q"].append(d.qpos[JIDX].copy()); rec["qvel"].append(d.qvel[JIDX].copy())
                    rec["Jx"].append(sim.J[:3, JIDX].ravel().copy()); rec["Jr"].append(sim.J[3:, JIDX].ravel().copy())
                    rec["M"].append(sim.M[np.ix_(JIDX, JIDX)].ravel().copy())
                    rec["torques"].append(np.array(ctl.action_to_torques(a.copy(), i == 0), dtype=np.float64))
                    sim.advance()

        ctl = cls(**dict(params[name]))
        ctl.reset()
        run(ctl, EdgeSim(rng), [RAMP_SECOND, RAMP_EP - RAMP_SECOND], True)
        for _ in range(2):
            ctl.reset()  # FurnitureEnv._reset (furniture.py:1885-1887): the same object
            run(ctl, EdgeSim(rng), [NSUB_EDGE, NSUB_EDGE], False)
        ctl = cls(**dict(params[name]))
        ctl.reset()
        run(ctl, EdgeSim(rng), [NSUB_EDGE, NSUB_EDGE], True)
        for k, v in rec.items():
            out["%s/%s" % (name, k)] = np.array(v)
        out["%s/control_dim" % name] = np.array(ctl.control_dim)
        print("edges", name, "records", len(rec["torques"]), "|torque| max", float(np.abs(out[name + "/torques"]).max()))
    return out


def main():
    import_reference()
    import hjson
    import mujoco_py  # the stub module of import_reference()

    def full_m(model, dst, qM):  # mujoco_py.cymj._mj_fullM(model, dst, qM): dense inertia from MuJoCo's sparse qM
        dst[:] = np.asarray(qM).ravel()

    mujoco_py.cymj = types.SimpleNamespace(_mj_fullM=full_m)
    from furniture.env.controllers import arm_controller as AC

    AC.mujoco_py = mujoco_py
    params = hjson.load(open("/root/reference/furniture/env/controllers/controller_config.hjson"))
    classes = {"position": AC.PositionController, "position_orientation": AC.PositionOrientationController, "joint_impedance": AC.JointImpedanceController,
               "joint_torque": AC.JointTorqueController, "joint_velocity": AC.JointVelocityController}
    rng = np.random.RandomState(20260926)
    out = {}
    for name, cls in classes.items():
        rec = {k: [] for k in ("reset", "policy_step", "action", "pos", "R", "velp", "velr", "q", "qvel", "Jx", "Jr", "M", "torques")}
        for ep in range(3):
            ctl = cls(**dict(params[name]))
            ctl.reset()
            sim = FakeSim(rng)
            for step in range(4):
                a = rng.uniform(-1.3, 1.3, size=ctl.control_dim)  # beyond [-1, 1] now and then: transform_action clips
                for i in range(NSUB):
                    ctl.update_model(sim, id_name="right_hand", joint_index=JIDX)
                    d = sim.data
                    rec["reset"].append(step == 0 and i == 0); rec["policy_step"].append(i == 0)
                    rec["action"].append(np.concatenate([a, np.zeros(6 - len(a))]) if len(a) < 7 else a[:7])
                    rec["pos"].append(d.body_xpos[3].copy()); rec["R"].append(d.body_xmat[3].copy()); rec["velp"].append(d.body_xvelp[3].copy())
                    rec["velr"].append(d.body_xvelr[3].copy()); rec["q"].append(d.qpos[JIDX].copy()); rec["qvel"].append(d.qvel[JIDX].copy())
                    rec["Jx"].append(sim.J[:3, JIDX].ravel().copy()); rec["Jr"].append(sim.J[3:, JIDX].ravel().copy())
                    rec["M"].append(sim.M[np.ix_(JIDX, JIDX)].ravel().copy())
                    rec["torques"].append(np.array(ctl.action_to_torques(a.copy(), i == 0), dtype=np.float64))
                    sim.advance()
        for k, v in rec.items():
            out["%s/%s" % (name, k)] = np.array(v)
        out["%s/control_dim" % name] = np.array(ctl.control_dim)
        print(name, "control_dim", ctl.control_dim, "records", len(rec["torques"]), "|torque| max", float(np.abs(out[name + "/torques"]).max()))
    savez(os.path.join(OUT, "controllers.npz"), **out, config_json=np.array(hjson.dumps(params)),
          source="reference furniture/env/controllers/arm_controller.py classes run unmodified on a stand-in simulator (tools/make_golden_controllers.py)")
    savez(os.path.join(OUT, "controllers_edges.npz"), **edge_records(classes, params), config_json=np.array(hjson.dumps(params)),
          source="reference furniture/env/controllers/arm_controller.py classes run unmodified on a stand-in simulator with near-singular "
                 "Jacobians, a ramp run to its end and reused controllers (tools/make_golden_controllers.py)")


if __name__ == "__main__":
    main()
