"""The five torque controllers of arm_controller.py (NEW_CONTROLLERS, SURVEY 8 f2).

Golden: tests/golden/controllers.npz = the reference's own controller classes with the parameters of controller_config.hjson, run on a
stand-in simulator (tools/make_golden_controllers.py), 600 mj_steps per controller (3 episodes x 4 env steps x 50);
tests/golden/controllers_edges.npz = the same classes where the first file never goes: the singular-value cut of update_model_opspace,
the end of the 2000-step goal ramp, Controller.reset() on a controller that lives on.
  * the numpy oracle (oracle/controller_oracle.py) reproduces the torques of both files
  * the device controllers (csrc/fe_ctl.h through fe_ctl_eval) reproduce them on the same records, on the emulated and the CUDA build
  * the env step under a controller (fe_env_ctl_step_kernel): per-substep ctrl against the float64 controller at many states, the
    controller state across auto-resets, and a short trajectory against the CPU env
"""
import os

import numpy as np
import pytest

from oracle.controller_oracle import ArmController

HERE = os.path.dirname(os.path.abspath(__file__))
MODES = ["joint_torque", "joint_velocity", "joint_impedance", "position_orientation", "position"]
CUT = 0.00025  # update_model_opspace's singular-value threshold (arm_controller.py:784-793)


def on_backends(modes):
    """(gpu, mode) parameters: the emulated build under the mode's name, the CUDA build (marked gpu) as cuda-<mode>"""
    return ([pytest.param(False, m, id=m) for m in modes]
            + [pytest.param(True, m, id="cuda-" + m, marks=pytest.mark.gpu) for m in modes])


def _load(name):
    g = np.load(os.path.join(HERE, "golden", name))
    return {m: {k.split("/")[1]: g[k] for k in g.files if k.startswith(m + "/")} for m in MODES}


@pytest.fixture(scope="module")
def golden():
    return _load("controllers.npz")


@pytest.fixture(scope="module")
def edges():
    return _load("controllers_edges.npz")


def _replay(G, mode, renew_every_reset=False):
    """the oracle through the records: a new controller where `renew` (every `reset` in controllers.npz), Controller.reset() where only `reset`"""
    renew = G["reset"] if renew_every_reset or "renew" not in G else G["renew"]
    out = np.zeros_like(G["torques"])
    for t in range(len(G["torques"])):
        if renew[t]:
            c = ArmController(mode)
        elif G["reset"][t]:
            c.reset()
        out[t] = c.torques(G["action"][t], bool(G["policy_step"][t]), G["pos"][t], G["R"][t].reshape(3, 3), G["velp"][t], G["velr"][t], G["q"][t], G["qvel"][t],
                           G["Jx"][t].reshape(3, 7), G["Jr"][t].reshape(3, 7), G["M"][t].reshape(7, 7))
    return out


def _rel_err(tau, want):
    return float((np.abs(tau - want) / np.maximum(1.0, np.abs(want).max(axis=1, keepdims=True))).max())


@pytest.mark.parametrize("mode", MODES)
def test_oracle_reproduces_the_reference_controllers(golden, mode):
    G = golden[mode]
    n = len(G["torques"])
    fast = 0
    for t in range(n):
        if G["reset"][t]:
            c = ArmController(mode)
        fast += np.linalg.norm(G["qvel"][t]) > 7.0
        tau = c.torques(G["action"][t], bool(G["policy_step"][t]), G["pos"][t], G["R"][t].reshape(3, 3), G["velp"][t], G["velr"][t], G["q"][t], G["qvel"][t],
                        G["Jx"][t].reshape(3, 7), G["Jr"][t].reshape(3, 7), G["M"][t].reshape(7, 7))
        assert np.abs(tau - G["torques"][t]).max() <= 1e-13 * max(1.0, np.abs(G["torques"][t]).max()), (mode, t)
    assert n == 600 and int(np.sum(G["policy_step"])) == 12 and int(np.sum(G["reset"])) == 3
    assert fast >= 3  # the joint impedance controller's velocity-norm branch is in the data
    assert np.abs(G["action"]).max() > 1.0  # so is the clipping of transform_action


@pytest.mark.parametrize("mode", MODES)
def test_oracle_reproduces_the_reference_controllers_at_the_edges(edges, mode):
    """the edge records reach what they are made for: eigenvalues of Jx M^-1 Jx^T / Jr M^-1 Jr^T on both sides of the cut (none within 10 %
    of it), a ramp held past its end before the next policy step, and episodes started by Controller.reset() on a living controller"""
    G = edges[mode]
    tau = _replay(G, mode)
    # numpy's inv / svd in place of scipy's, and 1 / s up to 1 / 2.8e-4: a few ulp of the torque scale times that gain
    assert _rel_err(tau, G["torques"]) < 1e-11, (mode, _rel_err(tau, G["torques"]))
    n = len(G["torques"])
    eig = np.array([[np.linalg.eigvalsh(J @ np.linalg.solve(M, J.T)) for J in (G["Jx"][t].reshape(3, 7), G["Jr"][t].reshape(3, 7))]
                    for t, M in enumerate(G["M"].reshape(n, 7, 7))])
    assert (np.abs(eig / CUT - 1.0) > 0.1).all()
    moving = np.ones(n, bool)
    moving[1:] = np.abs(np.diff(G["M"], axis=0)).max(axis=1) > 0  # records with readings of their own (the stand-in holds still in long env steps)
    assert ((eig > 1.2e-4) & (eig < CUT)).any(axis=(1, 2))[moving].sum() >= 40  # dropped values just below the cut
    assert ((eig > CUT) & (eig < 5e-4)).any(axis=(1, 2))[moving].sum() >= 40    # kept values just above it
    starts = np.flatnonzero(G["reset"])
    policy = np.flatnonzero(G["policy_step"])
    assert np.diff(np.append(starts, n)).max() >= 2003 and (np.diff(policy) >= 2001).any()  # the ramp reaches its last step and is held
    assert G["renew"][0] and G["renew"].sum() >= 2 and (G["reset"] & ~G["renew"]).sum() >= 2
    if mode == "position":  # the orientation goal survives Controller.reset(): a new controller per episode gives other torques
        assert _rel_err(_replay(G, mode, renew_every_reset=True), G["torques"]) > 1e-3


def _ctl_eval(eng, mode, G):
    """fe_ctl_eval on the records: one hook episode per controller life, reset byte 1 (new controller) or 2 (Controller.reset())"""
    from furniture_b200.controllers import ctl_config

    n = len(G["torques"])
    renew = G["renew"] if "renew" in G else G["reset"]
    reset = np.where(renew, 1, np.where(G["reset"], 2, 0)).astype(np.uint8)
    readings = np.concatenate([G["pos"], G["R"], G["velp"], G["velr"], G["q"], G["qvel"], G["Jx"], G["Jr"], G["M"]], axis=1)
    act = np.zeros((n, 7))
    act[:, : G["action"].shape[1]] = G["action"]
    starts = np.flatnonzero(renew)
    counts = np.diff(np.append(starts, n))
    return eng.ctl_eval(ctl_config(mode), starts, counts, reset, G["policy_step"], act, readings)


@pytest.mark.parametrize("gpu,mode", on_backends(MODES))
def test_device_controllers_reproduce_the_reference(golden, edges, gpu, mode):
    """csrc/fe_ctl.h (float64, Cholesky + Jacobi in place of scipy.linalg.inv / numpy.linalg.svd) on the golden and the edge records"""
    from furniture_b200 import mjcf
    from parity_util import make_engine

    eng = make_engine(mjcf.load_scene("None", "table_lack_0825"), 1, gpu)
    for name, G in (("controllers", golden[mode]), ("edges", edges[mode])):
        tau = _ctl_eval(eng, mode, G)
        scale = np.maximum(1.0, np.abs(G["torques"]).max(axis=1, keepdims=True))
        err = np.abs(tau - G["torques"])
        assert err.max() / scale.max() < 1e-9 and (err / scale).max() < 1e-9, (name, mode, err.max())


# ------------------------------------------------------------------ the env under a torque controller: device step against the CPU env
@pytest.fixture(scope="module")
def torque_sawyer():
    from furniture_b200 import mjcf

    return mjcf.load_scene("SawyerTorque", "table_lack_0825")


def _ctl_engine(m, n, gpu, mode, **cfg):
    from furniture_b200.controllers import ctl_config
    from furniture_b200.engine import Engine, default_config
    from parity_util import build_emu

    cc = ctl_config(mode, model=m)
    c = default_config(**cfg)
    eng = Engine(m, n, device=0, config=c, controller=cc) if gpu else Engine(m, n, config=c, lib_path=build_emu(), controller=cc)
    assert eng.act_dim == cc.control_dim + 2
    return eng


def _arm_command(a, ctl, move_speed=0.1):
    """the controller's command from an env action: _do_controller_step's scale and axis swap of action[:3] (furniture.py:3069-3071)"""
    arm = np.zeros(7)
    arm[: ctl.control_dim] = a[: ctl.control_dim]
    arm[:3] = arm[:3] * move_speed
    arm[:3] = [-arm[1], arm[0], arm[2]]
    return arm


def _arm_actuators(m):
    """(actuator, arm joint) pairs"""
    names = m.names["jnt"]
    return [(u, m.meta["robot_joints"].index(names[int(m.actuator_jntid[u])])) for u in range(m.nu) if names[int(m.actuator_jntid[u])] in m.meta["robot_joints"]]


# The emulated build's worst over 16 envs x 3 states per mode is 1.6e-6 .. 3.4e-6: the float32 kinematics (hand pose, Jacobian, inertia,
# bias) under float64 controller arithmetic; the CUDA build's on an H100 80GB HBM3 (700 W limit) is 0.8e-6 .. 2.4e-6.  The bound leaves a
# factor 6 above the worst of either.
SUBSTEP_CTRL_TOL = 2e-5


@pytest.mark.parametrize("gpu,mode", on_backends(MODES))
def test_controller_ctrl_matches_the_float64_controller_per_substep(torque_sawyer, gpu, mode):
    """one mj_step per env step, from per-env states written through the C-ABI (arm at robot_init_qpos +- 0.8 rad, joint speeds of
    N(0, 0.3) in half the envs and N(0, 4) in the other half, so that the joint impedance branch above 7 rad/s runs in the same block),
    actions in +-1.3 (clipped): ctrl of every arm actuator = qfrc_bias + torques of a fresh float64 controller fed from the float64
    simulator at the same state (fe_ctl_read's hand Jacobian from the motion subspaces and arm block of the inertia, fe_ctl_torques)"""
    from oracle.ref_env import OracleControllerEnv
    from test_env_parity import _sync_oracle_from_engine

    m, n = torque_sawyer, 16
    eng = _ctl_engine(m, n, gpu, mode, nsub=1)
    eng.env_reset()
    e = OracleControllerEnv(m, mode)
    arm_idx = np.array(e.arm_idx)
    acts = _arm_actuators(m)
    q0 = np.array(m.meta["robot_init_qpos"], dtype=np.float64)
    rng = np.random.RandomState(12)
    worst, fast = 0.0, 0
    for rep in range(3):
        q, v = eng.get("qpos"), np.zeros((n, m.nv), np.float32)
        q[:, arm_idx] = q0 + rng.uniform(-0.8, 0.8, (n, 7))
        v[:, arm_idx] = rng.normal(size=(n, 7)) * np.where(np.arange(n) < n // 2, 0.3, 4.0)[:, None]
        eng.set("qpos", q)
        eng.set("qvel", v)
        eng.set("qacc_warmstart", np.zeros(m.nv))
        eng.set("ctl_state", 0)
        eng.set("episode_length", 0)
        a = rng.uniform(-1.3, 1.3, (n, eng.act_dim)).astype(np.float32)
        a[:, -1] = -1.0
        want = np.zeros((n, len(acts)))
        for i in range(n):
            _sync_oracle_from_engine(e, eng, i)
            e._qvel_fwd = np.array(e.sim.qvel[arm_idx])
            fast += np.linalg.norm(e._qvel_fwd) > 7.0
            ctl = ArmController(mode, timestep=float(m.opt_timestep))
            tau = ctl.torques(_arm_command(a[i].astype(np.float64), ctl), True, *e.readings())
            want[i] = [e.sim.qfrc_bias[arm_idx[k]] + tau[k] for _, k in acts]
        eng.env_step_host(a)
        got = eng.get("ctrl")[:, [u for u, _ in acts]].astype(np.float64)
        err = (np.abs(got - want) / np.maximum(1.0, np.abs(want).max(axis=1, keepdims=True))).max(axis=1)
        worst = max(worst, float(err.max()))
        assert err.max() < SUBSTEP_CTRL_TOL, (mode, rep, err)
    assert fast >= n  # the fast half of the envs passes 7 rad/s in nearly every state
    print("%s worst relative ctrl error %.2e" % (mode, worst))


def _ctl_state(raw):
    """struct FeCtlState (csrc/fe_ctl.h) from its bytes"""
    i = np.frombuffer(raw[:16].tobytes(), np.int32)
    f = np.frombuffer(raw[16:].tobytes(), np.float64)
    out = dict(step=int(i[0]), ori_set=int(i[1]))
    off = 0
    for name, k in (("last", 7), ("start", 7), ("delta", 7), ("last_pos", 3), ("pos_start", 3), ("pos_delta", 3), ("last_ori", 9), ("ori_start", 9),
                    ("ori_delta", 3), ("ori_goal", 9)):
        out[name] = f[off : off + k]
        off += k
    assert off == len(f)
    return out


@pytest.mark.parametrize("gpu,mode", on_backends(["position", "joint_impedance"]))
def test_controller_state_follows_the_controller_across_auto_resets(torque_sawyer, gpu, mode):
    """reset + 5 env steps of 2 mj_steps with max_episode_steps 2 in even and 3 in odd envs, so that envs that start an episode and envs that
    go on share a block: after every step each env's controller state equals the float64 controller that has lived through the same
    episodes (Controller.reset() at each new one, furniture.py:1885-1887), fed at each policy step from the float64 simulator at the
    device's state.  The ramp state after an env step depends on the readings of its first mj_step only; the position controller's
    orientation goal is the one of the first episode, bit for bit"""
    from oracle.ref_env import OracleControllerEnv
    from test_env_parity import _sync_oracle_from_engine

    m, n = torque_sawyer, 8
    eng = _ctl_engine(m, n, gpu, mode, nsub=2, max_episode_steps=2)
    eng.set("max_episode_steps", np.where(np.arange(n) % 2 == 0, 2, 3)[:, None])
    eng.env_reset()
    e = OracleControllerEnv(m, mode)
    arm_idx = np.array(e.arm_idx)
    ctls = [ArmController(mode, timestep=float(m.opt_timestep)) for _ in range(n)]
    rng = np.random.RandomState(21)
    goal0, starts = [None] * n, np.zeros(n, int)
    for k in range(5):
        new = eng.get("episode_length")[:, 0] == 0
        starts += new
        a = rng.uniform(-1.3, 1.3, (n, eng.act_dim)).astype(np.float32)
        a[:, -1] = -1.0
        for i in range(n):
            _sync_oracle_from_engine(e, eng, i)
            e._qvel_fwd = np.array(e.sim.qvel[arm_idx])
            c = ctls[i]
            if new[i]:
                c.reset()
            r = e.readings()
            cmd = _arm_command(a[i].astype(np.float64), c)
            c.torques(cmd, True, *r)
            c.torques(cmd, False, *r)  # the second mj_step only advances the ramp
        obs, rew, done, info = eng.env_step_host(a)
        assert list(done) == [k % 2 == 1 if i % 2 == 0 else k == 2 for i in range(n)], (k, done)
        raw = eng.get("ctl_state")
        for i, c in enumerate(ctls):
            s = _ctl_state(raw[i])
            assert s["step"] == c.step == 2, (k, i)
            if mode == "joint_impedance":  # q and the action reach both exactly: float64 rounding only
                for f in ("last", "start", "delta"):
                    assert np.abs(s[f] - getattr(c, f)).max() <= 1e-12 * max(1.0, np.abs(getattr(c, f)).max()), (k, i, f)
            else:  # the hand pose of the float32 kinematics: the emulated build's worst is 3.6e-7 (pose), 1.8e-10 (ramp increments)
                for f, want in (("last_pos", c.last_pos), ("pos_start", c.pos_start), ("last_ori", c.last_ori.ravel()), ("ori_start", c.ori_start.ravel()),
                                ("ori_goal", c.ori_goal.ravel())):
                    assert np.abs(s[f] - want).max() < 2e-6, (k, i, f, np.abs(s[f] - want).max())
                for f, want in (("pos_delta", c.pos_delta), ("ori_delta", c.ori_delta)):  # differences over the 2000-step ramp
                    assert np.abs(s[f] - want).max() < 2e-9, (k, i, f, np.abs(s[f] - want).max())
                assert s["ori_set"] == 1
                if goal0[i] is None:
                    goal0[i] = s["ori_goal"].copy()
                assert np.array_equal(s["ori_goal"], goal0[i]), (k, i)  # fixed once per controller lifetime, not per episode
    assert (starts == [3, 2] * (n // 2)).all()


@pytest.mark.parametrize("gpu,mode", on_backends(MODES))
def test_controller_env_steps_match_the_cpu_env(torque_sawyer, gpu, mode):
    """reset + 3 env steps (3 x 10 mj_steps, a controller evaluation before each; short, because the torque-actuated arm is barely held
    in the first steps of the reference's 2000-step goal ramp and a falling arm separates the float32 and float64 trajectories quickly)
    on the torque-actuated Sawyer: torques reach the actuators as ctrl = qfrc_bias + torques, observation and reward of the device equal
    the CPU env (oracle physics + oracle controller).  The tolerances are those of the trajectory drift; the arithmetic is held to
    SUBSTEP_CTRL_TOL by the per-substep test above"""
    from oracle.ref_env import OracleControllerEnv
    from test_env_parity import _sync_oracle_from_engine

    m = torque_sawyer
    eng = _ctl_engine(m, 1, gpu, mode, nsub=10)
    eng.env_reset()
    eng.set("qvel", np.zeros(m.nv))  # the reset leaves the motor-driven arm collapsing at several rad/s: start the comparison from rest
    eng.set("qacc_warmstart", np.zeros(m.nv))
    eng.forward()
    e = OracleControllerEnv(m, mode)
    e.nsub = 10
    e.reset()
    _sync_oracle_from_engine(e, eng, 0)
    e.sim.qfrc_applied[: e.nr] = eng.get("qfrc_applied")[0]  # the gravity compensation written at the end of the reset stays in force: _pre_action never renews it
    rng = np.random.RandomState(8)
    for k in range(3):
        a = rng.uniform(-1, 1, (1, eng.act_dim)).astype(np.float32)
        a[0, -1] = -0.5
        obs, rew, done, info = eng.env_step_host(a)
        ob, r, d, inf = e.step(a[0].astype(np.float64))
        tau = np.array(e.torques[-1])
        ctrl = eng.get("ctrl")[0]
        want = e.sim.ctrl
        assert np.abs(ctrl - want).max() < 2e-3 * max(1.0, np.abs(want).max()), (mode, k, ctrl, want)
        assert np.abs(obs[0] - ob).max() < 2e-3, (mode, k, np.abs(obs[0] - ob).max())
        assert abs(rew[0] - r) < 1e-5 and bool(done[0]) == d and info[0][3] == k + 1
        assert np.isfinite(tau).all()
