"""control_freq and no_collision (config/furniture.py) per env inside the step and reset kernels.

The substep count is pinned to the reference's own _do_simulation loop bound by tests/golden/sim_options.npz
(tools/make_golden_sim_options.py).  The device, lane-emulated ([emu]) and on the GPU ([cuda]), is held to the CPU env oracle at the
bars of tests/test_env_parity.py, and a handle whose envs mix frequencies or no_collision is held bit for bit to handles that run
one value for all their envs.
"""
import os

import numpy as np
import pytest

from furniture_b200 import mjcf
from furniture_b200.engine import substep_count
from furniture_b200.env import build_engine, split_config
from parity_util import build_emu, make_engine
from test_env_parity import _sync_oracle_from_engine

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]
HERE = os.path.dirname(os.path.abspath(__file__))
TAG_FLOOR, TAG_ROBOT, TAG_PART_SHIFT = 1, 8, 8


def _engine(gpu, agent="Sawyer", n=4, **kw):
    return build_engine(agent, "table_lack_0825", n, **kw) if gpu else build_engine(agent, "table_lack_0825", n, lib_path=build_emu(), **kw)


def _rollout(eng, steps, seed=7):
    """reset + `steps` env steps with random actions; every output and the state after each call"""
    eng.env_reset()
    out = [(eng.get("obs"), eng.get("qpos"))]
    rng = np.random.RandomState(seed)
    for _ in range(steps):
        a = rng.uniform(-1, 1, (eng.N, eng.act_dim)).astype(np.float32)
        out.append(eng.env_step_host(a))
        out.append((eng.get("qpos"), eng.get("qvel"), eng.get("geom_contype")))
    return out


def _rows(out, i):
    """env i's rows of a _rollout"""
    return [tuple(None if x is None else np.asarray(x)[i] for x in (o if isinstance(o, tuple) else (o,))) for o in out]


def _same(a, b):
    return all(x is None and y is None or np.array_equal(x, y) for ra, rb in zip(a, b) for x, y in zip(ra, rb))


def _agent_geoms(eng):
    fm = eng.em.fm
    return np.array([not (t & TAG_FLOOR) and ((t >> TAG_PART_SHIFT) & 0x3FFFFF) == 0 for t in list(fm.geom_tag)[: fm.ngeom]])


# ------------------------------------------------------------------ substep counts
def test_substep_count_is_the_reference_loop_bound():
    g = np.load(os.path.join(HERE, "golden", "sim_options.npz"))
    timesteps = {float(mjcf.load_scene(a, f).opt_timestep) for a, f in (("Sawyer", "table_lack_0825"), ("Baxter", "table_lack_0825"),
                                                                          ("SawyerTorque", "table_lack_0825"), ("Sawyer", "swivel_chair_0700"))}
    assert timesteps <= set(g["timesteps"].tolist())
    for dt, row in zip(g["timesteps"], g["substeps"]):
        assert np.array_equal(substep_count(g["control_freq"], dt), row)
    assert substep_count(10, 0.002) == 50 and int((1.0 / 10) / float(np.float32(0.002))) == 49  # why the count is taken in float64


def test_refusals():
    with pytest.raises(ValueError):
        substep_count(501, 0.002)
    with pytest.raises(ValueError):
        substep_count(0, 0.002)
    with pytest.raises(ValueError):
        _engine(False, n=1, control_freq=20, nsub=10)
    with pytest.raises(ValueError):
        build_engine("Cursor", "toy_table", 1, lib_path=build_emu(), no_collision=True)
    with pytest.raises(ValueError):
        build_engine("Cursor", "toy_table", 1, lib_path=build_emu(), control_freq=20)
    eng = _engine(False, n=2)
    with pytest.raises(ValueError):
        eng.set_sim_options(control_freq=1000)
    with pytest.raises(RuntimeError):
        eng.set("substeps", 0)
    with pytest.raises(RuntimeError):
        eng.set("no_collision", 2)
    from furniture_b200.cursor_env import FurnitureCursorEnvB200

    with pytest.raises(ValueError):
        FurnitureCursorEnvB200(lib_path=build_emu(), no_collision=True)


def test_config_surface():
    name, over, ignored = split_config(dict(control_freq=20, no_collision=True, furniture_name="table_lack_0825"))
    assert over["control_freq"] == 20 and over["no_collision"] is True
    assert "control_freq" not in ignored and "no_collision" not in ignored
    _, over, ignored = split_config(dict(control_freq=10, no_collision=False))
    assert "control_freq" not in over and "no_collision" not in over and "control_freq" not in ignored
    eng = _engine(False, n=3, control_freq=[10, 20, 5], no_collision=[False, True, False])
    assert eng.get("substeps")[:, 0].tolist() == [50, 25, 100] and eng.get("no_collision")[:, 0].tolist() == [0, 1, 0]
    eng.set_sim_options(control_freq=4, envs=[1])
    assert eng.get("substeps")[:, 0].tolist() == [50, 125, 100]
    eng = _engine(False, n=2, control_freq=20)
    assert eng.cfg.nsub == 50 and eng.get("substeps")[:, 0].tolist() == [25, 25]  # FeConfig.nsub keeps its default; the envs run 25


@pytest.mark.gpu
def test_env_surfaces_take_both_keys():
    from furniture_b200.env import MixedFurnitureEnv, make_vec_env
    from furniture_b200.gym_api import FurnitureGymB200

    env = make_vec_env("IKEASawyer-v0", 2, dict(control_freq=20, no_collision=True))
    assert env.engine.get("substeps")[:, 0].tolist() == [25, 25] and env.engine.get("no_collision")[:, 0].tolist() == [1, 1]
    env.set_sim_options(control_freq=5, envs=[0])
    assert env.engine.get("substeps")[:, 0].tolist() == [100, 25]
    env.close()
    g = FurnitureGymB200("FurnitureSawyerEnv", control_freq=5)
    assert g.engine.get("substeps")[0, 0] == 100 and "control_freq" not in g.ignored_config
    g.set_sim_options(no_collision=True)
    assert g.engine.get("no_collision")[0, 0] == 1
    g.close()
    mix = MixedFurnitureEnv(["table_lack_0825", "chair_ingolf_0650"], 2, control_freq=20)
    mix.set_sim_options(control_freq=[5, 10], envs=[1, 2])
    assert [b.engine.get("substeps")[:, 0].tolist() for b in mix.buckets] == [[25, 100], [50, 25]]
    mix.close()


# ------------------------------------------------------------------ device vs the CPU env oracle
CASES = [("sparse", 20, False), ("sparse", 5, False), ("dense", 20, False), ("dense", 5, False), ("ik", 20, False), ("ik", 5, False),
         ("baxter", 20, False), ("sparse", 10, True)]


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("kind,control_freq,no_collision", CASES, ids=["%s-%dHz%s" % (k, f, "-no_collision" if c else "") for k, f, c in CASES])
def test_env_step_matches_cpu_env(sawyer_model, gpu, kind, control_freq, no_collision):
    """reset + 3 env steps at control_freq (25 / 100 mj_steps; the IK step runs them once per closed-loop repeat) or with the agent's
    collisions off: obs / reward / done of the device env equal the CPU env (nsub set to match, the agent's masks copied from the device)
    started from the same post-reset state, at the bars of tests/test_env_parity.py and, for the dense reward, tests/test_dense_reward.py"""
    from test_dense_reward import _adopt_device_anchors, _dense_state
    from test_obs_layout import _engine as layout_engine, _oracle, _sync_ik

    m = mjcf.load_scene("Baxter", "table_lack_0825") if kind == "baxter" else sawyer_model
    n = 2
    eng = layout_engine(m, n, gpu, dense=kind == "dense", ik=kind == "ik")
    eng.set_sim_options(control_freq=control_freq, no_collision=no_collision)
    eng.env_reset()
    agent = _agent_geoms(eng)
    if no_collision:
        assert (eng.get("geom_contype")[:, agent] == 0).all() and (eng.get("geom_conaffinity")[:, agent] == 0).all()
    envs = [_oracle(m, kind, {}) for _ in range(n)]
    for i, e in enumerate(envs):
        e.reset()
        e.nsub = int(substep_count(control_freq, m.opt_timestep))
        _sync_oracle_from_engine(e, eng, i)
        e.sim.qfrc_bias[: e.nr] = eng.get("qfrc_bias")[i]
        if kind == "dense":
            e.dense.begin_episode()
            _adopt_device_anchors(e.dense, _dense_state(eng, i))
        if kind == "ik":
            _sync_ik(e, eng, i)
    rng = np.random.RandomState(5)
    for k in range(3):
        a = rng.uniform(-1, 1, (n, eng.act_dim)).astype(np.float32)
        a[:, -1] = -0.5
        obs, rew, done, info = eng.env_step_host(a)
        for i, e in enumerate(envs):
            ob, r, d, _ = e.step(a[i].astype(np.float64))
            assert np.abs(obs[i] - ob).max() < 2e-4, (k, i, np.abs(obs[i] - ob).max())
            assert abs(rew[i] - r) < (2e-2 + 1e-5 * abs(r) if kind == "dense" else 1e-5) and bool(done[i]) == d, (k, i, rew[i], r)
    if no_collision:
        assert (eng.get("geom_contype")[:, agent] == 0).all()


# ------------------------------------------------------------------ one handle, mixed values
@pytest.mark.parametrize("gpu,control_type", [pytest.param(g, c, id="%s-%s" % ("cuda" if g else "emu", c), marks=[pytest.mark.gpu] if g else [])
                                                for g in (False, True) for c in ("impedance", "ik", "position")])
def test_mixed_frequencies_equal_uniform_handles(gpu, control_type):
    """envs at 10 / 20 / 5 / 10 Hz in one handle equal, bit for bit, the same envs of handles that run one frequency for all their envs,
    over reset + 5 steps with an auto-reset (max_episode_steps 3).  On the GPU the first step runs on the initial packing, envs 16 b ..
    16 b + 15 in block b, so every block of 16 holds all three counts; the packing of the later steps follows the predicted work."""
    if gpu:
        n = 64
    else:
        n = 4 if control_type == "impedance" else 2
    pattern = np.resize([10, 20, 5, 10], n)
    kw = dict(control_type=control_type, max_episode_steps=3)
    mixed = _rollout(_engine(gpu, n=n, control_freq=pattern, **kw), 5)
    for f in sorted(set(pattern.tolist())):
        ref = _rollout(_engine(gpu, n=n, control_freq=f, **kw), 5)
        for i in np.flatnonzero(pattern == f):
            assert _same(_rows(mixed, i), _rows(ref, i)), (control_type, f, i)


@pytest.mark.parametrize("gpu", BACKENDS)
def test_mixed_no_collision_equals_uniform_handles(gpu):
    n = 64 if gpu else 4
    flags = np.arange(n) % 2 == 1
    mixed = _rollout(_engine(gpu, n=n, no_collision=flags, max_episode_steps=3), 5)
    for f in (False, True):
        ref = _rollout(_engine(gpu, n=n, no_collision=f, max_episode_steps=3), 5)
        for i in np.flatnonzero(flags == f):
            assert _same(_rows(mixed, i), _rows(ref, i)), (f, i)


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("how", ["keywords", "set_sim_options"])
def test_defaults_change_nothing(gpu, how):
    n = 32 if gpu else 2
    plain = _rollout(_engine(gpu, n=n, max_episode_steps=3), 5)
    if how == "keywords":
        eng = _engine(gpu, n=n, max_episode_steps=3, control_freq=10, no_collision=False)
    else:
        eng = _engine(gpu, n=n, max_episode_steps=3)
        eng.set_sim_options(control_freq=10, no_collision=False)
    same = _rollout(eng, 5)
    assert all(_same(_rows(plain, i), _rows(same, i)) for i in range(n))


# ------------------------------------------------------------------ no_collision
@pytest.mark.parametrize("gpu", BACKENDS)
def test_no_collision_gripper_passes_through_a_part(sawyer_model, gpu):
    """a table leg planted on the gripper's fingers: with the agent's collisions on the fingers touch it; with no_collision no contact of
    the agent appears, and the steps give no touch or pick reward"""
    m = sawyer_model
    results = {}
    for off in (False, True):
        eng = make_engine(m, 1, gpu)
        eng.set_sim_options(no_collision=off)
        eng.env_reset()
        q = eng.get("qpos")
        fm = eng.em.fm
        finger = next(g for g in range(fm.ngeom) if fm.geom_tag[g] & 2)  # FE_TAG_LFINGER
        eng.forward()
        q[0, 9:12] = eng.get("link_xpos").reshape(-1, 3)[fm.geom_link[finger]]  # leg 0 onto the left finger's link
        eng.set_state(q, eng.get("qvel"))
        eng.forward()
        agent = _agent_geoms(eng)
        ncon = int(eng.get("ncon")[0, 0])
        cg = eng.get("con_geom")[0][:ncon]
        g1, g2 = cg & 0xFF, (cg >> 8) & 0xFF
        results[off] = bool(np.any(agent[g1] | agent[g2]))
        rews = []
        for _ in range(3):
            a = np.zeros((1, eng.act_dim), np.float32)
            a[:, -1] = -1
            _, rew, _, _ = eng.env_step_host(a)
            rews.append(float(rew[0]))
        if off:
            assert (eng.get("touched") == 0).all() and (eng.get("picked") == 0).all()
            assert all(r <= 0 for r in rews), rews  # only the control penalty: no touch or pick reward
    assert results[False] and not results[True], results


@pytest.mark.parametrize("gpu", BACKENDS)
def test_no_collision_off_restores_the_model_masks(sawyer_model, gpu):
    m = sawyer_model
    eng = make_engine(m, 2, gpu)
    fm = eng.em.fm
    ct0, ca0 = np.array(list(fm.geom_contype0)[: fm.ngeom]), np.array(list(fm.geom_conaffinity0)[: fm.ngeom])
    agent = _agent_geoms(eng)
    assert (agent & ((ct0 != 0) | (ca0 != 0))).sum() > 0
    eng.set_sim_options(no_collision=True, envs=[1])
    assert (eng.get("geom_contype")[1, agent] == 0).all() and np.array_equal(eng.get("geom_contype")[0], ct0)
    eng.env_reset()  # the reset saves the zeros of env 1
    eng.env_step_host(np.zeros((2, eng.act_dim), np.float32))
    assert (eng.get("geom_contype")[1, agent] == 0).all() and (eng.get("geom_conaffinity")[1, agent] == 0).all()
    eng.set_sim_options(no_collision=False, envs=[1])
    assert np.array_equal(eng.get("geom_contype")[1, agent], ct0[agent]) and np.array_equal(eng.get("geom_conaffinity")[1, agent], ca0[agent])
    eng.env_reset()
    c0, c1 = eng.get("geom_contype"), eng.get("geom_conaffinity")
    assert np.array_equal(c0[1], c0[0]) and np.array_equal(c1[1], c1[0])


@pytest.mark.parametrize("agent", ["Sawyer", "SawyerTorque", "Baxter"])
def test_agent_geoms_are_the_robots_worldbody(agent):
    """no_collision's geoms are every colliding geom of the robot's bodies (under mujoco_robot.worldbody, grippers included): neither a
    part's nor the floor's.  FE_TAG_ROBOT, what the reset switches off, is a subset."""
    m = mjcf.load_scene(agent, "table_lack_0825")
    from furniture_b200.engine_model import EngineModel

    em = EngineModel(m)
    fm = em.fm
    names = m.names["geom"]
    kept = [g for g in range(m.ngeom) if m.geom_contype[g] != 0 or m.geom_conaffinity[g] != 0 or "collision" in names[g]]
    parts = set(m.meta["part_names"])
    robot = {names[g] for g in kept if m.names["body"][m.geom_bodyid[g]] not in parts and m.geom_bodyid[g] != 0}
    tags = list(fm.geom_tag)[: fm.ngeom]
    agent_set = {names[g] for g, t in zip(kept, tags) if not (t & TAG_FLOOR) and ((t >> TAG_PART_SHIFT) & 0x3FFFFF) == 0}
    assert agent_set == robot
    assert {names[g] for g, t in zip(kept, tags) if t & TAG_ROBOT} <= agent_set
