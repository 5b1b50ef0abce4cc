"""Episodes that start from recorded states: set_init_qpos / --load_init_states / --load_demo (furniture.py:121-130, :315-316, :1433-1434,
:1505-1518, :1617, :2895), per env, inside the reset kernel.

`emu` runs the lane-emulated build on the CPU, `cuda` the sm_90a library (marked gpu).  The pick is checked against numpy's own
RandomState.rand / RandomState.choice over a list of dicts, the reference's expression; the reset against the CPU env oracle
(oracle/init_state_oracle.py).
"""
import os
import pickle

import numpy as np
import pytest

from furniture_b200 import mjcf
from oracle.init_state_oracle import InitStateDenseEnv, InitStateEnv
from oracle.ref_env import Cfg, DenseCfg
from parity_util import build_emu, make_engine, quat_err
from test_dense_reward import _adopt_device_anchors, _assert_same_machine, _dense_engine, _dense_state
from test_env_parity import _sync_oracle_from_engine
from test_preassembled import _welded_pairs

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]
SEED = 123  # default_config's seed
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def model():
    return mjcf.load_scene("Sawyer", "table_lack_0825")


@pytest.fixture(scope="module")
def golden():
    g = np.load(os.path.join(HERE, "golden", "init_states.npz"))
    return {k: g[k] for k in g.files}


def _engine(m, n, gpu, dense=False, **cfg):
    return _dense_engine(m, n, gpu, **cfg) if dense else make_engine(m, n, gpu, **cfg)


def _recorded_states(m, n=8, seed=5):
    """n settled states of the device's own resets (float32 values, as a demo of this engine records them)"""
    eng = make_engine(m, n, False, seed=seed)
    eng.env_reset()
    q, v = eng.get_state()
    eng.close()
    return [{"qpos": q[i].astype(np.float64), "qvel": v[i].astype(np.float64)} for i in range(n)]


def _mid_assembly_state(m):
    """the state of an episode two connections in: the first two legs of the recipe on the table (a preassembled reset of the device), a
    start the sampler never produces"""
    eng = make_engine(m, 1, False, seed=17)
    eng.set_subtask(2)
    eng.env_reset()
    q, v = eng.get_state()
    eng.close()
    return {"qpos": q[0].astype(np.float64), "qvel": v[0].astype(np.float64)}


def _replay_picks(env, states, nreset, start=-1):
    """the reference's pick (furniture.py:1433-1434) on numpy's RandomState(seed + 2**20 + env): the start after each reset, and the state"""
    rs = np.random.RandomState(SEED + 2**20 + env)
    tagged = [dict(s, index=i) for i, s in enumerate(states)]
    cur, out = start, []
    for _ in range(nreset):
        if rs.rand() > 0.2:
            cur = rs.choice(tagged)["index"]
        out.append(cur)
    return out, rs.get_state()


# ------------------------------------------------------------------ the oracle against the reference's own _reset (tests/golden/init_states.npz)
class _Tracer:
    """records the oracle env's reset in the vocabulary of tools/make_golden_init_states.py: simulator calls with the robot's collision
    flag, the reference's helper calls (_stop_objects / _slow_objects are one call for all parts there), the state set_env_state plants"""

    def __init__(self, e, tags):
        self.e, self.log, self.quiet = e, [], 0
        rc = lambda: int(e.sim.geom_contype[e.robot_geoms[0]] != 0)
        sim = e.sim
        for name in ("reset", "forward", "step"):
            f = getattr(sim, name)
            setattr(sim, name, self._wrap(f, lambda *a, name=name: name if name == "reset" else "%s:rc%d" % (name, rc())))
        e._stop = self._wrap(e._stop, lambda p, g: "stop_objects(%d)" % g if p == 0 else None)
        e._slow = self._wrap(e._slow, lambda p: "slow_objects" if p == 0 else None)
        e.place = self._wrap(e.place, lambda: "place_objects")
        e._init_robot = self._wrap(e._init_robot, lambda: "initialize_robot_pos")
        e._grav_comp = self._wrap(e._grav_comp, lambda: "grav_comp")
        names = e.m.names["site"]
        connect = e._connect

        def traced_connect(s1, s2):  # the reference's _connect is a recorder: its own steps are not in the trace
            self.emit("connect(%s,%s,auto_align=%d):rc%d" % (names[s1], names[s2], int(e.cfg.auto_align), rc()))
            self.quiet += 1
            try:
                connect(s1, s2)
            finally:
                self.quiet -= 1

        e._connect = traced_connect
        set_state = e._set_env_state

        def traced_set_state():
            set_state()
            self.emit("set_state(%d)" % tags[id(e.init_qpos)])

        e._set_env_state = traced_set_state

    def emit(self, ev):
        if ev is not None and not self.quiet:
            self.log.append(ev)

    def _wrap(self, f, event):
        def g(*a):
            self.emit(event(*a))
            return f(*a)

        return g


def _golden_trace(g, start, env, k, recipe):
    i = [j for j in range(len(g["case_k"])) if (str(g["case_start"][j]), int(g["case_env"][j]), int(g["case_k"][j]), bool(g["case_recipe"][j])) ==
         (start, env, k, recipe)]
    assert len(i) == 1
    return str(g["case_trace"][i[0]]).split("\n"), int(g["case_pick"][i[0]])


SETTLE = lambda rc: (["stop_objects(0)"] + ["forward:rc%d" % rc, "step:rc%d" % rc, "slow_objects"] * 10) * 10  # :1560-1566


@pytest.mark.parametrize("start,env", [("none", 0), ("fixed", 0), ("bank", 0), ("bank", 1)])
def test_oracle_reset_emits_the_reference_trace(model, golden, start, env):
    """the oracle's reset, call for call, against the reference's unmodified FurnitureEnv._reset: placement or set_env_state, when the robot's
    collisions come back relative to the preassembly, the preassembly's auto_align (True after placement, False on a recorded start), the
    settle loops, which state is planted and the pick.  The fixed start has tag 100, bank entry i tag i (tools/make_golden_init_states.py)."""
    m, g = model, golden
    fixed = _recorded_states(m, 3)
    bank = _recorded_states(m, 3, seed=6)
    tags = {id(fixed[0]): int(g["fixed_tag"])}
    tags.update({id(s): i for i, s in enumerate(bank)})
    for k in (0, 1, 2):
        cfg = Cfg()
        cfg.seed = SEED + env
        e = InitStateEnv(m, cfg)
        e.set_subtask(k)
        if start == "fixed":
            e.set_init_qpos(fixed[0])
        if start == "bank":
            e.load_init_states(bank)
        tr = _Tracer(e, tags)
        e.reset()
        pick = -1 if e.init_qpos is None else tags[id(e.init_qpos)]
        ref, ref_pick = _golden_trace(g, start, env, k, True)
        assert pick == ref_pick, (k, pick, ref_pick)
        if k == 0:  # the reference runs the settle loop after the preassembly whenever the furniture has a recipe; the oracle and the device
            # only when something was preassembled (DESIGN.md §9): the trace without a recipe is the oracle's, and the two differ by that loop
            plain, _ = _golden_trace(g, start, env, 0, False)
            assert tr.log == plain, (start, env, next(i for i, (x, y) in enumerate(zip(tr.log, plain)) if x != y))
            at = next(i for i, (x, y) in enumerate(zip(ref, plain)) if x != y)
            rc = int(ref[at + 1].endswith("rc1"))
            assert ref == plain[:at] + SETTLE(rc) + plain[at:]
        else:
            assert tr.log == ref, (start, env, k, next((i, x, y) for i, (x, y) in enumerate(zip(tr.log, ref)) if x != y) if len(tr.log) == len(ref) else (len(tr.log), len(ref)))
            no_recipe, _ = _golden_trace(g, start, env, k, False)  # preassembled without a recipe: the reference's eq_active-only branch, not built
            assert "merge_groups" in no_recipe and not any(x.startswith("connect") for x in no_recipe)


def test_picks_equal_the_reference(model, golden):
    """the oracle's pick generator against the reference's pick expression with np.random seeded as the device seeds env 0..7"""
    g = golden
    states = _recorded_states(model, 7)
    for S, env, want in zip(g["pick_S"], g["pick_env"], g["pick_picks"]):
        cfg = Cfg()
        cfg.seed = SEED + int(env)
        e = InitStateEnv(model, cfg)
        e.load_init_states(states[: int(S)])
        got = []
        for _ in range(20):
            e._pick()
            got.append(-1 if e.init_qpos is None else [id(s) for s in states].index(id(e.init_qpos)))
        assert got == list(want), (S, env)
        assert _replay_picks(int(env), states[: int(S)], 20)[0] == list(want)  # the replay the device tests use


# ------------------------------------------------------------------ the pick: numpy's stream, draw for draw
@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("S", [1, 3, 7])
def test_pick_follows_numpy_draw_for_draw(model, gpu, S):
    m, n = model, 8
    states = _recorded_states(m)[:S]
    eng = make_engine(m, n, gpu)
    eng.load_init_states(states)
    assert list(eng.get("init_pick")[:, 0]) == [S] * n and list(eng.get("init_state")[:, 0]) == [-1] * n
    mt0, pos0 = eng.get("mt_state").copy(), eng.get("mt_pos")[:, 0].copy()
    got = []
    for _ in range(20):
        eng.env_reset()
        got.append(eng.get("init_state")[:, 0].copy())
        assert (eng.get("flags") == 0).all()
    got = np.array(got)
    for i in range(n):
        want, st = _replay_picks(i, states, 20)
        assert list(got[:, i]) == want, (i, list(got[:, i]), want)
        assert np.array_equal(eng.get("init_mt_state")[i], st[1]) and int(eng.get("init_mt_pos")[i, 0]) == st[2], i
        if want[0] >= 0:  # every reset started from a state: the sampler's generator made no draw (furn_size_rand = 0)
            assert np.array_equal(eng.get("mt_state")[i], mt0[i]) and eng.get("mt_pos")[i, 0] == pos0[i], i
        else:
            assert eng.get("mt_pos")[i, 0] != pos0[i] or not np.array_equal(eng.get("mt_state")[i], mt0[i])
    if S > 1:
        assert len(np.unique(got[-1])) > 1  # the envs do not all pick alike
    eng.close()


# ------------------------------------------------------------------ the reset against the CPU env
RESET_CASES = [pytest.param(False, 0, False, id="emu-k0-sparse"), pytest.param(False, 2, False, id="emu-k2-sparse"),
               pytest.param(False, 1, True, id="emu-k1-dense"),
               pytest.param(True, 0, False, id="cuda-k0-sparse", marks=pytest.mark.gpu), pytest.param(True, 2, False, id="cuda-k2-sparse", marks=pytest.mark.gpu),
               pytest.param(True, 1, True, id="cuda-k1-dense", marks=pytest.mark.gpu)]


@pytest.mark.parametrize("gpu,k,dense", RESET_CASES)
def test_reset_from_a_recorded_state_matches_the_cpu_env(model, gpu, k, dense):
    """a mid-assembly start with k recipe steps preassembled (connected where the state has the parts, not aligned): welds, masks, groups,
    sites and both generators exactly, poses and weld data to fp32 tolerance, then 3 random steps"""
    m, n = model, 2
    state = _mid_assembly_state(m)
    eng = _engine(m, n, gpu, dense)
    if k:
        eng.set_subtask(k)
    eng.set_init_qpos(state)
    mt0 = eng.get("mt_state").copy(), eng.get("mt_pos").copy()
    eng.env_reset()
    assert (eng.get("flags") == 0).all() and list(eng.get("init_state")[:, 0]) == [0, 0]
    envs = []
    for i in range(n):
        cfg = DenseCfg() if dense else Cfg()
        cfg.seed = SEED + i
        e = InitStateDenseEnv(m, cfg) if dense else InitStateEnv(m, cfg)
        e.set_subtask(k)
        e.set_init_qpos(state)
        e.reset()
        envs.append(e)
        assert list(eng.get("eq_active")[i]) == list(e.sim.eq_active) and int(eng.get("eq_active")[i].sum()) == k
        ct, ca = eng.get("geom_contype")[i], eng.get("geom_conaffinity")[i]
        for j, g in enumerate(eng.em.geom_src):
            assert ct[j] == e.sim.geom_contype[g] and ca[j] == e.sim.geom_conaffinity[g], (i, j)
        assert int(eng.get("num_connected")[i, 0]) == e.num_connected == k
        assert set(np.flatnonzero(eng.get("site_connected")[i])) == e.connected_sites and list(eng.get("group")[i]) == e.group
        # no draw from either generator: the sampler's is where fe_create left it, the pick's was never used
        assert np.array_equal(eng.get("mt_state")[i], mt0[0][i]) and eng.get("mt_pos")[i, 0] == mt0[1][i, 0]
        st = e.rng.get_state()
        assert int(eng.get("mt_pos")[i, 0]) == 624 and np.array_equal(eng.get("mt_state")[i], st[1]) and st[2] == 624
        ps = e.pick_rng.get_state()
        assert np.array_equal(eng.get("init_mt_state")[i], ps[1]) and int(eng.get("init_mt_pos")[i, 0]) == ps[2]
        q = eng.get("qpos")[i]
        for p in range(e.npart):
            a = 9 + 7 * p
            assert np.abs(q[a : a + 3] - e.sim.qpos[a : a + 3]).max() < 5e-4 and quat_err(q[a + 3 : a + 7], e.sim.qpos[a + 3 : a + 7]) < 5e-4, (i, p)
        for w in np.flatnonzero(e.sim.eq_active):
            d, o = eng.get("eq_data")[i].reshape(-1, 7)[w], e.sim.eq_data[7 * w : 7 * w + 7]
            assert np.abs(d[:3] - o[:3]).max() < 5e-4 and quat_err(d[3:], o[3:]) < 5e-4, (i, w)
        assert np.abs(eng.get("obs")[i] - e.obs()).max() < 2e-4, (i, np.abs(eng.get("obs")[i] - e.obs()).max())
        if dense:
            ds = _dense_state(eng, i)
            assert (ds["subtask"], ds["phase"]) == (k, e.dense.phase) and e.dense.subtask == k
    assert len(_welded_pairs(eng, 0)) == k
    for i, e in enumerate(envs):  # continue from the device's state, as the step parity tests do
        _sync_oracle_from_engine(e, eng, i)
        e.sim.qfrc_bias[: e.nr] = eng.get("qfrc_bias")[i]
        if dense:
            e.dense.begin_episode()
            _assert_same_machine(_dense_state(eng, i), e.dense, ("reset", i), tol=5e-4)
            _adopt_device_anchors(e.dense, _dense_state(eng, i))
    rng = np.random.RandomState(3)
    for step in range(3):
        a = rng.uniform(-1, 1, (n, eng.act_dim)).astype(np.float32)
        a[:, -1] = -0.5
        obs, rew, done, info = eng.env_step_host(a)
        for i, e in enumerate(envs):
            ob, r, d, inf = e.step(a[i].astype(np.float64))
            assert np.abs(obs[i] - ob).max() < 2e-4, (step, i, np.abs(obs[i] - ob).max())
            assert abs(rew[i] - r) < (2e-2 + 1e-5 * abs(r) if dense else 1e-4) and bool(done[i]) == d and not d
            assert info[i][0] == k == inf["num_connected"]
    eng.close()


def test_baxter_resets_from_a_recorded_state_like_the_cpu_env():
    m = mjcf.load_scene("Baxter", "chair_ingolf_0650")
    eng = make_engine(m, 2, False)
    eng.env_reset()
    q, v = eng.get_state()
    state = {"qpos": q[1].astype(np.float64), "qvel": v[1].astype(np.float64)}
    eng.set_init_qpos(state)
    eng.env_reset()
    cfg = Cfg()
    e = InitStateEnv(m, cfg)
    e.set_init_qpos(state)
    e.reset()
    ob = e.obs()
    for i in range(2):
        assert np.abs(eng.get("obs")[i] - ob).max() < 2e-4, (i, np.abs(eng.get("obs")[i] - ob).max())
        assert eng.get("eq_active")[i].sum() == 0 and int(eng.get("num_connected")[i, 0]) == 0
    assert np.array_equal(eng.get("obs")[0], eng.get("obs")[1])  # no draw: both envs start alike
    eng.close()


# ------------------------------------------------------------------ persistence, and per env
def _snapshot(eng, i):
    return [eng.get("qpos")[i], eng.get("qvel")[i], eng.get("obs")[i], eng.get("eq_active")[i], eng.get("mt_state")[i], eng.get("mt_pos")[i],
            eng.get("init_mt_state")[i], eng.get("init_mt_pos")[i]]


@pytest.mark.parametrize("gpu", BACKENDS)
def test_a_fixed_start_persists_and_every_env_has_its_own(model, gpu):
    m = model
    states = _recorded_states(m)
    A, B = states[0], states[1]
    eng = make_engine(m, 1, gpu, nsub=2, max_episode_steps=2)
    eng.set_init_qpos(A)
    eng.env_reset()
    first = eng.get("obs").copy()
    a = np.zeros((1, eng.act_dim), np.float32)
    a[:, -1] = -1
    eng.env_step_host(a)
    obs, rew, done, info = eng.env_step_host(a)  # max_episode_steps: the auto-reset inside the step starts from A again
    assert done[0] and info[0][3] == 2 and int(eng.get("episode_length")[0, 0]) == 0
    assert np.array_equal(obs, first) and np.array_equal(eng.get("obs"), first)
    eng.close()
    # four envs: None, A, B, a pick from [A, B, states[2]]; each equals env 0 of a handle of its own set up alike, bit for bit
    eng = make_engine(m, 4, gpu, nsub=2)
    eng.set_init_qpos([None, A, B, None])
    eng.load_init_states(states[:3], envs=[3])
    assert list(eng.get("init_pick")[:, 0]) == [0, 0, 0, 3]
    for _ in range(2):
        eng.env_reset()
    for i in range(4):
        one = make_engine(m, 1, gpu, nsub=2, seed=SEED + i)
        one.set_init_qpos([None, A, B, None][i])
        if i == 3:
            one.load_init_states(states[:3])
        for _ in range(2):
            one.env_reset()
        for x, y in zip(_snapshot(eng, i), _snapshot(one, 0)):
            assert np.array_equal(x, y), i
        s, s1 = int(eng.get("init_state")[i, 0]), int(one.get("init_state")[0, 0])
        assert (s >= 0) == (s1 >= 0) == (i > 0 or s >= 0) and (i != 3 or s == s1), (i, s, s1)  # A and B sit at other bank indices than in `one`
        one.close()
    eng.close()


# ------------------------------------------------------------------ the unstable step clears the start (emulated build only)
def test_an_unstable_step_clears_the_start_and_each_reset_picks(model):
    m, n = model, 2
    states = _recorded_states(m)
    eng = make_engine(m, n, False, nsub=2)
    eng.set_init_qpos(states[0])  # env 0 and env 1: the fixed start, no list
    eng.env_reset()
    v = eng.get("qvel").copy()
    v[1, 0] = 1e8
    eng.set("qvel", v)
    a = np.zeros((n, eng.act_dim), np.float32)
    a[:, -1] = -1
    obs, rew, done, info = eng.env_step_host(a)
    assert done[1] and info[1][2] == 1 and not done[0]
    assert list(eng.get("init_state")[:, 0]) == [0, -1]
    cfg = Cfg()
    cfg.seed = SEED + 1
    e = InitStateEnv(m, cfg)  # both resets of the step drew from the sampler: two resets' worth of draws
    for _ in range(2):
        e.place()
        for _ in range(101):
            e.rng.uniform(-cfg.agent_xyz_rand, cfg.agent_xyz_rand, e.narm)
    s = e.rng.get_state()
    assert int(eng.get("mt_pos")[1, 0]) == s[2] and np.array_equal(eng.get("mt_state")[1], s[1])
    assert int(eng.get("mt_pos")[0, 0]) == 624
    eng.close()
    # with a list, each of the two resets makes its own pick draw, and the env ends on the state the last passing draw chose, or on the sampler
    outcomes = set()
    for seed_env in range(8):
        eng = make_engine(m, n, False, nsub=2, seed=SEED + seed_env)
        eng.load_init_states(states[:3])
        eng.env_reset()
        v = eng.get("qvel").copy()
        v[1, 0] = 1e8
        eng.set("qvel", v)
        eng.env_step_host(a)
        rs = np.random.RandomState(SEED + seed_env + 2**20 + 1)
        tagged = [dict(s, index=i) for i, s in enumerate(states[:3])]
        first_random = not rs.rand() > 0.2  # the reset before the step
        if not first_random:
            rs.choice(tagged)
        cur = -1  # cleared by the unstable step
        for _ in range(2):
            if rs.rand() > 0.2:
                cur = rs.choice(tagged)["index"]
        assert int(eng.get("init_state")[1, 0]) == cur, seed_env
        st = rs.get_state()
        assert np.array_equal(eng.get("init_mt_state")[1], st[1]) and int(eng.get("init_mt_pos")[1, 0]) == st[2]
        if cur >= 0:  # the env is where a reset from that bank entry puts it
            one = make_engine(m, 1, False, nsub=2)
            one.set_init_qpos(states[cur])
            one.env_reset()
            for name in ("qpos", "qvel", "obs"):
                assert np.array_equal(eng.get(name)[1], one.get(name)[0]), (seed_env, name)
            one.close()
        else:  # the sampler placed it: its generator spent the draws of both resets of the step (and of the first one if it was random)
            cfg = Cfg()
            cfg.seed = SEED + seed_env + 1
            e = InitStateEnv(m, cfg)
            for _ in range(2 + int(first_random)):
                e.place()
                for _ in range(101):
                    e.rng.uniform(-cfg.agent_xyz_rand, cfg.agent_xyz_rand, e.narm)
            s = e.rng.get_state()
            assert int(eng.get("mt_pos")[1, 0]) == s[2] and np.array_equal(eng.get("mt_state")[1], s[1]), seed_env
        outcomes.add(cur >= 0)
        eng.close()
    assert outcomes == {True, False}  # both endings were exercised


def test_the_oracle_clears_the_start_in_the_except_branch(model, golden):
    """the oracle's _simulate override against the reference's _do_simulation: the reset of the except branch starts from None"""
    assert list(golden["except_reset_start"]) == [-1] and bool(golden["except_fail"])
    cfg = Cfg()
    m = model
    e = InitStateEnv(m, cfg)
    e.nsub = 2
    state = _recorded_states(m, 1)[0]
    e.set_init_qpos(state)
    e.reset()
    seen = []
    reset = e.reset
    e.reset = lambda: (seen.append(e.init_qpos is None), reset())[1]
    e.sim.qvel[0] = 1e8
    a = np.zeros(e.dof)
    a[-1] = -1
    ob, r, d, info = e.step(a)
    assert info["unstable"] == 1 and d and seen == [True] and e.init_qpos is None


# ------------------------------------------------------------------ the untouched path
@pytest.mark.parametrize("gpu", BACKENDS)
def test_an_unused_bank_changes_nothing_and_ik_resets_alike(model, gpu):
    from furniture_b200.engine import Engine, default_config
    from furniture_b200.ik import ik_config

    m = model
    states = _recorded_states(m)
    runs = []
    for bank in (False, True):
        eng = make_engine(m, 2, gpu)
        if bank:
            eng.set_init_states(states)
        eng.env_reset()
        out = [eng.get("obs").copy()]
        rng = np.random.RandomState(9)
        for _ in range(5):
            out += list(eng.env_step_host(rng.uniform(-1, 1, (2, eng.act_dim)).astype(np.float32)))
        out += [eng.get("qpos"), eng.get("mt_state"), eng.get("mt_pos")]
        runs.append(out)
        eng.close()
    for x, y in zip(*runs):
        assert np.array_equal(x, y)
    imp = make_engine(m, 2, gpu)
    ik = Engine(m, 2, device=0, config=default_config(), ik=ik_config(m)) if gpu else Engine(m, 2, config=default_config(), lib_path=build_emu(), ik=ik_config(m))
    for eng in (imp, ik):
        eng.set_init_qpos([states[3], None])
        eng.env_reset()
    for name in ("qpos", "qvel", "obs"):
        assert np.array_equal(imp.get(name), ik.get(name)), name
    imp.close()
    ik.close()


def test_a_new_list_keeps_every_env_s_start(model):
    """load_init_states replaces the list to pick from; it never changes a start an env already has (the reference's _init_qpos survives a
    new list): a start picked from the old list and fixed starts stay where they were"""
    m = model
    st = _recorded_states(m, 6)
    A, B, C, D, E, F = st
    eng = make_engine(m, 3, False)
    eng.set_init_qpos([None, E, F])
    eng.load_init_states([A, B, C], envs=[0])
    eng.set("init_state", np.array([[2], [int(eng.get("init_state")[1, 0])], [int(eng.get("init_state")[2, 0])]], np.int32))  # env 0 picked C
    before = [eng.init_states()[0][s].copy() for s in eng.get("init_state")[:, 0]]
    for new in ([D], [], [A, B, C, D, E, F, A]):
        eng.load_init_states(new, envs=[0])
        q, v, npick = eng.init_states()
        assert npick == len(new) and np.array_equal(q[:npick], np.array([s["qpos"] for s in new], np.float32).reshape(-1, m.nq))
        for i, s in enumerate(eng.get("init_state")[:, 0]):
            assert s >= 0 and np.array_equal(q[s], before[i]), (len(new), i)
    eng.set_init_qpos([None, None, None])
    assert len(eng.init_states()[0]) == 7  # only the list is left


# ------------------------------------------------------------------ host surface
class _Recorded:
    """the face of an env that BatchDemoRecorder reads: num_envs and get_env_state"""

    def __init__(self, eng):
        self.eng, self.num_envs = eng, eng.N

    def get_env_state(self):
        q, v = self.eng.get_state()
        return {"qpos": q, "qvel": v}


def _write_files(m, tmp_path):
    """a demo file written by BatchDemoRecorder and an init-states pickle (a list of get_env_state dicts, furniture.py:127-130)"""
    from furniture_b200.demo import BatchDemoRecorder

    eng = make_engine(m, 2, False, seed=11)
    eng.env_reset()
    rec = BatchDemoRecorder(_Recorded(eng), demo_dir=str(tmp_path))
    rec.add_reset({"object_ob": eng.get("obs")[:, :35]})
    a = np.zeros((2, eng.act_dim), np.float32)
    obs, rew, _, _ = eng.env_step_host(a)
    rec.add_step(a, {"object_ob": obs[:, :35]}, rew)
    demo = rec.save("Sawyer_table_lack_0825_", envs=[1])[0]
    q, v = eng.get_state()
    states = [{"qpos": q[i].astype(np.float64), "qvel": v[i].astype(np.float64)} for i in range(2)]
    init = tmp_path / "init_states.pkl"
    with open(init, "wb") as f:
        pickle.dump(states, f)
    eng.close()
    with open(demo, "rb") as f:
        first = pickle.load(f)["states"][0]
    return demo, str(init), first, states


def test_config_keys_files_and_what_is_refused(model, tmp_path):
    from furniture_b200.env import split_config, split_dense_config
    from furniture_b200.gym_api import FurnitureGymB200

    m = model
    demo, init, first, states = _write_files(m, tmp_path)
    name, over, ignored = split_config(dict(load_init_states=init, load_demo=demo, port=1050))
    assert over == {"load_init_states": init, "load_demo": demo} and ignored == ["port"]
    assert split_config(dict(load_init_states=None, load_demo=None))[1:] == ({}, [])  # the reference's defaults
    assert split_dense_config(dict(load_demo=demo))[1]["load_demo"] == demo and split_dense_config(dict(load_demo=demo))[3] == []
    env = FurnitureGymB200(name="FurnitureSawyerEnv", lib_path=build_emu(), load_demo=demo, load_init_states=init)
    assert env.ignored_config == [] and int(env.engine.get("init_state")[0, 0]) >= 0
    bq, bv, npick = env.engine.init_states()
    assert npick == 2 and np.array_equal(bq[:2], np.array([s["qpos"] for s in states], np.float32))
    assert np.array_equal(bq[int(env.engine.get("init_state")[0, 0])], first["qpos"].astype(np.float32))
    env.close()
    env = FurnitureGymB200(name="FurnitureSawyerEnv", lib_path=build_emu(), load_demo=demo)
    ob = env.reset()
    assert int(env.engine.get("mt_pos")[0, 0]) == 624  # the demo's start: no random draw
    env.set_init_qpos(None)
    env.reset()
    assert int(env.engine.get("mt_pos")[0, 0]) != 624 and int(env.engine.get("init_state")[0, 0]) == -1
    eng = env.engine
    bad = [dict(qpos=first["qpos"][:-1], qvel=first["qvel"]), dict(qpos=first["qpos"], qvel=np.r_[first["qvel"], 0.0]),
           dict(qpos=np.where(np.arange(m.nq) == 3, np.nan, first["qpos"]), qvel=first["qvel"]), dict(qvel=first["qvel"]),
           dict(qpos=first["qpos"], qvel=np.full(m.nv, np.inf))]
    for b in bad:
        with pytest.raises(ValueError):
            eng.set_init_qpos(b)
        with pytest.raises(ValueError):
            eng.load_init_states([first, b])
    with pytest.raises(ValueError):
        eng.load_init_states([first], envs=[1])  # one env in this handle
    with pytest.raises(ValueError):
        eng.set_init_qpos([first, first])
    assert int(eng.get("init_state")[0, 0]) == -1 and eng.get("init_pick")[0, 0] == 0  # refusals leave the env as it was
    env.close()


@pytest.mark.gpu
def test_make_vec_env_takes_load_init_states_and_load_demo(model, tmp_path):
    from furniture_b200.env import make_vec_env

    demo, init, first, states = _write_files(model, tmp_path)
    env = make_vec_env("IKEASawyer-v0", num_env=3, config=dict(load_init_states=init, load_demo=demo, port=1050))
    assert env.ignored_config == ["port"] and list(env.engine.get("init_pick")[:, 0]) == [2, 2, 2]
    assert len(set(env.engine.get("init_state")[:, 0])) == 1 and env.engine.get("init_state")[0, 0] >= 0
    env.reset()
    env.set_init_qpos(None)
    env.load_init_states(None)
    env.reset()
    assert list(env.engine.get("init_state")[:, 0]) == [-1] * 3 and list(env.engine.get("init_pick")[:, 0]) == [0] * 3
    env.close()
