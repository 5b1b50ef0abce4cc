"""`assembled` (config/furniture.py:307-312) inside the reset kernel, per env: every weld on, the parts left at the model's qpos0 (the
furniture as assembled), all in one group (furniture.py:1501-1532).

The CPU env of tests/assembled_oracle.py is the yardstick; the device, lane-emulated ([emu]) and on the GPU ([cuda]), is held to it: welds,
groups, masks, subtask pair and generator exactly, poses and eq_data at the reset bar of tests/test_reset_options.py, then 3 steps at the
obs / reward bars of tests/test_sim_options.py.
"""
import ctypes as C
import os

import numpy as np
import pytest

from assembled_oracle import AssembledDenseEnv, AssembledIKEnv, AssembledInitStateEnv
from furniture_b200 import mjcf
from oracle.ref_env import DenseCfg
from parity_util import build_emu
from test_env_parity import _sync_oracle_from_engine
from test_reset_options import _cfg, _engine, _quat_err, _same_generator

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def lack():
    return mjcf.load_scene("Sawyer", "table_lack_0825")


def _oracle(m, kind, **kw):
    if kind == "dense":
        return AssembledDenseEnv(m, _cfg(DenseCfg), {}, **kw)
    if kind == "ik":
        return AssembledIKEnv(m, _cfg(), **kw)
    return AssembledInitStateEnv(m, _cfg(), **kw)


def _masks(eng, i, e):
    """the device's masks and the CPU env's, over the geoms the engine keeps"""
    src = list(eng.em.geom_src)
    dev = np.stack([eng.get("geom_contype")[i], eng.get("geom_conaffinity")[i]])
    cpu = np.array([[e.sim.geom_contype[g] for g in src], [e.sim.geom_conaffinity[g] for g in src]])
    return dev, cpu


def _assembled_state(m):
    """a recorded start that satisfies the welds: the state an assembled reset of the device settles to.  (A mid-assembly state with every
    weld turned on makes the solver fling the loose parts onto their weld targets, which an fp32-vs-fp64 comparison cannot follow.)"""
    eng = _engine(m, 1, False, cfg=dict(seed=17), assembled=True)
    eng.env_reset()
    q, v = eng.get_state()
    eng.close()
    return {"qpos": q[0].astype(np.float64), "qvel": v[0].astype(np.float64)}


def _pair(e):
    """_subtask_part1 / _subtask_part2 after the reset: _get_next_subtask, or in the dense env the parts of the reward's current subtask
    (furniture_sawyer_dense.py:149-162), which follows its recipe whatever the groups"""
    if getattr(e, "dense", None) is None:
        return e.subtask_pair()
    st = e.dense.sub[e.dense.subtask]
    return e.parts.index(st.leg), e.parts.index(st.table)


def _assert_reset_equal(eng, i, e, tag):
    """welds, groups, masks, subtask pair and generator exactly; part poses and eq_data at the reset bar, quaternions up to sign"""
    assert np.array_equal(eng.get("eq_active")[i], e.sim.eq_active), tag
    assert [int(g) for g in eng.get("group")[i]] == list(e.group), (tag, eng.get("group")[i], e.group)
    dev, cpu = _masks(eng, i, e)
    assert np.array_equal(dev, cpu), tag
    assert tuple(int(x) for x in eng.get("subtask_part")[i]) == _pair(e), tag
    assert _same_generator(eng, i, e), tag
    q = eng.get("qpos")[i]
    for p in range(e.npart):
        a = e.part_qadr[p]
        assert np.abs(q[a : a + 3] - e.sim.qpos[a : a + 3]).max() < 5e-4 and _quat_err(q[a + 3 : a + 7], e.sim.qpos[a + 3 : a + 7]) < 5e-4, (tag, p)
    ed = eng.get("eq_data")[i].reshape(-1, 7).astype(np.float64)
    od = np.asarray(e.sim.eq_data, np.float64).reshape(-1, 7)
    for w in range(len(ed)):
        assert np.abs(ed[w, :3] - od[w, :3]).max() < 5e-4 and _quat_err(ed[w, 3:], od[w, 3:]) < 5e-4, (tag, w)


def _steps_match(eng, envs, kind, n_steps=3):
    """the CPU envs synced from the device after its reset, then `n_steps` random steps at the obs and reward bars"""
    from test_dense_reward import _adopt_device_anchors, _dense_state
    from test_obs_layout import _sync_ik

    for i, e in enumerate(envs):
        _sync_oracle_from_engine(e, eng, i)
        e.sim.qfrc_bias[: e.nr] = eng.get("qfrc_bias")[i]
        if kind == "dense":
            e.dense.begin_episode()
            _adopt_device_anchors(e.dense, _dense_state(eng, i))
        if kind == "ik":
            _sync_ik(e, eng, i)
    rng = np.random.RandomState(5)
    for k in range(n_steps):
        a = rng.uniform(-1, 1, (len(envs), eng.act_dim)).astype(np.float32)
        a[:, -1] = -0.5
        obs, rew, done, info = eng.env_step_host(a)
        for i, e in enumerate(envs):
            ob, r, d, _ = e.step(a[i].astype(np.float64))
            assert np.abs(obs[i] - ob).max() < 2e-4, (k, i, np.abs(obs[i] - ob).max())
            assert abs(rew[i] - r) < (2e-2 + 1e-5 * abs(r) if kind == "dense" else 1e-5) and bool(done[i]) == d, (k, i, rew[i], r)


# ------------------------------------------------------------------ where an assembled start leaves the parts
def test_part_link_frames_are_qpos0():
    """the reset kernel plants an assembled part at its link frame in the model (fe_model.link_pos / link_quat), which must be sim.reset()'s
    qpos0 of the part's free joint in float32: checked for every part of every shipped scene"""
    import glob

    from furniture_b200.engine_model import EngineModel

    n = 0
    for path in sorted(glob.glob(os.path.join(ROOT, "furniture_b200", "compiled", "*.npz"))):
        agent, furn = os.path.basename(path)[:-4].split("_", 1)
        m = mjcf.load_scene(agent, furn)
        fm = EngineModel(m).fm
        for p in range(fm.npart):
            i = fm.nrlink + p
            qa = fm.link_qadr[i]
            frame = np.array(list(fm.link_pos[i]) + list(fm.link_quat[i]), np.float32)
            assert np.array_equal(frame, np.asarray(m.qpos0[qa : qa + 7], np.float32)), (agent, furn, p)
            n += 1
    assert n > 400


# ------------------------------------------------------------------ the oracle against the reference's own code
@pytest.fixture(scope="module")
def golden():
    g = np.load(os.path.join(HERE, "golden", "assembled.npz"))
    return {k: g[k] for k in g.files}


def _placement_words(e):
    """wrap the CPU env's place() to count the 32-bit words its placement draws"""
    from test_reset_options import _words

    e.place_words = 0
    place = e.place

    def counted():
        s0 = e.rng.get_state()
        out = place()
        e.place_words = _words(s0, e.rng.get_state())
        return out

    e.place = counted


def test_oracle_equals_the_reference(golden):
    """every golden case (assembled x random placement / fix_init over two resets / fix_init_parts / a recorded start x k = 0, 1, 2 on
    table_lack_0825, a furniture without a recipe, Baxter + chair_ingolf_0650, and connections followed by an assembled reset): the CPU env
    after each reset has the reference's eq_active, groups, planted parts, placement draws, init_pos (bit for bit), masks, num_connected,
    _success_num_conn and subtask pair; the welds no connection of the reset touched keep their eq_data bit for bit, as the model array
    does in the reference, and on an assembled first reset the ones the preassembly re-sets agree with it to 5e-3 (the stand-in does not
    simulate: its parts sit at qpos0, the CPU env's where the settle steps before the weld leave them)"""
    g = golden
    models = {}
    for c in range(len(g["case_start"])):
        agent, furn, start, k = str(g["case_agent"][c]), str(g["case_furniture"][c]), str(g["case_start"][c]), int(g["case_k"][c])
        m = models.setdefault((agent, furn), mjcf.load_scene(agent, furn))
        e = AssembledInitStateEnv(m, _cfg(), fix_init=start == "fix_init", fix_init_parts="1_part1,3_part3" if start == "fix_init_parts" else None)
        _placement_words(e)
        if start == "init_state":
            e.set_init_qpos(_assembled_state(m))
        if k:
            e.set_subtask(k)
        n, npart, neq, ng = e.npart, e.npart, m.neq, m.ngeom
        welds = [{e._part_of_body(m.eq_obj1id[w]), e._part_of_body(m.eq_obj2id[w])} for w in range(neq)]
        touched, connect = set(), e._connect

        def recorded(s1, s2, connect=connect, touched=touched, welds=welds):  # the welds a _connect re-sets (_activate_weld)
            pair = {e._part_of_body(m.site_bodyid[s1]), e._part_of_body(m.site_bodyid[s2])}
            touched.update(w for w in range(neq) if welds[w] <= pair)
            return connect(s1, s2)

        e._connect = recorded
        for r in range(int(g["case_nreset"][c])):
            touched.clear()
            tag = (agent, furn, start, k, r)
            e.assembled = bool(g["case_assembled"][c][r])
            e.place_words, e.moved = 0, []
            e.rng = np.random.RandomState(123)  # the stand-in's resets draw for the placement only: the CPU env's robot noise is skipped
            for _ in range(int(g["words"][c, :r].sum())):
                e.rng.bytes(4)
            before = np.array(e.sim.eq_data, np.float64).reshape(-1, 7)
            e.reset()
            assert list(e.sim.eq_active) == list(g["eq_active"][c, r][:neq]), tag
            ref_group = [int(x) for x in g["group"][c, r][:npart]]
            root = lambda grp, i: i if grp[i] == i else root(grp, grp[i])  # noqa: E731  (_find_group compresses paths, the oracle does not)
            assert [e._find(p) for p in range(n)] == [root(ref_group, p) for p in range(n)], (tag, e.group, ref_group)
            assert [p in e.moved for p in range(n)] == list(g["moved"][c, r][:npart]), tag
            assert e.place_words == int(g["words"][c, r]), (tag, e.place_words, g["words"][c, r])
            if start != "init_state":
                ip = np.array([np.concatenate([e.init_pos[nm], e.init_quat[nm]]) for nm in e.parts])
                assert np.array_equal(ip, g["init_pos"][c, r][:npart]), tag
            assert np.array_equal(np.array(e.sim.geom_contype), g["masks"][c, r][:ng, 0]), tag
            assert np.array_equal(np.array(e.sim.geom_conaffinity), g["masks"][c, r][:ng, 1]), tag
            assert e.num_connected == int(g["num_connected"][c, r]) and e.success_num_conn == int(g["success_num_conn"][c, r]), tag
            assert e.subtask_pair() == tuple(int(x) for x in g["subtask"][c, r]), tag
            kept = np.array([w not in touched for w in range(neq)])
            assert np.array_equal(g["eq_data"][c, r][:neq][kept], g["eq_data_before"][c, r][:neq][kept]), tag
            after = np.array(e.sim.eq_data, np.float64).reshape(-1, 7)
            assert np.array_equal(after[kept], before[kept]), tag
            # the stand-in neither aligns nor settles: compared where its parts sit where the CPU env's do, an assembled first reset (qpos0,
            # the compiled weld targets); later the CPU env's welds pull the parts onto the targets the last episode left in eq_data
            for w in np.flatnonzero(~kept) if e.assembled and r == 0 else []:
                ref = g["eq_data"][c, r][w]
                assert np.abs(after[w, :3] - ref[:3]).max() < 5e-3 and _quat_err(after[w, 3:], ref[3:]) < 5e-3, (tag, w, after[w], ref)
    assert (g["words"][:, 0] == 0).any() and (g["num_connected"] == 2).any() and (~np.all(g["eq_data"] == g["eq_data_before"], axis=-1)).any()


# ------------------------------------------------------------------ the device reset against the CPU env
@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("kind", ["sparse", "dense", "ik", "baxter"])
def test_assembled_reset_equals_the_cpu_env(lack, gpu, kind):
    """two envs with assembled: the reset equals the CPU env's, then 3 random steps"""
    m = mjcf.load_scene("Baxter", "chair_ingolf_0650") if kind == "baxter" else lack
    n = 2
    eng = _engine(m, n, gpu, dense=kind == "dense", ik=kind == "ik", assembled=True)
    eng.env_reset()
    envs = []
    for i in range(n):
        e = _oracle(m, kind, assembled=True)
        e.rng = np.random.RandomState(123 + i)
        e.reset()
        _assert_reset_equal(eng, i, e, (kind, i))
        assert (eng.get("eq_active")[i] == 1).all() and (eng.get("group")[i] == 0).all() and e.moved == []
        envs.append(e)
    _steps_match(eng, envs, kind)


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("start", ["preassembled", "init_state"])
def test_assembled_with_a_recipe_prefix_or_a_recorded_start(lack, gpu, start):
    """assembled with preassembled = 2 (two _connect calls inside group 0: every part's masks change, eq_data of the two legs is re-set,
    num_connected = 2) and with a recorded start of the welded furniture (every weld on, no group merged): the reset equals the CPU env's,
    then 3 steps"""
    eng = _engine(lack, 1, gpu, assembled=True)
    e = _oracle(lack, "sparse", assembled=True)
    if start == "init_state":
        st = _assembled_state(lack)
        eng.set_init_qpos(st)
        e.set_init_qpos(st)
    else:
        eng.set_subtask(2)
        e.set_subtask(2)
    eng.env_reset()
    e.reset()
    _assert_reset_equal(eng, 0, e, start)
    if start == "init_state":
        assert list(eng.get("group")[0]) == list(range(e.npart)) and (eng.get("eq_active")[0] == 1).all()
    else:
        assert int(eng.get("num_connected")[0, 0]) == e.num_connected == 2
    _steps_match(eng, [e], "sparse")


def test_the_furniture_stays_assembled(lack):
    """20 random steps of the bench workload from an assembled start: the relative pose of every welded pair stays as close to its eq_data
    on the device as in the CPU env run alongside it (lane-emulated build)"""
    from oracle import assembly_oracle as A

    eng = _engine(lack, 1, False, assembled=True)
    eng.env_reset()
    e = _oracle(lack, "sparse", assembled=True)
    e.reset()
    _sync_oracle_from_engine(e, eng, 0)
    e.sim.qfrc_bias[: e.nr] = eng.get("qfrc_bias")[0]
    m = lack
    pairs = [(e._part_of_body(m.eq_obj1id[w]), e._part_of_body(m.eq_obj2id[w])) for w in range(m.neq)]

    def drift(qpos, eq_data):
        out = []
        for w, (a, b) in enumerate(pairs):
            qa, qb = (np.asarray(qpos[e.part_qadr[p] : e.part_qadr[p] + 7], np.float64) for p in (a, b))
            rel = A.rel_pose(qa, qb)
            out.append(max(np.abs(rel[:3] - eq_data[7 * w : 7 * w + 3]).max(), _quat_err(rel[3:], eq_data[7 * w + 3 : 7 * w + 7])))
        return np.array(out)

    rng = np.random.RandomState(11)
    worst_dev, worst_cpu = 0.0, 0.0
    for k in range(20):
        a = rng.uniform(-1, 1, (1, eng.act_dim)).astype(np.float32)
        a[:, -1] = -0.5
        eng.env_step_host(a)
        e.step(a[0].astype(np.float64))
        dev = drift(eng.get("qpos")[0], eng.get("eq_data")[0].astype(np.float64))
        cpu = drift(e.sim.qpos, np.asarray(e.sim.eq_data, np.float64))
        worst_dev, worst_cpu = max(worst_dev, dev.max()), max(worst_cpu, cpu.max())
        assert (dev <= cpu + 1e-3).all(), (k, dev, cpu)
    assert worst_cpu < 5e-2 and worst_dev < 5e-2, (worst_dev, worst_cpu)


# ------------------------------------------------------------------ per env
def _rollout(eng, actions):
    """reset + one env step per entry of `actions` (rows: the envs of the handle); every output and the state after each call"""
    eng.env_reset()
    out = [eng.get("obs"), eng.get("qpos"), eng.get("eq_active"), eng.get("eq_data"), eng.get("group")]
    for a in actions:
        out += list(eng.env_step_host(np.ascontiguousarray(a)))
        out += [eng.get("qpos"), eng.get("qvel"), eng.get("eq_active"), eng.get("group"), eng.get("mt_state"), eng.get("mt_pos")]
    return out


@pytest.mark.parametrize("gpu", BACKENDS)
def test_options_per_env_equal_handles_of_their_own(lack, gpu):
    """envs with assembled / nothing / assembled + preassembled 1 / assembled + a recorded start in one handle equal, bit for bit, one-env
    handles seeded as those envs, over reset + 5 steps with an auto-reset (max_episode_steps 3); on the GPU 64 envs cycle through the four,
    so that every block mixes them"""
    st = _assembled_state(lack)
    kinds = ["assembled", "default", "prefix", "init_state"]
    n = 64 if gpu else 4

    def setup(eng, kind, envs):
        if kind != "default":
            eng.set_reset_options(assembled=True, envs=envs)
        if kind == "prefix":
            k = np.zeros(eng.N, np.int64)
            k[envs] = 1
            eng.set_subtask(k)

    cfg = dict(max_episode_steps=3)
    eng = _engine(lack, n, gpu, cfg=cfg)
    eng.set_init_qpos([st if kinds[i % 4] == "init_state" else None for i in range(n)])
    for j, kind in enumerate(kinds):
        setup(eng, kind, np.arange(j, n, 4))
    actions = np.random.RandomState(7).uniform(-1, 1, (5, n, eng.act_dim)).astype(np.float32)
    mixed = _rollout(eng, actions)
    assert (eng.get("episode_length")[:, 0] == 2).all()  # the auto-reset after step 3 ran
    for j in sorted({0, 1, 2, 3, n - 4, n - 3, n - 2, n - 1}):
        own = _engine(lack, 1, gpu, cfg=dict(cfg, seed=123 + j))
        if kinds[j % 4] == "init_state":
            own.set_init_qpos(st)
        setup(own, kinds[j % 4], [0])
        ref = _rollout(own, actions[:, j : j + 1])
        for x, y in zip(mixed, ref):
            assert np.array_equal(np.asarray(x)[j], np.asarray(y)[0]), (kinds[j % 4], j)


@pytest.mark.parametrize("gpu", BACKENDS)
def test_switching_assembled_off_returns_to_random_placement(lack, gpu):
    """an assembled reset, then the option off: the next reset places the parts at random again, and both resets draw from the generator
    exactly as the CPU env's does across the switch"""
    eng = _engine(lack, 1, gpu, assembled=True)
    e = _oracle(lack, "sparse", assembled=True)
    eng.env_reset()
    e.reset()
    _assert_reset_equal(eng, 0, e, "assembled")
    eng.set_reset_options(assembled=False)
    e.assembled = False
    eng.env_reset()
    e.reset()
    _assert_reset_equal(eng, 0, e, "off")
    assert (eng.get("eq_active")[0] == 0).all() and list(eng.get("group")[0]) == list(range(e.npart)) and e.moved == list(range(e.npart))


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("ik", [False, True], ids=["sparse", "ik"])
def test_default_changes_nothing(lack, gpu, ik):
    """assembled=False passed, or set, leaves reset + 5 steps bit-identical to an untouched handle"""
    from test_obs_layout import _run

    plain = _engine(lack, 2, gpu, ik=ik)
    passed = _engine(lack, 2, gpu, ik=ik, assembled=False)
    set_ = _engine(lack, 2, gpu, ik=ik)
    set_.set_reset_options(assembled=False)
    runs = [_run(x) for x in (plain, passed, set_)]
    for r in runs[1:]:
        for x, y in zip(runs[0], r):
            assert x.dtype == y.dtype and np.array_equal(x, y)


# ------------------------------------------------------------------ surfaces
def test_config_keys_and_refusals(lack):
    """split_config passes assembled on (and leaves it out at its default); the C-ABI refuses values outside {0, 1}; the Cursor env and an
    engine of the Cursor agent refuse it"""
    from furniture_b200.cursor_env import FurnitureCursorEnvB200
    from furniture_b200.engine import Engine
    from furniture_b200.env import build_engine, split_config, split_dense_config

    _, over, ignored = split_config(dict(assembled=True, port=1))
    assert over == dict(assembled=True) and ignored == ["port"]
    _, over, ignored = split_config(dict(assembled=False))
    assert over == {} and ignored == []
    _, over, _, ignored = split_dense_config(dict(assembled=True))
    assert over["assembled"] is True and ignored == []
    eng = _engine(lack, 2, False)
    assert (eng.get("assembled") == 0).all()
    for bad in (2, -1):
        with pytest.raises(RuntimeError):
            eng.set("assembled", bad)
    cursor = mjcf.load_scene("Cursor", "toy_table")
    ce = Engine(cursor, 1, lib_path=build_emu())
    with pytest.raises(ValueError):
        ce.set_reset_options(assembled=True)
    with pytest.raises(ValueError):
        Engine(cursor, 1, lib_path=build_emu(), assembled=True)
    with pytest.raises(ValueError):
        build_engine("Cursor", "toy_table", 1, lib_path=build_emu(), assembled=True)
    with pytest.raises(ValueError):
        FurnitureCursorEnvB200("toy_table", lib_path=build_emu(), assembled=True)


@pytest.mark.parametrize("gpu", BACKENDS)
def test_pair_only_object_ob_is_zero_on_an_assembled_start(lack, gpu):
    """object_ob_all=False: with every part in one group no subtask is left, so object_ob is 14 zeros"""
    from test_obs_layout import _engine as layout_engine

    eng = layout_engine(lack, 2, gpu, object_ob_all=False)
    eng.set_reset_options(assembled=True)
    eng.env_reset()
    cols, _ = eng.obs_columns()
    ob = eng.get("obs")[:, cols["object_ob"]]
    assert ob.shape == (2, 14) and (ob == 0).all() and (eng.get("subtask_part") == -1).all()


def test_scene_file_takes_the_field_through_the_c_abi(lack):
    """a handle created by fe_create_from_file from a shipped scene file takes `assembled` through fe_set_field, and its reset then equals
    the Python-built handle's: every weld on, the parts where the model's link frames put them"""
    from furniture_b200.engine import default_config

    L = C.CDLL(build_emu())
    L.fe_last_error.restype = C.c_char_p
    L.fe_last_error.argtypes = [C.c_void_p]
    cfg = default_config(maxcon=44)
    h = C.c_void_p()
    path = os.path.join(ROOT, "furniture_b200", "compiled", "Sawyer_table_lack_0825.feb").encode()
    assert L.fe_create_from_file(path, C.byref(cfg), 1, 0, C.byref(h)) == 0, L.fe_last_error(None)
    one = np.ones(1, np.int32)
    assert L.fe_set_field(h, b"assembled", one.ctypes.data_as(C.c_void_p), C.c_size_t(4)) == 0, L.fe_last_error(h)
    assert L.fe_env_reset(h, None, None, None) == 0
    q = np.empty(lack.nq, np.float32)
    assert L.fe_get_field(h, b"qpos", q.ctypes.data_as(C.c_void_p), C.c_size_t(q.nbytes)) == 0
    ea = np.empty(lack.neq, np.int32)
    assert L.fe_get_field(h, b"eq_active", ea.ctypes.data_as(C.c_void_p), C.c_size_t(ea.nbytes)) == 0
    L.fe_destroy(h)
    eng = _engine(lack, 1, False, cfg=dict(maxcon=44), assembled=True)
    eng.env_reset()
    assert (ea == 1).all() and np.array_equal(q, eng.get("qpos")[0])


@pytest.mark.gpu
def test_make_vec_env_gym_and_the_mixed_batch():
    """the config key through make_vec_env and the gym env, and every bucket of a mixed batch"""
    from furniture_b200.env import MixedFurnitureEnv, make_vec_env
    from furniture_b200.gym_api import FurnitureGymB200

    env = make_vec_env("IKEASawyer-v0", 2, dict(assembled=True, port=1))
    assert env.ignored_config == ["port"] and (env.engine.get("assembled") == 1).all()
    env.reset()
    assert (env.engine.get("eq_active") == 1).all()
    env.close()
    g = FurnitureGymB200("IKEASawyer-v0", assembled=True)
    assert int(g.engine.get("assembled")[0, 0]) == 1
    mixed = MixedFurnitureEnv(["table_lack_0825", "table_klubbo_0740"], 2, assembled=True)
    assert all((b.engine.get("assembled") == 1).all() for b in mixed.buckets)
    mixed.close()
