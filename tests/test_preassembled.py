"""Episodes that start part-way through the assembly: `preassembled` / set_subtask (furniture.py:204-213, :1477-1481, :1542-1566;
furniture_sawyer_dense.py:128-139), per env, inside the reset kernel.

Golden: tests/golden/preassembled.npz = the reference's own _project_connector_quat, _success_num_conn statement and
_reset_reward_variables / first _compute_reward (tools/make_golden_preassembled.py).  `emu` runs the lane-emulated build on the CPU,
`cuda` the sm_90a library (marked gpu).
"""
import json
import os

import numpy as np
import pytest

from furniture_b200 import mjcf
from oracle import assembly_oracle as A
from oracle import dense_oracle as D
from oracle.preassembled_oracle import PreassembledDenseEnv, PreassembledEnv, project_connector_quat
from oracle.ref_env import Cfg, DenseCfg
from parity_util import build_emu, make_engine, quat_err
from test_dense_reward import PREV_KEYS, _adopt_device_anchors, _assert_same_machine, _dense_engine, _dense_state
from test_env_parity import _grasp_and_align_state, _sync_oracle_from_engine

HERE = os.path.dirname(os.path.abspath(__file__))
BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]


@pytest.fixture(scope="module")
def golden():
    g = np.load(os.path.join(HERE, "golden", "preassembled.npz"))
    return {k: g[k] for k in g.files}


@pytest.fixture(scope="module")
def model():
    return mjcf.load_scene("Sawyer", "table_lack_0825")


# ------------------------------------------------------------------ the oracle and the device machine against the reference's answers
def test_project_connector_quat_equals_the_reference_bit_for_bit(golden):
    g = golden
    nan = 0
    with np.errstate(invalid="ignore"):
        for m1, m2, ang, has, want in zip(g["q_m1"], g["q_m2"], g["q_angle"], g["q_has_angle"], g["q_tq"]):
            got = project_connector_quat(m1, m2, float(ang) if has else None)
            assert np.array_equal(got, want, equal_nan=True), (m1, m2, ang, has, got, want)
            nan += int(np.isnan(want).any())
    assert nan > 20 and (~g["q_has_angle"]).sum() > 300  # the file does hold cosines that round past +-1


class StartWorld:
    """one golden start (a static world) by name; every grasp-target pair of a leg has its own position"""

    def __init__(self, g, t, recipe):
        self.g, self.t, self.names = g, t, {}
        n = len(recipe["recipe"])
        for s in range(n):
            leg = recipe["recipe"][s][0]
            self.names.setdefault(leg, ("leg_pos", s))
            self.names[recipe["site_recipe"][s][0]] = ("leg_site_pos", s)
            self.names[recipe["site_recipe"][s][1]] = ("table_site_pos", s)
            for i in range(n):
                self.names.setdefault("%s_ltgt_site%d" % (leg, i), ("gl", self.names[leg][1], i))
                self.names.setdefault("%s_rtgt_site%d" % (leg, i), ("gr", self.names[leg][1], i))

    def pos(self, name):
        if name == "griptip_site":
            return self.g["eef"][self.t].copy()
        key = self.names[name]
        return self.g[key[0]][self.t][key[1:]].copy()

    def _mat(self, name):
        if name == "grip_site":
            return self.g["grip_mat"][self.t].reshape(3, 3)
        kind, s = self.names[name][:2]
        return self.g["leg_site_mat" if kind == "leg_site_pos" else "table_site_mat"][self.t, s].reshape(3, 3)

    def up(self, name):
        return self._mat(name)[:, 2].copy()

    def forward(self, name):
        return self._mat(name)[:, 1].copy()

    def finger_contact(self, leg):
        b = bool(self.g["touch"][self.t, self.names[leg][1]])
        return b, b


def _start_cfg(g, t):
    cfg = {k: float(v) for k, v in zip(g["coef_names"], g["coefs"]) if k in D.DEFAULTS}
    cfg.update(diff_rew=bool(g["diff_rew"][t]), reset_robot_after_attach=bool(g["reset_robot_after_attach"][t]), early_termination=False, phase_ob=False)
    return cfg


def test_oracle_starts_an_episode_at_subtask_k_like_the_reference(golden):
    g = golden
    recipes = [json.loads(str(r)) for r in g["recipe_json"]]
    assert np.array_equal(g["goal_success_num_conn"], np.where(g["goal_num_connects"] >= 0, g["goal_num_connects"] + g["goal_k"], g["goal_nparts"] - 1))
    seen = set()
    for t in range(len(g["k"])):
        recipe, k = recipes[int(g["recipe"][t])], int(g["k"][t])
        nparts = len({p for row in recipe["recipe"] for p in row})
        nc = int(g["num_connects"][t])
        goal = nc + k if nc >= 0 else nparts - 1
        assert goal == int(g["success_num_conn"][t])
        orc = D.DenseOracle(StartWorld(g, t, recipe), recipe, _start_cfg(g, t), success_num_conn=goal, preassembled=range(k))
        orc.begin_episode()
        assert (orc.subtask, orc.phase) == (int(g["subtask0"][t]), int(g["phase0"][t])) and orc.subtask == k
        assert orc.gl == "%s_ltgt_site%d" % (recipe["recipe"][k][0], int(g["claimed"][t])), (t, orc.gl)
        r, done, info = orc.step(g["ac"][t], False)
        assert (done, orc.success, orc.phase, orc.subtask) == (bool(g["done"][t]), bool(g["success"][t]), int(g["phase"][t]), int(g["subtask"][t])), t
        assert abs(r - g["reward"][t]) <= 1e-11 * max(1.0, abs(g["reward"][t])), (t, r, g["reward"][t])
        seen.add((int(g["recipe"][t]), k))
    assert len(seen) == sum(len(r["recipe"]) for r in recipes)  # every k of every recipe


def _check_device_starts(eng, g):
    """the device machine through fe_dense_eval: a record with reset = 1 + k starts at subtask k.  Site ids: leg_site s, table_site 8 + s,
    g_l 16 + 4 leg + pair, g_r 32 + 4 leg + pair, griptip 48, grip_site 49; the packed recipe must hold, for subtask k, the pair the reference claimed"""
    from furniture_b200.dense import dense_config, pack_dense_recipe

    recipes = [json.loads(str(r)) for r in g["recipe_json"]]
    n = len(g["k"])
    for t in range(n):
        recipe, k = recipes[int(g["recipe"][t])], int(g["k"][t])
        S = len(recipe["recipe"])
        ids, legs = {}, []
        for s, (leg, _) in enumerate(recipe["recipe"]):
            if leg not in legs:
                legs.append(leg)
            ids[recipe["site_recipe"][s][0]], ids[recipe["site_recipe"][s][1]] = s, 8 + s
        first = {leg: [s for s in range(S) if recipe["recipe"][s][0] == leg][0] for leg in legs}  # the golden file keys a leg's arrays by its first subtask
        for leg in legs:
            for i in range(S):
                ids["%s_ltgt_site%d" % (leg, i)], ids["%s_rtgt_site%d" % (leg, i)] = 16 + 4 * first[leg] + i, 32 + 4 * first[leg] + i
        rc = pack_dense_recipe(recipe, ids.get, lambda leg: first[leg], 48, 49)
        assert rc.gl_site[k] == 16 + 4 * first[recipe["recipe"][k][0]] + int(g["claimed"][t]), (t, "the packed grasp pair of subtask k is not the one a k-prefix start claims")
        spos, smat = np.zeros((2, 50, 3)), np.zeros((2, 50, 9))
        spos[:, 0:4], spos[:, 8:12] = g["leg_site_pos"][t], g["table_site_pos"][t]
        smat[:, 0:4], smat[:, 8:12] = g["leg_site_mat"][t], g["table_site_mat"][t]
        spos[:, 16:32], spos[:, 32:48] = g["gl"][t].reshape(16, 3), g["gr"][t].reshape(16, 3)
        spos[:, 48], smat[:, 49] = g["eef"][t], g["grip_mat"][t]
        ppos = np.stack([g["leg_pos"][t]] * 2)
        touch = np.stack([g["touch"][t]] * 2).astype(np.uint8)
        cfg = _start_cfg(g, t)
        dc = dense_config(**{kk: v for kk, v in cfg.items() if not kk.startswith("alignment")})
        rew, done, info = eng.dense_eval(dc, rc, [0.02, 0.99, 0.99, 0.0], int(g["success_num_conn"][t]), [0], [2], spos, smat, ppos, touch, [1 + k, 0], [0, 0],
                                         np.stack([g["ac"][t]] * 2))
        assert (int(info[0, 0]), int(info[0, 1])) == (int(g["phase0"][t]), k), t
        assert (int(info[1, 0]), int(info[1, 1]), int(done[1] & 1), int(done[1] >> 1)) == (int(g["phase"][t]), int(g["subtask"][t]), int(g["done"][t]), int(g["success"][t])), t
        assert abs(rew[1] - g["reward"][t]) <= 1e-11 * max(1.0, abs(g["reward"][t])), (t, rew[1], g["reward"][t])


@pytest.mark.parametrize("gpu", BACKENDS)
def test_device_machine_starts_an_episode_at_subtask_k_like_the_reference(golden, gpu):
    _check_device_starts(make_engine(mjcf.load_scene("None", "table_lack_0825"), 1, gpu), golden)


# ------------------------------------------------------------------ the device reset against the CPU env
def _engine(m, n, gpu, dense, **cfg):
    return _dense_engine(m, n, gpu, **cfg) if dense else make_engine(m, n, gpu, **cfg)


def _welded_pairs(eng, i):
    sc = eng.scene
    return [(sc.eq_part1[q], sc.eq_part2[q]) for q in np.flatnonzero(eng.get("eq_active")[i])]


def _rel(q, a, b):
    return A.rel_pose(q[9 + 7 * a : 16 + 7 * a].astype(np.float64), q[9 + 7 * b : 16 + 7 * b].astype(np.float64))


RESET_CASES = [pytest.param(False, k, dense, id="emu-k%d-%s" % (k, "dense" if dense else "sparse")) for k in (1, 2, 3) for dense in (False, True)] + \
              [pytest.param(True, 2, dense, id="cuda-k2-%s" % ("dense" if dense else "sparse"), marks=pytest.mark.gpu) for dense in (False, True)]


@pytest.mark.parametrize("gpu,k,dense", RESET_CASES)
def test_preassembled_reset_matches_the_cpu_env(model, gpu, k, dense):
    """the reset kernel with k recipe steps preassembled against the CPU env's reset from the same seed: welds, masks, groups, sites and the
    random stream exactly, poses to fp32 tolerance; then 3 random env steps, whose first reward carries success_reward * k in the sparse env
    (prev_num_connected restarts at 0 while num_connected restarts at k, furniture.py:1473-1474, :525-528)"""
    m, n = model, 2
    eng = _engine(m, n, gpu, dense)
    eng.set_subtask(k)
    eng.env_reset()
    assert (eng.get("flags") == 0).all()
    envs = []
    for i in range(n):
        cfg = DenseCfg() if dense else Cfg()
        cfg.seed = 123 + i
        e = PreassembledDenseEnv(m, cfg) if dense else PreassembledEnv(m, cfg)
        e.set_subtask(k)
        e.reset()
        envs.append(e)
        # integers: exact
        assert list(eng.get("eq_active")[i]) == list(e.sim.eq_active) and int(eng.get("eq_active")[i].sum()) == k
        ct, ca = eng.get("geom_contype")[i], eng.get("geom_conaffinity")[i]
        for j, g in enumerate(eng.em.geom_src):
            assert ct[j] == e.sim.geom_contype[g] and ca[j] == e.sim.geom_conaffinity[g], (i, j)
        assert int(eng.get("num_connected")[i, 0]) == e.num_connected == k and int(eng.get("prev_num_connected")[i, 0]) == 0
        assert set(np.flatnonzero(eng.get("site_connected")[i])) == e.connected_sites and len(e.connected_sites) == 2 * k
        assert list(eng.get("group")[i]) == e.group
        # preassembly draws nothing: the env's generator is where numpy's RandomState(seed + env) is after one reset
        st = e.rng.get_state()
        assert np.array_equal(eng.get("mt_state")[i], st[1]) and int(eng.get("mt_pos")[i, 0]) == st[2]
        # poses: fp32 tolerance (quaternions up to sign: a leg turned by half a turn sits on a branch boundary of lookat_to_quat)
        q = eng.get("qpos")[i]
        for p in range(e.npart):
            a = 9 + 7 * p
            assert np.abs(q[a : a + 3] - e.sim.qpos[a : a + 3]).max() < 5e-4 and quat_err(q[a + 3 : a + 7], e.sim.qpos[a + 3 : a + 7]) < 5e-4, (i, p)
        for w in np.flatnonzero(e.sim.eq_active):
            d, o = eng.get("eq_data")[i].reshape(-1, 7)[w], e.sim.eq_data[7 * w : 7 * w + 7]
            assert np.abs(d[:3] - o[:3]).max() < 5e-4 and quat_err(d[3:], o[3:]) < 5e-4, (i, w)
        if dense:
            ds = _dense_state(eng, i)
            assert (ds["subtask"], ds["phase"]) == (k, e.dense.phase) and e.dense.subtask == k
    rel0 = [{pair: _rel(eng.get("qpos")[i], *pair) for pair in _welded_pairs(eng, i)} for i in range(n)]
    for i, e in enumerate(envs):  # continue from the device's state, as the step parity tests do
        _sync_oracle_from_engine(e, eng, i)
        e.sim.qfrc_bias[: e.nr] = eng.get("qfrc_bias")[i]
        if dense:
            e.dense.begin_episode()
            _assert_same_machine(_dense_state(eng, i), e.dense, ("reset", i), tol=5e-4)  # anchors of the last mj_step's forward pass against a fresh one, as in test_dense_reward
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
            if not dense:
                quirk = 100.0 * k if step == 0 else 0.0
                assert abs(rew[i] - (quirk - 1e-3 * float(np.square(a[i]).sum()))) < 1e-3, (step, i, rew[i])
            else:
                _assert_same_machine(_dense_state(eng, i), e.dense, (step, i))
    for i in range(n):  # every weld holds
        q = eng.get("qpos")[i]
        for pair, r0 in rel0[i].items():
            r1 = _rel(q, *pair)
            assert np.abs(r1[:3] - r0[:3]).max() < 2e-3 and quat_err(r1[3:], r0[3:]) < 2e-3, (i, pair)


# ------------------------------------------------------------------ finishing from a later subtask, and the auto-reset that follows
def _hold_leg_of_step(m, env, s):
    """the CPU env's state after a preassembled reset, rearranged so that the leg of recipe step s sits between the fingers with its connector
    on the table's; the table goes there with every part already welded to it"""
    recipe = json.loads(m.meta["recipe_json"])
    leg = env.parts.index(recipe["recipe"][s][0])
    table = env.parts.index(recipe["recipe"][s][1])
    old = env.sim.qpos.copy()
    grp = [p for p in range(env.npart) if env._find(p) == env._find(table) and p != table]
    q = _grasp_and_align_state(m, env, leg=leg, leg_site=recipe["site_recipe"][s][0], table_site=recipe["site_recipe"][s][1],
                               arm_qpos=[-0.28, -0.9, 0.0, 1.86, 0.0, 0.6, 1.57])
    part = lambda v, p: v[env.part_qadr[p] : env.part_qadr[p] + 7]
    for p in grp:
        rel = A.rel_pose(part(old, table), part(old, p))
        part(q, p)[:3] = part(q, table)[:3] + A._qrotate(part(q, table)[3:], rel[:3])
        part(q, p)[3:] = A._qmul(part(q, table)[3:], rel[3:])
    env.sim.qpos[:] = q
    return q


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("k,num_connects", [(3, None), (1, 1)], ids=["last-subtask", "num_connects-1"])
def test_connecting_from_subtask_k_ends_the_episode_and_the_auto_reset_preassembles_again(model, gpu, k, num_connects):
    """with k legs preassembled, the grasp -> connect script on the leg of recipe step k: the episode ends with success after that one
    connection (the last subtask, or num_connects = 1), and the auto-reset inside the step returns the env to k welded legs at subtask k"""
    m = model
    cfg = DenseCfg()
    cfg.auto_align = True
    env = PreassembledDenseEnv(m, cfg)
    env.set_subtask(k, num_connects)
    env.reset()
    assert env.success_num_conn == (4 if num_connects is None else k + 1) and env.num_subtask() == (4 if num_connects is None else 1)
    eng = _dense_engine(m, 2, gpu, nsub=1, auto_align=1)
    eng.set_subtask(k, num_connects)
    eng.env_reset()
    assert list(eng.num_subtask()) == [env.num_subtask()] * 2
    _sync_oracle_from_engine(env, eng, 0)  # the device's welds and masks
    q = _hold_leg_of_step(m, env, k)
    env.nsub = 1
    env.sim.qvel[:] = 0; env.sim.qacc_warmstart[:] = 0; env.sim.ctrl[:] = 0
    env.sim.forward()
    env.dense.begin_episode()
    assert env.dense.subtask == k
    eng.set("qpos", q); eng.set("qvel", np.zeros(m.nv)); eng.set("qacc_warmstart", np.zeros(m.nv))
    eng.forward()
    st = eng.get("dense_state").copy()
    raw = bytearray(st[0].tobytes())
    ints, dbl = np.frombuffer(raw[:32], np.int32).copy(), np.frombuffer(raw[32:], np.float64).copy()
    o = env.dense
    ints[:7] = [o.phase, o.subtask, 0, 0, 0, 0, 0]
    dbl[0:3], dbl[3:6], dbl[6:9], dbl[9:12] = o.table_site0, o.leg0, o.lift_target, getattr(o, "init_eef", np.zeros(3))
    for j, name in enumerate(PREV_KEYS):
        dbl[12 + j] = o.prev.get(name, 0.0)
    row = np.frombuffer(ints.tobytes() + dbl.tobytes(), np.uint8)
    eng.set("dense_state", np.stack([row, row]).view(st.dtype).reshape(st.shape))
    a = np.zeros((2, eng.act_dim), np.float32)
    a[:, -2], a[:, -1] = 1.0, -1.0
    obs, rew, done, info = eng.env_step_host(a)  # step 1: the held leg is noticed
    ob, r, d, inf = env.step(a[0].astype(np.float64))
    assert env.dense_info["skip_to_lift_leg"] == 1 and not d, "the CPU env did not see a safe grasp: test state is wrong"
    _assert_same_machine(_dense_state(eng, 0), env.dense, "grasp")
    assert not done.any() and (info[:, 0] == k).all()
    a[0, -1] = 1.0  # step 2: env 0 connects
    draws = eng.get("mt_pos")[:, 0].copy()
    obs, rew, done, info = eng.env_step_host(a)
    ob, r, d, inf = env.step(a[0].astype(np.float64))
    assert inf["num_connected"] == k + 1 and d and inf["success"] == 1, "the CPU env did not finish: test state is wrong"
    assert bool(done[0]) and info[0][0] == k + 1 and info[0][1] == 1 and not done[1] and info[1][0] == k
    assert abs(rew[0] - r) < 0.5 + 1e-4 * abs(r) and rew[0] > 9000
    # the auto-reset: k legs welded again, the machine back at subtask k; env 1 goes on
    assert int(eng.get("num_connected")[0, 0]) == k and int(eng.get("eq_active")[0].sum()) == k and int(eng.get("episode_length")[0, 0]) == 0
    assert _dense_state(eng, 0)["subtask"] == k and _dense_state(eng, 1)["subtask"] == k
    assert eng.get("mt_pos")[0, 0] != draws[0] and eng.get("mt_pos")[1, 0] == draws[1]
    z = eng.get("qpos")[0][9 + 2 :: 7]
    assert np.isfinite(eng.get("qpos")[0]).all() and z.min() > 0.0


# ------------------------------------------------------------------ per env, and the untouched path
def _snapshot(eng, i, dense):
    out = [eng.get("qpos")[i], eng.get("obs")[i], eng.get("eq_active")[i], eng.get("mt_state")[i], eng.get("mt_pos")[i]]
    return out + ([eng.get("dense_state")[i]] if dense else [])


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("dense", [False, True], ids=["sparse", "dense"])
def test_every_env_of_a_handle_has_its_own_subtask(model, gpu, dense):
    m = model
    eng = _engine(m, 4, gpu, dense, nsub=2)
    eng.set_subtask([0, 1, 2, 3], [-1, 1, -1, -1])
    assert list(eng.get("preassembled")[:, 0]) == [0, 1, 2, 3] and list(eng.num_subtask()) == [4, 1, 4, 4]
    eng.env_reset()
    assert list(eng.get("num_connected")[:, 0]) == [0, 1, 2, 3]
    for i in range(4):  # env i = env 0 of a handle of its own with scalar k = i and the seed of env i, bit for bit
        one = _engine(m, 1, gpu, dense, nsub=2, seed=123 + i)
        one.set_subtask(i, 1 if i == 1 else None)
        one.env_reset()
        for x, y in zip(_snapshot(eng, i, dense), _snapshot(one, 0, dense)):
            assert np.array_equal(x, y), i
        one.close()
    # set_subtask takes effect at an env's next reset only
    before = [_snapshot(eng, i, dense) for i in range(4)]
    eng.set_subtask(1)
    for i in range(4):
        for x, y in zip(before[i], _snapshot(eng, i, dense)):
            assert np.array_equal(x, y)
    a = np.zeros((4, eng.act_dim), np.float32)
    a[:, -1] = -1
    obs, rew, done, info = eng.env_step_host(a)
    assert list(info[:, 0]) == [0, 1, 2, 3] and not done.any()
    # a masked reset applies it to the masked envs only
    mask = np.array([0, 0, 1, 1], np.uint8)
    if gpu:
        import torch

        mask_dev = torch.as_tensor(mask).cuda()
        eng.env_reset(mask_dev=mask_dev.data_ptr())
    else:
        eng.env_reset(mask_dev=mask.ctypes.data)
    assert list(eng.get("num_connected")[:, 0]) == [0, 1, 1, 1] and list(eng.get("eq_active").sum(axis=1)) == [0, 1, 1, 1]


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("dense", [False, True], ids=["sparse", "dense"])
def test_set_subtask_zero_changes_nothing(model, gpu, dense):
    m = model
    runs = []
    for touch in (False, True):
        eng = _engine(m, 2, gpu, dense)
        if touch:
            eng.set_subtask(0)
        eng.env_reset()
        out = [eng.get("obs").copy()]
        rng = np.random.RandomState(9)
        for _ in range(5):
            a = rng.uniform(-1, 1, (2, eng.act_dim)).astype(np.float32)
            out += list(eng.env_step_host(a))
        out += [eng.get("qpos"), eng.get("mt_state"), eng.get("mt_pos")]
        runs.append(out)
        eng.close()
    for x, y in zip(*runs):
        assert np.array_equal(x, y)


# ------------------------------------------------------------------ host surface
def test_config_keys_and_what_is_refused(model):
    from furniture_b200.env import prefix_length, split_config, split_dense_config
    from furniture_b200.gym_api import FurnitureGymB200

    name, over, ignored = split_config(dict(preassembled=[0, 1], num_connects=1, port=1050))
    assert over == {"preassembled": [0, 1], "num_connects": 1} and ignored == ["port"]
    name, over, ignored = split_config(dict(preassembled=[], num_connects=None))  # the reference's defaults
    assert over == {} and ignored == []
    assert split_dense_config(dict(preassembled=range(3)))[1]["preassembled"] == [0, 1, 2] and prefix_length(None) == 0
    for bad in ([1], [0, 2], [1, 0]):
        with pytest.raises(ValueError):
            split_config(dict(preassembled=bad))
    # the single-env surface mirrors furniture.py:204-213
    env = FurnitureGymB200(name="FurnitureSawyerDenseRewardEnv", lib_path=build_emu(), nsub=1, preassembled=[0, 1])
    assert env.ignored_config == [] and env.num_subtask() == 4
    env.reset()
    assert _dense_state(env.engine, 0)["subtask"] == 2 and int(env.engine.get("num_connected")[0, 0]) == 2
    env.set_subtask(1, num_connects=2)
    assert env.num_subtask() == 2 and int(env.engine.get("num_connected")[0, 0]) == 2  # nothing moves before the next reset
    env.reset()
    assert _dense_state(env.engine, 0)["subtask"] == 1 and int(env.engine.get("eq_active")[0].sum()) == 1
    with pytest.raises(ValueError):
        env.set_subtask(4)  # the dense reward needs a subtask left
    with pytest.raises(ValueError):
        env.set_subtask(-1)
    env.close()
    with pytest.raises(NotImplementedError):  # a furniture without a recipe: the reference's eq_active-only branch is not built
        FurnitureGymB200(name="FurnitureSawyerEnv", furniture_name="swivel_chair_0700", lib_path=build_emu(), preassembled=[0])
    with pytest.raises(NotImplementedError):  # two arms: the scene packs no recipe
        FurnitureGymB200(name="FurnitureBaxterEnv", furniture_name="table_lack_0825", lib_path=build_emu(), preassembled=[0])
    sparse = FurnitureGymB200(name="FurnitureSawyerEnv", furniture_name="table_lack_0825", lib_path=build_emu(), nsub=1)
    sparse.set_subtask(4)  # the sparse env may start fully assembled: its first step reports success
    sparse.reset()
    a = np.zeros(sparse.dof); a[-1] = -1
    _, reward, done, info = sparse.step(a)
    assert done and info["episode_success"] == 1 and abs(reward - (400.0 - 1e-3)) < 1e-3  # success_reward * 4 on the first step, less the ctrl penalty
    sparse.close()


@pytest.mark.gpu
def test_make_vec_env_takes_preassembled():
    from furniture_b200.env import make_vec_env

    env = make_vec_env("IKEASawyerDense-v0", num_env=3, config=dict(preassembled=[0, 1], port=1050))
    assert env.ignored_config == ["port"] and list(env.num_subtask()) == [4, 4, 4]
    env.reset()
    assert [_dense_state(env.engine, i)["subtask"] for i in range(3)] == [2, 2, 2]
    env.set_subtask([0, 1, 3], num_connects=[-1, 1, -1])
    env.reset()
    assert [_dense_state(env.engine, i)["subtask"] for i in range(3)] == [0, 1, 3] and list(env.num_subtask()) == [4, 1, 4]
    env.close()
    with pytest.raises(ValueError):
        make_vec_env("IKEASawyer-v0", config=dict(preassembled=[1, 2]))
