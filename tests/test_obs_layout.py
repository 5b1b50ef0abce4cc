"""The observation flags robot_ob / object_ob / object_ob_all / subtask_ob (furniture.py:103-107, :215-252, :1344-1387) and each env's current
subtask (_get_next_subtask, :2723-2759; the dense env's _update_reward_variables, furniture_sawyer_dense.py:149-162), tracked inside the kernels.

`emu` runs the lane-emulated build on the CPU, `cuda` the sm_90a library (marked gpu).  The CPU env oracle (oracle/obs_layout_oracle.py) is
checked against the reference's own _get_obs / observation_space / _get_next_subtask (tests/golden/obs_layout.npz), the device against the
oracle.
"""
import os
import types

import numpy as np
import pytest

from furniture_b200 import mjcf
from furniture_b200.engine import OBS_DEFAULTS, Engine, default_config, obs_columns
from oracle.init_state_oracle import InitStateEnv
from oracle.obs_layout_oracle import ObsLayoutDenseEnv, ObsLayoutEnv, ObsLayoutIKEnv, ObsLayoutMixin
from oracle.ref_env import DenseCfg
from parity_util import build_emu
from test_dense_reward import DENSE_BASE, PREV_KEYS
from test_env_parity import _grasp_and_align_state, _sync_oracle_from_engine

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]
HERE = os.path.dirname(os.path.abspath(__file__))
FLAGS = ("robot_ob", "object_ob", "object_ob_all", "subtask_ob")
PAIR_ONLY = dict(object_ob_all=False, subtask_ob=True)
LAYOUTS = [dict(), PAIR_ONLY, dict(robot_ob=False, subtask_ob=True), dict(object_ob=False, subtask_ob=True), dict(object_ob_all=False)]
LAYOUT_IDS = ["default", "pair+subtask", "no_robot+subtask", "no_object+subtask", "pair"]


@pytest.fixture(scope="module")
def golden():
    g = np.load(os.path.join(HERE, "golden", "obs_layout.npz"))
    return {k: g[k] for k in g.files}


@pytest.fixture(scope="module")
def lack():
    return mjcf.load_scene("Sawyer", "table_lack_0825")


def _engine(m, n, gpu, dense=False, ik=False, cfg=None, **flags):
    from furniture_b200.dense import dense_config
    from furniture_b200.ik import ik_config

    kw = dict(config=default_config(**dict(DENSE_BASE if dense else {}, **(cfg or {}))), dense=dense_config() if dense else None, ik=ik_config(m) if ik else None,
              obs_layout=flags)
    return Engine(m, n, device=0, **kw) if gpu else Engine(m, n, lib_path=build_emu(), **kw)


def _pair(eng, i):
    return tuple(int(x) for x in eng.get("subtask_part")[i])


def _oracle_pair(e):
    return (e.subtask_part1, e.subtask_part2)


# ------------------------------------------------------------------ the oracle against the reference's own code
class _Tagged(InitStateEnv):
    """the base row of the stand-in of tools/make_golden_obs_layout.py: tagged part poses and robot readings"""

    def obs(self):
        parts = [100.0 * i + np.arange(1.0, 8.0) for i in range(self.npart)]
        robot = []
        for a, (arm, site) in enumerate(((0, 1), (20, 2))[: self.narms]):
            robot += [1000.0 + arm + np.arange(7), 2000.0 + arm + np.arange(7), 1000.0 + arm + 7 + np.arange(2), 3000.0 + 10 * site + np.arange(3),
                      4000.0 + 10 * a + np.array([1.0, 2.0, 3.0, 0.0]), 5000.0 + 10 * site + np.arange(3), 6000.0 + 10 * site + np.arange(3)]
        return np.concatenate(parts + robot)


class _TaggedLayoutEnv(ObsLayoutMixin, _Tagged):
    pass


def test_oracle_reproduces_the_reference_obs_layout(golden):
    """every golden case: the subtask pair after the scripted merges, and the obs dict's keys, order, shapes and values under the case's flags and
    control type; the host's column map (obs_columns) gives the reference's observation_space"""
    g = golden
    envs = {}
    for j in range(len(g["case_row"])):
        furniture, agent = str(g["case_furniture"][j]), str(g["case_agent"][j])
        if furniture not in envs:
            envs[furniture] = _TaggedLayoutEnv(mjcf.load_scene(agent, furniture))
        e = envs[furniture]
        e.group = list(range(e.npart))
        merges = [tuple(int(x) for x in ab.split("-")) for ab in str(g["case_merges"][j]).split(";") if ab]
        for a, b in merges:
            e.group[e._find(a)] = e._find(b)
            e._get_next_subtask()
        e._get_next_subtask()
        assert list(_oracle_pair(e)) == list(g["case_pair"][j]), (j, furniture, merges)
        flags = dict(zip(FLAGS, (bool(x) for x in g["case_flags"][j])))
        e.set_obs_layout(**flags)
        control = str(g["case_control"][j])
        d = e.obs_dict(e.obs(), control)
        assert ",".join(d) == str(g["case_keys"][j]), (j, list(d), g["case_keys"][j])
        assert ",".join(str(len(v)) for v in d.values()) == str(g["case_shapes"][j]), j
        want = [np.array([float(x) for x in s.split(",")]) if s else np.zeros(0) for s in str(g["case_row"][j]).split(";")] if d else []
        for (k, v), w in zip(d.items(), want):
            assert np.array_equal(v, w), (j, k, v, w)
        sc = types.SimpleNamespace(npart=e.npart, narms=e.narms, robot_ob_dim=e.narms * 29, phase_ob=0)
        cols = obs_columns(sc, 0 if control == "impedance" else 14, **flags)
        space = ",".join("%s:%d" % (k, len(range(1000)[c]) if isinstance(c, slice) else len(c)) for k, c in cols.items())
        assert space == str(g["case_space"][j]), (j, space, g["case_space"][j])


def test_oracle_dense_pairs_follow_the_recipe(golden, lack):
    """_update_reward_variables sets the recipe step's (leg, table): the oracle's dense env, started at every subtask k, holds the golden pair"""
    e = ObsLayoutDenseEnv(lack, DenseCfg())
    for k, want in enumerate(golden["dense_pairs"]):
        e.dense.preassembled = list(range(k))
        e.dense.begin_episode()
        assert list(_oracle_pair(e)) == list(want), k


# ------------------------------------------------------------------ the device against the CPU env
def _oracle(m, kind, flags):
    e = {"sparse": ObsLayoutEnv, "baxter": ObsLayoutEnv, "dense": lambda m: ObsLayoutDenseEnv(m, DenseCfg()), "ik": ObsLayoutIKEnv}[kind](m)
    e.set_obs_layout(**flags)
    return e


def _sync_ik(e, eng, i):
    hl, ikc = eng.scene.hand_link[0], eng.ik
    lpos, lquat = eng.get("link_xpos")[i], eng.get("link_xquat")[i]
    R = mjcf.q_to_mat(lquat[4 * hl : 4 * hl + 4].astype(np.float64))
    hp = lpos[3 * hl : 3 * hl + 3].astype(np.float64) + R @ np.array(ikc.hand_pos[:])
    hq = mjcf.q_norm(mjcf.q_mul(lquat[4 * hl : 4 * hl + 4].astype(np.float64), np.array(ikc.hand_quat[:], dtype=np.float64)))
    e.ik.sync(hp, hq)


@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("kind", ["sparse", "dense", "ik", "baxter"])
@pytest.mark.parametrize("flags", LAYOUTS[1:4], ids=LAYOUT_IDS[1:4])
def test_device_obs_equals_the_cpu_env(lack, gpu, kind, flags):
    """reset + 3 random steps: the row's layout, the pair and subtask_ob exactly, the poses at the parity tolerance"""
    m = mjcf.load_scene("Baxter", "table_lack_0825") if kind == "baxter" else lack
    n = 2
    eng = _engine(m, n, gpu, dense=kind == "dense", ik=kind == "ik", **flags)
    eng.env_reset()
    envs = [_oracle(m, kind, flags) for _ in range(n)]
    obs0 = eng.get("obs")
    for i, e in enumerate(envs):
        e.reset()
        _sync_oracle_from_engine(e, eng, i)
        e.sim.qfrc_bias[: e.nr] = eng.get("qfrc_bias")[i]
        if kind == "dense":
            e.dense.begin_episode()
        if kind == "ik":
            _sync_ik(e, eng, i)
        assert _pair(eng, i) == _oracle_pair(e), (i, _pair(eng, i), _oracle_pair(e))
        assert obs0.shape[1] == len(e.obs()), i  # the values after a reset differ by the synced oracle's fresh forward pass (test_env_parity)
    rng = np.random.RandomState(5)
    for k in range(3):
        a = rng.uniform(-1, 1, (n, eng.act_dim)).astype(np.float32)
        a[:, -1] = -0.5
        obs, rew, done, info = eng.env_step_host(a)
        for i, e in enumerate(envs):
            ob, r, d, _ = e.step(a[i].astype(np.float64))
            assert _pair(eng, i) == _oracle_pair(e)
            assert np.abs(obs[i] - ob).max() < 2e-4, (k, i, np.abs(obs[i] - ob).max())
            if flags.get("subtask_ob"):
                c = obs_columns(eng.scene, 0, **dict(OBS_DEFAULTS, **flags))["subtask_ob"]
                assert list(obs[i][c]) == [float(x + 1) for x in _oracle_pair(e)]


@pytest.mark.parametrize("gpu", BACKENDS)
def test_connect_moves_the_pair_in_that_env_only(lack, gpu):
    """grasp -> connect on env 0 (env 1 holds still): env 0's object_ob switches to the next weld's parts and its subtask_ob with it, as the CPU
    env's; env 1 keeps the first weld's pair"""
    m = lack
    env = ObsLayoutEnv(m)
    env.set_obs_layout(**PAIR_ONLY)
    env.reset()
    q = _grasp_and_align_state(m, env)
    env.nsub = 1
    env.sim.qvel[:] = 0; env.sim.qacc_warmstart[:] = 0; env.sim.ctrl[:] = 0
    env.sim.forward()
    eng = _engine(m, 2, gpu, cfg=dict(nsub=1), **PAIR_ONLY)
    eng.env_reset()
    before = _pair(eng, 0)
    assert before == _pair(eng, 1) == _oracle_pair(env)
    eng.set("qpos", q); eng.set("qvel", np.zeros(m.nv)); eng.set("qacc_warmstart", np.zeros(m.nv))
    eng.forward()
    a = np.zeros((2, eng.act_dim), np.float32)
    a[:, -2] = 1.0
    a[0, -1], a[1, -1] = 1.0, -1.0
    obs, rew, done, info = eng.env_step_host(a)
    ob, r, d, inf = env.step(a[0].astype(np.float64))
    assert inf["num_connected"] == 1 and info[0][0] == 1 and info[1][0] == 0
    assert _pair(eng, 0) == _oracle_pair(env) != before and _pair(eng, 1) == before
    assert list(obs[0][14:16]) == [float(x + 1) for x in _oracle_pair(env)] and list(obs[1][14:16]) == [float(x + 1) for x in before]
    assert np.abs(obs[0] - ob).max() < 1e-3


@pytest.mark.parametrize("gpu", BACKENDS)
def test_dense_connecting_step_shows_the_next_weld_then_the_recipe_pair(lack, gpu):
    """the dense env attaches the recipe's first leg: the connecting step's observation shows _get_next_subtask's pair (the observation is taken
    before _compute_reward, furniture_sawyer.py:66-84), the next step's the recipe's next (leg, table) -- device and CPU env alike"""
    m = lack
    cfg = DenseCfg()
    cfg.auto_align = True
    env = ObsLayoutDenseEnv(m, cfg)
    env.set_obs_layout(**PAIR_ONLY)
    env.reset()
    q = _grasp_and_align_state(m, env, leg=1, leg_site="leg-table,0,90,180,270,conn_site2", table_site="table-leg,0,90,180,270,conn_site2",
                               arm_qpos=[-0.28, -0.9, 0.0, 1.86, 0.0, 0.6, 1.57])
    env.nsub = 1
    env.sim.qvel[:] = 0; env.sim.qacc_warmstart[:] = 0; env.sim.ctrl[:] = 0
    env.sim.forward()
    env.dense.begin_episode()
    eng = _engine(m, 1, gpu, dense=True, cfg=dict(nsub=1, auto_align=1), **PAIR_ONLY)
    eng.env_reset()
    recipe0 = _pair(eng, 0)
    assert recipe0 == _oracle_pair(env) == (1, 4)
    eng.set("qpos", q); eng.set("qvel", np.zeros(m.nv)); eng.set("qacc_warmstart", np.zeros(m.nv))
    eng.forward()
    st = eng.get("dense_state").copy()
    raw = bytearray(st[0].tobytes())
    ints, dbl = np.frombuffer(raw[:32], np.int32).copy(), np.frombuffer(raw[32:], np.float64).copy()
    o = env.dense
    ints[:7] = [o.phase, o.subtask, 0, 0, 0, 0, 0]
    dbl[0:3], dbl[3:6], dbl[6:9] = o.table_site0, o.leg0, o.lift_target
    for k, name in enumerate(PREV_KEYS):
        dbl[12 + k] = o.prev.get(name, 0.0)
    eng.set("dense_state", np.frombuffer(ints.tobytes() + dbl.tobytes(), np.uint8)[None].view(st.dtype).reshape(st.shape))
    a = np.zeros((1, eng.act_dim), np.float32)
    a[:, -2], a[:, -1] = 1.0, -1.0
    obs, *_ = eng.env_step_host(a)  # the held leg is noticed
    ob, *_ = env.step(a[0].astype(np.float64))
    assert list(obs[0][14:16]) == list(ob[14:16]) == [2.0, 5.0]
    a[:, -1] = 1.0
    obs, rew, done, info = eng.env_step_host(a)  # connects: weld order's next pair in this step's observation
    ob, r, d, inf = env.step(a[0].astype(np.float64))
    assert inf["num_connected"] == 1 and env.dense.subtask == 1 and info[0][0] == 1 and not done[0]
    nxt = tuple(int(x) - 1 for x in ob[14:16])
    assert list(obs[0][14:16]) == list(ob[14:16]) and nxt != (2, 4), nxt
    assert _pair(eng, 0) == _oracle_pair(env) == (2, 4)  # the recipe's second (leg, table), shown from the next step on
    a[:, -1] = -1.0
    obs, *_ = eng.env_step_host(a)
    ob, *_ = env.step(a[0].astype(np.float64))
    assert list(obs[0][14:16]) == list(ob[14:16]) == [3.0, 5.0]
    assert np.abs(obs[0] - ob).max() < 1e-3


# ------------------------------------------------------------------ starts mid-assembly, per env
@pytest.mark.parametrize("gpu", BACKENDS)
@pytest.mark.parametrize("dense", [False, True], ids=["sparse", "dense"])
def test_preassembled_starts_hold_the_oracle_pair_per_env(lack, gpu, dense):
    """one handle, env i preassembled k = i: each env's pair after the reset is the oracle's for that k"""
    m = lack
    ks = [0, 1, 2]
    eng = _engine(m, 3, gpu, dense=dense, **PAIR_ONLY)
    eng.set_subtask(np.array(ks))
    eng.env_reset()
    obs = eng.get("obs")
    for i, k in enumerate(ks):
        e = ObsLayoutDenseEnv(m, DenseCfg()) if dense else ObsLayoutEnv(m)
        e.set_obs_layout(**PAIR_ONLY)
        e.set_subtask(k)
        e.reset()
        assert _pair(eng, i) == _oracle_pair(e), (k, _pair(eng, i), _oracle_pair(e))
        assert list(obs[i][14:16]) == [float(x + 1) for x in _oracle_pair(e)]
    if dense:
        assert [_pair(eng, i) for i in range(3)] == [(1, 4), (2, 4), (3, 4)]  # the recipe's steps k (tests/golden/obs_layout.npz dense_pairs)


@pytest.mark.parametrize("gpu", BACKENDS)
def test_start_from_a_recorded_mid_assembly_state_holds_the_oracle_pair(lack, gpu):
    """a recorded state two connections in, started with preassembled 2 and with the whole assembly preassembled: the pair is the oracle's,
    and the finished assembly shows the zero object_ob"""
    from test_init_states import _mid_assembly_state

    m = lack
    st = _mid_assembly_state(m)
    eng = _engine(m, 2, gpu, **PAIR_ONLY)
    eng.set_init_qpos(st)
    eng.set_subtask(np.array([2, 4]))
    eng.env_reset()
    obs = eng.get("obs")
    for i, k in enumerate((2, 4)):
        e = ObsLayoutEnv(m)
        e.set_obs_layout(**PAIR_ONLY)
        e.set_init_qpos(st)
        e.set_subtask(k)
        e.reset()
        assert _pair(eng, i) == _oracle_pair(e), (k, _pair(eng, i), _oracle_pair(e))
    assert _pair(eng, 1) == (-1, -1) and (obs[1][:14] == 0).all() and list(obs[1][14:16]) == [0.0, 0.0]


# ------------------------------------------------------------------ the default layout, the packed rows, the C-ABI
def _run(eng, steps=5, seed=3):
    eng.env_reset()
    out = [eng.get("obs")]
    rng = np.random.RandomState(seed)
    for _ in range(steps):
        a = rng.uniform(-1, 1, (eng.N, eng.act_dim)).astype(np.float32)
        a[:, -1] = -0.5
        out += list(eng.env_step_host(a))
    return out + list(eng.get_state()) + [eng.get("num_connected"), eng.get("episode_length")]


@pytest.mark.parametrize("gpu", BACKENDS)
def test_default_flags_change_nothing(lack, gpu):
    """an untouched handle, one with the default flags passed, one with fe_set_obs_layout(1, 1, 1, 0) called: bit-identical obs, reward, done,
    info and state over reset + 5 steps"""
    m = lack
    plain = _engine(m, 2, gpu)
    explicit = _engine(m, 2, gpu, **OBS_DEFAULTS)
    called = _engine(m, 2, gpu)
    called.set_obs_layout(True, True, True, False)
    assert called.scene.obs_layout == 0 and plain.obs_dim == explicit.obs_dim == called.obs_dim == 35 + 29
    ref = _run(plain)
    for eng in (explicit, called):
        for x, y in zip(ref, _run(eng)):
            assert x.dtype == y.dtype and np.array_equal(x, y)


@pytest.mark.gpu
def test_make_vec_env_with_the_reference_defaults_is_todays_env():
    """make_vec_env with the reference's default observation flags (config/furniture.py:228-258) builds today's env: same obs dict, bits and
    all, and the flags are no longer reported as ignored"""
    import argparse

    import torch

    from furniture_b200.env import make_vec_env

    ns = argparse.Namespace(furniture_name="table_lack_0825", robot_ob=True, object_ob=True, object_ob_all=True, subtask_ob=False, visual_ob=False,
                            port=1050, seed=7)
    a_env = make_vec_env("IKEASawyer-v0", 4, ns)
    b_env = make_vec_env("IKEASawyer-v0", 4, {"furniture_name": "table_lack_0825", "seed": 7})
    assert a_env.ignored_config == ["port", "visual_ob"] and list(a_env.observation_space) == ["object_ob", "robot_ob"]
    oa, ob_ = a_env.reset(), b_env.reset()
    for _ in range(5):
        act = torch.rand((4, a_env.act_dim), device=a_env.device) * 2 - 1
        act[:, -1] = -1
        oa, ra, da, ia = a_env.step(act)
        ob_, rb, db, ib = b_env.step(act)
        assert list(oa) == list(ob_) and all(torch.equal(oa[k], ob_[k]) for k in oa)
        assert torch.equal(ra, rb) and torch.equal(da, db) and torch.equal(ia, ib)
    a_env.close(); b_env.close()


@pytest.mark.gpu
def test_packed_rows_equal_the_step_obs_under_the_new_layout(lack):
    """fe_env_step_packed writes rows [obs | reward | done] of stride obs_dim + 2 under the new layout, equal to fe_env_step's"""
    import torch

    m = lack
    outs = []
    for packed in (False, True):
        eng = _engine(m, 4, True, **PAIR_ONLY)
        assert eng.obs_dim == 14 + 2 + 29
        eng.env_reset()
        rng = np.random.RandomState(2)
        for _ in range(3):
            a = torch.tensor(rng.uniform(-1, 1, (4, eng.act_dim)).astype(np.float32), device="cuda")
            a[:, -1] = -1
            if packed:
                p = torch.empty((4, eng.obs_dim + 2), device="cuda")
                eng.env_step_packed(a.data_ptr(), p.data_ptr())
                torch.cuda.synchronize()
                row = p.cpu().numpy()
                assert np.array_equal(row[:, : eng.obs_dim], eng.get("obs"))
            else:
                o = torch.empty((4, eng.obs_dim), device="cuda")
                r = torch.empty(4, device="cuda")
                d = torch.empty(4, dtype=torch.uint8, device="cuda")
                eng.env_step_dev(a.data_ptr(), o.data_ptr(), r.data_ptr(), d.data_ptr(), 0)
                torch.cuda.synchronize()
                row = np.concatenate([o.cpu().numpy(), r.cpu().numpy()[:, None], d.cpu().numpy()[:, None].astype(np.float32)], 1)
            outs.append(row)
        eng.close()
    for x, y in zip(outs[:3], outs[3:]):
        assert np.array_equal(x, y)


@pytest.mark.gpu
def test_mixed_batch_pair_only_is_14_wide_with_per_model_subtask_ob():
    """MixedFurnitureEnv over three models with object_ob_all=False: object_ob is 14 wide, nothing padded, and subtask_ob is each model's pair"""
    from furniture_b200.env import BatchedFurnitureEnv, MixedFurnitureEnv

    names = ["table_lack_0825", "chair_ingolf_0650", "block"]
    mixed = MixedFurnitureEnv(names, 2, **PAIR_ONLY)
    assert list(mixed.reset()) == ["object_ob", "subtask_ob", "robot_ob"] and mixed.object_ob_dim == 14 and mixed.obs_dim == 14 + 2 + 29
    obs = mixed.reset()
    for name, off, b in zip(names, mixed.offsets, mixed.buckets):
        alone = BatchedFurnitureEnv("Sawyer", name, 2, **PAIR_ONLY)
        od = alone.reset()
        pair = b.engine.get("subtask_part")
        assert (obs["subtask_ob"][off : off + 2].cpu().numpy() == pair + 1).all(), name
        assert obs["object_ob"].shape[1] == 14 and od["object_ob"].shape[1] == 14
        alone.close()
    mixed.close()


def test_the_entry_point_refuses_what_it_must(lack):
    """fe_set_obs_layout: a flag outside {0, 1} and any call after the first reset or step are refused; the gym surface and split_config take the
    flags, and hand subtask_ob out like the other entries"""
    from furniture_b200.env import split_config
    from furniture_b200.gym_api import FurnitureGymB200

    eng = _engine(lack, 1, False)
    for bad in ((2, 1, 1, 0), (1, -1, 1, 0), (1, 1, 1, 3)):
        with pytest.raises(RuntimeError, match="0 or 1"):
            eng.set_obs_layout(*bad)
    eng.set_obs_layout(True, True, False, True)
    assert eng.obs_dim == 14 + 2 + 29 and eng.field_info("obs")[0] == 45
    eng.env_reset()
    with pytest.raises(RuntimeError, match="fixed"):
        eng.set_obs_layout(True, True, True, False)
    assert eng.obs_dim == 45
    name, over, ignored = split_config(dict(robot_ob=True, object_ob=True, object_ob_all=False, subtask_ob=True, port=1))
    assert over == dict(object_ob_all=False, subtask_ob=True) and ignored == ["port"]
    env = FurnitureGymB200(name="FurnitureSawyerEnv", lib_path=build_emu(), nsub=1, object_ob_all=False, subtask_ob=True)
    ob = env.reset()
    assert list(ob) == ["object_ob", "subtask_ob", "robot_ob"] and ob["subtask_ob"].dtype == np.float64
    assert list(ob["subtask_ob"]) == [1.0, 5.0] and [v[0] for v in env.observation_space.values()] == [14, 2, 29]
    env.close()
    ik = FurnitureGymB200(name="FurnitureBaxterEnv", furniture_name="table_lack_0825", lib_path=build_emu(), nsub=1, control_type="ik", robot_ob=True,
                          subtask_ob=True, object_ob=False)
    ob = ik.reset()
    assert [len(v) for v in ob.values()] == [2, 30]  # each arm's 15-number tail after the two subtask numbers
    row = ik.engine.get("obs")[0]
    assert np.array_equal(ob["robot_ob"], np.concatenate([row[2 + 14 : 2 + 29], row[2 + 29 + 14 : 2 + 58]]).astype(np.float64))
    ik.close()
