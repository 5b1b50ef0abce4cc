"""The info dict of every env step (FurnitureEnv._compute_reward / _after_step, furniture.py:451-541): the sparse reward's four terms
(field "reward_info") and the record of the episode a step ends (field "episode_info"), written by the step kernels, and the surfaces
that return them as the reference's info dicts.

The CPU env's terms and records are pinned to the reference's own code by tests/golden/step_info.npz (tools/make_golden_step_info.py).
`emu` runs the lane-emulated build on the CPU, `cuda` the sm_90a library (marked gpu)."""
import ctypes as C
import os

import numpy as np
import pytest

from furniture_b200 import mjcf
from furniture_b200.engine import EPISODE_INFO_KEYS, INFO_DIM, REWARD_INFO_KEYS, default_config, packed_columns
from furniture_b200.env import build_engine
from oracle.preassembled_oracle import PreassembledEnv
from oracle.ref_env import Cfg, OracleFurnitureEnv
from parity_util import build_emu, make_engine
from step_info_oracle import EPISODE, TERMS, with_step_info
from test_env_parity import _sync_oracle_from_engine
from test_preassembled import _hold_leg_of_step
from test_reset_options import _cfg
from test_sharded_message import Buffers

BACKENDS = [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)]
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
COEF_KEYS = ("success_reward", "touch_reward", "pick_reward", "ctrl_penalty_coef", "unstable_penalty_coef")
KINDS = {"sparse": ("Sawyer", {}), "ik": ("Sawyer", dict(control_type="ik")), "joint_velocity": ("Sawyer", dict(control_type="joint_velocity")),
         "baxter": ("Baxter", {})}


def _lib(gpu):
    return None if gpu else build_emu()


def _terms_sum(ri):
    """the four terms added in the kernel's order, in float32"""
    return ((ri[:, 0] + ri[:, 1]) + ri[:, 2]) + ri[:, 3]


# ------------------------------------------------------------------ 1. the CPU env against the reference's own code
def test_oracle_step_info_equals_the_reference():
    """every golden step (one and two arms, four coefficient sets x episode lengths 2, 3, 5, 2000, scripted finger / floor contacts,
    connections and unstable steps): the CPU env's info dict has the reference's keys in its order, its terms and episode record equal
    the reference's (floats to 1e-12, integers exactly)"""
    g = np.load(os.path.join(HERE, "golden", "step_info.npz"))
    lack = mjcf.load_scene("Sawyer", "table_lack_0825")
    e = with_step_info(OracleFurnitureEnv)(lack)
    assert e.npart == g["bits"].shape[1]

    def new_episode():
        e.touched, e.picked = [False] * e.npart, [False] * e.npart
        e.num_connected = e.prev_num_connected = e.episode_len = 0
        e.episode_reward, e.episode_time = 0.0, 0.0

    e.reset, e.obs, e.connected_body1 = new_episode, lambda: np.zeros(1), None
    case = -1
    for k in range(len(g["reward"])):
        if g["case"][k] != case:
            case = g["case"][k]
            e.cfg = _cfg(**dict(zip(COEF_KEYS, g["coefs"][g["coef"][k]].tolist())), max_episode_steps=int(g["length"][k]))
            e.narms = int(g["arms"][k])
            new_episode()
        fail, bits = bool(g["fail"][k]), [int(b) for b in g["bits"][k]]
        e._simulate = lambda raw, fail=fail: (fail, fail)
        e.touch_bits = lambda bits=bits: bits
        if not fail:
            e.num_connected = int(g["num_connected"][k])
        ac = g["ac"][k][: 17 if e.narms == 2 else 9]
        _, r, d, _ = e.step(ac)
        info = e.step_info
        assert ",".join(info) == g["keys"][k], (k, list(info), g["keys"][k])
        assert r == pytest.approx(g["reward"][k], rel=1e-12, abs=1e-12) and d == bool(g["done"][k]), k
        for j, t in enumerate(TERMS):
            assert info[t] == pytest.approx(g["terms"][k][j], rel=1e-12, abs=1e-12), (k, t)
        if d:
            gold = dict(zip(g["episode_keys"].tolist(), g["episode"][k]))
            for t in ("episode_success", "episode_length", "episode_num_connected"):
                assert info[t] == int(gold[t]), (k, t)
            for t in ("episode_reward", "episode_unstable"):
                assert info[t] == pytest.approx(gold[t], rel=1e-12, abs=1e-12), (k, t, info[t], gold[t])
            assert ("episode_success_state" in info) == bool(g["success_state"][k])
            new_episode()
        if e.narms == 2:
            assert np.array_equal(info["ac"], ac)
    assert g["fail"].any() and g["success_state"].any() and set(g["arms"].tolist()) == {1, 2} and set(g["length"].tolist()) >= {2, 3, 5}


# ------------------------------------------------------------------ 2. the terms add up to the reward; the episode record
@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("gpu", BACKENDS)
def test_terms_add_up_to_the_reward_and_the_record_to_the_episode(gpu, kind):
    """random actions, episodes of 2, 3 or 5 steps per env: on every step the four terms added in the kernel's order are the returned reward
    bit for bit (on an unstable step, with episode_unstable added); at done, episode_reward is the float32 sum of the rewards the env
    returned over its episode (penalty included) bit for bit, episode_unstable the penalty; rows of envs that have not finished are NaN"""
    agent, opts = KINDS[kind]
    n, steps = (64, 300) if gpu else (3, 7)
    limits = np.array([2, 3, 5])[np.arange(n) % 3]
    eng = build_engine(agent, "table_lack_0825", n, lib_path=_lib(gpu), nsub=2, max_episode_steps=limits, **opts)
    eng.env_reset()
    rng = np.random.RandomState(11)
    acc = np.zeros(n, np.float32)
    finished = np.zeros(n, bool)
    for t in range(1, steps + 1):
        a = rng.uniform(-1, 1, (n, eng.act_dim)).astype(np.float32)
        a[:, -1] = rng.choice([-1.0, 1.0], n)
        obs, rew, done, info = eng.env_step_host(a)
        ri, ep = eng.reward_info(), eng.episode_info()
        unstable = info[:, 2] == 1
        s = _terms_sum(ri)
        assert np.array_equal(s[~unstable], rew[~unstable]), (kind, t)
        assert np.array_equal((s + ep[:, 1])[unstable], rew[unstable]), (kind, t)
        acc = np.where(unstable, np.float32(0), acc) + rew  # an unstable step's episode is that step alone
        d = done.astype(bool)
        assert np.array_equal(ep[d, 0], acc[d]), (kind, t)
        assert np.array_equal(ep[d, 1], np.where(unstable[d], -eng.cfg.unstable_penalty_coef, 0).astype(np.float32)), (kind, t)
        assert (info[d & unstable, 3] == 1).all()
        finished |= d
        assert np.isnan(ep[~finished]).all(), (kind, t)
        acc[d] = 0
    assert finished.all()


# ------------------------------------------------------------------ 3. against the CPU env
@pytest.mark.parametrize("gpu", BACKENDS)
def test_success_episode_against_the_cpu_env(gpu):
    """from a k = 3 preassembled start, the grasp -> connect script on the last leg ends env 0's episode with success: the terms equal the
    CPU env's (success / touch / pick exactly, ctrl_penalty at the reward bar), and so does the episode record"""
    m, k = mjcf.load_scene("Sawyer", "table_lack_0825"), 3
    cfg = Cfg()
    cfg.auto_align = True
    env = with_step_info(PreassembledEnv)(m, cfg)
    env.set_subtask(k)
    env.reset()
    eng = make_engine(m, 2, gpu, nsub=1, auto_align=1)
    eng.set_subtask(k)
    eng.env_reset()
    _sync_oracle_from_engine(env, eng, 0)
    q = _hold_leg_of_step(m, env, k)
    env.nsub = 1
    env.sim.qvel[:] = 0; env.sim.qacc_warmstart[:] = 0; env.sim.ctrl[:] = 0
    env.sim.forward()
    eng.set("qpos", q); eng.set("qvel", np.zeros(m.nv)); eng.set("qacc_warmstart", np.zeros(m.nv))
    eng.forward()
    a = np.zeros((2, eng.act_dim), np.float32)
    a[:, :7] = 0.3
    a[:, -2], a[:, -1] = 1.0, -1.0
    seen = set()
    for step in range(2):
        if step == 1:
            a[0, -1] = 1.0  # env 0 connects
        obs, rew, done, info = eng.env_step_host(a)
        ob, r, d, inf = env.step(a[0].astype(np.float64))
        ri, ep = eng.reward_info()[0], eng.episode_info()[0]
        want = env.step_info
        for j, t in enumerate(TERMS[:3]):
            assert ri[j] == np.float32(want[t]), (step, t, ri[j], want[t])
            if want[t]:
                seen.add(t)
        assert abs(ri[3] - want["ctrl_penalty"]) < 1e-5 and want["ctrl_penalty"] < 0
        assert abs(rew[0] - r) < 1e-5
    assert d and bool(done[0]) and info[0][1] == 1 and inf["success"] == 1
    assert {"success_reward", "touch_reward"} <= seen
    assert list(want)[4:] == list(EPISODE) + ["episode_success_state"]
    assert abs(ep[0] - want["episode_reward"]) < 1e-5 and ep[1] == 0 == want["episode_unstable"]
    assert info[0][3] == want["episode_length"] and info[0][0] == want["episode_num_connected"]


@pytest.mark.parametrize("gpu", BACKENDS)
def test_unstable_step_records_that_step_alone(gpu):
    """a diverged step resets inside the step (furniture.py:2889-2897): its episode record is that step's reward plus the penalty, with
    length 1, after two ordinary steps, as the CPU env's"""
    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    n, seed = 2, 321
    eng = make_engine(m, n, gpu, seed=seed, nsub=2)
    eng.env_reset()
    a = np.zeros((n, eng.act_dim), np.float32)
    a[:, :7], a[:, -1] = 0.5, -1
    for _ in range(2):
        eng.env_step_host(a)
    v = eng.get("qvel").copy()
    v[1, 0] = 1e8
    eng.set("qvel", v)
    obs, rew, done, info = eng.env_step_host(a)
    assert not done[0] and done[1] and info[1][2] == 1 and info[1][3] == 1
    ri, ep = eng.reward_info()[1], eng.episode_info()[1]
    assert ep[0] == rew[1] and ep[1] == -np.float32(Cfg.unstable_penalty_coef)
    assert ri[0] == ri[1] == ri[2] == 0 and _terms_sum(ri[None])[0] + ep[1] == rew[1]
    cfg = Cfg()
    cfg.seed = seed + 1
    e = with_step_info(OracleFurnitureEnv)(m, cfg)
    e.reset()
    e._simulate = lambda raw: (True, True)
    e.step(a[1].astype(np.float64))
    want = e.step_info
    assert want["episode_length"] == 1 and want["episode_unstable"] == -Cfg.unstable_penalty_coef
    assert abs(ep[0] - want["episode_reward"]) < 1e-5 and abs(ri[3] - want["ctrl_penalty"]) < 1e-5


# ------------------------------------------------------------------ 5. per env coefficients
@pytest.mark.parametrize("gpu", BACKENDS)
def test_mixed_coefficient_sets_equal_one_handle_per_set(gpu):
    """a handle whose envs take four coefficient sets (set_task_options) writes the rows that four handles with one set each through FeConfig
    write, bit for bit"""
    g = np.load(os.path.join(HERE, "golden", "step_info.npz"))
    sets = [dict(zip(COEF_KEYS, c.tolist())) for c in g["coefs"]]
    n = 4
    mixed = build_engine("Sawyer", "table_lack_0825", n, lib_path=_lib(gpu), nsub=2, max_episode_steps=3)
    for i, s in enumerate(sets):
        mixed.set_task_options(envs=[i], **s)
    singles = [build_engine("Sawyer", "table_lack_0825", n, lib_path=_lib(gpu), nsub=2, max_episode_steps=3, **s) for s in sets]
    for e in [mixed] + singles:
        e.env_reset()
    rng = np.random.RandomState(4)
    for t in range(4):
        a = rng.uniform(-1, 1, (n, mixed.act_dim)).astype(np.float32)
        a[:, -1] = -1
        rm = mixed.env_step_host(a)
        for i, e in enumerate(singles):
            rs = e.env_step_host(a)
            assert rm[1][i] == rs[1][i], (t, i)
            assert np.array_equal(mixed.reward_info()[i], e.reward_info()[i], equal_nan=True), (t, i)
            assert np.array_equal(mixed.episode_info()[i], e.episode_info()[i], equal_nan=True), (t, i)


# ------------------------------------------------------------------ 6. the three step entry points and the packed block
@pytest.mark.parametrize("kind", ["sparse", "dense"])
@pytest.mark.parametrize("gpu", BACKENDS)
def test_step_entry_points_and_packed_block(gpu, kind):
    """twin handles stepped by fe_env_step, fe_env_step_packed (with the step-info block) and fe_env_step_host leave the same reward_info and
    episode_info rows; the packed block's columns equal the fields (episode columns where done, the sentinel elsewhere until the env's first
    end; NaN terms on a dense handle)"""
    n = 64 if gpu else 3
    limits = np.array([2, 3, 5])[np.arange(n) % 3]
    mk = lambda: build_engine("Sawyer", "table_lack_0825", n, lib_path=_lib(gpu), nsub=2, max_episode_steps=limits, dense={} if kind == "dense" else None)
    engs = [mk() for _ in range(3)]
    for e in engs:
        e.env_reset()
    engs[1].set_packed_layout(info=True)
    engs[1].set_packed_step_info(True)
    cols = engs[1].packed_columns()
    assert list(cols)[-2:] == ["reward_info", "episode_info"] and engs[1].packed_dim() == engs[1].obs_dim + 2 + INFO_DIM + 6
    B = Buffers(gpu)
    od = engs[0].obs_dim
    obs, rew, done, info = B.zeros((n, od)), B.zeros(n), B.zeros(n, np.uint8), B.zeros((n, INFO_DIM), np.int32)
    packed = B.sentinel((n, engs[1].packed_dim()))
    rng = np.random.RandomState(3)
    ended = np.zeros(n, bool)
    for t in range(1, 6):
        a = rng.uniform(-1, 1, (n, engs[0].act_dim)).astype(np.float32)
        a[:, -1] = -1
        ad = B.upload(a)
        engs[0].env_step_dev(B.ptr(ad), B.ptr(obs), B.ptr(rew), B.ptr(done), B.ptr(info))
        engs[1].env_step_packed(B.ptr(ad), B.ptr(packed))
        ho, hr, hd, hi = engs[2].env_step_host(a)
        pk = B.host(packed)
        d = hd.astype(bool)
        ended |= d
        ep = [e.episode_info() for e in engs]
        assert np.array_equal(ep[0], ep[1], equal_nan=True) and np.array_equal(ep[0], ep[2], equal_nan=True), t
        pe = pk[:, cols["episode_info"]]
        assert np.array_equal(pe[ended], ep[0][ended]) and (pe[~ended].view(np.uint32) == 0x7FBADBAD).all(), t
        if kind == "sparse":
            ri = [e.reward_info() for e in engs]
            assert np.array_equal(ri[0], ri[1]) and np.array_equal(ri[0], ri[2]) and np.array_equal(pk[:, cols["reward_info"]], ri[0]), t
        else:
            assert np.isnan(pk[:, cols["reward_info"]]).all()
        assert np.array_equal(pk[:, cols["reward"]][:, 0], hr) and np.array_equal(pk[:, cols["obs"]], ho), t
    assert ended.all()


def test_existing_packed_layouts_keep_their_stride():
    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    eng = make_engine(m, 2, False, nsub=2)
    od = eng.obs_dim
    for info in (0, 1):
        for term in (0, 1):
            eng.set_packed_layout(info=info, terminal_obs=term)
            base = od + 2 + 6 * info + od * term
            assert eng.packed_dim() == base and eng.packed_columns() == packed_columns(od, info=info, terminal_obs=term)
            eng.set_packed_step_info(True)
            assert eng.packed_dim() == base + 6
            assert eng.packed_columns()["reward_info"] == slice(base, base + 4) and eng.packed_columns()["episode_info"] == slice(base + 4, base + 6)
            eng.set_packed_step_info(False)
            assert eng.packed_dim() == base


# ------------------------------------------------------------------ 7. surfaces and refusals
def test_c_abi_fields_and_refusals():
    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    eng = make_engine(m, 2, False, nsub=2)
    assert eng.field_info("reward_info") == (4, 4) and eng.field_info("episode_info") == (2, 4)
    assert np.isnan(eng.reward_info()).all() and np.isnan(eng.episode_info()).all()  # no step has written them
    for f in ("reward_info", "episode_info"):
        with pytest.raises(RuntimeError, match="read-only"):
            eng.set(f, np.zeros((2, eng.field_info(f)[0]), np.float32))
    assert all(eng.step_info_dev_ptrs())
    with pytest.raises(RuntimeError, match="step_info is 0 or 1"):
        eng.set_packed_step_info(2)
    assert eng.packed_dim() == eng.obs_dim + 2
    # a dense handle has no reward terms
    dense = build_engine("Sawyer", "table_lack_0825", 2, lib_path=build_emu(), nsub=2, dense={})
    with pytest.raises(RuntimeError, match="dense reward"):
        dense.reward_info()
    dense.env_reset()
    dense.env_step_host(np.zeros((2, dense.act_dim), np.float32))
    assert np.isnan(dense.get("reward_info")).all()  # a dense handle's steps write no terms
    assert dense.step_info_dev_ptrs()[0] is None and dense.step_info_dev_ptrs()[1]
    # a handle without a scene blob has no env step and none of the fields
    L, em = eng.L, eng.em
    cfg = default_config(nsub=2, maxcon=eng.cfg.maxcon)
    h = C.c_void_p()
    assert L.fe_create(C.byref(em.fm), C.c_size_t(C.sizeof(em.fm)), None, C.c_size_t(0), C.byref(cfg), 2, 0, C.byref(h)) == 0
    try:
        d, e = C.c_int(), C.c_int()
        for f in (b"reward_info", b"episode_info"):
            assert L.fe_field_dim(h, f, C.byref(d), C.byref(e)) == -3
        assert L.fe_reward_info_dev(h) is None and L.fe_episode_info_dev(h) is None
        assert L.fe_set_packed_step_info(h, 1) == -6 and b"without a scene blob" in L.fe_last_error(h)
    finally:
        L.fe_destroy(h)


def test_scene_file_handle_has_the_fields():
    from furniture_b200.engine import DEFAULT_LIB  # noqa: F401

    eng = make_engine(mjcf.load_scene("Sawyer", "table_lack_0825"), 2, False, nsub=2)
    L = eng.L
    path = os.path.join(ROOT, "furniture_b200", "compiled", "Sawyer_table_lack_0825.feb")
    cfg = default_config(nsub=2, maxcon=eng.cfg.maxcon)
    h = C.c_void_p()
    assert L.fe_create_from_file(path.encode(), C.byref(cfg), 2, 0, C.byref(h)) == 0, L.fe_last_error(None)
    try:
        d, e = C.c_int(), C.c_int()
        assert L.fe_field_dim(h, b"reward_info", C.byref(d), C.byref(e)) == 0 and d.value == 4
        assert L.fe_field_dim(h, b"episode_info", C.byref(d), C.byref(e)) == 0 and d.value == 2
        assert L.fe_set_packed_step_info(h, 1) == 0
    finally:
        L.fe_destroy(h)


@pytest.mark.parametrize("gpu", BACKENDS)
def test_gym_step_info(gpu):
    """FurnitureGymB200(step_info=True): the reference's keys on every step and at done, the terms and the record as the engine wrote them;
    the default gym returns the same rewards and its own info"""
    from furniture_b200.gym_api import FurnitureGymB200

    mk = lambda name, **kw: FurnitureGymB200(name=name, furniture_name="table_lack_0825", lib_path=_lib(gpu), nsub=2, max_episode_steps=3, **kw)
    for name in ("FurnitureSawyerEnv", "FurnitureBaxterEnv"):
        S, D = mk(name, step_info=True), mk(name)
        S.reset(), D.reset()
        rng = np.random.RandomState(5)
        total = np.float32(0)
        for t in range(3):
            a = rng.uniform(-1, 1, S.dof).astype(np.float32)
            a[-1] = -1
            (os_, rs, ds, i_s), (od, rd, dd, idd) = S.step(a), D.step(a)
            assert rs == rd and ds == dd
            total += np.float32(rs)
            keys = list(REWARD_INFO_KEYS) + (["ac"] if name == "FurnitureBaxterEnv" else [])
            if t < 2:
                assert list(i_s) == keys and idd == {}
            else:
                assert list(i_s) == keys + list(EPISODE) and ds
                assert i_s["episode_reward"] == total and i_s["episode_unstable"] == 0
                assert {k: i_s[k] for k in idd if k not in ("episode_reward", "episode_time")} == {k: v for k, v in idd.items() if k not in ("episode_reward", "episode_time")}
            assert np.float32(((i_s["success_reward"] + i_s["touch_reward"]) + i_s["pick_reward"]) + i_s["ctrl_penalty"]) == np.float32(rs) or t == 2
            if name == "FurnitureBaxterEnv":
                assert np.array_equal(i_s["ac"], a)


# ------------------------------------------------------------------ GPU surfaces: BatchedFurnitureEnv, MixedFurnitureEnv
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["sparse", "dense", "baxter"])
def test_batched_step_infos_have_the_reference_keys(case):
    import torch

    from furniture_b200.dense import INFO_KEYS as DENSE_KEYS
    from furniture_b200.env import BatchedFurnitureEnv

    agent = "Baxter" if case == "baxter" else "Sawyer"
    n = 6
    env = BatchedFurnitureEnv(agent, "table_lack_0825", n, nsub=2, max_episode_steps=[2, 3, 2, 3, 2, 3], dense={} if case == "dense" else None)
    env.reset()
    g = torch.Generator().manual_seed(1)
    for t in range(3):
        a = torch.rand((n, env.act_dim), generator=g) * 2 - 1
        a[:, -1] = -1
        ob, rew, done, info = env.step(a.cuda())
        infos = env.step_infos()
        torch.cuda.synchronize()
        d = done.cpu().numpy().astype(bool)
        base = list(DENSE_KEYS) if case == "dense" else list(REWARD_INFO_KEYS)
        if case == "baxter":
            base.append("ac")
        for i, row in enumerate(infos):
            want = base + (list(EPISODE) + (["episode_success_state"] if info[i, 1] else []) if d[i] else [])
            assert list(row) == want, (t, i, list(row))
            if d[i]:
                assert row["episode_reward"] == env.episode_record()["episode_reward"][i].item()
                assert row["episode_length"] == int(info[i, 3])
        if case == "dense":
            with pytest.raises(RuntimeError, match="dense reward"):
                env.reward_terms()
        else:
            terms = env.reward_terms()
            s = ((terms["success_reward"] + terms["touch_reward"]) + terms["pick_reward"]) + terms["ctrl_penalty"]
            assert torch.equal(s, rew)
    env.close()


@pytest.mark.gpu
def test_mixed_env_step_infos_in_global_order():
    import torch

    from furniture_b200.env import MixedFurnitureEnv

    names = ["table_lack_0825", "chair_ingolf_0650", "toy_table"]
    env = MixedFurnitureEnv(names, [3, 2, 4], nsub=2, max_episode_steps=2, pad_to=12)
    env.reset()
    for t in range(2):
        env.step(torch.zeros((env.num_envs, env.act_dim), device=env.device))
        terms, rec, infos = env.reward_terms(), env.episode_record(), env.step_infos()
        assert len(infos) == 12 and infos[9:] == ({},) * 3
        for b, off in zip(env.buckets, env.offsets):
            bt, be = b.reward_terms(), b.episode_record()
            for k in REWARD_INFO_KEYS:
                assert torch.equal(terms[k][off : off + b.num_envs], bt[k])
            for k in EPISODE_INFO_KEYS:
                assert torch.equal(rec[k][off : off + b.num_envs], be[k], ) or t == 0
            assert infos[off : off + b.num_envs] == b.step_infos() or t == 1
        assert torch.isnan(terms["ctrl_penalty"][9:]).all()
    env.close()


# ------------------------------------------------------------------ the sharded message over gloo, emulated shards
WORKER = r'''
import os, sys
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, "tests"))
import numpy as np, torch, torch.distributed as dist
from collections import OrderedDict
from furniture_b200.engine import EPISODE_INFO_KEYS, REWARD_INFO_KEYS
from furniture_b200.env import ShardedFurnitureEnv, build_engine
from parity_util import build_emu

class EmuShard:  # stand-in for BatchedFurnitureEnv with CPU tensors, stepped on the host path of ShardedFurnitureEnv
    def __init__(self, n, seed):
        self.engine = build_engine("Sawyer", "table_lack_0825", n, lib_path=build_emu(), seed=seed, nsub=2, max_episode_steps=list(2 + np.arange(n) %% 2))
        self.dense_cfg = None
        self.num_envs, self.obs_dim, self.act_dim = n, self.engine.obs_dim, self.engine.act_dim
        self.device = torch.device("cpu")
        self._obs = torch.zeros((n, self.obs_dim))
    def _obs_dict(self, obs):
        return OrderedDict(all=obs)
    def reset(self):
        self.engine.env_reset(); self._obs.copy_(torch.from_numpy(self.engine.get("obs"))); return self._obs_dict(self._obs)
    def step(self, a):
        obs, rew, done, info = self.engine.env_step_host(a.numpy())
        self._obs.copy_(torch.from_numpy(obs))
        return self._obs_dict(self._obs), torch.from_numpy(rew), torch.from_numpy(done), torch.from_numpy(info)
    def reward_terms(self):
        r = torch.from_numpy(self.engine.reward_info())
        return OrderedDict((k, r[:, j]) for j, k in enumerate(REWARD_INFO_KEYS))
    def episode_record(self):
        r = torch.from_numpy(self.engine.episode_info())
        return OrderedDict((k, r[:, j]) for j, k in enumerate(EPISODE_INFO_KEYS))

def gathered(x):
    parts = [torch.zeros_like(x) for _ in range(world)]
    dist.all_gather(parts, x.contiguous())
    return torch.cat(parts, 0)

dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
n = 3
seed = ShardedFurnitureEnv.shard_seed(123, rank, n)
env = ShardedFurnitureEnv(n, env=EmuShard(n, seed), gather_info=True, gather_step_info=True)
plain = ShardedFurnitureEnv(n, env=EmuShard(n, seed))
od = env.env.obs_dim
assert env.pack_dim == od + 2 + 6 + 6 and plain.pack_dim == od + 2
env.reset(); plain.reset()
rng = np.random.RandomState(rank)
for t in range(3):
    a = torch.from_numpy(rng.uniform(-1, 1, (n, env.env.act_dim)).astype(np.float32))
    a[:, -1] = -1
    ob, rew, done, info = env.step(a)
    plain.step(a)
    terms = torch.stack(list(env.reward_terms().values()), 1)
    assert torch.equal(terms, gathered(torch.from_numpy(env.env.engine.reward_info()))), t
    s = ((terms[:, 0] + terms[:, 1]) + terms[:, 2]) + terms[:, 3]
    assert torch.equal(s, rew), t
    rec = torch.stack(list(env.episode_record().values()), 1)
    want = gathered(torch.from_numpy(env.env.engine.episode_info()))
    assert done.any() or t == 0
    assert torch.equal(rec[done], want[done]), t
for what in ("reward_terms", "episode_record"):
    try:
        getattr(plain, what)()
        raise SystemExit("%%s did not raise" %% what)
    except ValueError as e:
        assert "gather_step_info" in str(e), str(e)
dist.barrier(); dist.destroy_process_group()
print("rank", rank, "ok")
'''


def test_two_ranks_gather_step_info_over_gloo(tmp_path):
    import subprocess
    import sys

    script = tmp_path / "worker.py"
    script.write_text(WORKER % {"root": ROOT})
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT="29541", WORLD_SIZE="2")
    procs = [subprocess.Popen([sys.executable, str(script)], env=dict(env, RANK=str(r), LOCAL_RANK=str(r)), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for r in range(2)]
    outs = [p.communicate(timeout=600)[0] for p in procs]
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, "rank %d failed:\n%s" % (r, o[-3000:])
        assert "rank %d ok" % r in o
