"""The sharded step's all-gather message under every layout of fe_set_packed_layout: the packed rows [obs | reward | done | info | dense_info |
terminal_obs] that the step kernel writes against what fe_env_step returns, the host-filled rows of a shard without that kernel, and
ShardedFurnitureEnv's gathered info, dense_info and terminal observation (the (ob, reward, done, info) that util/subproc_vec_env.py:100-113
sends back from every worker).

`emu` runs the lane-emulated build on the CPU, `cuda-*` the sm_90a library (marked gpu)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from furniture_b200 import mjcf
from furniture_b200.engine import INFO_DIM, default_config, packed_columns
from furniture_b200.env import build_engine
from parity_util import build_emu, make_engine
from test_terminal_obs import CASES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = np.uint32(0x7FBADBAD)  # a NaN no step writes
LAYOUTS = {"default": {}, "info": dict(info=True), "info-dense": dict(info=True, dense_info=True), "terminal": dict(terminal_obs=True),
           "all": dict(info=True, dense_info=True, terminal_obs=True)}


def on_backends(cases):
    """(gpu, case) parameters: the emulated build under the case's name, the CUDA build (marked gpu) as cuda-<case>"""
    return ([pytest.param(False, c, id=c) for c in cases]
            + [pytest.param(True, c, id="cuda-" + c, marks=pytest.mark.gpu) for c in cases])


class Buffers:
    """step buffers on the engine's side: torch tensors on cuda:0, or numpy arrays for the emulated build (whose device memory is host memory)"""

    def __init__(self, gpu):
        self.gpu = gpu
        if gpu:
            import torch

            self.torch = torch

    def zeros(self, shape, dtype=np.float32):
        if self.gpu:
            return self.torch.zeros(shape, dtype={np.float32: self.torch.float32, np.uint8: self.torch.uint8, np.int32: self.torch.int32}[dtype], device="cuda:0")
        return np.zeros(shape, dtype)

    def sentinel(self, shape):
        b = self.zeros(shape)
        if self.gpu:
            b.view(self.torch.int32).fill_(int(SENTINEL.view(np.int32)))
        else:
            b.view(np.uint32).fill(SENTINEL)
        return b

    def ptr(self, x):
        return x.data_ptr() if self.gpu else x.ctypes.data

    def host(self, x):
        if self.gpu:
            self.torch.cuda.synchronize()
            return x.cpu().numpy()
        return x.copy()

    def upload(self, a):
        if self.gpu:
            return self.torch.from_numpy(a).to("cuda:0")
        return np.ascontiguousarray(a)


def _is_sentinel(x):
    return x.view(np.uint32) == SENTINEL


def _layout(eng, name):
    """the layout `name` as this handle can have it: the dense_info block only on a dense handle"""
    return {k: v for k, v in LAYOUTS[name].items() if k != "dense_info" or eng.dense is not None}


# ------------------------------------------------------------------ 1. packed rows = the unpacked step, bit for bit, under every layout
@pytest.mark.parametrize("gpu,case", on_backends(list(CASES)))
def test_packed_rows_equal_the_unpacked_step(gpu, case):
    """twin handles, one stepped with fe_env_step and one per layout with fe_env_step_packed, same seed and actions; episodes end after 2, 3
    or 5 steps per env, so that finished and running envs share blocks.  Every block of every row equals the twin's output, the info block
    read as int32; the terminal slot equals terminal_obs where done and keeps the sentinel of an env that has not finished yet"""
    agent, furn, opts = CASES[case]
    n = 64 if gpu else 3
    limits = np.array([2, 3, 5])[np.arange(n) % 3]
    mk = lambda: build_engine(agent, furn, n, lib_path=None if gpu else build_emu(), nsub=2, max_episode_steps=limits, **opts)
    twin = mk()
    layouts = {}
    for name in LAYOUTS:  # on a sparse handle info-dense is info, and all is info + terminal
        lay = _layout(twin, name)
        if lay not in layouts.values():
            layouts[name] = lay
    engs = {name: mk() for name in layouts}
    B = Buffers(gpu)
    obs, rew, done, info = B.zeros((n, twin.obs_dim)), B.zeros(n), B.zeros(n, np.uint8), B.zeros((n, INFO_DIM), np.int32)
    packed = {}
    for name, eng in engs.items():
        eng.set_packed_layout(**layouts[name])
        cols = eng.packed_columns()
        assert eng.packed_dim() == next(reversed(cols.values())).stop
    for eng in [twin] + list(engs.values()):
        eng.env_reset()
    for name, eng in engs.items():
        packed[name] = B.sentinel((n, eng.packed_dim()))
    rng = np.random.RandomState(11)
    ended = np.zeros(n, bool)
    for t in range(1, 7):
        a = rng.uniform(-1, 1, (n, twin.act_dim)).astype(np.float32)
        a[:, -1] = -1.0
        ad = B.upload(a)
        twin.env_step_dev(B.ptr(ad), B.ptr(obs), B.ptr(rew), B.ptr(done), B.ptr(info))
        for name, eng in engs.items():
            eng.env_step_packed(B.ptr(ad), B.ptr(packed[name]))
        o, r, d, i = B.host(obs), B.host(rew), B.host(done), B.host(info)
        assert np.array_equal(d.astype(bool), t % limits == 0), (case, t)
        ended |= d.astype(bool)
        t_obs = twin.terminal_obs()
        for name, eng in engs.items():
            pk, c = B.host(packed[name]), eng.packed_columns()
            assert np.array_equal(pk[:, c["obs"]], o) and np.array_equal(pk[:, c["reward"]][:, 0], r), (case, name, t)
            assert np.array_equal(pk[:, c["done"]][:, 0], d.astype(np.float32)), (case, name, t)
            if "info" in c:
                assert np.array_equal(pk[:, c["info"]].view(np.int32), i), (case, name, t)
            if "dense_info" in c:
                assert np.array_equal(pk[:, c["dense_info"]], twin.get("dense_info")), (case, name, t)
            if "terminal_obs" in c:
                slot = pk[:, c["terminal_obs"]]
                now = d.astype(bool)
                assert np.array_equal(slot[now], t_obs[now]), (case, name, t)
                assert np.array_equal(slot[ended], eng.terminal_obs()[ended]), (case, name, t)  # a row is left as the step that wrote it
                assert _is_sentinel(slot[~ended]).all(), (case, name, t)
            assert np.array_equal(eng.terminal_obs()[ended], t_obs[ended]), (case, name, t)
    assert ended.all()


# ------------------------------------------------------------------ 2. the default layout writes [obs | reward | done] and nothing past it
@pytest.mark.parametrize("gpu", [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)])
def test_default_layout_writes_nothing_past_obs_reward_done(gpu):
    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    n = 64 if gpu else 3
    limits = 2 + np.arange(n) % 2
    twin, eng = make_engine(m, n, gpu, nsub=2), make_engine(m, n, gpu, nsub=2)
    B = Buffers(gpu)
    od = eng.obs_dim
    assert eng.packed_dim() == od + 2 and list(eng.packed_columns()) == ["obs", "reward", "done"]
    wide = B.sentinel((n, 2 * od + 2 + INFO_DIM + 12))  # as wide as the full layout, read with the default stride
    obs, rew, done = B.zeros((n, od)), B.zeros(n), B.zeros(n, np.uint8)
    for e in (twin, eng):
        e.set_task_options(max_episode_steps=limits)
        e.env_reset()
    rng = np.random.RandomState(4)
    for t in range(1, 4):
        a = rng.uniform(-1, 1, (n, eng.act_dim)).astype(np.float32)
        a[:, -1] = -1.0
        ad = B.upload(a)
        twin.env_step_dev(B.ptr(ad), B.ptr(obs), B.ptr(rew), B.ptr(done), 0)
        eng.env_step_packed(B.ptr(ad), B.ptr(wide))
        flat = B.host(wide).reshape(-1)
        used = n * (od + 2)
        rows = flat[:used].reshape(n, od + 2)
        assert _is_sentinel(flat[used:]).all(), t
        assert np.array_equal(rows[:, :od], B.host(obs)) and np.array_equal(rows[:, od], B.host(rew)), t
        assert np.array_equal(rows[:, od + 1], B.host(done).astype(np.float32)) and (B.host(done) == (limits == t)).all(), t


# ------------------------------------------------------------------ 3. an unstable step: the world of the reset inside the step
@pytest.mark.parametrize("gpu", [pytest.param(False, id="emu"), pytest.param(True, id="cuda", marks=pytest.mark.gpu)])
def test_unstable_step_terminal_slot_is_the_internal_reset(gpu):
    """the construction of test_terminal_obs: env 1's arm diverges, the step resets it inside _do_simulation's except branch and again
    for done; the terminal slot holds terminal_obs, the world of the first of those resets, and env 0's slot keeps the sentinel"""
    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    n, seed = 2, 321
    twin, eng = make_engine(m, n, gpu, seed=seed, nsub=2), make_engine(m, n, gpu, seed=seed, nsub=2)
    eng.set_packed_layout(info=True, terminal_obs=True)
    B = Buffers(gpu)
    pk = B.sentinel((n, eng.packed_dim()))
    for e in (twin, eng):
        e.env_reset()
        v = e.get("qvel").copy()
        v[1, 0] = 1e8
        e.set("qvel", v)
    a = np.zeros((n, eng.act_dim), np.float32)
    a[:, -1] = -1
    obs, rew, done, info = twin.env_step_host(a)
    eng.env_step_packed(B.ptr(B.upload(a)), B.ptr(pk))
    p, c = B.host(pk), eng.packed_columns()
    assert not done[0] and done[1] and info[1][2] == 1
    assert np.array_equal(p[:, c["info"]].view(np.int32), info) and np.array_equal(p[:, c["obs"]], obs)
    t_obs = twin.terminal_obs()
    assert np.array_equal(p[1, c["terminal_obs"]], t_obs[1]) and np.array_equal(eng.terminal_obs()[1], t_obs[1])
    assert not np.array_equal(t_obs[1], obs[1])  # the auto-reset drew a new world after it
    assert _is_sentinel(p[0, c["terminal_obs"]]).all()


# ------------------------------------------------------------------ 4. two ranks over gloo, emulated shards
WORKER = r'''
import os, sys
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, "tests"))
import numpy as np, torch, torch.distributed as dist
from collections import OrderedDict
from furniture_b200.env import ShardedFurnitureEnv, build_engine
from parity_util import build_emu

class EmuShard:  # stand-in for BatchedFurnitureEnv with CPU tensors, stepped on the host path of ShardedFurnitureEnv
    def __init__(self, n, seed, dense):
        self.engine = build_engine("Sawyer", "table_lack_0825", n, lib_path=build_emu(), seed=seed, nsub=2, max_episode_steps=list(2 + np.arange(n) %% 2),
                                   dense={} if dense else None)
        self.dense_cfg = self.engine.dense
        self.num_envs, self.obs_dim, self.act_dim = n, self.engine.obs_dim, self.engine.act_dim
        self.object_ob_dim = 7 * self.engine.scene.npart
        self.device = torch.device("cpu")
        self._obs = torch.zeros((n, self.obs_dim))
    def _obs_dict(self, obs):
        return OrderedDict(object_ob=obs[:, : self.object_ob_dim], rest=obs[:, self.object_ob_dim :])
    def reset(self):
        self.engine.env_reset(); self._obs.copy_(torch.from_numpy(self.engine.get("obs"))); return self._obs_dict(self._obs)
    def step(self, a):
        obs, rew, done, info = self.engine.env_step_host(a.numpy())
        self._obs.copy_(torch.from_numpy(obs))
        self.last_info = torch.from_numpy(info)
        return self._obs_dict(self._obs), torch.from_numpy(rew), torch.from_numpy(done), self.last_info
    def terminal_observation(self):
        return self._obs_dict(torch.from_numpy(self.engine.terminal_obs()))
    def dense_infos(self):
        return torch.from_numpy(self.engine.get("dense_info"))

def gathered(x):
    parts = [torch.zeros_like(x) for _ in range(world)]
    dist.all_gather(parts, x.contiguous())
    return torch.cat(parts, 0)

dist.init_process_group("gloo")
rank, world = dist.get_rank(), dist.get_world_size()
n = 3
seed = ShardedFurnitureEnv.shard_seed(123, rank, n)
full = ShardedFurnitureEnv(n, env=EmuShard(n, seed, False), gather_info=True, gather_terminal=True)
dense = ShardedFurnitureEnv(n, env=EmuShard(n, seed, True), gather_info=True)
plain = ShardedFurnitureEnv(n, env=EmuShard(n, seed, False))
od = full.env.obs_dim
assert full.pack_dim == 2 * od + 2 + 6 and dense.pack_dim == od + 2 + 6 + 12 and plain.pack_dim == od + 2
for env in (full, dense, plain):
    env.reset()
assert (full._all[:, od:] == 0).all()  # a reset zeroes the info and terminal columns
rng = np.random.RandomState(rank)
for t in range(3):
    a = torch.from_numpy(rng.uniform(-1, 1, (n, full.env.act_dim)).astype(np.float32))
    a[:, -1] = -1
    outs = {k: env.step(a) for k, env in (("full", full), ("dense", dense), ("plain", plain))}
    for k, env in (("full", full), ("dense", dense)):
        ob, rew, done, info = outs[k]
        assert info.dtype == torch.int32 and info.shape == (n * world, 6)
        assert info.data_ptr() == env._all.data_ptr() + 4 * (od + 2)  # a view of the message, not a conversion
        assert torch.equal(info, gathered(env.env.last_info)), (k, t)
    ob, rew, done, info = outs["full"]
    to = full.terminal_observation()
    assert list(to) == list(ob)
    rows, want = torch.cat(list(to.values()), 1), gathered(torch.from_numpy(full.env.engine.terminal_obs()))
    d = done.numpy()
    assert d.any() or t == 0
    assert torch.equal(rows[d], want[d]), t
    assert torch.equal(dense.dense_infos(), gathered(torch.from_numpy(dense.env.engine.get("dense_info")))), t
    pob, prew, pdone, pinfo = outs["plain"]
    assert pinfo.shape == (n, 6) and torch.equal(pinfo, plain.env.last_info) and torch.equal(pinfo, full.local_slice(info))  # local, as before
for env, what in ((plain, "terminal_observation"), (plain, "dense_infos"), (full, "dense_infos")):
    try:
        getattr(env, what)()
        raise SystemExit("%%s did not raise" %% what)
    except ValueError as e:
        assert ("gather_terminal" if what == "terminal_observation" else "gather_info") in str(e), str(e)
dist.barrier(); dist.destroy_process_group()
print("rank", rank, "ok")
'''


def test_two_ranks_gather_info_terminal_and_dense_over_gloo(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(WORKER % {"root": ROOT})
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT="29533", WORLD_SIZE="2")
    procs = [subprocess.Popen([sys.executable, str(script)], env=dict(env, RANK=str(r), LOCAL_RANK=str(r)), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for r in range(2)]
    outs = [p.communicate(timeout=600)[0] for p in procs]
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, "rank %d failed:\n%s" % (r, o[-3000:])
        assert "rank %d ok" % r in o


# ------------------------------------------------------------------ 5. a mixed shard on the host path, world-1 NCCL group
MIXED_WORKER = r"""
import os, sys
sys.path.insert(0, %(root)r)
import torch, torch.distributed as dist
from furniture_b200.env import MixedFurnitureEnv, ShardedFurnitureEnv
torch.cuda.set_device(0)
dist.init_process_group("nccl")
names = ["table_lack_0825", "chair_ingolf_0650", "toy_table"]
mixed = MixedFurnitureEnv(names, 4, nsub=2, max_episode_steps=2, pad_to=14)
env = ShardedFurnitureEnv(mixed.num_envs, env=mixed, gather_info=True, gather_terminal=True)
assert env.pack_dim == 2 * mixed.obs_dim + 2 + 6
env.reset()
g = torch.Generator().manual_seed(0)
for t in range(2):
    a = torch.rand((mixed.num_envs, mixed.act_dim), generator=g) * 2 - 1
    a[:, -1] = -1
    ob, rew, done, info = env.step(a.cuda())
    torch.cuda.synchronize()
    to = env.terminal_observation()
    assert list(to) == list(ob)
    for b, off in zip(mixed.buckets, mixed.offsets):
        sl = slice(off, off + b.num_envs)
        assert torch.equal(info[sl], b._info) and torch.equal(rew[sl], b._rew) and torch.equal(done[sl], b._done.bool()), (t, b.model.meta.get("furniture"))
        bo = b._obs_dict(b._obs)
        for k, v in b.terminal_observation().items():
            assert torch.equal(ob[k][sl, : v.shape[1]], bo[k]), (t, k)
            d = b._done.bool()
            assert torch.equal(to[k][sl, : v.shape[1]][d], v[d]), (t, k)
assert done[: mixed.real_envs].all()
try:
    env.dense_infos()
    raise SystemExit("dense_infos did not raise on a sparse shard")
except ValueError:
    pass
dist.destroy_process_group()
print("mixed ok")
"""


@pytest.mark.gpu
def test_mixed_shard_host_path_gathers_every_bucket(tmp_path):
    script = tmp_path / "mixed.py"
    script.write_text(MIXED_WORKER % {"root": ROOT})
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", MASTER_PORT="29537", WORLD_SIZE="1", RANK="0", LOCAL_RANK="0")
    p = subprocess.run([sys.executable, str(script)], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert p.returncode == 0 and "mixed ok" in p.stdout, p.stdout[-3000:]


@pytest.mark.gpu
def test_mixed_env_dense_infos_in_global_order():
    """MixedFurnitureEnv.dense_infos: each bucket's dense_info rows at its offsets, zero rows for the padding"""
    import torch

    from furniture_b200.env import MixedFurnitureEnv

    env = MixedFurnitureEnv(["table_lack_0825", "table_lack_0825"], [3, 5], nsub=2, pad_to=10, dense={})
    env.reset()
    env.step(torch.zeros((env.num_envs, env.act_dim), device=env.device))
    rows = env.dense_infos()
    assert rows.shape == (10, 12) and rows.device == env.device
    for b, off in zip(env.buckets, env.offsets):
        assert np.array_equal(rows[off : off + b.num_envs].cpu().numpy(), b.engine.get("dense_info"))
    assert (rows[8:] == 0).all()
    env.close()


# ------------------------------------------------------------------ 6. the C-ABI
def test_packed_dim_and_refusals():
    m = mjcf.load_scene("Sawyer", "table_lack_0825")
    sparse = make_engine(m, 2, False, nsub=2)
    dense = build_engine("Sawyer", "table_lack_0825", 2, lib_path=build_emu(), nsub=2, dense={})
    for eng in (sparse, dense):
        od = eng.obs_dim
        for info in (0, 1):
            for di in ((0, 1) if eng is dense else (0,)):
                for term in (0, 1):
                    eng.set_packed_layout(info=info, dense_info=di, terminal_obs=term)
                    want = od + 2 + 6 * info + 12 * di + od * term
                    assert eng.packed_dim() == want == next(reversed(eng.packed_columns().values())).stop, (info, di, term)
                    assert list(eng.packed_columns()) == [k for k, f in (("obs", 1), ("reward", 1), ("done", 1), ("info", info),
                                                                          ("dense_info", di), ("terminal_obs", term)) if f]
    # the stride follows fe_set_obs_layout
    eng = make_engine(m, 2, False, nsub=2)
    eng.set_packed_layout(info=True, terminal_obs=True)
    eng.set_obs_layout(object_ob_all=False, subtask_ob=True)
    od = eng.obs_dim
    assert od == 14 + 2 + eng.scene.robot_ob_dim and eng.packed_dim() == 2 * od + 2 + 6
    assert eng.packed_columns() == packed_columns(od, info=True, terminal_obs=True)
    # refusals
    for bad in (dict(info=2), dict(dense_info=-1), dict(terminal_obs=3)):
        with pytest.raises(RuntimeError, match="each flag is 0 or 1"):
            dense.set_packed_layout(**bad)
    with pytest.raises(RuntimeError, match="dense_info needs a handle with the dense reward"):
        sparse.set_packed_layout(info=True, dense_info=True)
    assert sparse.packed_dim() == 2 * sparse.obs_dim + 2 + 6  # a refused layout leaves the last one (info, terminal_obs) in place
    L, em = sparse.L, sparse.em
    h = C.c_void_p()
    cfg = default_config(nsub=2, maxcon=sparse.cfg.maxcon)
    assert L.fe_create(C.byref(em.fm), C.c_size_t(C.sizeof(em.fm)), None, C.c_size_t(0), C.byref(cfg), 2, 0, C.byref(h)) == 0
    try:
        assert L.fe_set_packed_layout(h, 1, 0, 0) == -6 and b"without a scene blob" in L.fe_last_error(h)
    finally:
        L.fe_destroy(h)
