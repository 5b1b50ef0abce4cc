"""The mixed-furniture case (BASELINE.json config 5, SURVEY.md 8d): FurnitureSawyerEnv over every furniture XML of the asset
tree (64 models; 3 of them with mesh colliders, which collide through their convex hulls) -- ragged nq/nv/nefc, 2 to 14
parts, 1 to 37 welds, boxes, cylinders and hulls.  For each model: device reset (settle protocol of furniture.py:1406-1663), then
env steps with random actions compared with the CPU env oracle started from the same post-reset state.

`emu` = lane-emulated harness build of the kernel source (CPU); `cuda` = the sm_90a library (marked gpu, a subset that
spans the shapes: most parts, most geoms, cylinders, smallest)."""
import glob
import os

import numpy as np
import pytest

from furniture_b200 import mjcf
from furniture_b200.engine import FLAG_CONTACT_FULL
from oracle.ref_env import OracleFurnitureEnv
from parity_util import make_engine
from test_env_parity import _sync_oracle_from_engine

HERE = os.path.dirname(os.path.abspath(__file__))
COMPILED = os.path.join(os.path.dirname(HERE), "furniture_b200", "compiled")
NAMES = sorted(os.path.basename(p)[len("Sawyer_") : -len(".npz")] for p in glob.glob(os.path.join(COMPILED, "Sawyer_*.npz")))

# Seven models carry no `*_initpos` numerics: the reference drops those parts at z = 0.01 wherever the sampler puts them
# (placement_sampler.py:68-104), i.e. large panels start half inside the floor and are pushed out during the reset; all seven
# come out of the reset still moving, so steps are compared loosely (chaotic contact).  During that push-out three of them
# have more simultaneous contacts than the engine's per-env contact capacity (auto_maxcon; the reference runs with
# nconmax=5000) and raise the overflow flag at this draw (the others may, depending on the draw).
UNLISTED = {"bookcase_billy_0191", "bookcase_grevback_0484", "cabinet_akurum_0021", "chair_agam_0005", "table_hemnes_0539", "table_klubbo_0740", "table_liden_0921"}
OVERFLOW = {"bookcase_grevback_0484", "table_hemnes_0539", "table_liden_0921"}
GPU_SUBSET = ["bookcase_expedit_0376", "chair_ingolf_0650", "table_dockstra_0279", "toy_table_flip", "three_blocks_peg", "bookcase_hensvik_0565", "chair_bertil_0148"]


def _run(name, gpu, n=2, steps=2):
    m = mjcf.load_scene("Sawyer", name)
    eng = make_engine(m, n, gpu)
    assert eng.obs_dim == 7 * len(m.meta["part_names"]) + 29
    eng.env_reset()
    flags = eng.get("flags")[:, 0]
    q = eng.get("qpos")
    assert np.isfinite(q).all()
    if name in UNLISTED:
        assert ((flags & ~FLAG_CONTACT_FULL) == 0).all(), flags  # at most the capacity bit
        if name in OVERFLOW or (flags != 0).any():  # how deep the panels start inside the floor depends on the draw
            eng.close()
            return
    assert (flags == 0).all(), flags
    assert np.allclose(np.linalg.norm(q[:, 9:].reshape(n, -1, 7)[:, :, 3:], axis=2), 1, atol=1e-5)  # unit quaternions
    if name not in UNLISTED:
        assert np.abs(eng.get("qvel")[:, 9:]).max() < 0.5  # parts (nearly) at rest after the settle phase
    envs = [OracleFurnitureEnv(m) for _ in range(n)]
    for i, e in enumerate(envs):
        e.reset()
        _sync_oracle_from_engine(e, eng, i)
        e.sim.qfrc_bias[: e.nr] = eng.get("qfrc_bias")[i]
    rng = np.random.RandomState(5)
    # analytic pairs (plane/sphere/box) agree to fp32 round-off; cylinder pairs go through MPR (portal tolerance), as in
    # test_engine_parity; parts still in motion after the reset amplify round-off through contact (loose bound)
    has_cyl = bool(np.isin(np.asarray(m.geom_type), (5, 7)).any())  # cylinders and mesh hulls collide through MPR
    tol = 2e-2 if name in UNLISTED else (1e-3 if has_cyl else 5e-5)
    for k in range(steps):
        a = rng.uniform(-1, 1, (n, eng.act_dim)).astype(np.float32)
        a[:, -1] = -0.5
        obs, rew, done, info = eng.env_step_host(a)
        assert (eng.get("flags")[:, 0] == 0).all()
        for i, e in enumerate(envs):
            ob, r, d, inf = e.step(a[i].astype(np.float64))
            assert np.abs(obs[i] - ob).max() < tol, (name, k, i, np.abs(obs[i] - ob).max())
            assert abs(rew[i] - r) < 1e-5 and bool(done[i]) == d
            assert info[i][0] == inf["num_connected"] and info[i][3] == inf["episode_length"]
    eng.close()


def test_compiled_tables_cover_the_supported_models():
    # all 64 furniture XMLs of the asset tree, the three with mesh colliders (convex hulls) included
    assert len(NAMES) == 64 and "toy_table" in NAMES and "table_lack_0825" in NAMES and "swivel_chair_0700" in NAMES
    assert {"chair_agne_0010", "chair_bertil_0148", "shelf_liden_0922"} <= set(NAMES)


@pytest.mark.parametrize("name", NAMES)
def test_env_parity_every_furniture_emu(name):
    _run(name, False)


@pytest.mark.gpu
@pytest.mark.parametrize("name", GPU_SUBSET)
def test_env_parity_mixed_furniture_cuda(name):
    _run(name, True, n=4)


@pytest.mark.gpu
def test_mixed_batch_buckets_are_independent_and_layout_switching_is_ordered():
    """MixedFurnitureEnv steps one engine handle per furniture model from one stream; the slice-layout table (one
    __constant__ object per process) is switched between buckets by a stream-ordered upload.  Every bucket must come out
    bit-identical to the same envs stepped alone, whatever is interleaved with it."""
    import torch

    from furniture_b200.env import BatchedFurnitureEnv, MixedFurnitureEnv

    names = ["table_lack_0825", "bookcase_expedit_0376", "toy_table_flip", "chair_ingolf_0650"]
    counts = [16, 8, 12, 8]
    env = MixedFurnitureEnv(names, counts, seed=77)
    obs = env.reset()
    assert obs["object_ob"].shape == (sum(counts), 7 * 11) and obs["robot_ob"].shape == (sum(counts), 29)
    g = torch.Generator(device="cuda").manual_seed(3)
    acts = [torch.rand((sum(counts), env.act_dim), device="cuda", generator=g) * 2 - 1 for _ in range(3)]
    for a in acts:
        obs, rew, done, info = env.step(a)
    torch.cuda.synchronize()
    mixed = {k: v.clone() for k, v in obs.items()}
    assert torch.isfinite(mixed["object_ob"]).all() and (info[:, 3] == 3).all()
    assert env.bucket_of(16) == ("bookcase_expedit_0376", 0) and env.bucket_of(35) == ("toy_table_flip", 11)
    off = 0
    for name, n in zip(names, counts):
        alone = BatchedFurnitureEnv("Sawyer", name, n, seed=77 + off)
        alone.reset()
        for a in acts:
            od, _, _, _ = alone.step(a[off : off + n].contiguous())
        torch.cuda.synchronize()
        assert torch.equal(od["object_ob"], mixed["object_ob"][off : off + n, : alone.object_ob_dim]), name
        assert torch.equal(od["robot_ob"], mixed["robot_ob"][off : off + n]), name
        assert (mixed["object_ob"][off : off + n, alone.object_ob_dim :] == 0).all()
        alone.close()
        off += n
    env.close()


def test_furniture_buckets_are_spread_over_ranks_by_cost():
    """mixed batch over several GPUs (SURVEY.md 8e): whole buckets per rank, balanced by envs * nv^3, same answer on every rank"""
    from furniture_b200.env import shard_furniture

    nv = {n: mjcf.load_scene("Sawyer", n).nv for n in NAMES}
    owned = shard_furniture(NAMES, 128, 8, nv=[nv[n] for n in NAMES])
    assert sorted(n for r in owned for n, _ in r) == NAMES and all(c == 128 for r in owned for _, c in r)
    load = [sum(c * nv[n] ** 3 for n, c in r) for r in owned]
    assert max(load) < 1.15 * (sum(load) / 8)  # LPT keeps the heaviest rank within 15 % of the mean here
    assert owned == shard_furniture(NAMES, 128, 8, nv=[nv[n] for n in NAMES])
    one = shard_furniture(["table_lack_0825", "toy_table"], [10, 20], 1, nv=[39, 39])
    assert one == [[("toy_table", 20), ("table_lack_0825", 10)]]
