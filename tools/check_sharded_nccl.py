"""Multi-GPU check of ShardedFurnitureEnv over NCCL (run under torchrun, one rank per GPU):
  torchrun --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tools/check_sharded_nccl.py
Every rank steps its own shard; the all-gathered [obs | reward | done] must contain every rank's local tensors bit for
bit, the shards must differ (per-rank seeds), and a shard must be bit-identical to the same envs stepped alone.  The full message
(gather_info, gather_terminal; episodes of 2 steps) must carry every rank's info and, where done, terminal observation bit for bit."""
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch
import torch.distributed as dist

from furniture_b200.env import BatchedFurnitureEnv, ShardedFurnitureEnv

local = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
rank, world = dist.get_rank(), dist.get_world_size()
n = 64
env = ShardedFurnitureEnv(n)
env.timing = True
# the same envs run alone with the same seed and actions are the truth for this rank's slice (no cross-rank coupling)
alone = BatchedFurnitureEnv("Sawyer", "table_lack_0825", n, device=local, seed=ShardedFurnitureEnv.shard_seed(123, rank, n))
od = env.reset()
alone.reset()
assert od["object_ob"].shape == (n * world, 35) and od["robot_ob"].shape == (n * world, 29)
assert torch.equal(torch.cat([od["object_ob"], od["robot_ob"]], 1)[rank * n : (rank + 1) * n], alone._obs)
gen = torch.Generator(device=dev).manual_seed(rank)
for k in range(3):
    a = torch.rand((n, env.env.act_dim), device=dev, generator=gen) * 2 - 1
    od, rew, done, info = env.step(a)
    alone.step(a)
    full = torch.cat([od["object_ob"], od["robot_ob"]], 1)
    mine = full[rank * n : (rank + 1) * n]
    assert torch.equal(mine, alone._obs), "my slice of the gathered tensor is not my shard"
    assert torch.equal(env.local_slice(rew), alone._rew) and torch.equal(env.local_slice(done), alone._done > 0)
    # every rank holds the same gathered tensor
    chk = [torch.zeros_like(full) for _ in range(world)]
    dist.all_gather(chk, full.contiguous())
    for c in chk:
        assert torch.equal(c, full)
    other = full[((rank + 1) % world) * n : ((rank + 1) % world + 1) * n]
    assert not torch.allclose(other[:, :2], mine[:, :2]), "shards with different seeds placed parts identically"
    assert torch.isfinite(full).all()
# the full message: [obs | reward | done | info | terminal_obs]
full = ShardedFurnitureEnv(n, gather_info=True, gather_terminal=True, max_episode_steps=2)
alone = BatchedFurnitureEnv("Sawyer", "table_lack_0825", n, device=local, seed=ShardedFurnitureEnv.shard_seed(123, rank, n), max_episode_steps=2)
full.reset()
alone.reset()
for k in range(3):
    a = torch.rand((n, full.env.act_dim), device=dev, generator=gen) * 2 - 1
    od, rew, done, info = full.step(a)
    alone.step(a)
    assert info.shape == (n * world, 6) and info.dtype == torch.int32
    parts = [torch.zeros_like(alone._info) for _ in range(world)]
    dist.all_gather(parts, alone._info)
    assert torch.equal(info, torch.cat(parts, 0)), "the gathered info is not every rank's info"
    mine = torch.cat(list(alone.terminal_observation().values()), 1).contiguous()
    parts = [torch.zeros_like(mine) for _ in range(world)]
    dist.all_gather(parts, mine)
    to = torch.cat(list(full.terminal_observation().values()), 1)
    d = done.bool()
    assert d.any() == (k == 1) and torch.equal(to[d], torch.cat(parts, 0)[d]), "the gathered terminal rows are not every rank's"
km, gm = env.pop_timing()
assert len(km) == 3 and all(v > 0 for v in km + gm)
dist.barrier()
dist.destroy_process_group()
print("rank %d of %d ok (kernel %.2f ms, gather %.3f ms)" % (rank, world, sum(km) / 3, sum(gm) / 3))
