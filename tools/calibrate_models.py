"""Measures, on one GPU, the step time of every compiled furniture model (Sawyer + furniture, N envs, random actions) and writes
furniture_b200/compiled/cost.json: microseconds of GPU time per env-step per env.  shard_furniture balances the buckets of a
mixed batch with these numbers instead of the nv^3 guess."""
import json, os, sys
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import torch
from furniture_b200.engine import FLAG_CONTACT_FULL
from furniture_b200.env import BatchedFurnitureEnv

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
cdir = os.path.join(ROOT, "furniture_b200", "compiled")
names = sorted(f[len("Sawyer_"):-4] for f in os.listdir(cdir) if f.startswith("Sawyer_") and f.endswith(".npz"))
N = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
out = {}
for name in names:
    env = BatchedFurnitureEnv("Sawyer", name, N, seed=123)
    env.reset()
    g = torch.Generator(device="cuda").manual_seed(0)
    acts = [torch.rand((N, env.act_dim), device="cuda", generator=g) * 2 - 1 for _ in range(7)]
    for a in acts[:3]:
        env.step(a)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for a in acts[3:]:
        env.step(a)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 4
    out[name] = {"us_per_env_step": ms * 1e3 / N, "ms_per_step_at_%d" % N: ms, "nv": int(env.model.nv), "smem_bytes_per_env": int(env.engine.L.fe_smem_bytes_per_env(env.engine.h)),
                 "overflow_envs": int((env.engine.get("flags")[:, 0] & FLAG_CONTACT_FULL).sum())}
    print(name, out[name], flush=True)
    env.close()
json.dump(out, open(os.path.join(ROOT, "gpurun_out", "model_cost.json"), "w"), indent=1)
