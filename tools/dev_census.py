"""Developer script: how often does the per-env contact capacity overflow under the bench workload (random actions)?"""
import sys, os
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import numpy as np, torch
from furniture_b200 import mjcf
from furniture_b200.engine import FLAG_CONTACT_FULL, Engine, default_config
N = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 30
m = mjcf.load_scene("Sawyer", "table_lack_0825")
eng = Engine(m, N, 0, default_config(maxcon=int(os.environ.get("FE_MAXCON", "0"))))
eng.env_reset()
g = torch.Generator(device="cuda").manual_seed(0)
obs = torch.empty((N, eng.obs_dim), device="cuda"); rew = torch.empty(N, device="cuda"); done = torch.empty(N, dtype=torch.uint8, device="cuda"); info = torch.empty((N, 6), dtype=torch.int32, device="cuda")
hist = np.zeros(200, int)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for k in range(steps):
    act = torch.rand((N, eng.act_dim), device="cuda", generator=g) * 2 - 1
    if k == 5: e0.record()
    eng.env_step_dev(act.data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
    nc = info[:, 4].cpu().numpy()
    hist += np.bincount(np.minimum(nc, 199), minlength=200)
e1.record(); torch.cuda.synchronize()
fl = eng.get("flags")[:, 0]
print("maxcon", eng.cfg.maxcon, "after", steps, "steps: envs with overflow bit", int((fl & FLAG_CONTACT_FULL).sum()), "other bits", int((fl & ~FLAG_CONTACT_FULL != 0).sum()), "of", N)
print("ncon at step end: p50 %d p90 %d p99 %d max %d; share of (env,step) with ncon >= 36: %.3f%%, >= 40: %.3f%%" % (
    np.searchsorted(np.cumsum(hist), 0.5 * hist.sum()), np.searchsorted(np.cumsum(hist), 0.9 * hist.sum()), np.searchsorted(np.cumsum(hist), 0.99 * hist.sum()),
    np.nonzero(hist)[0].max(), 100 * hist[36:].sum() / hist.sum(), 100 * hist[40:].sum() / hist.sum()))
print("ms per step (steps 5..): %.2f" % (e0.elapsed_time(e1) / (steps - 5)))
