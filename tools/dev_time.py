"""Developer script: time env steps on the GPU (device-resident actions)."""
import sys, os, time
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
import numpy as np, torch
from furniture_b200 import mjcf
from furniture_b200 import engine as E
from furniture_b200.engine import Engine, default_config
N = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
scale = float(sys.argv[3]) if len(sys.argv) > 3 else 1.0
m = mjcf.load_scene("Sawyer", "table_lack_0825")
eng = Engine(m, N, 0, default_config(maxcon=int(os.environ.get("FE_MAXCON", "0"))))
t = time.time(); eng.env_reset(); torch.cuda.synchronize(); print("reset wall %.3f s" % (time.time() - t), "flags nonzero", int((eng.get("flags") != 0).sum()))
g = torch.Generator(device="cuda").manual_seed(0)
act = (torch.rand((N, eng.act_dim), device="cuda", generator=g) * 2 - 1) * scale
obs = torch.empty((N, eng.obs_dim), device="cuda"); rew = torch.empty(N, device="cuda"); done = torch.empty(N, dtype=torch.uint8, device="cuda"); info = torch.empty((N, 6), dtype=torch.int32, device="cuda")
for w in range(2):
    eng.env_step_dev(act.data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for k in range(steps):
    act = (torch.rand((N, eng.act_dim), device="cuda", generator=g) * 2 - 1) * scale
    eng.env_step_dev(act.data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
e1.record(); torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / steps
print("N=%d  %.3f ms/env-step-batch  => %.0f env-steps/s  (%.2f us per mj_step batch)" % (N, ms, N / ms * 1e3, ms * 1e3 / 50))
print("mean ncon %.1f mean niter %.2f done %d unstable %d" % (info[:, 4].float().mean().item(), info[:, 5].float().mean().item(), int(done.sum()), int(info[:, 2].sum())))
st = eng.get("stats")
print("per env-step (50 substeps): coupled substeps mean %.2f  Newton solves mean %.2f  Newton iterations mean %.2f; envs with any coupled %.1f%%" % (st[:,E.STAT_COUPLED].mean(), st[:,E.STAT_NEWTON_SOLVES].mean(), st[:,E.STAT_NEWTON_ITERS].mean(), 100*(st[:,E.STAT_COUPLED]>0).mean()))
import numpy as np
print("coupled histogram", np.bincount(np.minimum(st[:,E.STAT_COUPLED], 50)//10, minlength=6), " Newton-solve histogram", np.bincount(np.minimum(st[:,E.STAT_NEWTON_SOLVES],50)//10, minlength=6))
names = ["kin_smooth", "collide", "assemble", "solve", "integrate", "barrier_wait"]
cyc = st[:, [E.STAT_KIN, E.STAT_COLLIDE, E.STAT_ASSEMBLE, E.STAT_SOLVE, E.STAT_INTEGRATE, E.STAT_WAIT]].astype(np.float64) * 16
solve = st[:, E.STAT_SOLVE].astype(np.float64) * 16
tot = cyc.sum(1)
print("cycles per env-step per warp: total mean %.0f max %.0f" % (tot.mean(), tot.max()))
for i, nme in enumerate(names): print("  %-13s mean %9.0f (%.1f%%)  p99 %9.0f  max %9.0f" % (nme, cyc[:, i].mean(), 100 * cyc[:, i].mean() / tot.mean(), np.percentile(cyc[:, i], 99), cyc[:, i].max()))
it = st[:, E.STAT_NEWTON_ITERS]
print("Newton iterations per env-step: max %d  p99 %d  p90 %d ; envs > 200: %d" % (it.max(), np.percentile(it, 99), np.percentile(it, 90), (it > 200).sum()))
worst = np.argsort(-solve)[:5]
for e in worst: print("  env %d: solve cycles %.0f coupled %d Newton solves %d Newton iters %d ncon %d" % (e, solve[e], st[e, E.STAT_COUPLED], st[e, E.STAT_NEWTON_SOLVES], st[e, E.STAT_NEWTON_ITERS], info[e, 4].item()))
print("parts-solver iterations (max over parts, summed over 50 substeps): mean %.1f p99 %d max %d" % (st[:,E.STAT_PART_ITERS].mean(), np.percentile(st[:,E.STAT_PART_ITERS],99), st[:,E.STAT_PART_ITERS].max()))
robot = st[:,E.STAT_ROBOT_ONLY]
print("substeps whose coupled component is the robot block alone (it touches something, no part coupled): mean %.2f, envs with any %.1f%%, hist" % (robot.mean(), 100*(robot>0).mean()), np.bincount(np.minimum(robot,50)//10, minlength=6))
mx = st[:,E.STAT_SOLVE_MAX].astype(np.float64)*16
print("slowest single-substep solve per env: mean %.0f p50 %.0f p90 %.0f p99 %.0f max %.0f cycles" % (mx.mean(), np.percentile(mx,50), np.percentile(mx,90), np.percentile(mx,99), mx.max()))
fastenv = st[:,E.STAT_COUPLED]==0
print("never-coupled envs: solve cycles mean %.0f p50 %.0f p90 %.0f p99 %.0f ; slowest substep p50 %.0f p90 %.0f p99 %.0f" % (solve[fastenv].mean(), np.percentile(solve[fastenv],50), np.percentile(solve[fastenv],90), np.percentile(solve[fastenv],99), np.percentile(mx[fastenv],50), np.percentile(mx[fastenv],90), np.percentile(mx[fastenv],99)))
print("never-coupled envs with no robot contact: solve mean %.0f, with: %.0f" % (solve[fastenv & (robot==0)].mean(), solve[fastenv & (robot>0)].mean()))
bw = st[:, [E.STAT_WAIT_KIN, E.STAT_WAIT_COLLIDE, E.STAT_WAIT_ASSEMBLE, E.STAT_WAIT_SOLVE, E.STAT_WAIT_INTEGRATE]].astype(np.float64) * 16
print("wait at the barrier before kin/collide/assemble/solve/integrate: mean", " ".join("%.0f" % v for v in bw.mean(0)), "| never-coupled:", " ".join("%.0f" % v for v in bw[fastenv].mean(0)))
heavy = np.argsort(-solve)[:40]
cc = st[heavy][:, [E.STAT_NEWTON_SETUP, E.STAT_NEWTON_START, E.STAT_NEWTON_GRAD, E.STAT_NEWTON_HESSIAN, E.STAT_NEWTON_CHOL, E.STAT_NEWTON_PRODUCTS, E.STAT_NEWTON_LS]].astype(np.float64) * 16
its = st[heavy][:, E.STAT_NEWTON_ITERS].astype(np.float64)
pre = st[heavy][:, [E.STAT_SOLVE_PRE, E.STAT_SOLVE_GROUPED, E.STAT_SOLVE_COMP]].astype(np.float64) * 16
nsol = st[heavy][:, E.STAT_NEWTON_SOLVES].astype(np.float64)
print("40 heaviest envs: component solves %.0f, Newton iterations mean %.0f; cycles per solve: preamble %.0f grouped+limits %.0f component %.0f | inside the component solver, per solve: setup %.0f candidates %.0f ; per iteration: forces+JTf+grad %.0f H rows+pairs %.0f cholesky+solves %.0f M s, J s %.0f line search %.0f" % ((nsol.mean(), its.mean()) + tuple(pre.sum(0) / nsol.sum()) + tuple(cc[:, :2].sum(0) / nsol.sum()) + tuple(cc[:, 2:].sum(0) / its.sum())))
if os.environ.get("FE_DUMP_STATS"):
    order_k = eng.get("order")  # the order the next step will run with
    act = (torch.rand((N, eng.act_dim), device="cuda", generator=g) * 2 - 1) * scale
    eng.env_step_dev(act.data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
    torch.cuda.synchronize()
    np.savez(os.environ["FE_DUMP_STATS"], st_prev=st, order=order_k, st=eng.get("stats"))
