"""Developer script: every env holds a table leg between the finger tips (the coupled-component solve in every mj_step);
prints the cycle counters of the component solver for a few batch sizes (1 env = one warp alone on the GPU)."""
import sys, os
sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", "tests"))
import numpy as np, torch
from furniture_b200 import mjcf
from furniture_b200 import engine as E
from furniture_b200.engine import Engine, default_config
from oracle.ref_env import OracleFurnitureEnv
from test_env_parity import _grasp_and_align_state
m = mjcf.load_scene("Sawyer", "table_lack_0825")
env = OracleFurnitureEnv(m); env.reset()
q = _grasp_and_align_state(m, env)
from parity_util import settled_state
qs = settled_state(m, 0, dz=0.0)
q2 = qs.copy(); q2[:9] = q[:9]; q2[9:16] = q[9:16]  # leg 0 between the pads; the other parts rest on the floor
q = q2
for N in [int(a) for a in sys.argv[1:]] or [1, 7, 132 * 7, 4096]:
    eng = Engine(m, N, 0, default_config(), lib_path=os.environ.get("FE_LIB"))
    eng.env_reset()
    eng.set("qpos", q); eng.set("qvel", np.zeros(m.nv)); eng.set("qacc_warmstart", np.zeros(m.nv)); eng.forward()
    a = torch.zeros((N, eng.act_dim), device="cuda"); a[:, -2] = 1.0; a[:, -1] = -1.0
    obs = torch.empty((N, eng.obs_dim), device="cuda"); rew = torch.empty(N, device="cuda"); done = torch.empty(N, dtype=torch.uint8, device="cuda"); info = torch.empty((N, 6), dtype=torch.int32, device="cuda")
    for k in range(3):
        eng.env_step_dev(a.data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(3):
        eng.env_step_dev(a.data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
    e1.record(); torch.cuda.synchronize()
    st = eng.get("stats").astype(np.float64)
    nsol, its = st[:, E.STAT_NEWTON_SOLVES].sum(), st[:, E.STAT_NEWTON_ITERS].sum()
    cyc = st[:, [E.STAT_KIN, E.STAT_COLLIDE, E.STAT_ASSEMBLE, E.STAT_SOLVE, E.STAT_INTEGRATE, E.STAT_WAIT]] * 16
    pre = st[:, [E.STAT_SOLVE_PRE, E.STAT_SOLVE_GROUPED, E.STAT_SOLVE_COMP]] * 16
    cc = st[:, [E.STAT_NEWTON_SETUP, E.STAT_NEWTON_START, E.STAT_NEWTON_GRAD, E.STAT_NEWTON_HESSIAN, E.STAT_NEWTON_CHOL, E.STAT_NEWTON_PRODUCTS, E.STAT_NEWTON_LS]] * 16
    print("N=%d: %.2f ms per env-step batch; solves/env %.0f iterations/solve %.2f ncon %.0f | phases per mj_step: kin %.0f collide %.0f assemble %.0f solve %.0f integrate %.0f wait %.0f" % ((N, e0.elapsed_time(e1) / 3, nsol / N, its / max(nsol, 1), info[:, 4].float().mean().item()) + tuple(cyc.mean(0) / 50)))
    print("   per solve: preamble %.0f grouped+limits %.0f component %.0f (setup %.0f candidates %.0f) | per iteration: forces+JTf+grad %.0f H rows+pairs %.0f cholesky+solves %.0f Ms,Js %.0f line search %.0f" % (tuple(pre.sum(0) / max(nsol, 1)) + tuple(cc[:, :2].sum(0) / max(nsol, 1)) + tuple(cc[:, 2:].sum(0) / max(its, 1))))
    eng.close()
