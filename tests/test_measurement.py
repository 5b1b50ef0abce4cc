"""Source-level invariants of the kernels that are benched."""
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ik_step_restates_the_stock_step_blocks_verbatim():
    """csrc/fe_ik.h carries its own copy of the control-mapping block and of everything that follows the simulation in fe_env_step_one
    (fe_env.h is frozen as the profiled build, see fe_ik.h's header).  The copies may differ from the original only where they say so:
    the policy action's length is a parameter, and the reset after a failed simulation is decided by the caller."""
    csrc = os.path.join(ROOT, "furniture_b200", "csrc")
    env = open(os.path.join(csrc, "fe_env.h")).read()
    ik = open(os.path.join(csrc, "fe_ik.h")).read()
    body = env[env.index("FE_FN void fe_env_step_one("):env.index("// per-env context set-up shared by the CUDA kernels")]
    ctrl = body[body.index("  LANES_BEGIN\n    for (int u = lane; u < m->nu; u += 32) { // _setup_action"):body.index("  for (int i = 0; i < cfg->nsub; ++i) fe_substep_lockstep(w); // _do_simulation")]
    after = body[body.index("  FE_SYNC;\n  if (fail) {"):body.rindex("}")]
    assert ctrl in ik, "fe_ik_controls no longer equals the _setup_action block of fe_env_step_one"
    want = after.replace("sc->act_dim", "act_dim").replace("  FE_SYNC;\n  if (fail) {", "  FE_SYNC;\n  if (reset_now) {", 1)
    assert want in ik, "fe_ik_finish no longer equals the post-simulation part of fe_env_step_one"
