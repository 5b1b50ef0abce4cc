"""Run on an H100: the paths that were written after this round's GPU budget was spent and have only run on the lane-emulated build --
the torque controllers (arithmetic hook + env steps) and control_type="ik_quaternion".  Prints one line per check; exit code 1 if any fails.
Once they pass, give the corresponding tests a `cuda` parameter (pytest.mark.gpu) like the other parity tests.

  python tools/check_cuda_pending.py
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402


def main():
    import parity_util
    import test_controllers as TC
    import test_ik as TI
    from furniture_b200 import mjcf
    from furniture_b200.engine import Engine

    # make the test helpers build CUDA engines instead of emulated ones
    parity_util.build_emu = lambda: None
    real_init = Engine.__init__

    def cuda_init(self, *a, lib_path=None, **k):
        real_init(self, *a, lib_path=None, **k)

    Engine.__init__ = cuda_init
    golden = {m: None for m in TC.MODES}
    g = np.load(os.path.join(ROOT, "tests", "golden", "controllers.npz"))
    golden = {m: {k.split("/")[1]: g[k] for k in g.files if k.startswith(m + "/")} for m in TC.MODES}
    torque = mjcf.load_scene("SawyerTorque", "table_lack_0825")
    sawyer = mjcf.load_scene("Sawyer", "table_lack_0825")
    checks = [("controller arithmetic %s" % m, lambda m=m: TC.test_device_controllers_reproduce_the_reference_emu.__wrapped__(golden, m)
               if hasattr(TC.test_device_controllers_reproduce_the_reference_emu, "__wrapped__") else TC.test_device_controllers_reproduce_the_reference_emu(golden, m)) for m in TC.MODES]
    checks += [("controller env %s" % m, lambda m=m: TC.test_controller_env_steps_match_the_cpu_env(torque, m)) for m in TC.MODES]
    checks += [("baxter ik env", lambda: TI.test_baxter_ik_env_steps_match_the_cpu_env(0)), ("baxter ik_quaternion env", lambda: TI.test_baxter_ik_env_steps_match_the_cpu_env(1)),
               ("ik_quaternion env", lambda: TI.test_ik_env_steps_match_the_cpu_env(sawyer, "emu-quaternion")),
               ("ik + dense env", lambda: TI.test_dense_reward_under_ik_control_matches_the_cpu_env(sawyer)),
               ("ik unstable step", lambda: TI.test_unstable_ik_step_resets_mid_step_and_once_more_at_the_end(sawyer))]
    bad = 0
    for name, fn in checks:
        try:
            fn()
            print("PASS", name)
        except Exception as e:  # noqa: BLE001
            bad += 1
            print("FAIL", name, "--", type(e).__name__, str(e)[:300])
    print("%d checks, %d failed" % (len(checks), bad))
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
