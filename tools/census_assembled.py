"""Contact census of assembled starts on the lane-emulated build: for every compiled robot scene, one env with `assembled` on, reset + 20
random env steps; per scene the contact capacity (auto_maxcon), the largest `ncon` seen after the reset and after each step, and whether
FE_FLAG_CONTACT_FULL was ever raised.  One JSON line per scene.

  python tools/census_assembled.py [--steps 20] [--only Sawyer_table_lack_0825 ...]
"""
import argparse
import glob
import json
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
from furniture_b200 import mjcf  # noqa: E402
from furniture_b200.engine import FLAG_CONTACT_FULL, Engine  # noqa: E402
from parity_util import build_emu  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--only", nargs="*")
    args = ap.parse_args()
    scenes = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(ROOT, "furniture_b200", "compiled", "*.npz")))
    for scene in scenes:
        agent, furniture = scene.split("_", 1)
        if agent == "Cursor" or (args.only and scene not in args.only):  # the Cursor env's reset is host logic: no assembled start
            continue
        eng = Engine(mjcf.load_scene(agent, furniture), 1, lib_path=build_emu(), assembled=True)
        eng.set("flags", 0)
        eng.env_reset()
        ncon, full = [int(eng.get("ncon")[0, 0])], bool(eng.get("flags")[0, 0] & FLAG_CONTACT_FULL)
        rng = np.random.RandomState(0)
        for _ in range(args.steps):
            a = rng.uniform(-1, 1, (1, eng.act_dim)).astype(np.float32)
            eng.env_step_host(a)
            ncon.append(int(eng.get("ncon")[0, 0]))
            full |= bool(eng.get("flags")[0, 0] & FLAG_CONTACT_FULL)
        print(json.dumps({"scene": scene, "npart": int(eng.scene.npart), "maxcon": int(eng.cfg.maxcon), "max_ncon": max(ncon), "contact_full": full}),
              flush=True)
        eng.close()


if __name__ == "__main__":
    main()
