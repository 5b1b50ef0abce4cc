"""Golden vectors for control_freq, made by running the REFERENCE'S OWN Python, unmodified.

Runs only where the reference checkout is (make_golden_assembly.REF); writes tests/golden/sim_options.npz, which travels.
What is executed from the reference: furniture/env/furniture.py FurnitureEnv.initialize_time (:2849-2855), which sets
_control_timestep = 1.0 / control_freq and _model_timestep = sim.model.opt.timestep, and FurnitureEnv._do_simulation (:2857-2897), on a
stand-in whose sim counts the sim.step() calls of the `for _ in range(int(self._control_timestep / self._model_timestep))` loop.
Recorded: that count for every integer control_freq from 1 to 500 and every model timestep of the compiled scenes (the XML's
`timestep` attribute read as MuJoCo does, a float64).
"""
import glob
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
import make_golden_assembly as G  # noqa: E402

OUT = os.path.join(HERE, "..", "tests", "golden")
FREQS = np.arange(1, 501)


def scene_timesteps():
    from furniture_b200 import mjcf

    dts = set()
    for f in sorted(glob.glob(os.path.join(HERE, "..", "furniture_b200", "compiled", "*.npz"))):
        agent, furniture = os.path.basename(f)[:-4].split("_", 1)
        dts.add(float(mjcf.load_scene(agent, furniture).opt_timestep))
    return sorted(dts)


def main():
    _, FurnitureEnv = G.import_reference()

    class Sim:
        def __init__(self, dt):
            self.model = types.SimpleNamespace(opt=types.SimpleNamespace(timestep=dt))
            self.data = types.SimpleNamespace(ctrl=None)
            self.steps = 0

        def forward(self):
            pass

        def step(self):
            self.steps += 1

    dts = scene_timesteps()
    counts = np.zeros((len(dts), len(FREQS)), np.int64)
    for i, dt in enumerate(dts):
        for j, cf in enumerate(FREQS):
            env = object.__new__(FurnitureEnv)
            env.sim, env._control_freq, env._agent_type, env._unity = Sim(dt), int(cf), "Sawyer", None
            FurnitureEnv.initialize_time(env)
            env._fail = False
            FurnitureEnv._do_simulation(env, None)
            assert not env._fail, (dt, cf)
            counts[i, j] = env.sim.steps
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, "sim_options.npz"), timesteps=np.array(dts, np.float64), control_freq=FREQS, substeps=counts,
                        source="reference FurnitureEnv.initialize_time / _do_simulation run unmodified on a step-counting stand-in "
                               "(tools/make_golden_sim_options.py)")
    for dt, row in zip(dts, counts):
        print(dt, row[[0, 4, 9, 19, 499]])


if __name__ == "__main__":
    main()
