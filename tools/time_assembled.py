"""Step time of one batch whose episodes start from random placement, one whose episodes start from the assembled furniture, and one
with half its envs each (interleaved: env i assembled for odd i), so that every block of the step launch holds both at first.  CUDA events
around every env step; the three batches are timed in turn, `--rounds` times, so that the spread between rounds shows next to the
differences.  Per batch it also reports, from the `stats` field of the timed steps, the mean over envs and steps of FE_STAT_COUPLED (solves
whose coupled component holds a free part), FE_STAT_SOLVE and FE_STAT_SOLVE_COMP (cycles / 16 of the constraint solve and of the register
solver of the component) and FE_STAT_SOLVE_MAX (cycles / 16 of the slowest solve).  One JSON line with the card's name, power limit and SM
clock, read right after the timed steps.

  python tools/time_assembled.py --envs 4096 --steps 20 --warmup 5 --rounds 2
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from furniture_b200.engine import STAT_COUPLED, STAT_SOLVE, STAT_SOLVE_COMP, STAT_SOLVE_MAX  # noqa: E402

STATS = {"coupled": STAT_COUPLED, "solve": STAT_SOLVE, "solve_comp": STAT_SOLVE_COMP, "solve_max": STAT_SOLVE_MAX}


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"], text=True)
        return [x.strip() for x in out.strip().splitlines()[0].split(",")]
    except Exception:
        return None, None, None


def main():
    import torch

    from furniture_b200.env import BatchedFurnitureEnv

    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--furniture", default="table_lack_0825")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_assembled.py needs a CUDA device")
    n = args.envs
    batches = {"default": np.zeros(n, bool), "assembled": np.ones(n, bool), "mixed": np.arange(n) % 2 == 1}
    envs = {}
    for k, flags in batches.items():
        env = envs[k] = BatchedFurnitureEnv("Sawyer", args.furniture, n)
        env.set_reset_options(assembled=True, envs=np.flatnonzero(flags))
    gen = torch.Generator(device="cuda").manual_seed(0)
    times = {k: [] for k in batches}
    stats = {k: {s: [] for s in STATS} for k in batches}
    for env in envs.values():
        env.reset()
        for _ in range(args.warmup):
            env.step(torch.rand((n, env.act_dim), device="cuda", generator=gen) * 2 - 1)
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for k, env in envs.items():
            ms = []
            for _ in range(args.steps):
                a = torch.rand((n, env.act_dim), device="cuda", generator=gen) * 2 - 1
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                env.step(a)
                e.record()
                e.synchronize()
                ms.append(s.elapsed_time(e))
                st = env.engine.get("stats")
                for name, col in STATS.items():
                    stats[k][name].append(float(st[:, col].mean()))
            times[k].append(float(np.median(ms)))
    name, power, clock = card()
    print(json.dumps({"envs": n, "furniture": args.furniture, "steps": args.steps, "gpu": name, "power_limit": power, "sm_clock_after": clock,
                      "median_step_ms_per_round": times,
                      "stats_mean_per_env_step": {k: {s: float(np.mean(v)) for s, v in d.items()} for k, d in stats.items()}}))
    for env in envs.values():
        env.close()


if __name__ == "__main__":
    main()
