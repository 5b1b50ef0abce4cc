"""Step time of one batch at 10 Hz, at 20 Hz, and with half its envs at each (interleaved: env i at 10 Hz for even i), so that every
block of the step launch holds both substep counts at first.  CUDA events around every env step; the three batches are timed in
turn, `--rounds` times, so that the spread between rounds shows next to the differences.  One JSON line with the card's name and
power limit.

  python tools/time_control_freq.py --envs 4096 --steps 20 --warmup 5 --rounds 2
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip().splitlines()[0]
        name, power = (x.strip() for x in out.split(","))
        return name, power
    except Exception:
        return None, None


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
        raise SystemExit("time_control_freq.py needs a CUDA device")
    n = args.envs
    batches = {"10Hz": 10, "20Hz": 20, "mixed_10_20": np.where(np.arange(n) % 2 == 0, 10, 20)}
    envs = {k: BatchedFurnitureEnv("Sawyer", args.furniture, n, control_freq=v) for k, v in batches.items()}
    gen = torch.Generator(device="cuda").manual_seed(0)
    times = {k: [] for k in batches}
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
            times[k].append(float(np.median(ms)))
    name, power = card()
    print(json.dumps({"envs": n, "furniture": args.furniture, "steps": args.steps, "gpu": name, "power_limit": power,
                      "median_step_ms_per_round": times}))
    for env in envs.values():
        env.close()


if __name__ == "__main__":
    main()
