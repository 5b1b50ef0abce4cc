"""Time the env step in which every env of a batch finishes its episode, against the ordinary steps around it (CUDA events, one GPU).

  python tools/time_episode_end.py [--envs 4096] [--max-steps 10] [--episodes 4]

Every env starts its episode at the same reset and has max_episode_steps = --max-steps, so the last step of each episode ends every env's
episode at once: that launch runs the auto-reset (301 mj_steps per env) and, where the build has them, the writes of the terminal
observation and state.  Only the BatchedFurnitureEnv surface is used, so the script runs on builds with or without those writes.  The
first episode is a warm-up.  Prints one JSON line: the finishing steps' and the ordinary steps' times in milliseconds (median, min, max
over the episodes after the first), a checksum of the observations the finishing steps return, and the card's name, power limit and the SM
clock read right after the timed steps, which belong beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--max-steps", type=int, default=10)
    ap.add_argument("--episodes", type=int, default=4)
    args = ap.parse_args()
    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("time_episode_end needs a CUDA device: a step time measured anywhere else says nothing")
    from furniture_b200.env import BatchedFurnitureEnv

    env = BatchedFurnitureEnv("Sawyer", "table_lack_0825", args.envs, max_episode_steps=args.max_steps)
    rng = np.random.RandomState(0)
    acts = torch.from_numpy(rng.uniform(-1, 1, (args.max_steps, args.envs, env.act_dim)).astype(np.float32)).to(env.device)
    acts[:, :, -1] = -1.0  # no connect request: every episode ends at the time limit
    env.reset()
    end_ms, ord_ms, checksum = [], [], 0.0
    for ep in range(args.episodes):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(args.max_steps + 1)]
        ev[0].record()
        for t in range(args.max_steps):
            ob, rew, done, info = env.step(acts[t])
            ev[t + 1].record()
            if t == args.max_steps - 1:
                d = done.bool()
                obs_sum = float(sum(v.double().sum() for v in ob.values()))
        torch.cuda.synchronize()
        assert bool(d.all()), "not every env finished at the time limit"
        ms = [ev[t].elapsed_time(ev[t + 1]) for t in range(args.max_steps)]
        if ep == 0:
            continue  # warm-up episode
        end_ms.append(ms[-1])
        ord_ms += ms[1:-1]  # the first step of an episode follows the host's reads of the last one
        checksum += obs_sum
    stat = lambda x: {"median": float(np.median(x)), "min": float(np.min(x)), "max": float(np.max(x)), "n": len(x)}
    out = {"envs": args.envs, "max_episode_steps": args.max_steps, "finishing_step_ms": stat(end_ms), "ordinary_step_ms": stat(ord_ms),
           "finishing_obs_checksum": checksum, "gpu": torch.cuda.get_device_name(0)}
    try:  # read right after the timed steps, so that the SM clock is the one they ran at
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"], text=True).strip()
        out["power_limit"], out["sm_clock_after"] = [x.strip() for x in q.split(",")]
    except Exception:
        out["power_limit"] = out["sm_clock_after"] = None
    print(json.dumps(out))


if __name__ == "__main__":
    main()
