"""Time the env step under the default observation layout and under object_ob_all=False, subtask_ob=True (CUDA events, one GPU).

  python tools/time_obs_layout.py [--envs 4096] [--steps 20] [--warmup 5] [--rounds 2]

Prints one JSON line: milliseconds per env step (median, min, max over the timed steps) for each layout, in alternating rounds on the same
card, with the card's name, power limit and the SM clock read right after the timed steps, which belong beside the numbers.  Both handles
start from the same seed and take the same random actions, so that they step the same physics.
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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("time_obs_layout needs a CUDA device: a step time measured anywhere else says nothing")
    from furniture_b200.env import BatchedFurnitureEnv

    layouts = {"default": {}, "pair_subtask": dict(object_ob_all=False, subtask_ob=True)}
    envs = {k: BatchedFurnitureEnv("Sawyer", "table_lack_0825", args.envs, **v) for k, v in layouts.items()}
    out = {"envs": args.envs, "gpu": torch.cuda.get_device_name(0), "obs_dim": {k: e.obs_dim for k, e in envs.items()}}
    ms = {k: [] for k in layouts}
    for _ in range(args.rounds):
        for key, env in envs.items():
            env.reset()
            g = torch.Generator(device="cuda").manual_seed(0)
            for s in range(args.warmup + args.steps):
                a = torch.rand((args.envs, env.act_dim), device=env.device, generator=g) * 2 - 1
                a[:, -1] = -1
                b, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                b.record()
                env.step(a)
                e.record()
                e.synchronize()
                if s >= args.warmup:
                    ms[key].append(b.elapsed_time(e))
    for key, v in ms.items():
        v.sort()
        out[key + "_ms"] = {"median": v[len(v) // 2], "min": v[0], "max": v[-1]}
    try:  # read right after the timed steps, so that the SM clock is the one they ran at
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"], text=True).strip()
        out["power_limit"], out["sm_clock_after"] = [x.strip() for x in q.split(",")]
    except Exception:
        out["power_limit"] = out["sm_clock_after"] = None
    print(json.dumps(out))


if __name__ == "__main__":
    main()
