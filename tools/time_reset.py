"""Time one fe_env_reset of a batch with nothing preassembled and with k recipe steps preassembled (CUDA events, one GPU).

  python tools/time_reset.py [--envs 4096] [--k 3] [--repeats 5] [--reward sparse|dense]

Prints one JSON line: milliseconds per reset launch for k = 0 and for k (median and spread over the repeats, after one warm-up
reset of each), with the card's name and power limit, which belong beside the numbers.
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
    ap.add_argument("--k", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--reward", default="sparse", choices=["sparse", "dense"])
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("time_reset needs a CUDA device: a reset time measured anywhere else says nothing")
    from furniture_b200.env import BatchedFurnitureEnv

    env = BatchedFurnitureEnv("Sawyer", "table_lack_0825", args.envs, dense={} if args.reward == "dense" else None)
    out = {"envs": args.envs, "reward": args.reward, "gpu": torch.cuda.get_device_name(0)}
    try:
        out["power_limit"] = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], text=True).strip()
    except Exception:
        out["power_limit"] = None
    for k in (0, args.k):
        env.set_subtask(k)
        env.reset()  # warm-up: module load, and the first reset from creation state
        ms = []
        for _ in range(args.repeats):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            env.reset()
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
        ms.sort()
        out["k%d_ms" % k] = {"median": ms[len(ms) // 2], "min": ms[0], "max": ms[-1]}
        assert int(env.engine.get("num_connected").min()) == k
    print(json.dumps(out))


if __name__ == "__main__":
    main()
