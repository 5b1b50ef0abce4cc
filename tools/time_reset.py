"""Time one fe_env_reset of a batch with nothing preassembled and with k recipe steps preassembled (CUDA events, one GPU).

  python tools/time_reset.py [--envs 4096] [--k 3] [--repeats 5] [--reward sparse|dense] [--init-state] [--assembled]

Prints one JSON line: milliseconds per reset launch for k = 0 and for k (median and spread over the repeats, after one warm-up
reset of each), with the card's name, power limit and the SM clock read right after the timed launches, which belong beside the numbers.  --init-state adds the same two
times for a batch whose envs all start from a recorded state (set_init_qpos): the state env 0 reached by the random reset with the
same k, so that the recipe's connectors already touch where the preassembly connects them.  --assembled adds the two times again with
every env's `assembled` option on (the welded furniture left at qpos0).
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
    ap.add_argument("--init-state", action="store_true")
    ap.add_argument("--assembled", action="store_true")
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("time_reset needs a CUDA device: a reset time measured anywhere else says nothing")
    from furniture_b200.env import BatchedFurnitureEnv

    env = BatchedFurnitureEnv("Sawyer", "table_lack_0825", args.envs, dense={} if args.reward == "dense" else None)
    out = {"envs": args.envs, "reward": args.reward, "gpu": torch.cuda.get_device_name(0)}
    def timed(key, k):
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
        out[key] = {"median": ms[len(ms) // 2], "min": ms[0], "max": ms[-1]}
        assert int(env.engine.get("num_connected").min()) == k

    for k in (0, args.k):
        env.set_subtask(k)
        env.set_init_qpos(None)
        timed("k%d_ms" % k, k)
        if args.init_state:
            st = env.get_env_state()
            env.set_init_qpos({"qpos": st["qpos"][0], "qvel": st["qvel"][0]})
            timed("init_state_k%d_ms" % k, k)
    if args.assembled:
        env.set_init_qpos(None)
        env.set_reset_options(assembled=True)
        for k in (0, args.k):
            env.set_subtask(k)
            timed("assembled_k%d_ms" % k, k)
    try:  # read right after the timed launches, so that the SM clock is the one they ran at
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"], text=True).strip()
        out["power_limit"], out["sm_clock_after"] = [x.strip() for x in q.split(",")]
    except Exception:
        out["power_limit"] = out["sm_clock_after"] = None
    print(json.dumps(out))


if __name__ == "__main__":
    main()
