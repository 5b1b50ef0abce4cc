"""Time fe_env_step_packed under the default message layout [obs | reward | done] against the full one [obs | reward | done | info |
terminal_obs] (CUDA events, one GPU): what widening ShardedFurnitureEnv's all-gather message with gather_info / gather_terminal costs the
step kernel that writes it.

  python tools/time_sharded_message.py [--envs 4096] [--max-steps 10] [--episodes 5]

Two handles of Sawyer + table_lack_0825 with the same seed and actions, one per layout, run whole episodes in turn (default, full, default,
...), so that drift of the card's clock falls on both alike.  Every env has max_episode_steps = --max-steps, so the last step of each
episode ends every env's episode at once and writes every terminal slot: it is timed apart from the ordinary steps, as in
tools/time_episode_end.py.  The first episode of each handle is a warm-up.  The obs, reward and done columns of the two handles' rows are
compared bit for bit after the last step of every episode.  Prints one JSON line: per layout the row width and the finishing and ordinary steps' times in
milliseconds (median, min, max), and the card's name, power limit and the SM clock read right after the timed steps.
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
    ap.add_argument("--episodes", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("time_sharded_message needs a CUDA device: a step time measured anywhere else says nothing")
    from furniture_b200.env import build_engine

    torch.cuda.set_device(0)
    torch.zeros(1, device="cuda:0")
    n, T = args.envs, args.max_steps
    layouts = {"default": {}, "full": dict(info=True, terminal_obs=True)}
    engs, bufs = {}, {}
    for name, lay in layouts.items():
        engs[name] = e = build_engine("Sawyer", "table_lack_0825", n, max_episode_steps=T)
        e.set_packed_layout(**lay)
        bufs[name] = torch.zeros((n, e.packed_dim()), dtype=torch.float32, device="cuda:0")
        e.env_reset()
    od = engs["default"].obs_dim
    rng = np.random.RandomState(0)
    acts = torch.from_numpy(rng.uniform(-1, 1, (T, n, engs["default"].act_dim)).astype(np.float32)).to("cuda:0")
    acts[:, :, -1] = -1.0  # no connect request: every episode ends at the time limit
    stream = torch.cuda.current_stream().cuda_stream
    times = {name: {"finishing": [], "ordinary": []} for name in layouts}
    rows = {}
    for ep in range(args.episodes):
        for name, e in engs.items():
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(T + 1)]
            ev[0].record()
            for t in range(T):
                e.env_step_packed(acts[t].data_ptr(), bufs[name].data_ptr(), stream=stream)
                ev[t + 1].record()
            torch.cuda.synchronize()
            rows[name] = bufs[name][:, : od + 2].clone()
            assert bool((bufs[name][:, od + 1] == 1).all()), "not every env finished at the time limit"
            if ep == 0:
                continue  # warm-up episode
            ms = [ev[t].elapsed_time(ev[t + 1]) for t in range(T)]
            times[name]["finishing"].append(ms[-1])
            times[name]["ordinary"] += ms[1:-1]  # the first step of an episode follows the host's reads of the last one
        assert torch.equal(rows["default"], rows["full"]), "the two layouts disagree on [obs | reward | done]"
    stat = lambda x: {"median": float(np.median(x)), "min": float(np.min(x)), "max": float(np.max(x)), "n": len(x)}
    out = {"envs": n, "max_episode_steps": T}
    for name, e in engs.items():
        out[name] = {"row_floats": e.packed_dim(), "MB_per_rank": round(4 * n * e.packed_dim() / 1e6, 3),
                     "finishing_step_ms": stat(times[name]["finishing"]), "ordinary_step_ms": stat(times[name]["ordinary"])}
    out["gpu"] = torch.cuda.get_device_name(0)
    try:  # read right after the timed steps, so that the SM clock is the one they ran at
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"], text=True).strip()
        out["power_limit"], out["sm_clock_after"] = [x.strip() for x in q.split(",")]
    except Exception:
        out["power_limit"] = out["sm_clock_after"] = None
    print(json.dumps(out))


if __name__ == "__main__":
    main()
