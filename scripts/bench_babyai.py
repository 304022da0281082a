"""BabyAI GoTo env-steps/s on the GPU, and the cost of the BabyAI branch to the existing roomgrid kinds.

    python scripts/bench_babyai.py [--ids ID,...] [--parent DIR] [--ab-ids ID,...] [--repeats 3] [--steps 400]

Runs `bench.py --env ID --no-configs --no-cpu-baseline` (262144 envs, desynchronised NEXT_STEP episodes, CUDA graphs)
as a subprocess per measurement and prints one JSON line: the headline value of every BabyAI id in --ids (default IDS),
and, with --parent pointing at a built checkout of an earlier revision, the A/B of every id in --ab-ids (default
AB_IDS: the DoorKey-8x8 headline and KeyCorridorS6R3) between that checkout and this one, the two alternated
`--repeats` times. The GPU's name and power
limit are read in the same run. Writes nothing to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDS = ["BabyAI-GoToLocal-v0", "BabyAI-GoToRedBallGrey-v0", "BabyAI-GoToRedBlueBall-v0"]
AB_IDS = ["MiniGrid-DoorKey-8x8-v0", "MiniGrid-KeyCorridorS6R3-v0"]


def bench(tree, env_id, steps, warmup):
    cmd = [sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", str(warmup),
           "--env", env_id, "--no-configs", "--no-cpu-baseline"]
    out = subprocess.run(cmd, cwd=tree, check=True, capture_output=True, text=True).stdout
    line = json.loads([ln for ln in out.splitlines() if ln.startswith("{")][-1])
    return {"value": line["value"], "ms_per_step": line["ms_per_step"], "sm_mhz": line["clocks"]["sm_mhz"],
            "autoreset_fraction_per_step": line["run"]["autoreset_fraction_per_step"]}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, sm_max = (s.strip() for s in q.split(","))
    return {"gpu": name, "power_limit_w": float(power), "sm_max_mhz": float(sm_max)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ids", default=",".join(IDS), help="comma-separated ids to measure")
    ap.add_argument("--parent", help="a built checkout of the revision to compare against")
    ap.add_argument("--ab-ids", default=",".join(AB_IDS), help="comma-separated ids of the A/B against --parent")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=50)
    args = ap.parse_args()
    res = {**gpu_info(), "envs": 262144, "steps": args.steps, "babyai": {}}
    for env_id in args.ids.split(","):
        res["babyai"][env_id] = bench(ROOT, env_id, args.steps, args.warmup)
    if args.parent:
        args.parent = os.path.abspath(args.parent)
        ab_ids = args.ab_ids.split(",")
        res["ab"] = {env_id: {"parent": [], "this": []} for env_id in ab_ids}
        for _ in range(args.repeats):
            for env_id in ab_ids:
                for side, tree in (("parent", args.parent), ("this", ROOT)):
                    res["ab"][env_id][side].append(bench(tree, env_id, args.steps, args.warmup)["value"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
