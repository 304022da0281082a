"""What per-episode missions cost on the GPU: BabyAI env-steps/s with missions off and on, and the render kernels.

    python scripts/bench_missions.py [--ids ID,...] [--envs 262144] [--rounds 3] [--steps 300] [--warmup 50]

For every id, `--rounds` alternated A/B rounds: a missions=False and a missions=True MinigridVecEnv of the same id, each
stepped `--steps` times (after `--warmup` steps) with uniform random actions from a pool of 16 device tensors, timed with
CUDA events around the whole loop (NEXT_STEP autoreset, so the resets of every ended episode are inside the loop). Then
the time per call of the three render kernels (mg_mission_text, mg_mission_indices through DictObservationSpaceWrapper,
mg_obs_flat_missions through FlatObsWrapper) on the missions=True handle, averaged over 50 calls. Prints one JSON line,
with the GPU's name and power limit read in the same run. Writes nothing to the tree.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
IDS = ["BabyAI-GoToLocal-v0", "BabyAI-PutNextLocal-v0", "BabyAI-OpenDoorsOrderN4-v0", "BabyAI-UnlockLocalDist-v0"]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power, sm_max = (s.strip() for s in q.split(","))
    return {"gpu": name, "power_limit_w": float(power), "sm_max_mhz": float(sm_max)}


def steps_per_s(env, pool, steps, warmup):
    import torch

    env.reset(seed=0)
    for t in range(warmup):
        env.step(pool[t % len(pool)])
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for t in range(steps):
        env.step(pool[t % len(pool)])
    e.record()
    e.synchronize()
    return env.num_envs * steps / (s.elapsed_time(e) / 1e3)


def time_call(fn, calls=50):
    import torch

    fn()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(calls):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / calls * 1e3  # us per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ids", default=",".join(IDS))
    ap.add_argument("--envs", type=int, default=262144)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=50)
    args = ap.parse_args()
    import torch

    import minigrid_b200 as mb

    n = args.envs
    g = torch.Generator(device="cuda").manual_seed(0)
    pool = [torch.randint(0, 7, (n,), device="cuda", dtype=torch.int32, generator=g) for _ in range(16)]
    res = {**gpu_info(), "envs": n, "steps": args.steps, "rounds": args.rounds, "ids": {}}
    for env_id in args.ids.split(","):
        envs = {False: mb.MinigridVecEnv(env_id, n, missions=False), True: mb.MinigridVecEnv(env_id, n, missions=True)}
        r = {"off": [], "on": []}
        for _ in range(args.rounds):
            for on in (False, True):
                r["on" if on else "off"].append(steps_per_s(envs[on], pool, args.steps, args.warmup))
        env = envs[True]
        obs = env._obs()
        text = torch.empty((n, 96), dtype=torch.uint8, device="cuda")
        dict_w = None if env_id not in mb_dict_ids() else mb.DictObservationSpaceWrapper(env)
        flat_w = mb.FlatObsWrapper(env)
        r["render_us"] = {"text": time_call(lambda: env.mission_text(out=text)),
                          "flat": time_call(lambda: flat_w.observation(obs))}
        if dict_w is not None:
            r["render_us"]["indices"] = time_call(lambda: dict_w.observation(obs))
        for k in ("off", "on"):
            r[k + "_median"] = sorted(r[k])[len(r[k]) // 2]
        r["on_over_off"] = r["on_median"] / r["off_median"]
        res["ids"][env_id] = r
        for e in envs.values():
            e.close()
    print(json.dumps(res))


def mb_dict_ids():
    from minigrid_b200 import specs
    from minigrid_b200.wrappers import MINIGRID_WORDS

    return {i for i in list(specs.BABYAI_REGISTRY) + list(specs.BABYAI_PICKUP_PUTNEXT_REGISTRY) + list(specs.BABYAI_OPEN_REGISTRY)
            if specs.babyai_mission_words(specs.get(i)) <= set(MINIGRID_WORDS)}


if __name__ == "__main__":
    main()
