"""k_hash (MinigridVecEnv.hash_digest, MiniGridEnv.hash) on the GPU: one JSON line with, per workload, the device-event
time of a call, SHA-256 blocks per second and the share of the SMs' issue slots. Writes nothing to the tree.

    python scripts/bench_hash.py [--envs 262144] [--calls 50]

The state is what 40 forward-heavy random steps after a seeded reset leave. The blocks of an env are its prefix blocks
plus the one or two final blocks of its tail, counted for the numpy-int form of agent_pos (the form after any forward
move). The issue share takes SASS_PER_BLOCK warp instructions per 32 blocks against 4 issue slots per SM per clock.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# SASS instructions of one prefix block of k_hash: the static length of the block loop's body in `cuobjdump -sass` of
# the sm_90a build (mg_hash.cu, the loop that ends in the backward branch around the first sha256_compress). The digit
# slots behind warp-uniform branches make it an upper bound per block.
SASS_PER_BLOCK = 1796
ENVS = ["MiniGrid-DoorKey-8x8-v0", "MiniGrid-FourRooms-v0"]


def sm_clock_and_power(dev_index):
    """(a function that reads the SM clock in MHz, the power limit in W) through NVML, or (None, None)."""
    try:
        import pynvml

        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(dev_index)
        return (lambda: float(pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)),
                pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000)
    except Exception:  # noqa: BLE001
        return None, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=262144)
    ap.add_argument("--calls", type=int, default=50)
    args = ap.parse_args()
    import torch

    from minigrid_b200 import MinigridVecEnv

    if not torch.cuda.is_available():
        raise SystemExit("bench_hash.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    props = torch.cuda.get_device_properties(dev)
    clock, power = sm_clock_and_power(0)
    out = {"kernel": "k_hash (K4, MiniGridEnv.hash)", "gpu": props.name, "power_limit_w": power, "sms": props.multi_processor_count,
           "sass_instructions_per_block": SASS_PER_BLOCK, "calls": args.calls, "envs": []}
    n = args.envs
    for env_id in ENVS:
        e = MinigridVecEnv(env_id, n, device=dev)
        e.reset(seed=0)
        g = torch.Generator(device=dev).manual_seed(1)
        for _ in range(40):
            a = torch.where(torch.rand(n, generator=g, device=dev) < 0.5, 2, torch.randint(0, 7, (n,), generator=g, device=dev))
            e.step(a.to(torch.int32))
        d = torch.empty((n, 32), dtype=torch.uint8, device=dev)
        for _ in range(3):
            e.hash_digest(d)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.calls):
            e.hash_digest(d)
        t1.record()
        mhz = [clock() for _ in range(5)] if clock else []  # sampled while the calls run
        torch.cuda.synchronize()
        us = t0.elapsed_time(t1) * 1e3 / args.calls
        L = 11 * e.width * e.height + 2 * e.width
        xy = e.get_state()["agent"][:, :2].cpu().numpy()
        tail = 27 + (xy[:, 0] >= 10) + (xy[:, 1] >= 10)  # "(np.int64(x), np.int64(y))" + the direction digit
        blocks = int(np.sum(L // 64 + ((L % 64 + tail + 9 + 63) // 64)))
        sm_mhz = float(np.median(mhz)) if mhz else None
        issue = (SASS_PER_BLOCK * blocks / 32) / (props.multi_processor_count * 4 * sm_mhz * 1e6 * us * 1e-6) if sm_mhz else None
        out["envs"].append({"env": env_id, "envs": n, "us_per_call": us, "sha256_blocks_per_call": blocks,
                            "blocks_per_s": blocks / (us * 1e-6), "sm_mhz": sm_mhz, "issue_bound_share": issue})
        del e, d
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
