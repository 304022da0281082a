"""The record of the reference's single-room BabyAI Pickup and PutNext levels. TEST INFRASTRUCTURE ONLY.

Runs the UNMODIFIED reference (oracle/ref_loader.py) on every id of minigrid_b200.specs.BABYAI_PICKUP_PUTNEXT_REGISTRY
and writes what tests/test_babyai_pickup_cpu.py and tests/test_gpu_babyai_pickup.py compare against, in the format of
oracle/ref_babyai.py's record: the dims, lockstep rollout traces in both autoreset modes, the mission after each of 50
seeded resets, the hash checks, DictObservationSpaceWrapper's mission indices of the ids whose mission is constant and
the observation-wrapper traces. Random actions almost never complete a PutNext, so it also holds scripted rollouts: the
actions of tests/babyai_pickup_oracle.py's ScriptedPolicy (a BFS on the reference env's own state: pick the target up,
or carry the move object next to the fixed one; every other env first moves the fixed object away) and the traces of
the reference under them. The reference prints "Sampling rejected: ..." for every rejected level; that output is
swallowed. Rewrite the record with

    python -m oracle.ref_babyai_pickup        (needs the reference tree, see oracle/ref_loader.py)
"""
from __future__ import annotations

import contextlib
import io
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RECORD = os.path.join(ROOT, "tests", "golden", "ref_babyai_pickup_traces.json")
N_ENVS, SEED, ACT_SEED, STEPS = 6, 1000, 77, 250
SCRIPT_SEED, SCRIPT_STEPS = 300, 200
MISSION_SEEDS = range(50)
CONSTANT_MISSION_IDS = ["BabyAI-OneRoomS8-v0", "BabyAI-OneRoomS12-v0", "BabyAI-OneRoomS16-v0", "BabyAI-OneRoomS20-v0"]
OBS_WRAPPER_IDS = ["BabyAI-OneRoomS8-v0", "BabyAI-OneRoomS20-v0", "BabyAI-PickupDistDebug-v0", "BabyAI-PutNextLocalS5N3-v0"]


def load_record():
    with open(RECORD) as f:
        return json.load(f)


def _instr(e):
    """The instruction as ScriptedPolicy reads it: ("pickup", (type, colour)) or ("putnext", move, fixed)."""
    ins = e.instrs
    if hasattr(ins, "desc_move"):
        return ("putnext", (ins.desc_move.type, ins.desc_move.color), (ins.desc_fixed.type, ins.desc_fixed.color))
    return ("pickup", (ins.desc.type, ins.desc.color))


def scripted_actions(ref, n, seed, steps):
    """ScriptedPolicy's actions on the reference's envs (ReferenceVecEnv, NEXT_STEP: the traces replay them in that
    mode): [steps][n] ints."""
    import numpy as np
    from babyai_pickup_oracle import ScriptedPolicy

    ref.reset(seed=seed)
    pols = [ScriptedPolicy(displace_fixed=i % 2 == 0) for i in range(n)]
    seen = [None] * n
    out = []
    for _ in range(steps):
        acts = []
        for i, e in enumerate(ref.envs):
            if seen[i] is not e.instrs:  # gen_mission makes a new instruction at every reset
                seen[i] = e.instrs
                pols[i].start(_instr(e))
            c = e.carrying
            acts.append(int(pols[i].act(e.grid.encode(), int(e.agent_pos[0]), int(e.agent_pos[1]), int(e.agent_dir),
                                        None if c is None else (c.type, c.color))))
        out.append(acts)
        ref.step(np.asarray(acts))
    return out


def record():
    from oracle import ref_trace as rt
    from oracle.ref_babyai import _reference_views, observation_wrappers
    from minigrid_b200.specs import BABYAI_PICKUP_PUTNEXT_REGISTRY
    from oracle.ref_loader import ReferenceVecEnv, load

    gym, _ = load()
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import hash_support as hs
    from babyai_pickup_oracle import scripted_rollout

    from minigrid.wrappers import DictObservationSpaceWrapper

    out = {"dims": {}, "lockstep": {}, "missions": {}, "hash_rollout": {}, "hash_walk": {}, "dict_missions": {},
           "obs_wrappers": {}, "scripted": {}}
    for env_id in BABYAI_PICKUP_PUTNEXT_REGISTRY:
        e = gym.make(env_id).unwrapped
        e.reset(seed=0)  # max_steps is set by the first reset (roomgrid_level.py:71-85)
        out["dims"][env_id] = [e.width, e.height, e.max_steps, bool(e.see_through_walls)]
        missions = []
        for s in MISSION_SEEDS:
            e.reset(seed=s)
            missions.append(e.mission)
        out["missions"][env_id] = missions
        for mode in rt.MODES:
            out["lockstep"][rt.key(env_id, mode)] = rt.rollout(ReferenceVecEnv(env_id, N_ENVS, autoreset=mode), N_ENVS,
                                                               SEED, ACT_SEED, STEPS)
            out["hash_rollout"][rt.key(env_id, mode)] = hs.hash_rollout(hs.HashedReference(env_id, N_ENVS, autoreset=mode),
                                                                        N_ENVS)
        out["hash_walk"][env_id] = hs.hash_walk(hs.HashedReference(env_id, N_ENVS), N_ENVS)
        acts = scripted_actions(ReferenceVecEnv(env_id, N_ENVS), N_ENVS, SCRIPT_SEED, SCRIPT_STEPS)
        out["scripted"][env_id] = {"actions": acts,
                                   "trace": scripted_rollout(ReferenceVecEnv(env_id, N_ENVS), N_ENVS, SCRIPT_SEED, acts)}
    for env_id in CONSTANT_MISSION_IDS:
        obs, _ = DictObservationSpaceWrapper(gym.make(env_id)).reset(seed=0)
        out["dict_missions"][env_id] = [int(i) for i in obs["mission"]]
    for env_id in OBS_WRAPPER_IDS:
        out["obs_wrappers"][env_id] = observation_wrappers(ReferenceVecEnv(env_id, N_ENVS), N_ENVS,
                                                           _reference_views(env_id in CONSTANT_MISSION_IDS))
    return out


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    with contextlib.redirect_stdout(io.StringIO()):
        rec = record()
    with open(RECORD, "w") as f:
        json.dump(rec, f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"wrote {RECORD}")
