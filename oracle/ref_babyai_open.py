"""The record of the reference's BabyAI Open and UnlockLocal levels. TEST INFRASTRUCTURE ONLY.

Runs the UNMODIFIED reference (oracle/ref_loader.py) on every id of minigrid_b200.specs.BABYAI_OPEN_REGISTRY and writes
what tests/test_babyai_open_cpu.py and tests/test_gpu_babyai_open.py compare against, in the format of
oracle/ref_babyai_pickup.py's record: the dims, lockstep rollout traces in both autoreset modes, the mission after each of
50 seeded resets, the hash checks, DictObservationSpaceWrapper's mission indices of the ids whose mission is constant,
the observation-wrapper traces and scripted rollouts. Random actions rarely open a locked door with its key or two doors
in order, so the scripted rollouts hold the actions of tests/babyai_open_oracle.py's ScriptedPolicy (a BFS on the
reference env's own state: face the instruction's door and toggle it, fetching the key of a locked door first; by env,
open a door no instruction names first, close an opened first door again, or open the second door before the first)
and the traces of the reference under them. Rewrite the record with

    python -m oracle.ref_babyai_open        (needs the reference tree, see oracle/ref_loader.py)
"""
from __future__ import annotations

import contextlib
import io
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RECORD = os.path.join(ROOT, "tests", "golden", "ref_babyai_open_traces.json")
N_ENVS, SEED, ACT_SEED, STEPS = 6, 1000, 77, 250
SCRIPT_ENVS, SCRIPT_SEED, SCRIPT_STEPS = 8, 300, 300
MISSION_SEEDS = range(50)
CONSTANT_MISSION_IDS = ["BabyAI-OpenRedDoor-v0", "BabyAI-OpenRedBlueDoors-v0", "BabyAI-OpenRedBlueDoorsDebug-v0",
                        "BabyAI-UnlockLocal-v0", "BabyAI-UnlockLocalDist-v0"]
OBS_WRAPPER_IDS = ["BabyAI-OpenRedDoor-v0", "BabyAI-OpenDoorLoc-v0", "BabyAI-OpenDoorsOrderN4-v0",
                   "BabyAI-UnlockLocalDist-v0"]


def load_record():
    with open(RECORD) as f:
        return json.load(f)


def _door_cells(instr):
    return [tuple(int(v) for v in d.cur_pos) for d in instr.desc.obj_set]


def scripted_actions(ref, n, seed, steps):
    """ScriptedPolicy's actions on the reference's envs (ReferenceVecEnv, NEXT_STEP: the traces replay them in that
    mode), env i in style STYLES[i % 4]: [steps][n] ints."""
    import numpy as np
    from babyai_open_oracle import STYLES, ScriptedPolicy

    ref.reset(seed=seed)
    pols = [ScriptedPolicy(STYLES[i % len(STYLES)]) for i in range(n)]
    seen = [None] * n
    out = []
    for _ in range(steps):
        acts = []
        for i, e in enumerate(ref.envs):
            if seen[i] is not e.instrs:  # gen_mission makes a new instruction at every reset
                seen[i] = e.instrs
                ins = e.instrs
                if hasattr(ins, "instr_a"):  # BeforeInstr completes a first, AfterInstr b
                    first, second = (ins.instr_a, ins.instr_b) if type(ins).__name__ == "BeforeInstr" else (ins.instr_b, ins.instr_a)
                else:
                    first, second = ins, None
                g = e.grid.encode()
                doors = [(int(x), int(y)) for x, y in zip(*np.nonzero(g[:, :, 0] == 4))]
                pols[i].start(_door_cells(first), _door_cells(second) if second else [], doors)
            c = e.carrying
            acts.append(int(pols[i].act(e.grid.encode(), int(e.agent_pos[0]), int(e.agent_pos[1]), int(e.agent_dir),
                                        None if c is None else (c.type, c.color))))
        out.append(acts)
        ref.step(np.asarray(acts))
    return out


def record():
    from oracle import ref_trace as rt
    from oracle.ref_babyai import _reference_views, observation_wrappers
    from minigrid_b200.specs import BABYAI_OPEN_REGISTRY
    from oracle.ref_loader import ReferenceVecEnv, load

    gym, _ = load()
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import hash_support as hs
    from babyai_open_oracle import scripted_rollout

    from minigrid.wrappers import DictObservationSpaceWrapper

    out = {"dims": {}, "lockstep": {}, "missions": {}, "hash_rollout": {}, "hash_walk": {}, "dict_missions": {},
           "obs_wrappers": {}, "scripted": {}}
    for env_id in BABYAI_OPEN_REGISTRY:
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
        acts = scripted_actions(ReferenceVecEnv(env_id, SCRIPT_ENVS), SCRIPT_ENVS, SCRIPT_SEED, SCRIPT_STEPS)
        out["scripted"][env_id] = {"actions": acts,
                                   "trace": scripted_rollout(ReferenceVecEnv(env_id, SCRIPT_ENVS), SCRIPT_ENVS, SCRIPT_SEED,
                                                             acts)}
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
