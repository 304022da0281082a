"""The record of the reference's BabyAI maze levels (GoToObjMaze*, FindObjS*, KeyCorridor*). TEST INFRASTRUCTURE ONLY.

Runs the UNMODIFIED reference (oracle/ref_loader.py) on every id of minigrid_b200.specs.BABYAI_MAZE_REGISTRY and writes
what tests/test_babyai_maze_cpu.py and tests/test_gpu_babyai_maze.py compare against, in the format of
oracle/ref_babyai_open.py's record: the dims, lockstep rollout traces in both autoreset modes, the mission after each of
50 seeded resets, the hash checks and scripted rollouts, plus the number of RejectSampling retries over REJECT_SEEDS
seeded resets (RoomGridLevel._gen_grid prints "Sampling rejected" for each). Random actions rarely reach an object
three rooms away, so the scripted rollouts hold the actions of tests/babyai_maze_oracle.py's ScriptedPolicy (a BFS on
the reference env's own state that toggles closed doors on its way, and in KeyCorridor fetches the key, unlocks the
door and drops the key; on odd envs it presses pickup in front of the ball while still carrying the key) and the traces
of the reference under them. Rewrite the record with

    python -m oracle.ref_babyai_maze        (needs the reference tree, see oracle/ref_loader.py)
"""
from __future__ import annotations

import contextlib
import io
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RECORD = os.path.join(ROOT, "tests", "golden", "ref_babyai_maze_traces.json")
N_ENVS, SEED, ACT_SEED, STEPS = 6, 1000, 77, 250
SCRIPT_ENVS, SCRIPT_SEED, SCRIPT_STEPS = 8, 300, 300
MISSION_SEEDS = range(50)
REJECT_SEEDS = range(2000)


def load_record():
    with open(RECORD) as f:
        return json.load(f)


def scripted_actions(ref, n, seed, steps):
    """ScriptedPolicy's actions on the reference's envs (ReferenceVecEnv, NEXT_STEP: the traces replay them in that
    mode), env i pressing pickup while carrying when i is odd: [steps][n] ints."""
    import numpy as np
    from babyai_maze_oracle import ScriptedPolicy

    ref.reset(seed=seed)
    pols = [ScriptedPolicy(press_while_carrying=bool(i % 2)) for i in range(n)]
    seen = [None] * n
    out = []
    for _ in range(steps):
        acts = []
        for i, e in enumerate(ref.envs):
            if seen[i] is not e.instrs:  # gen_mission makes a new instruction at every reset
                seen[i] = e.instrs
                pols[i].start((e.instrs.desc.type, e.instrs.desc.color))
            c = e.carrying
            acts.append(int(pols[i].act(e.grid.encode(), int(e.agent_pos[0]), int(e.agent_pos[1]), int(e.agent_dir),
                                        None if c is None else (c.type, c.color),
                                        type(e.instrs).__name__ == "GoToInstr")))
        out.append(acts)
        ref.step(np.asarray(acts))
    return out


def rejections(gym, env_id):
    """RejectSampling retries over the REJECT_SEEDS seeded resets, counted from what _gen_grid prints."""
    buf = io.StringIO()
    e = gym.make(env_id).unwrapped
    with contextlib.redirect_stdout(buf):
        for s in REJECT_SEEDS:
            e.reset(seed=s)
    return buf.getvalue().count("Sampling rejected")


def record():
    from oracle import ref_trace as rt
    from minigrid_b200.specs import BABYAI_MAZE_REGISTRY
    from oracle.ref_loader import ReferenceVecEnv, load

    gym, _ = load()
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import hash_support as hs
    from babyai_pickup_oracle import scripted_rollout

    out = {"dims": {}, "lockstep": {}, "missions": {}, "hash_rollout": {}, "hash_walk": {}, "scripted": {},
           "rejections": {}}
    for env_id in BABYAI_MAZE_REGISTRY:
        out["rejections"][env_id] = rejections(gym, env_id)
        with contextlib.redirect_stdout(io.StringIO()):
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
                out["hash_rollout"][rt.key(env_id, mode)] = hs.hash_rollout(
                    hs.HashedReference(env_id, N_ENVS, autoreset=mode), N_ENVS)
            out["hash_walk"][env_id] = hs.hash_walk(hs.HashedReference(env_id, N_ENVS), N_ENVS)
            acts = scripted_actions(ReferenceVecEnv(env_id, SCRIPT_ENVS), SCRIPT_ENVS, SCRIPT_SEED, SCRIPT_STEPS)
            out["scripted"][env_id] = {"actions": acts,
                                       "trace": scripted_rollout(ReferenceVecEnv(env_id, SCRIPT_ENVS), SCRIPT_ENVS,
                                                                 SCRIPT_SEED, acts)}
    return out


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    rec = record()
    with open(RECORD, "w") as f:
        json.dump(rec, f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"wrote {RECORD}")
