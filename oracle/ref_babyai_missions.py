"""The record of the reference's per-episode missions on the 43 BabyAI ids of the engine. TEST INFRASTRUCTURE ONLY.

Runs the UNMODIFIED reference (oracle/ref_loader.py) and writes what tests/test_babyai_missions_cpu.py and
tests/test_gpu_babyai_missions.py compare against:
  - "missions": for every id of minigrid_b200.specs' three BabyAI registries in both autoreset modes, N_ENVS envs reset
    with SEED and stepped with tests/babyai_mission_oracle.record_actions (half the actions are the level's verb, so
    that successes end episodes as well as truncations) until every env has ended three episodes, i.e. passed at least
    two autoresets: the number of steps, each env's mission after the reset and every change of an env's mission as
    [step, env, mission];
  - "dict": DictObservationSpaceWrapper's mission indices after DICT_SEEDS resets of every id whose grammar stays in the
    Minigrid vocabulary, with those missions;
  - "flat": FlatObsWrapper rows of FLAT_IDS in oracle.ref_babyai.observation_wrappers' form.
Rewrite the record with

    python -m oracle.ref_babyai_missions        (needs the reference tree, see oracle/ref_loader.py)
"""
from __future__ import annotations

import contextlib
import io
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RECORD = os.path.join(ROOT, "tests", "golden", "ref_babyai_mission_traces.json")
N_ENVS, SEED, ACT_SEED, MAX_STEPS, ENDS = 6, 3000, 91, 6000, 3
DICT_SEEDS = range(20)
FLAT_IDS = ["BabyAI-GoToLocal-v0", "BabyAI-PickupDist-v0", "BabyAI-PutNextLocal-v0", "BabyAI-OpenDoorLoc-v0",
            "BabyAI-OpenDoorsOrderN4-v0"]


def load_record():
    with open(RECORD) as f:
        return json.load(f)


def babyai_ids():
    from minigrid_b200.specs import BABYAI_OPEN_REGISTRY, BABYAI_PICKUP_PUTNEXT_REGISTRY, BABYAI_REGISTRY

    return list(BABYAI_REGISTRY) + list(BABYAI_PICKUP_PUTNEXT_REGISTRY) + list(BABYAI_OPEN_REGISTRY)


def dict_ids():
    """The ids whose mission grammar has only words of DictObservationSpaceWrapper's vocabulary."""
    from minigrid_b200 import specs
    from minigrid_b200.wrappers import MINIGRID_WORDS

    return [i for i in babyai_ids() if specs.babyai_mission_words(specs.get(i)) <= set(MINIGRID_WORDS)]


def mission_rollout(ref, env_id, mode):
    import numpy as np
    from babyai_mission_oracle import record_actions

    acts = record_actions(env_id, N_ENVS, MAX_STEPS, ACT_SEED)
    ref.reset(seed=SEED)
    cur = [e.mission for e in ref.envs]
    initial, changes = list(cur), []
    ends = np.zeros(N_ENVS, int)
    t = 0
    while t < MAX_STEPS and ends.min() < ENDS:
        _, _, _, te, tr = ref.step(acts[t])
        ends += np.asarray(te) | np.asarray(tr)
        for i, e in enumerate(ref.envs):
            if e.mission != cur[i]:
                cur[i] = e.mission
                changes.append([t, i, e.mission])
        t += 1
    return {"steps": t, "initial": initial, "changes": changes, "ends": [int(v) for v in ends]}


def record():
    import numpy as np

    from oracle.ref_babyai import observation_wrappers
    from oracle.ref_loader import ReferenceVecEnv, load
    from oracle.ref_trace import MODES, key

    gym, _ = load()
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from minigrid.wrappers import DictObservationSpaceWrapper

    out = {"missions": {}, "dict": {}, "flat": {}}
    for env_id in babyai_ids():
        for mode in MODES:
            out["missions"][key(env_id, mode)] = mission_rollout(ReferenceVecEnv(env_id, N_ENVS, autoreset=mode), env_id, mode)
    for env_id in dict_ids():
        w = DictObservationSpaceWrapper(gym.make(env_id))
        rows = []
        for s in DICT_SEEDS:
            obs, _ = w.reset(seed=s)
            rows.append([w.unwrapped.mission, [int(i) for i in obs["mission"]]])
        out["dict"][env_id] = rows
    for env_id in FLAT_IDS:
        out["flat"][env_id] = observation_wrappers(ReferenceVecEnv(env_id, N_ENVS), N_ENVS,
                                                   lambda ref: [np.asarray(ref.flat_obs(), np.float32)])
    return out


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    with contextlib.redirect_stdout(io.StringIO()):
        rec = record()
    with open(RECORD, "w") as f:
        json.dump(rec, f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"wrote {RECORD}")
