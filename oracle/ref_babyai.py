"""The record of the reference's single-room BabyAI GoTo levels. TEST INFRASTRUCTURE ONLY.

Runs the UNMODIFIED reference (oracle/ref_loader.py) on every id of minigrid_b200.specs.BABYAI_REGISTRY and writes what
tests/test_babyai_cpu.py and tests/test_gpu_babyai.py compare against: the dims, lockstep rollout traces in both
autoreset modes (oracle/ref_trace.py's format), the mission after each of 50 seeded resets, the hash checks of
tests/hash_support.py, and DictObservationSpaceWrapper's mission indices of the ids whose mission is constant.
The reference prints "Sampling rejected: ..." for every rejected level; that output is swallowed. Rewrite the record with

    python -m oracle.ref_babyai        (needs the reference tree, see oracle/ref_loader.py)
"""
from __future__ import annotations

import contextlib
import io
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
RECORD = os.path.join(ROOT, "tests", "golden", "ref_babyai_traces.json")
N_ENVS, SEED, ACT_SEED, STEPS = 6, 1000, 77, 250
MISSION_SEEDS = range(50)
CONSTANT_MISSION_IDS = ["BabyAI-GoToRedBallGrey-v0", "BabyAI-GoToRedBallNoDists-v0"]


OBS_WRAPPER_IDS = ["BabyAI-GoToRedBallGrey-v0", "BabyAI-GoToRedBallNoDists-v0", "BabyAI-GoToLocal-v0",
                   "BabyAI-GoToRedBlueBall-v0"]


def load_record():
    with open(RECORD) as f:
        return json.load(f)


def observation_wrappers(env, n, views):
    """A seeded reset and 40 random-action steps; every 10 steps, views(env) (FullyObsWrapper, RGBImgPartialObsWrapper,
    RGBImgObsWrapper and, for a constant mission, FlatObsWrapper, as uint8 / uint8 / uint8 / float32 arrays) into a
    ref_trace.Trace. `views` is the side-specific part: the reference's wrapper classes or the engine's."""
    import numpy as np

    from oracle.ref_trace import Trace

    tr = Trace()
    env.reset(seed=41)
    rng = np.random.default_rng(6)
    for t in range(40):
        env.step(rng.integers(0, 7, n))
        if t % 10 == 9:
            tr.add(*views(env))
            tr.mark(f"step {t}")
    return tr.marks


def _reference_views(flat):
    import numpy as np

    def views(ref):
        out = [ref.full_obs(), ref.rgb_partial_obs(), ref.rgb_full_obs()]
        return out + ([np.asarray(ref.flat_obs(), np.float32)] if flat else [])
    return views


def record():
    from oracle import ref_trace as rt
    from minigrid_b200.specs import BABYAI_REGISTRY
    from oracle.ref_loader import ReferenceVecEnv, load

    gym, _ = load()
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import hash_support as hs

    from minigrid.wrappers import DictObservationSpaceWrapper

    out = {"dims": {}, "lockstep": {}, "missions": {}, "hash_rollout": {}, "hash_walk": {}, "dict_missions": {},
           "obs_wrappers": {}}
    for env_id in BABYAI_REGISTRY:
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
