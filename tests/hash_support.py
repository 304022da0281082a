"""MiniGridEnv.hash (minigrid_env.py:159-170) on the test side: the oracle's and the reference's hashes, and the hash
checks as procedures that run on the engine, the oracle or the reference alike (same interface: reset / step / hash).
TEST INFRASTRUCTURE ONLY. tests/golden/ref_hash_traces.json holds the reference's traces of the checks; rewrite it with

    python tests/hash_support.py        (needs the reference tree, see oracle/ref_loader.py)
"""
from __future__ import annotations

import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.oracle import ENV_SPECS, KIND, OracleVecEnv  # noqa: E402
from oracle.ref_trace import MODES, Trace, key  # noqa: E402

RECORD = os.path.join(ROOT, "tests", "golden", "ref_hash_traces.json")


def load_record():
    with open(RECORD) as f:
        return json.load(f)


def oracle_spec(env_id):
    """The oracle's spec of any id the engine registers (the oracle's own table, else restated from minigrid_b200.specs)."""
    from minigrid_b200 import specs

    if env_id in ENV_SPECS:
        return ENV_SPECS[env_id]
    s = specs.get(env_id)
    name = {v: k for k, v in KIND.items()}[s.kind]
    return (name, s.width, s.height, s.max_steps, bool(s.see_through_walls), list(s.params))


class HashedOracle:
    """The C oracle plus what MiniGridEnv.hash needs beyond its state: whether agent_pos was last assigned by a forward
    move (minigrid_env.py:553, a tuple of numpy ints) or by the kind's generator. A forward move that succeeds always
    changes the position and nothing else moves the agent, so within a step that does not reset an env, "moved" is
    "the position changed". Autoresets follow SyncVectorEnv: NEXT_STEP resets the envs pending before the step,
    SAME_STEP the envs that ended in it. Injected agent records count as moved, as in the engine."""

    def __init__(self, env_id=None, num_envs=1, *, spec=None, autoreset="next_step"):
        self.o = OracleVecEnv(None, num_envs, spec=spec if spec is not None else oracle_spec(env_id), autoreset=autoreset)
        self.num_envs, self.autoreset = int(num_envs), autoreset
        self.moved = np.zeros(self.num_envs, bool)

    def reset(self, seed=None):
        self.moved[:] = False
        return self.o.reset(seed=seed)

    def step(self, actions):
        before = self.o.get_state()
        r = self.o.step(actions)
        after = self.o.get_state()
        changed = np.any(before["agent"][:, :2] != after["agent"][:, :2], axis=1)
        if self.autoreset == "next_step":
            reset = before["pending"] != 0
        elif self.autoreset == "same_step":
            reset = np.asarray(r[3], bool) | np.asarray(r[4], bool)
        else:
            reset = np.zeros(self.num_envs, bool)
        self.moved = np.where(reset, False, self.moved | changed)
        return r

    def get_state(self):
        return self.o.get_state()

    def set_state(self, grid=None, agent=None, rng=None, pending=None):
        self.o.set_state(grid=grid, agent=agent, rng=rng, pending=pending)
        if agent is not None:
            self.moved[:] = True

    def reset_form(self):
        """How the reference's generator of this kind assigns agent_pos: "tuple" (agent_start_pos, empty.py:109,
        distshift.py:115, dynamicobstacles.py:123), "array" (np.array, crossing.py:141, lavagap.py:110, memory.py:129) or
        "npint" (place_agent / place_obj, minigrid_env.py:347-350, 383-395)."""
        kind, prm = self.o.kind, self.o.params
        if (kind == "empty" and not prm[0]) or kind == "distshift" or (kind == "dynobstacles" and not prm[1]):
            return "tuple"
        if kind in ("crossing", "lavagap", "memory"):
            return "array"
        return "npint"

    def hash(self, size=16, envs=None):
        """MiniGridEnv.hash(size) of every env (or of `envs`): the Python objects the reference would hold, printed with
        str() and hashed with hashlib, as the reference does."""
        st = self.o.get_state()
        form = self.reset_form()
        out = []
        for i in range(self.num_envs) if envs is None else envs:
            x, y, d = (int(v) for v in st["agent"][i, :3])
            if self.moved[i] or form == "npint":
                pos = (np.int64(x), np.int64(y))
            elif form == "tuple":
                pos = (x, y)
            else:
                pos = np.array((x, y))
            h = hashlib.sha256()
            for item in [st["grid"][i].tolist(), pos, d]:
                h.update(str(item).encode("utf8"))
            out.append(h.hexdigest()[:size])
        return out

    def forms(self):
        """Per env: 0 tuple of ints, 1 tuple of numpy ints, 2 ndarray (the numbering of mg_hash.cuh)."""
        f0 = {"tuple": 0, "npint": 1, "array": 2}[self.reset_form()]
        return np.where(self.moved, 1, f0).astype(np.int32)


class HashedReference:
    """The reference's own envs (oracle/ref_loader.py) with MiniGridEnv.hash."""

    def __init__(self, env_id, num_envs, autoreset="next_step"):
        from oracle.ref_loader import ReferenceVecEnv

        self.r = ReferenceVecEnv(env_id, num_envs, autoreset=autoreset)

    def reset(self, seed=None):
        return self.r.reset(seed=seed)

    def step(self, actions):
        return self.r.step(actions)

    def hash(self, size=16):
        return [e.hash(size) for e in self.r.envs]


def _hashes(env):
    return np.array(env.hash(64), dtype="S64")


def hash_rollout(env, n, seed=1000, act_seed=78, steps=120):
    """MiniGridEnv.hash(64) of every env after a seeded reset and after every step of forward-heavy random actions
    (forward moves change how the reference prints agent_pos)."""
    tr = Trace()
    env.reset(seed=seed)
    tr.add(_hashes(env))
    tr.mark("reset")
    rng = np.random.default_rng(act_seed)
    for t in range(steps):
        env.step(np.where(rng.random(n) < 0.5, 2, rng.integers(0, 7, n)))
        tr.add(_hashes(env))
        if (t + 1) % 20 == 0:
            tr.mark(f"step {t}")
    return tr.marks


HASH_WALK = [2, 0, 0, 2, 0, 0]  # forward, turn around, forward, turn around: back where it started, facing the same way


def hash_walk(env, n, seed=5):
    """The hashes after a reset and after walking away and back (HASH_WALK): the state is the reset state again wherever
    the first forward move succeeded, but agent_pos is now a tuple of numpy ints."""
    tr = Trace()
    env.reset(seed=seed)
    tr.add(_hashes(env))
    tr.mark("reset")
    for a in HASH_WALK:
        env.step(np.full(n, a))
    tr.add(_hashes(env))
    tr.mark("walk")
    return tr.marks


def record():
    """Runs the hash checks on the reference for every id the engine registers. Returns the record the tests read."""
    from minigrid_b200 import specs

    out = {"rollout": {}, "walk": {}}
    for env_id in specs.REGISTRY:
        for mode in MODES:
            out["rollout"][key(env_id, mode)] = hash_rollout(HashedReference(env_id, 6, autoreset=mode), 6)
        out["walk"][env_id] = hash_walk(HashedReference(env_id, 6), 6)
    return out


if __name__ == "__main__":
    rec = record()
    with open(RECORD, "w") as f:
        json.dump(rec, f, indent=0, sort_keys=True)
        f.write("\n")
    print(f"wrote {RECORD}")
