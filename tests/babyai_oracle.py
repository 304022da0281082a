"""The oracle of the single-room BabyAI GoTo levels. TEST INFRASTRUCTURE ONLY.

`BabyAIOracle` has the surface of oracle.oracle.OracleVecEnv. The parts that are the same for every MiniGrid env (the
transition, gen_obs, FullyObs, truncation) run on the C oracle (oracle/mg_oracle.c) in its `disabled` autoreset mode.
The BabyAI parts are restated here, close to the reference's own code:
  - RoomGridLevel._gen_grid (babyai/core/roomgrid_level.py:119-144) with the gen_mission of the GoTo levels
    (babyai/goto.py:67-78, 133-141, 192-193, 256-260, 333-338, 661-677), drawing from numpy's own PCG64 Generator;
  - GoToInstr's verifier (verifier.py:290-316): success when front_pos is one of the positions that
    find_matching_objs recorded at reset;
  - the SyncVectorEnv autoresets.
Each generated level is written into the C oracle with mgo_vec_set_state, so get_state / full_obs / gen_obs see it.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.oracle import OracleVecEnv  # noqa: E402

REDBALL_GREY, REDBALL, OBJ, LOCAL, REDBLUEBALL = 0, 1, 2, 3, 4


def _spec(level, room_size=8, num_dists=7):
    """One room, room_size^2 steps (roomgrid_level.py:71-85); params {7, room_size, 1, 1, level, num_dists}"""
    return ("roomgrid", room_size, room_size, room_size * room_size, False, [7, room_size, 1, 1, level, num_dists])


# __init__.py:573-665
BABYAI_SPECS = {
    "BabyAI-GoToRedBallGrey-v0": _spec(REDBALL_GREY),
    "BabyAI-GoToRedBall-v0": _spec(REDBALL),
    "BabyAI-GoToRedBallNoDists-v0": _spec(REDBALL, 8, 0),
    "BabyAI-GoToObj-v0": _spec(OBJ, 8, 1),
    "BabyAI-GoToObjS4-v0": _spec(OBJ, 4, 1),
    "BabyAI-GoToObjS6-v1": _spec(OBJ, 6, 1),
    "BabyAI-GoToLocal-v0": _spec(LOCAL, 8, 8),
    **{f"BabyAI-GoToLocalS{s}N{n}-v0": _spec(LOCAL, s, n)
       for s, n in [(5, 2), (6, 2), (6, 3), (6, 4), (7, 4), (7, 5), (8, 2), (8, 3), (8, 4), (8, 5), (8, 6), (8, 7)]},
    "BabyAI-GoToRedBlueBall-v0": _spec(REDBLUEBALL),
}

# constants.py: COLOR_NAMES (sorted) as COLOR_TO_IDX values; OBJECT_TO_IDX
COLOR_NAMES = ["blue", "green", "grey", "purple", "red", "yellow"]
COLOR_TO_IDX = {"red": 0, "green": 1, "blue": 2, "purple": 3, "yellow": 4, "grey": 5}
OBJECT_TO_IDX = {"key": 5, "ball": 6, "box": 7}
NONE, WALL = (1, 0, 0), (2, 5, 0)  # Grid.encode of None and of Wall()
DIR_TO_VEC = [(1, 0), (0, 1), (-1, 0), (0, -1)]


class RejectSampling(Exception):
    pass


def rng_row(g):
    """numpy's PCG64 state as the oracle's rng record {state_hi, state_lo, inc_hi, inc_lo, has_uint32, uinteger}"""
    st = g.bit_generator.state
    s, inc, m = st["state"]["state"], st["state"]["inc"], (1 << 64) - 1
    return [s >> 64, s & m, inc >> 64, inc & m, st["has_uint32"], st["uinteger"]]


class Level:
    """One GoTo level as RoomGridLevel builds it: the encoded grid, the agent and GoToInstr's obj_poss."""

    def __init__(self, spec, g):
        _, self.W, self.H, _, _, params = spec
        self.S, self.level, self.num_dists = params[1], params[4], params[5]
        self.g = g
        self.rejections = 0
        while True:  # roomgrid_level.py:119-140
            try:
                self._room_grid()
                self._gen_mission()
                break
            except RejectSampling:
                self.rejections += 1
        # GoToInstr.reset_verifier -> find_matching_objs: i over the width, then j over the height
        self.obj_poss = [(i, j) for i in range(self.W) for j in range(self.H)
                         if tuple(self.grid[i, j, :2]) == self.target]

    def _rand_int(self, lo, hi):
        return int(self.g.integers(lo, hi))

    def _rand_elem(self, lst):
        return lst[self._rand_int(0, len(lst))]

    def _room_grid(self):  # RoomGrid._gen_grid (roomgrid.py:123-177) for one room: no door positions are drawn
        self.grid = np.empty((self.W, self.H, 3), np.uint8)
        self.grid[:] = NONE
        self.grid[0, :] = self.grid[-1, :] = self.grid[:, 0] = self.grid[:, -1] = WALL
        self.agent_pos = (self.S // 2, self.S // 2)
        self.agent_dir = 0

    def _is_none(self, x, y):
        return tuple(self.grid[x, y]) == NONE

    def _place_obj(self, obj, reject_next_to):  # minigrid_env.py:313-372 over the room (0, 0, S, S)
        while True:
            pos = (self._rand_int(0, min(self.S, self.W)), self._rand_int(0, min(self.S, self.H)))
            if not self._is_none(*pos):
                continue
            if pos == tuple(self.agent_pos):
                continue
            if reject_next_to and abs(self.agent_pos[0] - pos[0]) + abs(self.agent_pos[1] - pos[1]) < 2:  # roomgrid.py:11-20
                continue
            break
        if obj is not None:
            self.grid[pos] = (OBJECT_TO_IDX[obj[0]], COLOR_TO_IDX[obj[1]], 0)
        return pos

    def _place_agent(self):  # RoomGrid.place_agent (roomgrid.py:313-334), i and j drawn from a range of one
        self._rand_int(0, 1)
        self._rand_int(0, 1)
        while True:
            self.agent_pos = (-1, -1)
            self.agent_pos = self._place_obj(None, False)
            self.agent_dir = self._rand_int(0, 4)
            dx, dy = DIR_TO_VEC[self.agent_dir]
            front = tuple(self.grid[self.agent_pos[0] + dx, self.agent_pos[1] + dy])
            if front in (NONE, WALL):
                break

    def _add_object(self, kind, color):  # RoomGrid.add_object (roomgrid.py:196-224) with kind and colour given
        pos = self._place_obj((kind, color), True)
        self.objs.append((kind, color, pos))
        return kind, color, pos

    def _add_distractors(self, num, all_unique):  # roomgrid.py:396-438
        existing = [(k, c) for k, c, _ in self.objs]
        dists = []
        while len(dists) < num:
            color = self._rand_elem(COLOR_NAMES)
            kind = self._rand_elem(["key", "ball", "box"])
            if all_unique and (kind, color) in existing:
                continue
            self._rand_int(0, 1)
            self._rand_int(0, 1)
            dists.append(self._add_object(kind, color))
            existing.append((kind, color))
        return dists

    def _check_objs_reachable(self):  # roomgrid_level.py:250-302
        reachable, stack = set(), [tuple(self.agent_pos)]
        while stack:
            i, j = stack.pop()
            if i < 0 or i >= self.W or j < 0 or j >= self.H or (i, j) in reachable:
                continue
            reachable.add((i, j))
            if not self._is_none(i, j) and self.grid[i, j, 0] != 4:  # anything but a door blocks
                continue
            stack += [(i + 1, j), (i - 1, j), (i, j + 1), (i, j - 1)]
        for i in range(self.W):
            for j in range(self.H):
                if not self._is_none(i, j) and self.grid[i, j, 0] != 2 and (i, j) not in reachable:
                    raise RejectSampling

    def _gen_mission(self):
        self.objs = []
        self._place_agent()
        lv = self.level
        if lv in (REDBALL_GREY, REDBALL):
            obj = self._add_object("ball", "red")
        dists = self._add_distractors(self.num_dists, all_unique=lv == OBJ)
        if lv == REDBALL_GREY:  # dist.color = "grey"
            for _, _, pos in dists:
                self.grid[pos][1] = COLOR_TO_IDX["grey"]
        if lv == OBJ:
            obj = dists[0]
        if lv == REDBLUEBALL:
            if any(k == "ball" and c in ("red", "blue") for k, c, _ in dists):
                raise RejectSampling
            obj = self._add_object("ball", self._rand_elem(["red", "blue"]))
        if lv != OBJ:
            self._check_objs_reachable()
        if lv == LOCAL:
            obj = self._rand_elem(dists)
        self.target = (OBJECT_TO_IDX[obj[0]], COLOR_TO_IDX[obj[1]])


class BabyAIOracle:
    """N GoTo envs in lockstep with SyncVectorEnv autoresets (see the module docstring)."""

    def __init__(self, env_id=None, num_envs=1, *, spec=None, autoreset="next_step", n_threads=1):
        self.spec = spec if spec is not None else BABYAI_SPECS[env_id]
        kind, W, H, max_steps, see_through, params = self.spec
        self.kind, self.width, self.height = kind, W, H
        self.max_steps, self.see_through, self.params = max_steps, see_through, list(params)
        self.num_envs = n = int(num_envs)
        self.autoreset = autoreset
        self.c = OracleVecEnv(None, n, spec=self.spec, autoreset="disabled", n_threads=n_threads)
        self.gens = [np.random.default_rng(i) for i in range(n)]  # the engine and the C oracle seed env i with i
        self.obj_poss = [[] for _ in range(n)]
        self.pending = np.zeros(n, bool)
        self.n_rejections = 0

    def rejections(self):
        """Generation attempts thrown away by RejectSampling, over all envs since creation."""
        return self.n_rejections

    def _regenerate(self, envs):
        if len(envs) == 0:
            return
        st = self.c.get_state()
        for i in envs:
            lv = Level(self.spec, self.gens[i])
            self.n_rejections += lv.rejections
            st["grid"][i] = lv.grid
            st["agent"][i] = [lv.agent_pos[0], lv.agent_pos[1], lv.agent_dir, -1, 0, 0]
            self.obj_poss[i] = lv.obj_poss
            self.pending[i] = False
        st["rng"][:] = [rng_row(g) for g in self.gens]
        self.c.set_state(grid=st["grid"], agent=st["agent"], rng=st["rng"])

    def reset(self, seed=None, mask=None):
        sel = np.arange(self.num_envs) if mask is None else np.nonzero(np.asarray(mask))[0]
        if seed is not None:
            seeds = np.arange(self.num_envs, dtype=np.uint64) + np.uint64(seed) if np.isscalar(seed) else np.asarray(seed, np.uint64)
            for i in sel:
                self.gens[i] = np.random.default_rng(int(seeds[i]))
        self._regenerate(sel)
        obs, d = self.c.gen_obs()
        return obs, d

    def step(self, actions):
        a = np.ascontiguousarray(actions, dtype=np.int32)
        fresh = self.pending.copy() if self.autoreset == "next_step" else np.zeros(self.num_envs, bool)
        _, _, r, te, tr = self.c.step(a)
        r, te, tr = r.copy(), te.copy(), tr.copy()
        agent = self.c.get_state()["agent"]
        for i in np.nonzero(~fresh)[0]:  # RoomGridLevel.step: instrs.verify after every step (roomgrid_level.py:87-104)
            x, y, d = (int(v) for v in agent[i, :3])
            if (x + DIR_TO_VEC[d][0], y + DIR_TO_VEC[d][1]) in self.obj_poss[i]:
                te[i] = True
                r[i] = 1.0 - 0.9 * (int(agent[i, 5]) / self.max_steps)  # _reward(), minigrid_env.py:240-245
        r[fresh], te[fresh], tr[fresh] = 0.0, False, False
        done = (te | tr) & ~fresh
        if self.autoreset == "next_step":
            self._regenerate(np.nonzero(fresh)[0])
            self.pending = done
        elif self.autoreset == "same_step":
            self._regenerate(np.nonzero(done)[0])
        obs, d = self.c.gen_obs()
        return obs, d, r, te, tr

    def get_state(self):
        st = self.c.get_state()
        st["pending"] = self.pending.astype(np.uint8)
        return st

    def full_obs(self):
        return self.c.full_obs()

    def gen_obs(self):
        return self.c.gen_obs()


def hashed(env_id, num_envs=1, autoreset="next_step"):
    """hash_support.HashedOracle (MiniGridEnv.hash on the oracle's states) over a BabyAIOracle."""
    import hash_support as hs

    h = hs.HashedOracle.__new__(hs.HashedOracle)
    h.o = BabyAIOracle(env_id, num_envs, autoreset=autoreset)
    h.num_envs, h.autoreset = int(num_envs), autoreset
    h.moved = np.zeros(h.num_envs, bool)
    return h
