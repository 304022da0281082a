"""The oracle of the BabyAI maze levels: GoToObjMaze*, FindObjS* and KeyCorridor*. TEST INFRASTRUCTURE ONLY.

`MazeOracle` is tests/babyai_oracle.py's BabyAIOracle (the transition, gen_obs, FullyObs and truncation on the C oracle,
the SyncVectorEnv autoresets in Python) with the generators and verifiers of these levels restated in the reference's
own form, on numpy's own PCG64 Generator:
  - RoomGrid._gen_grid (core/roomgrid.py:123-177) and RoomGridLevel._gen_grid (babyai/core/roomgrid_level.py:119-144),
    a RejectSampling starting again from RoomGrid._gen_grid;
  - place_agent() in a random room, remove_wall, connect_all and add_distractors (roomgrid.py:276-438),
    check_objs_reachable over all rooms and open_all_doors (roomgrid_level.py:238-302);
  - the gen_mission of GoTo with one object (goto.py:416-426), FindObjS5 (other.py:169-177) and KeyCorridor
    (other.py:252-272);
  - GoToInstr (verifier.py:290-316) and PickupInstr (verifier.py:319-363) on the objects, compared by identity.
"""
from __future__ import annotations

import collections

import numpy as np

from babyai_oracle import COLOR_NAMES, COLOR_TO_IDX, DIR_TO_VEC, NONE, OBJECT_TO_IDX, WALL, BabyAIOracle, RejectSampling, rng_row
from babyai_open_oracle import OpenLevel
from babyai_pickup_oracle import _bfs_first_action

GOTO, FINDOBJ, KEYCORRIDOR = 0, 1, 2
A_LEFT, A_FORWARD, A_PICKUP, A_DROP, A_TOGGLE = 0, 2, 3, 4, 5
IDX_TO_TYPE = {5: "key", 6: "ball", 7: "box"}


def _spec(level, room_size, rows, cols, max_steps, arg=0):
    """params {10, room_size, num_rows, num_cols, level, arg}"""
    return ("roomgrid", (room_size - 1) * cols + 1, (room_size - 1) * rows + 1, max_steps, False,
            [10, room_size, rows, cols, level, int(arg)])


def _goto(s=8, rows=3, cols=3, doors_open=False):  # one navigation: room_size^2 rows cols (roomgrid_level.py:71-85)
    return _spec(GOTO, s, rows, cols, s * s * rows * cols, doors_open)


# __init__.py:692-732, 1001-1057
MAZE_SPECS = {
    "BabyAI-GoToObjMaze-v0": _goto(),
    "BabyAI-GoToObjMazeOpen-v0": _goto(doors_open=True),
    "BabyAI-GoToObjMazeS4R2-v0": _goto(4, 2, 2),
    **{f"BabyAI-GoToObjMazeS{s}-v0": _goto(s) for s in (4, 5, 6, 7)},
    **{f"BabyAI-FindObjS{s}-v0": _spec(FINDOBJ, s, 3, 3, 20 * s * s) for s in (5, 6, 7)},
    "BabyAI-KeyCorridor-v0": _spec(KEYCORRIDOR, 6, 3, 3, 30 * 36),
    **{f"BabyAI-KeyCorridorS{s}R{r}-v0": _spec(KEYCORRIDOR, s, r, 3, 30 * s * s)
       for s, r in [(3, 1), (3, 2), (3, 3), (4, 3), (5, 3), (6, 3)]},
}


class Obj:
    """Key, Ball or Box: compared by identity, as the verifiers compare them."""

    def __init__(self, kind, color, pos):
        self.type, self.color, self.cur_pos = kind, color, tuple(pos)


class MazeLevel(OpenLevel):
    """One maze level as RoomGridLevel builds it, then its objects and instruction as the reference holds them."""

    def __init__(self, spec, g):
        _, self.W, self.H, _, _, params = spec
        self.S, self.rows, self.cols, self.level, self.arg = params[1], params[2], params[3], params[4], params[5]
        self.g = g
        self.rejections = 0
        self.connect_doors = 0  # doors added by connect_all in the accepted attempt
        while True:  # roomgrid_level.py:119-140
            try:
                self._room_grid()
                self._gen_mission()
                break
            except RejectSampling:
                self.rejections += 1
        self.world = {o.cur_pos: o for o in self.obj_list}
        self.carrying = self.pre_carrying = None
        kind, color = self.desc
        # find_matching_objs at reset: every object of the descriptor (a door never matches a key, ball or box)
        self.obj_set = [self.world[p] for p in sorted(self.world)
                        if self.world[p].type == kind and (color is None or self.world[p].color == color)]
        self.obj_poss = [o.cur_pos for o in self.obj_set]

    def _room_grid(self):
        super()._room_grid()
        self.obj_list = []
        for row in self.room_grid:
            for room in row:
                room.locked = False

    def _add_door(self, i, j, door_idx=None, color=None, locked=None):
        door = super()._add_door(i, j, door_idx, color, locked)
        self.room_grid[j][i].locked = door.is_locked
        return door

    def _add_object(self, i, j, kind=None, color=None):  # roomgrid.py:196-224
        if kind is None:
            kind = self._rand_elem(["key", "ball", "box"])
        if color is None:
            color = self._rand_elem(COLOR_NAMES)
        pos = self._place_obj(i, j, (kind, color), True)
        obj = Obj(kind, color, pos)
        self.obj_list.append(obj)
        return obj

    def _place_agent_room(self, i=None, j=None):  # RoomGrid.place_agent: a random room when none is given
        if i is None:
            i = self._rand_int(0, self.cols)
        if j is None:
            j = self._rand_int(0, self.rows)
        self._place_agent(i, j)

    def _remove_wall(self, i, j, wall_idx):  # roomgrid.py:276-311, wall_idx 3 (up) only
        room = self.room_grid[j][i]
        tx, ty = room.top
        for k in range(1, self.S - 1):
            self.grid[tx + k, ty] = NONE
        room.doors[wall_idx] = True
        room.neighbors[wall_idx].doors[(wall_idx + 2) % 4] = True

    def _connect_all(self):  # roomgrid.py:336-394
        start = self.room_from_pos(*self.agent_pos)

        def find_reach():
            reach, stack = [], [start]
            while stack:
                room = stack.pop()
                if any(room is r for r in reach):
                    continue
                reach.append(room)
                stack += [room.neighbors[k] for k in range(4) if room.doors[k]]
            return reach

        while True:
            if len(find_reach()) == self.rows * self.cols:
                break
            i, j, k = self._rand_int(0, self.cols), self._rand_int(0, self.rows), self._rand_int(0, 4)
            room = self.room_grid[j][i]
            if not room.door_pos[k] or room.doors[k]:
                continue
            if room.locked or room.neighbors[k].locked:
                continue
            self._add_door(i, j, k, self._rand_elem(COLOR_NAMES), False)
            self.connect_doors += 1

    def _check_objs_reachable(self):  # roomgrid_level.py:250-302
        reachable, stack = set(), [tuple(self.agent_pos)]
        while stack:
            i, j = stack.pop()
            if i < 0 or i >= self.W or j < 0 or j >= self.H or (i, j) in reachable:
                continue
            reachable.add((i, j))
            if tuple(self.grid[i, j]) != NONE and self.grid[i, j, 0] != 4:  # anything but a door blocks
                continue
            stack += [(i + 1, j), (i - 1, j), (i, j + 1), (i, j - 1)]
        for i in range(self.W):
            for j in range(self.H):
                if tuple(self.grid[i, j]) not in (NONE, WALL) and (i, j) not in reachable:
                    raise RejectSampling("unreachable object at " + str((i, j)))

    def _gen_mission(self):
        if self.level == GOTO:
            self._place_agent_room()
            self._connect_all()
            # add_distractors(num_distractors=1, all_unique=False): colour, type, then a random room
            color = self._rand_elem(COLOR_NAMES)
            kind = self._rand_elem(["key", "ball", "box"])
            obj = self._add_object(self._rand_int(0, self.cols), self._rand_int(0, self.rows), kind, color)
            self._check_objs_reachable()
            obj = self._rand_elem([obj])
            self.desc = (obj.type, obj.color)  # GoToInstr(ObjDesc(obj.type, obj.color))
            if self.arg:  # open_all_doors()
                for pos in self.doors:
                    self.grid[pos][2] = 0
        elif self.level == FINDOBJ:
            i, j = self._rand_int(0, self.rows), self._rand_int(0, self.cols)
            obj = self._add_object(i, j)
            self._place_agent(1, 1)
            self._connect_all()
            self.desc = (obj.type, None)  # PickupInstr(ObjDesc(obj.type))
        else:
            for j in range(1, self.rows):
                self._remove_wall(1, j, 3)
            room_idx = self._rand_int(0, self.rows)
            door = self._add_door(2, room_idx, 2, locked=True)
            obj = self._add_object(2, room_idx, "ball")
            self._add_object(0, self._rand_int(0, self.rows), "key", door.color)
            self._place_agent(1, self.rows // 2)
            self._connect_all()
            self.desc = (obj.type, None)

    def mission(self):
        kind, color = self.desc
        what = f"the {color} {kind}" if color else f"the {kind}"  # one object matches: "the"
        return ("go to " if self.level == GOTO else "pick up ") + what

    # ---- RoomGridLevel.step after super().step (roomgrid_level.py:87-104) ----
    def verify(self, action, front, carried_before, carried_after):
        if self.level == GOTO:  # GoToInstr.verify_action: front_pos is one of obj_poss
            return "success" if front in self.obj_poss else "continue"
        if action == A_PICKUP and carried_before < 0 <= carried_after:  # the C oracle picked up the object at front
            self.carrying = self.world.pop(front)
            self.carrying.cur_pos = (-1, -1)
        elif action == A_DROP and carried_after < 0 <= carried_before:
            self.carrying.cur_pos = front
            self.world[front] = self.carrying
            self.carrying = None
        pre = self.pre_carrying  # PickupInstr.verify_action (strict=False)
        self.pre_carrying = self.carrying
        if action != A_PICKUP:
            return "continue"
        for obj in self.obj_set:
            if pre is None and self.carrying is obj:
                return "success"
        self.pre_carrying = self.carrying
        return "continue"


class MazeOracle(BabyAIOracle):
    """N maze envs in lockstep with SyncVectorEnv autoresets (see the module docstring). `events` counts what the tests
    need to have happened: rejections, doors added by connect_all, successes, pickups pressed while carrying."""

    def __init__(self, env_id=None, num_envs=1, *, spec=None, autoreset="next_step", n_threads=1):
        super().__init__(None, num_envs, spec=spec if spec is not None else MAZE_SPECS[env_id], autoreset=autoreset,
                         n_threads=n_threads)
        self.levels = [None] * self.num_envs
        self.events = collections.Counter()

    def _regenerate(self, envs):
        if len(envs) == 0:
            return
        st = self.c.get_state()
        for i in envs:
            lv = MazeLevel(self.spec, self.gens[i])
            self.n_rejections += lv.rejections
            self.events["rejections"] += lv.rejections
            self.events["connect_doors"] += lv.connect_doors
            st["grid"][i] = lv.grid
            st["agent"][i] = [lv.agent_pos[0], lv.agent_pos[1], lv.agent_dir, -1, 0, 0]
            self.levels[i] = lv
            self.pending[i] = False
        st["rng"][:] = [rng_row(g) for g in self.gens]
        self.c.set_state(grid=st["grid"], agent=st["agent"], rng=st["rng"])

    def missions(self):
        return [lv.mission() for lv in self.levels]

    def mission_codes(self):
        """The device's MIS_* layout (mg_common.cuh): GOTO 1 / PICKUP 2, ObjDesc type:3 colour:3 (0 none, 1 + index)."""
        out = []
        for lv in self.levels:
            kind, color = lv.desc
            d = ["key", "ball", "box"].index(kind) + 1 | ((0 if color is None else COLOR_TO_IDX[color] + 1) << 3)
            out.append((1 if lv.level == GOTO else 2) | (d << 3))
        return np.asarray(out, np.uint32)

    def step(self, actions):
        a = np.ascontiguousarray(actions, dtype=np.int32)
        fresh = self.pending.copy() if self.autoreset == "next_step" else np.zeros(self.num_envs, bool)
        before = self.c.get_state()["agent"].copy()
        _, _, r, te, tr = self.c.step(a)
        r, te, tr = r.copy(), te.copy(), tr.copy()
        after = self.c.get_state()["agent"]
        for i in np.nonzero(~fresh)[0]:
            lv, act = self.levels[i], int(a[i])
            x, y, d = (int(v) for v in before[i, :3])
            front = (x + DIR_TO_VEC[d][0], y + DIR_TO_VEC[d][1])
            nx, ny, nd = (int(v) for v in after[i, :3])
            if act == A_PICKUP and before[i, 3] >= 0:
                self.events["pickup_while_carrying"] += 1
            status = lv.verify(act, (nx + DIR_TO_VEC[nd][0], ny + DIR_TO_VEC[nd][1]) if lv.level == GOTO else front,
                               int(before[i, 3]), int(after[i, 3]))
            if status == "success":
                te[i] = True
                r[i] = 1.0 - 0.9 * (int(after[i, 5]) / self.max_steps)  # _reward(), minigrid_env.py:240-245
                self.events["success"] += 1
        r[fresh], te[fresh], tr[fresh] = 0.0, False, False
        done = (te | tr) & ~fresh
        if self.autoreset == "next_step":
            self._regenerate(np.nonzero(fresh)[0])
            self.pending = done
        elif self.autoreset == "same_step":
            self._regenerate(np.nonzero(done)[0])
        obs, dd = self.c.gen_obs()
        return obs, dd, r, te, tr

    def inject(self, i, pos=None, d=None, carry=None):
        """Env i's agent moved to the empty cell pos facing d, and / or the object at cell `carry` put in its hands as if
        picked up in an earlier step, in the C oracle and in the level's objects alike (copy get_state()'s grid and
        agent into the engine to give it the same)."""
        st = self.c.get_state()
        lv = self.levels[i]
        if pos is not None:
            st["agent"][i, :3] = (pos[0], pos[1], d)
        if carry is not None:
            obj = lv.world.pop(tuple(carry))
            obj.cur_pos = (-1, -1)
            lv.carrying = lv.pre_carrying = obj
            st["grid"][i][tuple(carry)] = NONE
            st["agent"][i, 3:5] = (OBJECT_TO_IDX[obj.type], COLOR_TO_IDX[obj.color])
        self.c.set_state(grid=st["grid"], agent=st["agent"])


def hashed(env_id, num_envs=1, autoreset="next_step"):
    """hash_support.HashedOracle (MiniGridEnv.hash on the oracle's states) over a MazeOracle."""
    import hash_support as hs

    h = hs.HashedOracle.__new__(hs.HashedOracle)
    h.o = MazeOracle(env_id, num_envs, autoreset=autoreset)
    h.num_envs, h.autoreset = int(num_envs), autoreset
    h.moved = np.zeros(h.num_envs, bool)
    return h


# ---- the scripted policy of the reference record's scripted rollouts (oracle/ref_babyai_maze.py) ----
def _bfs_through_doors(grid, ax, ay, adir, cells):
    """_bfs_first_action with closed doors passable: the plan goes through them, and the agent toggles one when it is
    the next cell."""
    g = grid.copy()
    closed = (g[:, :, 0] == 4) & (g[:, :, 2] != 2)
    g[closed] = NONE
    act = _bfs_first_action(g, ax, ay, adir, cells)
    fx, fy = ax + DIR_TO_VEC[adir][0], ay + DIR_TO_VEC[adir][1]
    if act == A_FORWARD and closed[fx, fy] and int(grid[fx, fy, 2]) == 1:
        return A_TOGGLE
    return act


class ScriptedPolicy:
    """Goes to the GoTo target, or picks up the Pickup target, toggling the closed doors on its way. In KeyCorridor it
    first fetches the key of the locked door, unlocks the door, and drops the key in front of it on an empty cell;
    with press_while_carrying it presses pickup in front of the ball once while still holding the key. Reads only what a
    reference env shows: Grid.encode(), the agent, what it carries and the instruction's descriptor. Call start() at
    every reset."""

    def __init__(self, press_while_carrying=False):
        self.press = press_while_carrying
        self.start(None)

    def start(self, desc):
        self.desc, self.pressed = desc, False

    def act(self, grid, ax, ay, adir, carrying, goto):
        kind, color = self.desc
        tgt = {(int(x), int(y)) for x, y in zip(*np.nonzero((grid[:, :, 0] == OBJECT_TO_IDX[kind]) &
                                                              ((grid[:, :, 1] == COLOR_TO_IDX[color]) if color else True)))}
        fx, fy = ax + DIR_TO_VEC[adir][0], ay + DIR_TO_VEC[adir][1]
        if goto:
            return self._go(grid, ax, ay, adir, tgt, A_LEFT)
        locked = {(int(x), int(y)) for x, y in zip(*np.nonzero((grid[:, :, 0] == 4) & (grid[:, :, 2] == 2)))}
        if locked:
            if carrying is None:
                keys = {(int(x), int(y)) for x, y in zip(*np.nonzero((grid[:, :, 0] == OBJECT_TO_IDX["key"])))}
                return self._go(grid, ax, ay, adir, keys, A_PICKUP)
            return self._go(grid, ax, ay, adir, locked, A_TOGGLE)
        if carrying is not None:
            if self.press and not self.pressed and (fx, fy) in tgt:
                self.pressed = True
                return A_PICKUP
            if self.press and not self.pressed:
                return self._go(grid, ax, ay, adir, tgt, A_PICKUP)
            return A_DROP if int(grid[fx, fy, 0]) == 1 else A_LEFT
        return self._go(grid, ax, ay, adir, tgt, A_PICKUP)

    @staticmethod
    def _go(grid, ax, ay, adir, cells, final):
        fx, fy = ax + DIR_TO_VEC[adir][0], ay + DIR_TO_VEC[adir][1]
        if (fx, fy) in cells:
            return final
        act = _bfs_through_doors(grid, ax, ay, adir, cells)
        return A_LEFT if act is None else act
