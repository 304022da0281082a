"""The oracle of the BabyAI Open and UnlockLocal levels. TEST INFRASTRUCTURE ONLY.

`OpenOracle` is tests/babyai_oracle.py's BabyAIOracle (the transition, gen_obs, FullyObs and truncation on the C oracle,
the SyncVectorEnv autoresets in Python) with the generators and verifiers of these levels restated in the reference's
own form:
  - RoomGrid._gen_grid (core/roomgrid.py:123-177) on 1 x 2 or 3 x 3 rooms and RoomGridLevel._gen_grid
    (babyai/core/roomgrid_level.py:119-177) with the gen_mission of OpenRedDoor, OpenDoor, OpenTwoDoors, OpenDoorsOrder
    (babyai/open.py:143-146, 210-229, 306-324, 399-423) and UnlockLocal (babyai/unlock.py:168-175), on numpy's own PCG64
    Generator;
  - every door is a Python object (compared by identity) whose is_open follows the C oracle's toggles;
  - ObjDesc.find_matching_objs with locations relative to the agent at reset (verifier.py:105-171), OpenInstr
    (verifier.py:254-287), BeforeInstr and AfterInstr (verifier.py:451-530) line by line, the re-verify of the second
    instruction on the action that completes the first included.
The device reduces the verifiers to predicates on the front cell's code and one progress bit (mg_postfilter.cuh); the
tests compare the two.
"""
from __future__ import annotations

import collections

import numpy as np

from babyai_oracle import COLOR_NAMES, COLOR_TO_IDX, DIR_TO_VEC, NONE, OBJECT_TO_IDX, WALL, BabyAIOracle, rng_row
from babyai_pickup_oracle import _bfs_first_action, scripted_rollout  # noqa: F401  (re-exported for the tests)

OPENREDDOOR, OPENDOOR, OPENTWODOORS, OPENDOORSORDER, UNLOCKLOCAL = 0, 1, 2, 3, 4
LOC_NAMES = ["left", "right", "front", "behind"]
A_PICKUP, A_TOGGLE = 3, 5
IDX_TO_COLOR = {v: k for k, v in COLOR_TO_IDX.items()}


def _spec(level, room_size=8, rows=3, cols=3, arg=0, strict=False, max_steps=None):
    """params {9, room_size, num_rows, num_cols, level, arg, strict}; max_steps = room_size^2 rows cols (one navigation,
    roomgrid_level.py:71-85) unless the level fixes it"""
    return ("roomgrid", (room_size - 1) * cols + 1, (room_size - 1) * rows + 1,
            max_steps or room_size * room_size * rows * cols, False,
            [9, room_size, rows, cols, level, int(arg), int(strict)])


# __init__.py:774-844, 957-965
OPEN_SPECS = {
    "BabyAI-OpenRedDoor-v0": _spec(OPENREDDOOR, 5, 1, 2),
    "BabyAI-OpenDoor-v0": _spec(OPENDOOR, arg=2),
    "BabyAI-OpenDoorDebug-v0": _spec(OPENDOOR, arg=2, strict=True),
    "BabyAI-OpenDoorColor-v0": _spec(OPENDOOR, arg=0),
    "BabyAI-OpenDoorLoc-v0": _spec(OPENDOOR, arg=1),
    "BabyAI-OpenTwoDoors-v0": _spec(OPENTWODOORS, 6, max_steps=720),
    "BabyAI-OpenRedBlueDoors-v0": _spec(OPENTWODOORS, 6, arg=1, max_steps=720),
    "BabyAI-OpenRedBlueDoorsDebug-v0": _spec(OPENTWODOORS, 6, arg=1, strict=True, max_steps=720),
    "BabyAI-OpenDoorsOrderN2-v0": _spec(OPENDOORSORDER, 6, arg=2, max_steps=720),
    "BabyAI-OpenDoorsOrderN4-v0": _spec(OPENDOORSORDER, 6, arg=4, max_steps=720),
    "BabyAI-OpenDoorsOrderN2Debug-v0": _spec(OPENDOORSORDER, 6, arg=2, strict=True, max_steps=720),
    "BabyAI-OpenDoorsOrderN4Debug-v0": _spec(OPENDOORSORDER, 6, arg=4, strict=True, max_steps=720),
    "BabyAI-UnlockLocal-v0": _spec(UNLOCKLOCAL),
    "BabyAI-UnlockLocalDist-v0": _spec(UNLOCKLOCAL, arg=1),
}


class Door:
    """Door(color, is_locked) (world_object.py), compared by identity; cur_pos never changes."""
    type = "door"

    def __init__(self, color, pos, locked):
        self.color, self.cur_pos, self.is_locked, self.is_open = color, tuple(pos), bool(locked), False


class Room:
    def __init__(self, top, size):
        self.top, self.size = top, size
        self.doors = [None] * 4
        self.neighbors = [None] * 4
        self.door_pos = [None] * 4

    def pos_inside(self, x, y):  # roomgrid.py:47-63: the walls included
        return self.top[0] <= x < self.top[0] + self.size[0] and self.top[1] <= y < self.top[1] + self.size[1]


class ObjDesc:  # verifier.py:44-171, for doors
    def __init__(self, type, color=None, loc=None):
        self.type, self.color, self.loc = type, color, loc
        self.obj_set, self.obj_poss = [], []

    def surface(self, env):
        self.find_matching_objs(env)
        assert len(self.obj_set) > 0, "no object matching description"
        s = str(self.type) if self.type else "object"
        if self.color:
            s = self.color + " " + s
        if self.loc:
            if self.loc == "front":
                s = s + " in front of you"
            elif self.loc == "behind":
                s = s + " behind you"
            else:
                s = s + " on your " + self.loc
        return ("a " if len(self.obj_set) > 1 else "the ") + s

    def find_matching_objs(self, env, use_location=True):
        if use_location:
            self.obj_set = []
        self.obj_poss = []
        agent_room = env.room_from_pos(*env.agent_pos)
        for i in range(env.W):
            for j in range(env.H):
                cell = env.doors.get((i, j))  # only doors can match: the descriptor's type is "door"
                if cell is None:
                    continue
                if not use_location and not any(cell is obj for obj in self.obj_set):
                    continue
                if self.type is not None and cell.type != self.type:
                    continue
                if self.color is not None and cell.color != self.color:
                    continue
                if use_location and self.loc in LOC_NAMES:
                    if not agent_room.pos_inside(i, j):
                        continue
                    v = (i - env.agent_pos[0], j - env.agent_pos[1])
                    d1 = DIR_TO_VEC[env.agent_dir]
                    d2 = (-d1[1], d1[0])
                    pos_matches = {"left": v[0] * d2[0] + v[1] * d2[1] < 0, "right": v[0] * d2[0] + v[1] * d2[1] > 0,
                                   "front": v[0] * d1[0] + v[1] * d1[1] > 0, "behind": v[0] * d1[0] + v[1] * d1[1] < 0}
                    if not pos_matches[self.loc]:
                        continue
                if use_location:
                    self.obj_set.append(cell)
                self.obj_poss.append((i, j))
        return self.obj_set, self.obj_poss


class OpenInstr:  # verifier.py:254-287 (ActionInstr.verify without BABYAI_DONE_ACTIONS)
    def __init__(self, obj_desc, strict=False):
        assert obj_desc.type == "door"
        self.desc, self.strict = obj_desc, strict

    def surface(self, env):
        return "open " + self.desc.surface(env)

    def reset_verifier(self, env):
        self.env = env
        self.desc.find_matching_objs(env)

    def verify(self, action):
        return self.verify_action(action)

    def verify_action(self, action):
        if action != A_TOGGLE:
            return "continue"
        front_cell = self.env.doors.get(self.env.front_pos())  # a key, ball or box is never one of obj_set's doors
        for door in self.desc.obj_set:
            if front_cell and front_cell is door and door.is_open:
                return "success"
        if self.strict:
            if front_cell and front_cell.type == "door":
                return "failure"
        return "continue"


class BeforeInstr:  # verifier.py:451-489 (SeqInstr strict=False)
    def __init__(self, instr_a, instr_b, strict=False):
        self.instr_a, self.instr_b, self.strict = instr_a, instr_b, strict

    def surface(self, env):
        return self.instr_a.surface(env) + ", then " + self.instr_b.surface(env)

    def reset_verifier(self, env):
        self.env = env
        self.instr_a.reset_verifier(env)
        self.instr_b.reset_verifier(env)
        self.a_done = False
        self.b_done = False

    def first_done(self):
        return self.a_done == "success"

    def verify(self, action):
        if self.a_done == "success":
            self.b_done = self.instr_b.verify(action)
            if self.b_done == "failure":
                return "failure"
            if self.b_done == "success":
                return "success"
        else:
            self.a_done = self.instr_a.verify(action)
            if self.a_done == "failure":
                return "failure"
            if self.a_done == "success":
                return self.verify(action)
            if self.strict:
                if self.instr_b.verify(action) == "success":
                    return "failure"
        return "continue"


class AfterInstr:  # verifier.py:492-530 (SeqInstr strict=False)
    def __init__(self, instr_a, instr_b, strict=False):
        self.instr_a, self.instr_b, self.strict = instr_a, instr_b, strict

    def surface(self, env):
        return self.instr_a.surface(env) + " after you " + self.instr_b.surface(env)

    def reset_verifier(self, env):
        self.env = env
        self.instr_a.reset_verifier(env)
        self.instr_b.reset_verifier(env)
        self.a_done = False
        self.b_done = False

    def first_done(self):
        return self.b_done == "success"

    def verify(self, action):
        if self.b_done == "success":
            self.a_done = self.instr_a.verify(action)
            if self.a_done == "success":
                return "success"
            if self.a_done == "failure":
                return "failure"
        else:
            self.b_done = self.instr_b.verify(action)
            if self.b_done == "failure":
                return "failure"
            if self.b_done == "success":
                return self.verify(action)
            if self.strict:
                if self.instr_a.verify(action) == "success":
                    return "failure"
        return "continue"


def ordered(instrs):
    """(the OpenInstr to complete first, the one to complete second or None)"""
    if isinstance(instrs, BeforeInstr):
        return instrs.instr_a, instrs.instr_b
    if isinstance(instrs, AfterInstr):
        return instrs.instr_b, instrs.instr_a
    return instrs, None


class OpenLevel:
    """One Open / UnlockLocal level as RoomGridLevel builds it, then its doors and instruction as the reference holds them."""

    def __init__(self, spec, g):
        _, self.W, self.H, _, _, params = spec
        self.S, self.rows, self.cols = params[1], params[2], params[3]
        self.level, self.arg, self.strict = params[4], params[5], bool(params[6])
        self.g = g
        self.rejections = 0  # none of these levels rejects
        self._room_grid()
        self._gen_mission()
        self.mission_str = self.instrs.surface(self)  # roomgrid_level.py:142-144
        self.instrs.reset_verifier(self)              # RoomGridLevel.reset

    # ---- MiniGridEnv / RoomGrid helpers ----
    def _rand_int(self, lo, hi):
        return int(self.g.integers(lo, hi))

    def _rand_elem(self, lst):
        return lst[self._rand_int(0, len(lst))]

    def _rand_subset(self, lst, n):  # minigrid_env.py:277-292
        lst, out = list(lst), []
        while len(out) < n:
            e = self._rand_elem(lst)
            lst.remove(e)
            out.append(e)
        return out

    def room_from_pos(self, x, y):
        return self.room_grid[y // (self.S - 1)][x // (self.S - 1)]

    def front_pos(self):
        return (self.agent_pos[0] + DIR_TO_VEC[self.agent_dir][0], self.agent_pos[1] + DIR_TO_VEC[self.agent_dir][1])

    def _room_grid(self):  # RoomGrid._gen_grid (roomgrid.py:123-177)
        S = self.S
        self.grid = np.empty((self.W, self.H, 3), np.uint8)
        self.grid[:] = NONE
        self.room_grid = []
        for j in range(self.rows):
            row = []
            for i in range(self.cols):
                room = Room((i * (S - 1), j * (S - 1)), (S, S))
                row.append(room)
                x0, y0 = room.top
                self.grid[x0:x0 + S, y0] = self.grid[x0:x0 + S, y0 + S - 1] = WALL
                self.grid[x0, y0:y0 + S] = self.grid[x0 + S - 1, y0:y0 + S] = WALL
            self.room_grid.append(row)
        for j in range(self.rows):
            for i in range(self.cols):
                room = self.room_grid[j][i]
                x_l, y_l = room.top[0] + 1, room.top[1] + 1
                x_m, y_m = room.top[0] + S - 1, room.top[1] + S - 1
                if i < self.cols - 1:
                    room.neighbors[0] = self.room_grid[j][i + 1]
                    room.door_pos[0] = (x_m, self._rand_int(y_l, y_m))
                if j < self.rows - 1:
                    room.neighbors[1] = self.room_grid[j + 1][i]
                    room.door_pos[1] = (self._rand_int(x_l, x_m), y_m)
                if i > 0:
                    room.neighbors[2] = self.room_grid[j][i - 1]
                    room.door_pos[2] = room.neighbors[2].door_pos[0]
                if j > 0:
                    room.neighbors[3] = self.room_grid[j - 1][i]
                    room.door_pos[3] = room.neighbors[3].door_pos[1]
        self.agent_pos = ((self.cols // 2) * (S - 1) + S // 2, (self.rows // 2) * (S - 1) + S // 2)
        self.agent_dir = 0
        self.doors = {}  # grid position -> Door
        self.objs = []   # (type, colour) of Room.objs, in creation order

    def _place_obj(self, i, j, obj, reject_next_to):  # minigrid_env.py:313-372 over room (i, j)
        top = self.room_grid[j][i].top
        while True:
            pos = (self._rand_int(top[0], min(top[0] + self.S, self.W)), self._rand_int(top[1], min(top[1] + self.S, self.H)))
            if tuple(self.grid[pos]) != NONE:
                continue
            if pos == tuple(self.agent_pos):
                continue
            if reject_next_to and abs(self.agent_pos[0] - pos[0]) + abs(self.agent_pos[1] - pos[1]) < 2:
                continue
            break
        if obj is not None:
            self.grid[pos] = (OBJECT_TO_IDX[obj[0]], COLOR_TO_IDX[obj[1]], 0)
        return pos

    def _place_agent(self, i, j):  # RoomGrid.place_agent (roomgrid.py:313-334)
        while True:
            self.agent_pos = (-1, -1)
            self.agent_pos = self._place_obj(i, j, None, False)
            self.agent_dir = self._rand_int(0, 4)
            if tuple(self.grid[self.front_pos()]) in (NONE, WALL):
                break

    def _add_door(self, i, j, door_idx=None, color=None, locked=None):  # roomgrid.py:226-273
        room = self.room_grid[j][i]
        if door_idx is None:
            while True:
                door_idx = self._rand_int(0, 4)
                if room.neighbors[door_idx] and room.doors[door_idx] is None:
                    break
        if color is None:
            color = self._rand_elem(COLOR_NAMES)
        if locked is None:
            locked = self._rand_int(0, 2) == 0
        assert room.doors[door_idx] is None, "door already exists"
        pos = room.door_pos[door_idx]
        door = Door(color, pos, locked)
        self.grid[pos] = (4, COLOR_TO_IDX[color], 2 if locked else 1)
        self.doors[pos] = door
        room.doors[door_idx] = door
        room.neighbors[door_idx].doors[(door_idx + 2) % 4] = door
        return door

    def _add_object(self, i, j, kind, color):  # roomgrid.py:196-224 (kind and colour given)
        self._place_obj(i, j, (kind, color), True)
        self.objs.append((kind, color))

    def _add_distractors(self, i, j, num):  # roomgrid.py:396-438, all_unique=True, room given
        objs = list(self.objs)
        n = 0
        while n < num:
            color = self._rand_elem(COLOR_NAMES)
            kind = self._rand_elem(["key", "ball", "box"])
            if (kind, color) in objs:
                continue
            self._add_object(i, j, kind, color)
            objs.append((kind, color))
            n += 1

    def _gen_mission(self):
        lv = self.level
        if lv == OPENREDDOOR:
            self._add_door(0, 0, 0, "red", locked=False)
            self._place_agent(0, 0)
            self.instrs = OpenInstr(ObjDesc("door", "red"))
        elif lv == OPENDOOR:
            door_colors = self._rand_subset(COLOR_NAMES, 4)
            objs = [self._add_door(1, 1, door_idx=i, color=c, locked=False) for i, c in enumerate(door_colors)]
            select_by = {0: "color", 1: "loc", 2: None}[self.arg]
            if select_by is None:
                select_by = self._rand_elem(["color", "loc"])
            if select_by == "color":
                desc = ObjDesc(objs[0].type, color=objs[0].color)
            else:
                desc = ObjDesc(objs[0].type, loc=self._rand_elem(LOC_NAMES))
            self._place_agent(1, 1)
            self.instrs = OpenInstr(desc, strict=self.strict)
        elif lv == OPENTWODOORS:
            colors = self._rand_subset(COLOR_NAMES, 2)
            first, second = ("red", "blue") if self.arg else (colors[0], colors[1])
            door1 = self._add_door(1, 1, 2, color=first, locked=False)
            door2 = self._add_door(1, 1, 0, color=second, locked=False)
            self._place_agent(1, 1)
            self.instrs = BeforeInstr(OpenInstr(ObjDesc(door1.type, door1.color), strict=self.strict),
                                      OpenInstr(ObjDesc(door2.type, door2.color)))
        elif lv == OPENDOORSORDER:
            colors = self._rand_subset(COLOR_NAMES, self.arg)
            doors = [self._add_door(1, 1, color=colors[i], locked=False) for i in range(self.arg)]
            self._place_agent(1, 1)
            door1, door2 = self._rand_subset(doors, 2)
            desc1, desc2 = ObjDesc(door1.type, door1.color), ObjDesc(door2.type, door2.color)
            self.mode = self._rand_int(0, 3)
            if self.mode == 0:
                self.instrs = OpenInstr(desc1, strict=self.strict)
            elif self.mode == 1:
                self.instrs = BeforeInstr(OpenInstr(desc1, strict=self.strict), OpenInstr(desc2, strict=self.strict))
            else:
                self.instrs = AfterInstr(OpenInstr(desc1, strict=self.strict), OpenInstr(desc2, strict=self.strict))
        else:
            door = self._add_door(1, 1, locked=True)
            self._add_object(1, 1, "key", door.color)
            if self.arg:
                self._add_distractors(1, 1, 3)
            self._place_agent(1, 1)
            self.instrs = OpenInstr(ObjDesc(door.type))

    def mission(self):
        return self.mission_str


class OpenOracle(BabyAIOracle):
    """N Open / UnlockLocal envs in lockstep with SyncVectorEnv autoresets (see the module docstring). `events` counts what
    the tests need to have happened (successes, strict failures, progress, closes of an open target, ...)."""

    def __init__(self, env_id=None, num_envs=1, *, spec=None, autoreset="next_step", n_threads=1):
        super().__init__(None, num_envs, spec=spec if spec is not None else OPEN_SPECS[env_id], autoreset=autoreset,
                         n_threads=n_threads)
        self.levels = [None] * self.num_envs
        self.events = collections.Counter()

    def _regenerate(self, envs):
        if len(envs) == 0:
            return
        st = self.c.get_state()
        for i in envs:
            lv = OpenLevel(self.spec, self.gens[i])
            first, _ = ordered(lv.instrs)
            if first.desc.loc is not None:
                self.events["loc_matches_%d" % len(first.desc.obj_set)] += 1
            st["grid"][i] = lv.grid
            st["agent"][i] = [lv.agent_pos[0], lv.agent_pos[1], lv.agent_dir, -1, 0, 0]
            self.levels[i] = lv
            self.pending[i] = False
        st["rng"][:] = [rng_row(g) for g in self.gens]
        self.c.set_state(grid=st["grid"], agent=st["agent"], rng=st["rng"])

    def step(self, actions):
        a = np.ascontiguousarray(actions, dtype=np.int32)
        fresh = self.pending.copy() if self.autoreset == "next_step" else np.zeros(self.num_envs, bool)
        _, _, r, te, tr = self.c.step(a)
        r, te, tr = r.copy(), te.copy(), tr.copy()
        after = self.c.get_state()
        for i in np.nonzero(~fresh)[0]:
            lv, act = self.levels[i], int(a[i])
            lv.agent_pos, lv.agent_dir = (int(after["agent"][i, 0]), int(after["agent"][i, 1])), int(after["agent"][i, 2])
            door = lv.doors.get(lv.front_pos())
            was_open = door is not None and door.is_open
            if door is not None:  # Door.toggle (world_object.py:222-236) as the C oracle did it
                state = int(after["grid"][i][door.cur_pos][2])
                door.is_open, door.is_locked = state == 0, state == 2
            status = self._verify(lv, act, door, was_open)
            if status == "success":
                te[i] = True
                r[i] = 1.0 - 0.9 * (int(after["agent"][i, 5]) / self.max_steps)  # _reward(), minigrid_env.py:240-245
                self.events["success"] += 1
            elif status == "failure":
                te[i] = True
                r[i] = 0.0
                self.events["failure"] += 1
        r[fresh], te[fresh], tr[fresh] = 0.0, False, False
        done = (te | tr) & ~fresh
        if self.autoreset == "next_step":
            self._regenerate(np.nonzero(fresh)[0])
            self.pending = done
        elif self.autoreset == "same_step":
            self._regenerate(np.nonzero(done)[0])
        obs, d = self.c.gen_obs()
        return obs, d, r, te, tr

    def _verify(self, lv, act, door, was_open):
        """instrs.verify(action), counting the events around it"""
        first, second = ordered(lv.instrs)
        seq = second is not None
        done_before = seq and lv.instrs.first_done()
        if act == A_TOGGLE and door is not None:
            if was_open and not door.is_open and any(door is d for ins in (first, second) if ins for d in ins.desc.obj_set):
                self.events["closed_target"] += 1
            if seq and not done_before and door.is_open and any(door is d for d in second.desc.obj_set):
                self.events["second_opened_first"] += 1
            if door.is_open and door.is_locked is False and lv.level == UNLOCKLOCAL:
                self.events["unlocked"] += 1
        status = lv.instrs.verify(act)
        if seq and not done_before and lv.instrs.first_done():
            self.events["progress"] += 1
            if status == "failure":
                self.events["failure_on_first_open"] += 1
        if status == "failure" and not seq:
            self.events["strict_failure_single"] += 1
        return status

    def inject(self, i, pos=None, d=None, door_states=None, carry=None):
        """Env i's agent moved to the empty cell pos facing d, door cells set to states (0 open, 1 closed, 2 locked),
        and / or a key of colour `carry` put in its hands, in the C oracle and in the level's doors alike: the tests'
        injected states (copy get_state()'s grid and agent into the engine to give it the same)."""
        st = self.c.get_state()
        lv = self.levels[i]
        if pos is not None:
            st["agent"][i, :3] = (pos[0], pos[1], d)
        for cell, state in (door_states or {}).items():
            door = lv.doors[tuple(cell)]
            door.is_open, door.is_locked = state == 0, state == 2
            st["grid"][i][tuple(cell)][2] = state
        if carry is not None:
            st["agent"][i, 3:5] = (OBJECT_TO_IDX["key"], COLOR_TO_IDX[carry])
        self.c.set_state(grid=st["grid"], agent=st["agent"])


def hashed(env_id, num_envs=1, autoreset="next_step"):
    """hash_support.HashedOracle (MiniGridEnv.hash on the oracle's states) over an OpenOracle."""
    import hash_support as hs

    h = hs.HashedOracle.__new__(hs.HashedOracle)
    h.o = OpenOracle(env_id, num_envs, autoreset=autoreset)
    h.num_envs, h.autoreset = int(num_envs), autoreset
    h.moved = np.zeros(h.num_envs, bool)
    return h


# ---- the scripted policy of the reference record's scripted rollouts (oracle/ref_babyai_open.py) ----
STYLES = ["plain", "wrong_first", "close_again", "reverse"]


class ScriptedPolicy:
    """Toggles door cells in a planned order, fetching the key of a locked door first. `style`: "plain" opens the
    first instruction's door, then the second's; "wrong_first" first toggles a door neither instruction names;
    "close_again" toggles the first door three times (open, close, open) before the second; "reverse" opens the second
    door, then the first, then toggles the second twice (it closes, then opens). Reads only what a reference env shows:
    Grid.encode(), the agent, what it carries and the door cells of the instructions' obj_sets. Call start() at every
    reset; once the plan is done it turns left."""

    def __init__(self, style="plain"):
        self.style = style
        self.plan = []

    def start(self, first, second, doors):
        """first / second: the door cells of the first / second OpenInstr's obj_set (second empty for one
        instruction); doors: every door cell"""
        t1, t2 = first[0], (second[0] if second else None)
        plan = []
        if self.style == "wrong_first":
            plan += [c for c in doors if c not in first and c not in second][:1]
        if self.style == "reverse" and t2:
            plan.append(t2)
        plan.append(t1)
        if self.style == "close_again":
            plan += [t1, t1]
        if t2:
            plan += [t2, t2, t2] if self.style == "reverse" else [t2]
        self.plan = plan

    def act(self, grid, ax, ay, adir, carrying):
        if not self.plan:
            return 0
        tgt = self.plan[0]
        if int(grid[tgt][2]) == 2 and carrying is None:  # locked: fetch its key
            keys = {(int(x), int(y)) for x, y in zip(*np.nonzero((grid[:, :, 0] == OBJECT_TO_IDX["key"]) &
                                                                   (grid[:, :, 1] == grid[tgt][1])))}
            return self._go(grid, ax, ay, adir, keys, A_PICKUP)
        act = self._go(grid, ax, ay, adir, {tgt}, A_TOGGLE)
        if act == A_TOGGLE:
            self.plan.pop(0)
        return act

    @staticmethod
    def _go(grid, ax, ay, adir, cells, final):
        fx, fy = ax + DIR_TO_VEC[adir][0], ay + DIR_TO_VEC[adir][1]
        if (fx, fy) in cells:
            return final
        act = _bfs_first_action(grid, ax, ay, adir, cells)
        return 0 if act is None else act
