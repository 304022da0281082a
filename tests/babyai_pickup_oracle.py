"""The oracle of the single-room BabyAI Pickup and PutNext levels. TEST INFRASTRUCTURE ONLY.

`PickupOracle` is tests/babyai_oracle.py's BabyAIOracle (the transition, gen_obs, FullyObs and truncation on the C
oracle, the SyncVectorEnv autoresets in Python) with the generators and verifiers of these levels restated in the
reference's own form:
  - RoomGridLevel._gen_grid (babyai/core/roomgrid_level.py:119-177) with the gen_mission of OneRoomS* (other.py:329-332),
    PickupDist (pickup.py:275-290) and PutNextLocal (putnext.py:71-80) and validate_instrs' "objs already next to each
    other", on numpy's own PCG64 Generator;
  - every object is a Python object whose identity follows the C oracle's pickups, drops and box toggles, with the
    cur_pos the reference keeps ((-1, -1) while carried);
  - PickupInstr (verifier.py:319-363): obj_set by identity, preCarrying, strict;
  - PutNextInstr (verifier.py:366-435): obj_set by identity, preCarrying, obj_poss refreshed on every drop
    (RoomGridLevel.step's update_objs_poss), cur_pos of the move object.
The device reduces both verifiers to predicates on cell codes (mg_postfilter.cuh); the tests compare the two.
"""
from __future__ import annotations

import collections

import numpy as np

from babyai_oracle import COLOR_NAMES, COLOR_TO_IDX, DIR_TO_VEC, OBJECT_TO_IDX, BabyAIOracle, Level, RejectSampling, rng_row

ONEROOM, PICKUPDIST, PUTNEXTLOCAL = 0, 1, 2
A_PICKUP, A_DROP, A_TOGGLE = 3, 4, 5


def _spec(level, room_size, num_objs, num_navs, strict=False):
    """One room, num_navs * room_size^2 steps (roomgrid_level.py:71-85); params {8, room_size, 1, 1, level, num_objs,
    strict}"""
    return ("roomgrid", room_size, room_size, num_navs * room_size * room_size, False,
            [8, room_size, 1, 1, level, num_objs, int(strict)])


# __init__.py:864-873, 883-898, 1059-1081
PICKUP_SPECS = {
    **{f"BabyAI-OneRoomS{s}-v0": _spec(ONEROOM, s, 1, 1) for s in (8, 12, 16, 20)},
    "BabyAI-PickupDist-v0": _spec(PICKUPDIST, 7, 5, 1),
    "BabyAI-PickupDistDebug-v0": _spec(PICKUPDIST, 7, 5, 1, strict=True),
    "BabyAI-PutNextLocal-v0": _spec(PUTNEXTLOCAL, 8, 8, 2),
    "BabyAI-PutNextLocalS5N3-v0": _spec(PUTNEXTLOCAL, 5, 3, 2),
    "BabyAI-PutNextLocalS6N4-v0": _spec(PUTNEXTLOCAL, 6, 4, 2),
}


class Obj:
    """A WorldObj of these rooms (Key, Ball or Box): compared by identity, as the verifiers compare them."""

    def __init__(self, kind, color, pos):
        self.type, self.color, self.cur_pos = kind, color, tuple(pos)


def pos_next_to(a, b):  # verifier.py:29-39
    return abs(a[0] - b[0]) + abs(a[1] - b[1]) == 1


class PickupLevel(Level):
    """One Pickup / PutNext level as RoomGridLevel builds it, then its objects and verifier as the reference holds them."""

    def __init__(self, spec, g):
        _, self.W, self.H, _, _, params = spec
        self.S, self.level, self.num_objs, self.strict = params[1], params[4], params[5], bool(params[6])
        self.g = g
        self.rejections = self.next_rejections = 0
        while True:  # roomgrid_level.py:119-140
            try:
                self._room_grid()
                self._gen_mission()
                self._validate()
                break
            except RejectSampling as e:
                self.rejections += 1
                self.next_rejections += str(e) == "objs already next to each other"
        self.world = {pos: Obj(k, c, pos) for k, c, pos in self.objs}  # grid position -> object
        self.carrying = None
        self.pre_carrying = None
        if self.level == PUTNEXTLOCAL:
            self.move_set = self._matching(*self.move[:2])
            self.fixed_set = self._matching(*self.fixed[:2])
            self.fixed_poss = [o.cur_pos for o in self.fixed_set]
        else:
            self.obj_set = self._matching(*self.desc)

    def _gen_mission(self):
        self.objs = []
        if self.level == ONEROOM:  # add_object(0, 0, kind="ball"): the colour is drawn; then place_agent()
            self._add_object("ball", self._rand_elem(COLOR_NAMES))
            self._place_agent()
            self.desc = ("ball", None)
            self.select_by = "type"
        elif self.level == PICKUPDIST:  # placed around the default room centre, then place_agent(0, 0)
            objs = self._add_distractors(self.num_objs, all_unique=True)
            self._place_agent()
            kind, color, _ = self._rand_elem(objs)
            self.select_by = self._rand_elem(["type", "color", "both"])
            self.desc = (None if self.select_by == "color" else kind, None if self.select_by == "type" else color)
        else:
            self._place_agent()
            objs = self._add_distractors(self.num_objs, all_unique=True)
            self._check_objs_reachable()
            lst = list(objs)  # _rand_subset(objs, 2)
            self.move = self._rand_elem(lst)
            lst.remove(self.move)
            self.fixed = self._rand_elem(lst)

    def _validate(self):  # validate_instrs (roomgrid_level.py:160-177) for a PutNextInstr
        if self.level == PUTNEXTLOCAL and pos_next_to(self.move[2], self.fixed[2]):
            raise RejectSampling("objs already next to each other")

    def _matching(self, kind, color):
        """ObjDesc.find_matching_objs's obj_set over the objects (x-major, as it scans). Walls match a colour-only grey
        descriptor too; they can never be carried, so the verifiers do not need them (the mission counts them)."""
        return [self.world[p] for p in sorted(self.world)
                if (kind is None or self.world[p].type == kind) and (color is None or self.world[p].color == color)]

    def mission(self):
        """instrs.surface(env) (verifier.py:64-100, 331-332, 378-384)."""
        def surface(kind, color):
            n = len(self._matching(kind, color))
            if kind is None and color == "grey":  # find_matching_objs scans every cell: the walls are grey
                n += 2 * (self.W + self.H) - 4
            s = (color + " " if color else "") + (kind or "object")
            return ("a " if n > 1 else "the ") + s
        if self.level == PUTNEXTLOCAL:
            return "put " + surface(*self.move[:2]) + " next to " + surface(*self.fixed[:2])
        return "pick up " + surface(*self.desc)

    # ---- what the C oracle's transition did to the objects (minigrid_env.py:555-588) ----
    def transition(self, action, front, carried_before, carried_after, front_after):
        if action == A_PICKUP and carried_before < 0 <= carried_after:
            self.carrying = self.world.pop(front)
            self.carrying.cur_pos = (-1, -1)
        elif action == A_DROP and carried_after < 0 <= carried_before:
            self.carrying.cur_pos = front
            self.world[front] = self.carrying
            self.carrying = None
        elif action == A_TOGGLE and front in self.world and self.world[front].type == "box" and front_after == 1:
            del self.world[front]  # Box.toggle: replaced by its contents, None here

    # ---- RoomGridLevel.step after super().step (roomgrid_level.py:87-104) ----
    def verify(self, action):
        if self.level == PUTNEXTLOCAL:
            if action == A_DROP:  # update_objs_poss: find_matching_objs(use_location=False) on the tracked objects
                self.fixed_poss = [p for p in sorted(self.world) if any(self.world[p] is o for o in self.fixed_set)]
            return self._verify_putnext(action)
        return self._verify_pickup(action)

    def _verify_pickup(self, action):  # PickupInstr.verify_action
        pre = self.pre_carrying
        self.pre_carrying = self.carrying
        if action != A_PICKUP:
            return "continue"
        for obj in self.obj_set:
            if pre is None and self.carrying is obj:
                return "success"
        if self.strict and self.carrying:
            return "failure"
        self.pre_carrying = self.carrying
        return "continue"

    def _verify_putnext(self, action):  # PutNextInstr.verify_action (strict=False)
        pre = self.pre_carrying
        self.pre_carrying = self.carrying
        if action != A_DROP:
            return "continue"
        for obj_a in self.move_set:
            if pre is not obj_a:
                continue
            for pos_b in self.fixed_poss:
                if pos_next_to(obj_a.cur_pos, pos_b):
                    return "success"
        return "continue"


class PickupOracle(BabyAIOracle):
    """N Pickup / PutNext envs in lockstep with SyncVectorEnv autoresets (see the module docstring). `events` counts what
    the tests need to have happened (successes, strict failures, drops next to the fixed object, ...)."""

    def __init__(self, env_id=None, num_envs=1, *, spec=None, autoreset="next_step", n_threads=1):
        super().__init__(None, num_envs, spec=spec if spec is not None else PICKUP_SPECS[env_id], autoreset=autoreset,
                         n_threads=n_threads)
        self.levels = [None] * self.num_envs
        self.fixed_moved = np.zeros(self.num_envs, bool)
        self.events = collections.Counter()

    def _regenerate(self, envs):
        if len(envs) == 0:
            return
        st = self.c.get_state()
        for i in envs:
            lv = PickupLevel(self.spec, self.gens[i])
            self.n_rejections += lv.rejections
            self.events["next_rejections"] += lv.next_rejections
            if lv.level == PICKUPDIST:
                self.events["select_by_" + lv.select_by] += 1
            st["grid"][i] = lv.grid
            st["agent"][i] = [lv.agent_pos[0], lv.agent_pos[1], lv.agent_dir, -1, 0, 0]
            self.levels[i] = lv
            self.fixed_moved[i] = False
            self.pending[i] = False
        st["rng"][:] = [rng_row(g) for g in self.gens]
        self.c.set_state(grid=st["grid"], agent=st["agent"], rng=st["rng"])

    def step(self, actions):
        a = np.ascontiguousarray(actions, dtype=np.int32)
        fresh = self.pending.copy() if self.autoreset == "next_step" else np.zeros(self.num_envs, bool)
        before = self.c.get_state()["agent"].copy()
        _, _, r, te, tr = self.c.step(a)
        r, te, tr = r.copy(), te.copy(), tr.copy()
        after = self.c.get_state()
        for i in np.nonzero(~fresh)[0]:
            lv, act = self.levels[i], int(a[i])
            x, y, d = (int(v) for v in before[i, :3])
            front = (x + DIR_TO_VEC[d][0], y + DIR_TO_VEC[d][1])
            lv.transition(act, front, int(before[i, 3]), int(after["agent"][i, 3]), int(after["grid"][i][front][0]))
            if lv.level == PUTNEXTLOCAL:
                self._count_putnext(i, lv, act, front, before[i], after["agent"][i])
            status = lv.verify(act)
            if status == "success":
                te[i] = True
                r[i] = 1.0 - 0.9 * (int(after["agent"][i, 5]) / self.max_steps)  # _reward(), minigrid_env.py:240-245
                self.events["success"] += 1
                self.events["success_after_fixed_moved"] += int(self.fixed_moved[i])
            elif status == "failure":
                te[i] = True
                r[i] = 0.0
                self.events["failure"] += 1
                self.events["failure_while_carrying"] += int(before[i, 3] >= 0)
        r[fresh], te[fresh], tr[fresh] = 0.0, False, False
        done = (te | tr) & ~fresh
        if self.autoreset == "next_step":
            self._regenerate(np.nonzero(fresh)[0])
            self.pending = done
        elif self.autoreset == "same_step":
            self._regenerate(np.nonzero(done)[0])
        obs, d = self.c.gen_obs()
        return obs, d, r, te, tr

    def inject(self, i, pos=None, d=None, carry=None):
        """Env i's agent moved to the empty cell pos facing d, and / or the object at cell `carry` put in its hands as if
        picked up in an earlier step (preCarrying included), in the C oracle and in the level's objects alike: the tests'
        injected states (copy get_state()'s grid and agent into the engine to give it the same)."""
        st = self.c.get_state()
        lv = self.levels[i]
        if pos is not None:
            st["agent"][i, :3] = (pos[0], pos[1], d)
        if carry is not None:
            obj = lv.world.pop(tuple(carry))
            obj.cur_pos = (-1, -1)
            lv.carrying = lv.pre_carrying = obj
            st["grid"][i][tuple(carry)] = (1, 0, 0)
            st["agent"][i, 3:5] = (OBJECT_TO_IDX[obj.type], COLOR_TO_IDX[obj.color])
            if lv.level == PUTNEXTLOCAL and obj is lv.fixed_set[0]:
                self.fixed_moved[i] = True
        self.c.set_state(grid=st["grid"], agent=st["agent"])

    def _count_putnext(self, i, lv, act, front, before, after):
        fixed = lv.fixed_set[0]
        if act == A_PICKUP and lv.carrying is fixed:
            self.fixed_moved[i] = True
        if act == A_DROP and before[3] >= 0 and after[3] >= 0 and lv.carrying is lv.move_set[0] and fixed.cur_pos != (-1, -1) \
                and pos_next_to(front, fixed.cur_pos):
            self.events["occupied_drop_next_to_fixed"] += 1


def hashed(env_id, num_envs=1, autoreset="next_step"):
    """hash_support.HashedOracle (MiniGridEnv.hash on the oracle's states) over a PickupOracle."""
    import hash_support as hs

    h = hs.HashedOracle.__new__(hs.HashedOracle)
    h.o = PickupOracle(env_id, num_envs, autoreset=autoreset)
    h.num_envs, h.autoreset = int(num_envs), autoreset
    h.moved = np.zeros(h.num_envs, bool)
    return h


# ---- the scripted policy of the reference record's scripted rollouts (oracle/ref_babyai_pickup.py) ----
def _bfs_first_action(grid, ax, ay, adir, goal_cells):
    """The first of the fewest left / right / forward actions that leave the agent facing one of goal_cells, moving
    through empty cells only; None when none is reachable. grid is Grid.encode() ([x, y] -> (type, colour, state))."""
    start = (ax, ay, adir)
    seen = {start: None}
    queue = collections.deque([start])
    while queue:
        s = queue.popleft()
        x, y, d = s
        if (x + DIR_TO_VEC[d][0], y + DIR_TO_VEC[d][1]) in goal_cells:
            if s == start:
                return None
            while seen[s][0] != start:
                s = seen[s][0]
            return seen[s][1]
        fx, fy = x + DIR_TO_VEC[d][0], y + DIR_TO_VEC[d][1]
        nxt = [((x, y, (d + 3) % 4), 0), ((x, y, (d + 1) % 4), 1)]
        if int(grid[fx, fy, 0]) == 1:
            nxt.append(((fx, fy, d), 2))
        for t, act in nxt:
            if t not in seen:
                seen[t] = (s, act)
                queue.append(t)
    return None


def _cells(grid, kind, color):
    return {(int(x), int(y)) for x, y in zip(*np.nonzero(
        (grid[:, :, 0] == OBJECT_TO_IDX[kind] if kind else np.isin(grid[:, :, 0], [5, 6, 7])) &
        (grid[:, :, 1] == COLOR_TO_IDX[color] if color else True)))}


class ScriptedPolicy:
    """Picks up the Pickup target, or carries the PutNext move object to a free cell next to the fixed object. With
    displace_fixed, a PutNext episode first picks the fixed object up and drops it at least two cells from where it
    was. Reads only what a reference env shows: Grid.encode(), the agent, what it carries and the instruction's
    descriptors (type, colour). Stateful per episode: call start() at every reset."""

    def __init__(self, displace_fixed=False):
        self.displace_fixed = displace_fixed
        self.start(None)

    def start(self, instr):
        self.instr = instr
        self.displaced = not self.displace_fixed
        self.fixed_origin = None

    def act(self, grid, ax, ay, adir, carrying):
        """carrying: (type, colour) names or None; returns an action."""
        kind, ins = self.instr[0], self.instr[1:]
        if kind == "pickup":
            return self._go(grid, ax, ay, adir, _cells(grid, *ins[0]), A_PICKUP) if carrying is None else A_DROP
        move, fixed = ins
        if not self.displaced:
            if carrying is None:
                cells = _cells(grid, *fixed)
                if self.fixed_origin is None and cells:
                    self.fixed_origin = next(iter(cells))
                return self._go(grid, ax, ay, adir, cells, A_PICKUP)
            if tuple(carrying) == tuple(fixed):
                ox, oy = self.fixed_origin
                face = {(int(x), int(y)) for x, y in zip(*np.nonzero(grid[:, :, 0] == 1)) if abs(x - ox) + abs(y - oy) >= 2}
                act = self._go(grid, ax, ay, adir, face, A_DROP)
                if act == A_DROP:
                    self.displaced = True
                return act
        if carrying is None:
            return self._go(grid, ax, ay, adir, _cells(grid, *move), A_PICKUP)
        fc = _cells(grid, *fixed)
        face = {(x + dx, y + dy) for x, y in fc for dx, dy in DIR_TO_VEC if int(grid[x + dx, y + dy, 0]) == 1}
        return self._go(grid, ax, ay, adir, face, A_DROP)

    @staticmethod
    def _go(grid, ax, ay, adir, cells, final):
        fx, fy = ax + DIR_TO_VEC[adir][0], ay + DIR_TO_VEC[adir][1]
        if (fx, fy) in cells:
            return final
        act = _bfs_first_action(grid, ax, ay, adir, cells)
        return 0 if act is None else act  # nothing reachable: turn (the episode runs into its step limit)


def scripted_rollout(env, n, seed, actions):
    """A seeded reset and the given per-step actions ([steps][n]), traced as oracle/ref_trace.rollout traces its
    random ones (outputs after every step, then the state and FullyObs)."""
    from oracle.ref_trace import Trace, _end

    tr = Trace()
    tr.add(*env.reset(seed=seed))
    tr.mark("reset")
    for t, a in enumerate(actions):
        tr.add(*env.step(np.asarray(a)))
        if (t + 1) % 25 == 0 or t + 1 == len(actions):
            tr.mark(f"step {t}")
    _end(env, tr, True)
    return tr.marks
