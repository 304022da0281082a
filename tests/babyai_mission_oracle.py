"""Per-env missions of the three BabyAI oracles. TEST INFRASTRUCTURE ONLY.

`make(env_id, n, autoreset)` returns the GoTo, Pickup or Open oracle of an id with two additions, kept up to date through
both autoreset modes and reset_mask:
  - missions():      [env.mission for every env], from the oracle's own instruction objects (Level / PickupLevel /
                     OpenLevel, their ObjDesc restatements and obj_set / obj_poss);
  - mission_codes(): the same missions in the device's layout (minigrid_b200/csrc/mg_common.cuh, MIS_*), built from those
                     objects, not from anything the device computes.
Also here: the actions of the missions record (biased toward the level's verb) and the renderer of a code back into
text, restated in Python from verifier.py's surface() methods for the tests that check the device's renderer.
"""
from __future__ import annotations

import numpy as np

from babyai_oracle import BABYAI_SPECS, BabyAIOracle, Level, rng_row
from babyai_open_oracle import OPEN_SPECS, AfterInstr, BeforeInstr, OpenOracle
from babyai_pickup_oracle import PICKUP_SPECS, PICKUPDIST, PUTNEXTLOCAL, PickupOracle

# mg_common.cuh: forms, ObjDesc fields
GOTO, PICKUP, OPEN, PUTNEXT, BEFORE, AFTER = 1, 2, 3, 4, 5, 6
TYPES = [None, "key", "ball", "box", "door"]
COLORS_BY_IDX = ["red", "green", "blue", "purple", "yellow", "grey"]  # COLOR_TO_IDX order
LOCS = [None, "left", "right", "front", "behind"]
IDX = {"red": 0, "green": 1, "blue": 2, "purple": 3, "yellow": 4, "grey": 5}
IDX_TO_TYPE = {5: "key", 6: "ball", 7: "box"}
IDX_TO_COLOR = {v: k for k, v in IDX.items()}


def desc_code(kind, color, loc, plural):
    return TYPES.index(kind) | ((0 if color is None else IDX[color] + 1) << 3) | (LOCS.index(loc) << 6) | (int(plural) << 9)


def code(form, a, b=0):
    return form | (a << 3) | (b << 13)


def surface(c):
    """Instr.surface of a mission code, restated from verifier.py (the device renders it with mission_words)."""
    def desc(d):
        kind, color, loc = TYPES[d & 7], (d >> 3) & 7, LOCS[(d >> 6) & 7]
        s = ("a " if (d >> 9) & 1 else "the ") + (COLORS_BY_IDX[color - 1] + " " if color else "") + (kind or "object")
        return s + {None: "", "front": " in front of you", "behind": " behind you"}.get(loc, f" on your {loc}")
    form, a, b = c & 7, (c >> 3) & 1023, (c >> 13) & 1023
    return {GOTO: lambda: "go to " + desc(a), PICKUP: lambda: "pick up " + desc(a), OPEN: lambda: "open " + desc(a),
            PUTNEXT: lambda: "put " + desc(a) + " next to " + desc(b),
            BEFORE: lambda: "open " + desc(a) + ", then open " + desc(b),
            AFTER: lambda: "open " + desc(a) + " after you open " + desc(b)}.get(form, lambda: "")()


def all_codes():
    """Every code the BabyAI grammars can produce (and a few more: any article on any descriptor)."""
    descs = [desc_code(k, c, None, p) for k in TYPES[:4] for c in [None] + COLORS_BY_IDX for p in (0, 1) if k or c]
    doors = [desc_code("door", c, None, p) for c in [None] + COLORS_BY_IDX for p in (0, 1)]
    doors += [desc_code("door", None, loc, p) for loc in LOCS[1:] for p in (0, 1)]
    out = [code(f, d) for f in (GOTO, PICKUP) for d in descs] + [code(OPEN, d) for d in doors]
    out += [code(PUTNEXT, a, b) for a in descs[::3] for b in descs[::5]]
    out += [code(f, a, b) for f in (BEFORE, AFTER) for a in doors for b in doors[:14]]
    return out


# ---- GoTo: Level keeps target and obj_poss; GoToInstr(ObjDesc(type, colour)) ----
def goto_code(lv):
    kind, color = IDX_TO_TYPE[lv.target[0]], IDX_TO_COLOR[lv.target[1]]
    return code(GOTO, desc_code(kind, color, None, len(lv.obj_poss) > 1))


def goto_mission(lv):
    kind, color = IDX_TO_TYPE[lv.target[0]], IDX_TO_COLOR[lv.target[1]]
    return "go to " + ("a " if len(lv.obj_poss) > 1 else "the ") + f"{color} {kind}"


class GoToMissionOracle(BabyAIOracle):
    """BabyAIOracle that keeps each env's Level (its _regenerate, restated with the level kept)."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.levels = [None] * self.num_envs

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
            self.levels[i] = lv
            self.pending[i] = False
        st["rng"][:] = [rng_row(g) for g in self.gens]
        self.c.set_state(grid=st["grid"], agent=st["agent"], rng=st["rng"])

    def missions(self):
        return [goto_mission(lv) for lv in self.levels]

    def mission_codes(self):
        return np.asarray([goto_code(lv) for lv in self.levels], np.uint32)


# ---- Pickup / PutNext: PickupLevel.desc / move / fixed, counted as its mission() counts them ----
def pickup_code(lv):
    def desc(kind, color):
        n = len(lv._matching(kind, color))
        if kind is None and color == "grey":
            n += 2 * (lv.W + lv.H) - 4
        return desc_code(kind, color, None, n > 1)
    if lv.level == PUTNEXTLOCAL:
        return code(PUTNEXT, desc(*lv.move[:2]), desc(*lv.fixed[:2]))
    return code(PICKUP, desc(*lv.desc))


class _AtReset:
    """missions() / mission_codes() as RoomGridLevel._gen_grid left them: taken when a level is generated, because
    PickupLevel.mission() counts the objects where they are now (a pickup takes one off the grid)."""

    def _regenerate(self, envs):
        super()._regenerate(envs)
        if not hasattr(self, "_mis"):
            self._mis, self._codes = [""] * self.num_envs, np.zeros(self.num_envs, np.uint32)
        for i in envs:
            self._mis[i], self._codes[i] = self.levels[i].mission(), self._code(self.levels[i])

    def missions(self):
        return list(self._mis)

    def mission_codes(self):
        return self._codes.copy()


class PickupMissionOracle(_AtReset, PickupOracle):
    _code = staticmethod(pickup_code)


# ---- Open: the instruction objects themselves ----
def open_code(lv):
    def desc(instr):
        d = instr.desc
        return desc_code(d.type, d.color, d.loc, len(d.obj_set) > 1)
    ins = lv.instrs
    if isinstance(ins, BeforeInstr):
        return code(BEFORE, desc(ins.instr_a), desc(ins.instr_b))
    if isinstance(ins, AfterInstr):  # the surface order: instr_a, " after you ", instr_b
        return code(AFTER, desc(ins.instr_a), desc(ins.instr_b))
    return code(OPEN, desc(ins))


class OpenMissionOracle(_AtReset, OpenOracle):
    _code = staticmethod(open_code)


ALL_SPECS = {**BABYAI_SPECS, **PICKUP_SPECS, **OPEN_SPECS}
IDS = list(ALL_SPECS)


def make(env_id, num_envs=1, autoreset="next_step"):
    if env_id in BABYAI_SPECS:
        return GoToMissionOracle(env_id, num_envs, autoreset=autoreset)
    if env_id in PICKUP_SPECS:
        return PickupMissionOracle(env_id, num_envs, autoreset=autoreset)
    return OpenMissionOracle(env_id, num_envs, autoreset=autoreset)


# ---- the actions of the missions record ----
def verb_actions(env_id):
    """The level's verbs: toggle for Open / UnlockLocal (and pickup, for the key), pickup for Pickup, pickup and drop
    for PutNext, none for GoTo (facing the target ends its episode)."""
    if env_id in OPEN_SPECS:
        return [5, 5, 3] if "Unlock" in env_id else [5]
    if env_id in PICKUP_SPECS:
        return [3, 4] if ALL_SPECS[env_id][5][4] == PUTNEXTLOCAL else [3]
    return []


def record_actions(env_id, n, steps, seed):
    """[steps][n] actions: half the time one of the level's verbs, otherwise uniform over left / right / forward."""
    rng = np.random.default_rng(seed)
    verbs = verb_actions(env_id)
    move = rng.integers(0, 3, (steps, n))
    if not verbs:
        return move
    use = rng.random((steps, n)) < 0.5
    verb = np.asarray(verbs)[rng.integers(0, len(verbs), (steps, n))]
    return np.where(use, verb, move)


__all__ = ["make", "IDS", "ALL_SPECS", "surface", "all_codes", "record_actions", "PICKUPDIST"]
