"""The BabyAI Open and UnlockLocal levels without a GPU: the oracle (tests/babyai_open_oracle.py) against the reference's
record (tests/golden/ref_babyai_open_traces.json, written by oracle/ref_babyai_open.py), the device generator compiled by
g++ (tests/host_emu) against the oracle, the device post-filter's Open branch compiled by g++ against the oracle's
OpenInstr / BeforeInstr / AfterInstr, mg_create's parameter checks, and the events the record is only worth something
with, counted on the oracle rather than assumed."""
import ctypes as C
import itertools
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import hash_support as hs
from oracle import ref_babyai_open as rec_mod
from oracle import ref_trace as rt
from babyai_oracle import BABYAI_SPECS, COLOR_TO_IDX
from babyai_pickup_oracle import PICKUP_SPECS
from babyai_open_oracle import (A_TOGGLE, OPEN_SPECS, AfterInstr, BeforeInstr, Door, ObjDesc, OpenInstr, OpenLevel,
                                OpenOracle, hashed, scripted_rollout)

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "host_emu"))
from emu import EmuVecEnv  # noqa: E402

REC = rec_mod.load_record()
IDS = list(OPEN_SPECS)
MODES = ["next_step", "same_step"]
COLORS = ["red", "green", "blue", "purple", "yellow", "grey"]


def test_ids_and_tables_agree():
    from minigrid_b200 import specs

    assert len(IDS) == 14
    assert set(specs.BABYAI_OPEN_REGISTRY) == set(IDS) == set(REC["dims"])
    assert not set(IDS) & (set(specs.REGISTRY) | set(specs.BABYAI_REGISTRY) | set(specs.BABYAI_PICKUP_PUTNEXT_REGISTRY) |
                           set(BABYAI_SPECS) | set(PICKUP_SPECS))
    assert len(specs.REGISTRY) + len(specs.BABYAI_REGISTRY) + len(specs.BABYAI_PICKUP_PUTNEXT_REGISTRY) + len(IDS) == 119
    for env_id, (kind, w, h, ms, st, prm) in OPEN_SPECS.items():
        s = specs.get(env_id)
        assert (s.kind, s.width, s.height, s.max_steps, s.see_through_walls) == (specs.KIND_ROOMGRID, w, h, ms, st), env_id
        assert list(s.params) == list(prm), env_id
        assert [w, h, ms, st] == REC["dims"][env_id], env_id
    with pytest.raises(KeyError, match="BabyAI-OpenDoor-v0"):
        specs.get("BabyAI-OpenDoor-v1")


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_oracle_rollout_matches_reference(env_id, mode):
    orc = OpenOracle(env_id, rec_mod.N_ENVS, autoreset=mode)
    got = rt.rollout(orc, rec_mod.N_ENVS, rec_mod.SEED, rec_mod.ACT_SEED, rec_mod.STEPS)
    assert got == REC["lockstep"][rt.key(env_id, mode)]


@pytest.mark.parametrize("env_id", IDS)
def test_oracle_scripted_rollout_matches_reference(env_id):
    sc = REC["scripted"][env_id]
    assert len(sc["actions"]) == rec_mod.SCRIPT_STEPS
    orc = OpenOracle(env_id, rec_mod.SCRIPT_ENVS)
    assert scripted_rollout(orc, rec_mod.SCRIPT_ENVS, rec_mod.SCRIPT_SEED, sc["actions"]) == sc["trace"]


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_oracle_hash_rollout_matches_reference(env_id, mode):
    assert hs.hash_rollout(hashed(env_id, 6, autoreset=mode), 6) == REC["hash_rollout"][rt.key(env_id, mode)]


@pytest.mark.parametrize("env_id", IDS)
def test_oracle_hash_walk_matches_reference(env_id):
    assert hs.hash_walk(hashed(env_id, 6), 6) == REC["hash_walk"][env_id]


def _mission_pattern(mission):
    """A template's {article}, {color} and {location} fields, and [a | b] for one of two optional endings."""
    alt = {"article": "(the|a)", "color": "(" + "|".join(COLORS) + ")",
           "location": "(on your left|on your right|in front of you|behind you)"}
    s = re.escape(mission)
    s = re.sub(r"\\\[(.*?)\\\]", lambda m: "(" + "|".join(m.group(1).split("\\|")) + ")?", s)
    s = re.sub(r"\\\{(\w+)\\\}", lambda m: alt[m.group(1)], s)
    if mission.startswith("open {article} {color} door"):  # OpenDoor: a colour or a location, not both
        return re.compile(r"open (the ({c}) door|(the|a) door {l})\Z".format(c=alt["color"][1:-1], l=alt["location"]))
    return re.compile(s.replace("\\ ", " ") + r"\Z")


def test_recorded_missions_match_the_spec_and_the_oracle():
    """Every recorded mission matches its spec's template (a constant one is the recorded string after every reset);
    the oracle's surface form is the recorded string exactly, "a" and "the" included; every form of OpenDoor and
    OpenDoorsOrder occurs."""
    from minigrid_b200 import specs

    forms = set()
    for env_id in IDS:
        mission, got = specs.get(env_id).mission, REC["missions"][env_id]
        assert len(got) == 50
        if "{" not in mission:
            assert set(got) == {mission}, env_id
        pat = _mission_pattern(mission)
        for m in got:
            assert pat.match(m), (env_id, m)
        assert [OpenLevel(OPEN_SPECS[env_id], np.random.default_rng(s)).mission() for s in rec_mod.MISSION_SEEDS] == got
        if env_id.startswith("BabyAI-OpenDoor-") or env_id.startswith("BabyAI-OpenDoorsOrder"):
            forms |= {("order" if "Order" in env_id else "door", "your" in m or "front" in m or "behind" in m,
                       ", then" in m, " after you " in m, m.split()[1]) for m in got}
    assert {f[1:4] for f in forms if f[0] == "door"} == {(False, False, False), (True, False, False)}
    assert {f[2:4] for f in forms if f[0] == "order"} == {(False, False), (True, False), (False, True)}
    assert {f[4] for f in forms if f[1]} == {"a", "the"}


def test_dict_observation_indices_of_the_constant_missions():
    from minigrid_b200 import specs
    from minigrid_b200.wrappers import mission_to_indices

    assert set(REC["dict_missions"]) == {i for i in IDS if "{" not in specs.get(i).mission} == set(rec_mod.CONSTANT_MISSION_IDS)
    for env_id, want in REC["dict_missions"].items():
        assert mission_to_indices(specs.get(env_id).mission) == want, env_id


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("layout", [0, 1], ids=["tiled", "window"])
def test_emu_generator_vs_oracle(env_id, layout):
    """The device's generator and fill (g++ build of the headers) against the oracle: a seeded reset, then unseeded
    resets that continue every env's stream; obs, direction, grid, agent record and RNG."""
    n = 45
    emu = EmuVecEnv(OPEN_SPECS[env_id], n, autoreset="next_step", layout=layout)
    orc = OpenOracle(env_id, n)
    for k in range(6):
        seed = 31 if k == 0 else None
        eo, ed = emu.reset(seed=seed)
        oo, od = orc.reset(seed=seed)
        np.testing.assert_array_equal(eo, oo, err_msg=f"obs, reset {k}")
        np.testing.assert_array_equal(ed, od, err_msg=f"dir, reset {k}")
        es, os_ = emu.get_state(), orc.get_state()
        for key in ("grid", "agent", "rng"):
            np.testing.assert_array_equal(es[key], os_[key], err_msg=f"{key}, reset {k}")


# ---- the device post-filter (mg_postfilter.cuh) under g++, against the oracle's verifiers ----
_PF_SRC = r"""
#include <cstdlib>
#include <cstring>
#include "mg_common.cuh"
#include "mg_postfilter.cuh"
using namespace mg;
extern "C" void pf_open(int action, unsigned front, int tx, int ty, unsigned aux, int *out) {
  PostIn in;
  in.action = action; in.ax = in.ay = 3; in.dir = 0;
  in.carry_before = in.carry = 0; in.tx = tx; in.ty = ty; in.aux = aux;
  in.red_before = in.blue_before = in.red_after = in.blue_after = false;
  in.variant = RG_BABYAI_OPEN; in.door_open = false; in.front = front; in.level = 0; in.next_to = 0;
  const PostOut o = post_filter<KIND_ROOMGRID>(in, 0u);
  out[0] = (int)o.terminated; out[1] = o.reward; out[2] = (int)o.aux;
}
"""


@pytest.fixture(scope="module")
def pf(tmp_path_factory):
    d = tmp_path_factory.mktemp("pf")
    src, lib = d / "pf.cpp", d / "libpf.so"
    src.write_text(_PF_SRC)
    csrc = os.path.join(os.path.dirname(HERE), "minigrid_b200", "csrc")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-I", csrc, "-o", str(lib),
                           str(src)])
    L = C.CDLL(str(lib))
    L.pf_open.argtypes = [C.c_int, C.c_uint, C.c_int, C.c_int, C.c_uint, C.c_void_p]

    def call(*args):
        out = (C.c_int * 3)()
        L.pf_open(*args, out)
        return {(0, 0): "continue", (1, 1): "success", (1, 2): "failure"}[(out[0], out[1])], out[2]
    return call


class _Env:
    """What OpenInstr reads of the env: the doors by position and front_pos"""

    def __init__(self, doors, front):
        self.doors, self._front = doors, front

    def front_pos(self):
        return self._front


# room (1, 1) of a 3 x 3 grid of rooms of 6: one door per side (right, down, left, up), each its own colour
SIDE_CELLS = [(10, 7), (7, 10), (5, 7), (7, 5)]
SIDE_COLORS = ["red", "green", "blue", "grey"]
OPEN_AUX = {"seq": 1, "strict1": 2, "strict2": 4, "done": 8}


def _front_cases():
    """(front cell position, its code, its door state or None): each side's door open / closed / locked, a wall, an empty
    cell and a key of a door's colour"""
    out = []
    for k, cell in enumerate(SIDE_CELLS):
        for state, t4 in ((0, 4), (1, 11), (2, 12)):
            out.append((cell, t4 | COLOR_TO_IDX[SIDE_COLORS[k]] << 4 | (0x80 if state else 0), state))
    return out + [((0, 0), 0xD2, None), ((7, 7), 1, None), ((8, 8), 5 | COLOR_TO_IDX["red"] << 4, None)]


def _mask(sides):
    return sum(1 << COLOR_TO_IDX[SIDE_COLORS[k]] for k in sides)


def test_post_filter_open_vs_oracle_verifier(pf):
    """Every action × front cell (each side's door in each state, a wall, an empty cell, a key) × descriptor (the set of
    sides obj_set holds) × mode (one OpenInstr, BeforeInstr, AfterInstr) × strict flags × progress bit: the device
    predicate and its progress bit against the reference's verifiers on doors compared by identity."""
    side_sets = [s for r in range(1, 5) for s in itertools.combinations(range(4), r)]
    seq_sets = [(k,) for k in range(4)] + [(0, 2), (0, 1, 2, 3)]
    n = {"success": 0, "failure": 0, "done_set": 0}
    cases = [("single", d1, (), s1, False, False) for d1 in side_sets for s1 in (False, True)]
    cases += [(m, d1, d2, s1, s2, p) for m in ("before", "after") for d1 in seq_sets for d2 in seq_sets
              for s1 in (False, True) for s2 in (False, True) for p in (False, True)]
    for (mode, d1, d2, s1, s2, prog), (front, code, state), action in itertools.product(cases, _front_cases(), range(7)):
        doors = {cell: Door(SIDE_COLORS[k], cell, False) for k, cell in enumerate(SIDE_CELLS)}
        if state is not None:
            doors[front].is_open, doors[front].is_locked = state == 0, state == 2
        env = _Env(doors, front)

        def instr(sides, strict):
            desc = ObjDesc("door")
            desc.obj_set = [doors[SIDE_CELLS[k]] for k in sides]
            ins = OpenInstr(desc, strict=strict)
            ins.env = env
            return ins
        if mode == "single":
            ins = instr(d1, s1)
            first_sides, second_sides, st1, st2 = d1, (), s1, False
        else:
            a, b = instr(d1, s1), instr(d2, s2)
            ins = (BeforeInstr if mode == "before" else AfterInstr)(a, b)
            ins.a_done = ins.b_done = False
            if prog:
                if mode == "before":
                    ins.a_done = "success"
                else:
                    ins.b_done = "success"
            first_sides, second_sides, st1, st2 = (d1, d2, s1, s2) if mode == "before" else (d2, d1, s2, s1)
        want = ins.verify(action)
        want_done = mode != "single" and ins.first_done()
        aux = ((OPEN_AUX["seq"] if mode != "single" else 0) | (OPEN_AUX["strict1"] if st1 else 0) |
               (OPEN_AUX["strict2"] if st2 else 0) | (OPEN_AUX["done"] if prog else 0))
        got, got_aux = pf(action, code, _mask(first_sides), _mask(second_sides), aux)
        assert (got, bool(got_aux & OPEN_AUX["done"])) == (want, want_done), (mode, d1, d2, s1, s2, prog, front, code,
                                                                               action)
        assert got_aux & ~OPEN_AUX["done"] == aux & ~OPEN_AUX["done"]
        n[want] = n.get(want, 0) + 1
        n["done_set"] += want_done and not prog
    assert n["success"] > 0 and n["failure"] > 0 and n["done_set"] > 0


def test_post_filter_debug_sequence_fails_on_the_first_correct_open(pf):
    """BeforeInstr / AfterInstr of two strict OpenInstrs: the toggle that opens the first door re-verifies the second,
    which sees a door that is not its own: failure (the reference's behaviour, kept)."""
    red_open = 4 | COLOR_TO_IDX["red"] << 4
    aux = OPEN_AUX["seq"] | OPEN_AUX["strict1"] | OPEN_AUX["strict2"]
    assert pf(A_TOGGLE, red_open, _mask([0]), _mask([2]), aux) == ("failure", aux | OPEN_AUX["done"])
    aux = OPEN_AUX["seq"] | OPEN_AUX["strict1"]
    assert pf(A_TOGGLE, red_open, _mask([0]), _mask([2]), aux) == ("continue", aux | OPEN_AUX["done"])


# ---- mg_create ----
def _create(L, params, w=None, h=None, max_steps=64):
    S = params[1] if len(params) > 1 else 8
    w = (S - 1) * (params[3] if len(params) > 3 else 1) + 1 if w is None else w
    h = (S - 1) * (params[2] if len(params) > 2 else 1) + 1 if h is None else h
    prm = (C.c_int32 * len(params))(*params)
    hd = C.c_void_p()
    rc = L.mg_create(16, w, h, max_steps, 0, prm, len(params), 4, 0, 0, C.byref(hd))
    if hd.value:
        L.mg_destroy(hd)
    return rc


@pytest.mark.parametrize("params", [
    [9, 8, 1, 1, 0, 1, 0],           # one room: a door needs a neighbour
    [9, 8, 1, 1, 1, 2, 0],
    [9, 5, 1, 2, 0, 0],              # strict missing
    [9, 5, 3, 3, 0, 0, 0],           # OpenRedDoor is 1 x 2 rooms
    [9, 8, 1, 2, 1, 2, 0],           # the others are 3 x 3
    [9, 8, 2, 2, 4, 0, 0],
    [9, 4, 3, 3, 1, 0, 0],           # rooms of 5..8
    [9, 9, 3, 3, 1, 0, 0],
    [9, 8, 3, 3, 5, 0, 0],           # unknown level
    [9, 8, 3, 3, -1, 0, 0],
    [9, 5, 1, 2, 0, 1, 0],           # OpenRedDoor has no arg
    [9, 5, 1, 2, 0, 0, 1],           # nor a strict flag
    [9, 8, 3, 3, 1, 3, 0],           # select_by 0..2
    [9, 6, 3, 3, 2, 2, 0],           # fixed red / blue: 0 or 1
    [9, 6, 3, 3, 3, 1, 0],           # num_doors 2..4
    [9, 6, 3, 3, 3, 5, 0],
    [9, 8, 3, 3, 4, 2, 0],           # distractors 0 or 1
    [9, 8, 3, 3, 4, 0, 1],           # UnlockLocal is never strict
    [9, 8, 3, 3, 1, 0, 2],
    [10, 8, 3, 3, 1, 0, 0],          # no variant 10
])
def test_create_refuses_malformed_params(params):
    from minigrid_b200 import _lib

    L = _lib.load()
    assert _create(L, params) == -1, params
    assert b"babyai" in L.mg_last_error() or b"roomgrid" in L.mg_last_error()


def test_create_accepts_the_registered_params():
    """Valid parameters pass the checks (MG_OK on a GPU, MG_ERR_NO_DEVICE without one, never MG_ERR_INVALID_ARG)."""
    from minigrid_b200 import _lib, specs

    L = _lib.load()
    for env_id in IDS:
        s = specs.get(env_id)
        assert _create(L, list(s.params), s.width, s.height, s.max_steps) in (0, -4), env_id
    for prm in ([9, 5, 3, 3, 4, 1, 0], [9, 6, 3, 3, 1, 1, 1], [9, 7, 3, 3, 3, 3, 1], [9, 8, 1, 2, 0, 0, 0]):
        assert _create(L, prm) in (0, -4), prm


# ---- the events the record is only worth something with ----
def _random_events(env_id, n=256, steps=300, seed=123):
    """Random actions with toggles made likely: forward 40 %, toggle 30 %, the rest uniform."""
    orc = OpenOracle(env_id, n)
    orc.reset(seed=seed)
    rng = np.random.default_rng(9)
    for _ in range(steps):
        u = rng.random(n)
        orc.step(np.where(u < 0.4, 2, np.where(u < 0.7, A_TOGGLE, rng.integers(0, 7, n))).astype(np.int32))
    return orc.events


@pytest.mark.parametrize("env_id", IDS)
def test_oracle_runs_are_not_vacuous(env_id):
    """Counted on the oracle over the recorded scripted actions and random ones: successes on every id; strict failures
    on the Debug ids and none elsewhere; on the sequences, first instructions completed (the progress bit) and a second
    door opened before the first; on OpenDoorsOrder*Debug, failures on the very toggle that completes the first
    instruction; closes of an open target door; location descriptors that match two or more doors."""
    sc = REC["scripted"][env_id]["actions"]
    orc = OpenOracle(env_id, rec_mod.SCRIPT_ENVS)
    scripted_rollout(orc, rec_mod.SCRIPT_ENVS, rec_mod.SCRIPT_SEED, sc)
    ev = orc.events + _random_events(env_id)
    assert orc.events["success"] > 0
    strict = OPEN_SPECS[env_id][5][6]
    assert (ev["failure"] > 0) == bool(strict)
    level = OPEN_SPECS[env_id][5][4]
    if level in (2, 3):
        assert ev["progress"] > 0 and ev["second_opened_first"] > 0
    if level == 2 or (level == 3 and not strict):  # a strict sequence fails before any door can be closed again
        assert ev["closed_target"] > 0
    if level == 3 and strict:
        assert ev["failure_on_first_open"] > 0
    if env_id == "BabyAI-OpenRedBlueDoorsDebug-v0":  # only door1's OpenInstr is strict: no failure on the first open
        assert ev["failure_on_first_open"] == 0 and ev["strict_failure_single"] == 0
    if level == 4:
        assert orc.events["unlocked"] > 0
    if env_id in ("BabyAI-OpenDoorLoc-v0", "BabyAI-OpenDoor-v0"):
        assert ev["loc_matches_1"] > 0 and ev["loc_matches_2"] + ev["loc_matches_3"] > 0
