"""The single-room BabyAI Pickup and PutNext levels without a GPU: the oracle (tests/babyai_pickup_oracle.py) against the
reference's record (tests/golden/ref_babyai_pickup_traces.json, written by oracle/ref_babyai_pickup.py), the device
generator compiled by g++ (tests/host_emu) against the oracle, the device post-filter's Pickup and PutNext branches
compiled by g++ against the oracle's verifiers, mg_create's parameter checks, and the events the record is only worth
something with, counted on the oracle rather than assumed."""
import ctypes as C
import itertools
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import hash_support as hs
from oracle import ref_babyai_pickup as rec_mod
from oracle import ref_trace as rt
from babyai_oracle import BABYAI_SPECS
from babyai_pickup_oracle import (A_DROP, A_PICKUP, COLOR_TO_IDX, OBJECT_TO_IDX, PICKUP_SPECS, Obj, PickupLevel,
                                  PickupOracle, hashed, scripted_rollout)

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "host_emu"))
from emu import EmuVecEnv  # noqa: E402

REC = rec_mod.load_record()
IDS = list(PICKUP_SPECS)
MODES = ["next_step", "same_step"]
COLORS = ["red", "green", "blue", "purple", "yellow", "grey"]
TYPES = ["key", "ball", "box"]


def test_ids_and_tables_agree():
    from minigrid_b200 import specs

    assert len(IDS) == 9
    assert set(specs.BABYAI_PICKUP_PUTNEXT_REGISTRY) == set(IDS) == set(REC["dims"])
    assert not set(IDS) & (set(specs.REGISTRY) | set(specs.BABYAI_REGISTRY) | set(BABYAI_SPECS))
    for env_id, (kind, w, h, ms, st, prm) in PICKUP_SPECS.items():
        s = specs.get(env_id)
        assert (s.kind, s.width, s.height, s.max_steps, s.see_through_walls) == (specs.KIND_ROOMGRID, w, h, ms, st), env_id
        assert list(s.params) == list(prm), env_id
        assert [w, h, ms, st] == REC["dims"][env_id], env_id
    with pytest.raises(KeyError, match="BabyAI-OneRoomS8-v0"):
        specs.get("BabyAI-OneRoomS9-v0")


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_oracle_rollout_matches_reference(env_id, mode):
    orc = PickupOracle(env_id, rec_mod.N_ENVS, autoreset=mode)
    got = rt.rollout(orc, rec_mod.N_ENVS, rec_mod.SEED, rec_mod.ACT_SEED, rec_mod.STEPS)
    assert got == REC["lockstep"][rt.key(env_id, mode)]


@pytest.mark.parametrize("env_id", IDS)
def test_oracle_scripted_rollout_matches_reference(env_id):
    sc = REC["scripted"][env_id]
    assert len(sc["actions"]) == rec_mod.SCRIPT_STEPS
    orc = PickupOracle(env_id, rec_mod.N_ENVS)
    assert scripted_rollout(orc, rec_mod.N_ENVS, rec_mod.SCRIPT_SEED, sc["actions"]) == sc["trace"]


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_oracle_hash_rollout_matches_reference(env_id, mode):
    assert hs.hash_rollout(hashed(env_id, 6, autoreset=mode), 6) == REC["hash_rollout"][rt.key(env_id, mode)]


@pytest.mark.parametrize("env_id", IDS)
def test_oracle_hash_walk_matches_reference(env_id):
    assert hs.hash_walk(hashed(env_id, 6), 6) == REC["hash_walk"][env_id]


def _mission_pattern(mission):
    """PickupDist's descriptor drops the colour or the type ("object"), so its template stands for three forms."""
    alt = {"article": "(the|a)", "color": "(" + "|".join(COLORS) + ")", "type": "(" + "|".join(TYPES) + ")"}
    if mission == "pick up {article} {color} {type}":
        return re.compile(r"pick up (the|a) ({color} {type}|{color} object|{type})\Z".format(**alt))
    return re.compile(re.sub(r"\\\{(\w+)\\\}", lambda m: alt[m.group(1)], re.escape(mission)) + r"\Z")


def test_recorded_missions_match_the_spec_and_the_oracle():
    """Every recorded mission matches its spec's template (a constant one is the recorded string after every reset);
    the oracle's surface form is the recorded string exactly, "a" and "the" included."""
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
        assert [PickupLevel(PICKUP_SPECS[env_id], np.random.default_rng(s)).mission() for s in rec_mod.MISSION_SEEDS] == got
        if env_id.startswith("BabyAI-PickupDist"):
            forms |= {("object" in m, any(c in m.split() for c in COLORS), m.split()[2]) for m in got}
    # type only, colour only (an object: "a grey object" as the walls match too), both; with both articles
    assert {(f[0], f[1]) for f in forms} == {(False, False), (True, True), (False, True)}
    assert {f[2] for f in forms} == {"a", "the"}


def test_dict_observation_indices_of_the_constant_missions():
    from minigrid_b200 import specs
    from minigrid_b200.wrappers import mission_to_indices

    assert set(REC["dict_missions"]) == {i for i in IDS if "{" not in specs.get(i).mission}
    for env_id, want in REC["dict_missions"].items():
        assert mission_to_indices(specs.get(env_id).mission) == want, env_id


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("layout", [0, 1], ids=["tiled", "window"])
def test_emu_generator_vs_oracle(env_id, layout):
    """The device's generator and fill (g++ build of the headers) against the oracle: a seeded reset, then unseeded
    resets that continue every env's stream through the rejection loops; obs, direction, grid, agent record and RNG."""
    n = 45
    emu = EmuVecEnv(PICKUP_SPECS[env_id], n, autoreset="next_step", layout=layout)
    orc = PickupOracle(env_id, n)
    for k in range(6):
        seed = 31 if k == 0 else None
        eo, ed = emu.reset(seed=seed)
        oo, od = orc.reset(seed=seed)
        np.testing.assert_array_equal(eo, oo, err_msg=f"obs, reset {k}")
        np.testing.assert_array_equal(ed, od, err_msg=f"dir, reset {k}")
        es, os_ = emu.get_state(), orc.get_state()
        for key in ("grid", "agent", "rng"):
            np.testing.assert_array_equal(es[key], os_[key], err_msg=f"{key}, reset {k}")
    if PICKUP_SPECS[env_id][5][4] == 2:
        assert orc.rejections() > 0 and orc.events["next_rejections"] > 0


# ---- the device post-filter (mg_postfilter.cuh) under g++, against the oracle's verifiers ----
_PF_SRC = r"""
#include <cstdlib>
#include <cstring>
#include "mg_common.cuh"
#include "mg_postfilter.cuh"
using namespace mg;
extern "C" void pf_babyai(int level, int action, unsigned carry_before, unsigned carry, int tx, int ty, unsigned aux,
                          unsigned next_to, int *out) {
  PostIn in;
  in.action = action; in.ax = in.ay = 3; in.dir = 0;
  in.carry_before = carry_before; in.carry = carry; in.tx = tx; in.ty = ty; in.aux = aux;
  in.red_before = in.blue_before = in.red_after = in.blue_after = false;
  in.variant = RG_BABYAI_PICKUP_PUTNEXT; in.door_open = false; in.level = level; in.next_to = next_to;
  const PostOut o = post_filter<KIND_ROOMGRID>(in, 0u);
  out[0] = (int)o.terminated; out[1] = o.reward;
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
    L.pf_babyai.argtypes = [C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_int, C.c_int, C.c_uint, C.c_uint, C.c_void_p]

    def call(*args):
        out = (C.c_int * 2)()
        L.pf_babyai(*args, out)
        return {(0, 0): "continue", (1, 1): "success", (1, 2): "failure"}[(out[0], out[1])]
    return call


def _code(kind, color):
    return OBJECT_TO_IDX[kind] | COLOR_TO_IDX[color] << 4


OBJS = [(k, c) for k in TYPES for c in ("red", "grey", "blue")]
WALL = 0xD2


def _verifier_level(level, strict=False):
    """A PickupLevel with only its verifier state, for objects the test places itself"""
    lv = PickupLevel.__new__(PickupLevel)
    lv.level, lv.strict = level, strict
    lv.pre_carrying = lv.carrying = None
    lv.world = {}
    return lv


def test_post_filter_pickup_vs_oracle_verifier(pf):
    """Every action, every pair (carried before, carried after) among nothing and nine objects, every descriptor form
    and strictness: the device predicate against PickupInstr.verify_action on objects compared by identity."""
    n = 0
    for (tk, tc), select_by, strict in itertools.product(OBJS, ["type", "color", "both"], [False, True]):
        desc = (None if select_by == "color" else tk, None if select_by == "type" else tc)
        aux = (0 if select_by == "color" else 1) | (0 if select_by == "type" else 2) | (4 if strict else 0)
        for before, after, action in itertools.product([None] + OBJS, [None] + OBJS, range(7)):
            lv = _verifier_level(1, strict=strict)
            objs = {o: Obj(o[0], o[1], (1 + i, 1)) for i, o in enumerate(OBJS)}
            lv.obj_set = [objs[o] for o in OBJS if (desc[0] in (None, o[0])) and (desc[1] in (None, o[1]))]
            lv.pre_carrying = None if before is None else objs[before]
            lv.carrying = None if after is None else objs[after]
            want = lv.verify(action)
            got = pf(1, action, 0 if before is None else _code(*before), 0 if after is None else _code(*after),
                     OBJECT_TO_IDX[tk], COLOR_TO_IDX[tc], aux, 0)
            assert got == want, (desc, strict, before, after, action)
            n += want != "continue"
    assert n > 0


def test_post_filter_putnext_vs_oracle_verifier(pf):
    """Drops (and every other action) of the move object or another one, succeeded or not, with the fixed object in each
    of the 8 cells around the drop cell or elsewhere, and the other neighbours walls, empty or other objects: the
    device predicate on the three neighbour codes against PutNextInstr.verify_action with cur_pos and obj_poss."""
    move, fixed, other = ("ball", "red"), ("key", "blue"), ("box", "grey")
    front = (4, 4)  # the agent stands on (3, 4), facing +x
    around = [(5, 4), (4, 3), (4, 5)]  # beyond, and the two beside: K1's byte order
    spots = around + [(5, 3), (5, 5), (3, 3), (3, 5), (6, 4), (4, 6), (1, 6)]  # the fixed object's cell
    n_succ = 0
    for action, carried, dropped, spot, filler in itertools.product(range(7), [move, other, None], [True, False],
                                                                    spots, [1, WALL, _code(*other)]):
        om, of = Obj(*move, (1, 1)), Obj(*fixed, spot)
        lv = _verifier_level(2)
        lv.move_set, lv.fixed_set = [om], [of]
        lv.world = {of.cur_pos: of}
        carried_obj = {move: om, other: Obj(*other, (6, 6)), None: None}[carried]
        lv.pre_carrying = carried_obj
        ok_drop = action == A_DROP and carried_obj is not None and dropped
        if carried_obj is not None:
            carried_obj.cur_pos = (-1, -1)
        lv.carrying = carried_obj
        if ok_drop:
            lv.transition(A_DROP, front, 0, -1, 0)
        want = lv.verify(action)
        codes = [(_code(*fixed) if c == spot else filler) for c in around]
        nxt = codes[0] | codes[1] << 8 | codes[2] << 16
        cb = 0 if carried is None else _code(*carried)
        ca = 0 if ok_drop or carried is None else cb
        got = pf(2, action, cb, ca, OBJECT_TO_IDX[move[0]], COLOR_TO_IDX[move[1]], _code(*fixed), nxt)
        assert got == want, (action, carried, dropped, spot, filler)
        n_succ += want == "success"
    assert n_succ > 0


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
    [8, 8, 1, 1, 0, 1],              # strict missing
    [8, 8, 1, 2, 2, 3, 0],           # two rooms
    [8, 8, 2, 1, 1, 5, 0],
    [8, 8, 1, 1, 3, 2, 0],           # unknown level
    [8, 8, 1, 1, -1, 2, 0],
    [8, 8, 1, 1, 0, 2, 0],           # OneRoom places one ball
    [8, 8, 1, 1, 2, 1, 0],           # PutNext needs two objects
    [8, 7, 1, 1, 1, 0, 0],           # PickupDist draws its target from the objects
    [8, 8, 1, 1, 2, 9, 0],           # more than 8 objects
    [8, 5, 1, 1, 2, 5, 0],           # a room of 5: 4 cells in the worst case
    [8, 4, 1, 1, 2, 2, 0],           # a room of 4 has one cell away from the agent
    [8, 12, 1, 1, 2, 3, 0],          # PutNext: the fill is a 64-bit mask
    [8, 12, 1, 1, 1, 5, 0],          # only OneRoom goes past 8
    [8, 21, 1, 1, 0, 1, 0],          # nor OneRoom past 20
    [8, 3, 1, 1, 0, 1, 0],
    [8, 8, 1, 1, 0, 1, 1],           # strict only on PickupDist
    [8, 8, 1, 1, 2, 3, 1],
    [8, 7, 1, 1, 1, 5, 2],
    [7, 12, 1, 1, 3, 2],             # GoTo stays <= 8
    [3, 9, 3, 3],                    # and every other variant
    [0, 12, 1, 2],
    [9, 8, 1, 1, 0, 1, 0],           # no variant 9
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
    for prm in ([8, 4, 1, 1, 0, 1, 0], [8, 20, 1, 1, 0, 1, 0], [8, 8, 1, 1, 1, 8, 1], [8, 6, 1, 1, 2, 2, 0]):
        assert _create(L, prm) in (0, -4), prm


# ---- the events the record is only worth something with ----
def _random_events(env_id, n=256, steps=400, seed=123, forward=0.4):
    orc = PickupOracle(env_id, n)
    orc.reset(seed=seed)
    rng = np.random.default_rng(9)
    for _ in range(steps):
        orc.step(np.where(rng.random(n) < forward, 2, rng.integers(0, 7, n)).astype(np.int32))
    return orc.events


@pytest.mark.parametrize("env_id", IDS)
def test_oracle_runs_are_not_vacuous(env_id):
    """Counted on the oracle: successes on every id (random actions for Pickup, the recorded scripted actions for
    PutNext); strict failures on PickupDistDebug, one of them while already carrying; every select_by form; for PutNext
    a success after the fixed object was moved, a drop next to the fixed object that failed because the cell was
    occupied, and levels rejected because the two objects were already next to each other."""
    level = PICKUP_SPECS[env_id][5][4]
    sc = REC["scripted"][env_id]["actions"]
    orc = PickupOracle(env_id, rec_mod.N_ENVS)
    scripted_rollout(orc, rec_mod.N_ENVS, rec_mod.SCRIPT_SEED, sc)
    assert orc.events["success"] > 0
    ev = _random_events(env_id, steps=150 if level == 0 else 400)
    if level != 2:
        assert ev["success"] > 0
    if env_id == "BabyAI-PickupDistDebug-v0":
        # a strict failure ends the episode at its first pickup, so a pickup while carrying needs an injected carry:
        # the target itself in half of the envs, another object in the others
        assert ev["failure"] > 0
        n = 64
        orc = PickupOracle(env_id, n)
        orc.reset(seed=4)
        for i, lv in enumerate(orc.levels):
            pick = lv.obj_set[0] if i % 2 == 0 else next(o for o in lv.world.values() if o not in lv.obj_set)
            orc.inject(i, carry=pick.cur_pos)
        _, _, r, te, _ = orc.step(np.full(n, A_PICKUP, np.int32))
        assert te.all() and not r.any() and orc.events["failure_while_carrying"] == n
    else:
        assert ev["failure"] == 0
    if level == 1:
        assert all(ev["select_by_" + s] > 0 for s in ("type", "color", "both"))
    if level == 2:
        assert orc.events["success_after_fixed_moved"] > 0
        assert ev["occupied_drop_next_to_fixed"] + orc.events["occupied_drop_next_to_fixed"] > 0
        assert ev["next_rejections"] > 0
