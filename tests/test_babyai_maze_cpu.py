"""The BabyAI maze levels (GoToObjMaze*, FindObjS*, KeyCorridor*) without a GPU: the oracle (tests/babyai_maze_oracle.py)
against the reference's record (tests/golden/ref_babyai_maze_traces.json, written by oracle/ref_babyai_maze.py), the
device generator compiled by g++ (tests/host_emu) against the oracle, mg_create's parameter checks, and the events the
record is only worth something with, counted on the oracle rather than assumed."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import hash_support as hs
from oracle import ref_babyai_maze as rec_mod
from oracle import ref_trace as rt
from babyai_maze_oracle import FINDOBJ, GOTO, KEYCORRIDOR, MAZE_SPECS, MazeLevel, MazeOracle, hashed
from babyai_pickup_oracle import scripted_rollout

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "host_emu"))
from emu import EmuVecEnv  # noqa: E402

REC = rec_mod.load_record()
IDS = list(MAZE_SPECS)
MODES = ["next_step", "same_step"]


def test_ids_and_tables_agree():
    from minigrid_b200 import specs

    assert len(IDS) == 17
    assert set(specs.BABYAI_MAZE_REGISTRY) == set(IDS) == set(REC["dims"])
    others = (set(specs.REGISTRY) | set(specs.BABYAI_REGISTRY) | set(specs.BABYAI_PICKUP_PUTNEXT_REGISTRY) |
              set(specs.BABYAI_OPEN_REGISTRY))
    assert not set(IDS) & others
    assert len(others) + len(IDS) == 136
    for env_id, (kind, w, h, ms, st, prm) in MAZE_SPECS.items():
        s = specs.get(env_id)
        assert (s.kind, s.width, s.height, s.max_steps, s.see_through_walls) == (specs.KIND_ROOMGRID, w, h, ms, st), env_id
        assert list(s.params) == list(prm), env_id
        assert [w, h, ms, st] == REC["dims"][env_id], env_id
        assert specs.is_babyai(s)
    # BabyAI's KeyCorridor is MiniGrid's generator on the same grid and step limit
    for env_id in [i for i in IDS if "KeyCorridor" in i]:
        b = specs.get(env_id)
        m = specs.get("MiniGrid-KeyCorridorS6R3-v0" if env_id == "BabyAI-KeyCorridor-v0" else env_id.replace("BabyAI", "MiniGrid"))
        assert (b.width, b.height, b.max_steps, b.params[1:4]) == (m.width, m.height, m.max_steps, m.params[1:4])


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_oracle_rollout_matches_reference(env_id, mode):
    orc = MazeOracle(env_id, rec_mod.N_ENVS, autoreset=mode)
    got = rt.rollout(orc, rec_mod.N_ENVS, rec_mod.SEED, rec_mod.ACT_SEED, rec_mod.STEPS)
    assert got == REC["lockstep"][rt.key(env_id, mode)]


@pytest.mark.parametrize("env_id", IDS)
def test_oracle_scripted_rollout_matches_reference(env_id):
    sc = REC["scripted"][env_id]
    assert len(sc["actions"]) == rec_mod.SCRIPT_STEPS
    orc = MazeOracle(env_id, rec_mod.SCRIPT_ENVS)
    assert scripted_rollout(orc, rec_mod.SCRIPT_ENVS, rec_mod.SCRIPT_SEED, sc["actions"]) == sc["trace"]


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_oracle_hash_rollout_matches_reference(env_id, mode):
    assert hs.hash_rollout(hashed(env_id, 6, autoreset=mode), 6) == REC["hash_rollout"][rt.key(env_id, mode)]


@pytest.mark.parametrize("env_id", IDS)
def test_oracle_hash_walk_matches_reference(env_id):
    assert hs.hash_walk(hashed(env_id, 6), 6) == REC["hash_walk"][env_id]


@pytest.mark.parametrize("env_id", IDS)
def test_missions_and_rejections_match_reference(env_id):
    """The oracle's mission after each recorded seeded reset is the reference's, and its RejectSampling retries over the
    recorded seeds are as many as the reference printed."""
    from minigrid_b200 import specs

    got = [MazeLevel(MAZE_SPECS[env_id], np.random.default_rng(s)).mission() for s in rec_mod.MISSION_SEEDS]
    assert got == REC["missions"][env_id]
    words = specs.babyai_mission_words(specs.get(env_id))
    assert all(set(m.split()) <= words for m in got)
    assert all(m.split()[2] == "the" for m in got)  # one object: "the"
    n = sum(MazeLevel(MAZE_SPECS[env_id], np.random.default_rng(s)).rejections for s in rec_mod.REJECT_SEEDS)
    assert n == REC["rejections"][env_id]


def test_recorded_rejections():
    """The reference rejects the GoTo mazes (most on small rooms) and never FindObj or KeyCorridor."""
    rej = REC["rejections"]
    for env_id in IDS:
        assert (rej[env_id] > 0) == ("GoToObjMaze" in env_id), env_id
    assert rej["BabyAI-GoToObjMazeS4R2-v0"] > rej["BabyAI-GoToObjMazeS5-v0"] > rej["BabyAI-GoToObjMaze-v0"]


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("layout", [0, 1], ids=["tiled", "window"])
def test_emu_generator_vs_oracle(env_id, layout):
    """The device's generator and fill (g++ build of the headers) against the oracle: a seeded reset of 200 envs, then
    unseeded resets that continue every env's stream; obs, direction, grid, agent record and RNG."""
    n = 200
    emu = EmuVecEnv(MAZE_SPECS[env_id], n, autoreset="next_step", layout=layout)
    orc = MazeOracle(env_id, n)
    for k in range(3):
        seed = 31 if k == 0 else None
        eo, ed = emu.reset(seed=seed)
        oo, od = orc.reset(seed=seed)
        np.testing.assert_array_equal(eo, oo, err_msg=f"obs, reset {k}")
        np.testing.assert_array_equal(ed, od, err_msg=f"dir, reset {k}")
        es, os_ = emu.get_state(), orc.get_state()
        for key in ("grid", "agent", "rng"):
            np.testing.assert_array_equal(es[key], os_[key], err_msg=f"{key}, reset {k}")
    if MAZE_SPECS[env_id][5][4] == GOTO and MAZE_SPECS[env_id][5][1] <= 5:
        assert orc.events["rejections"] > 0


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
    [10, 8, 3, 3, 0],                # arg missing
    [10, 8, 3, 3, 0, 0, 0],          # a seventh parameter
    [10, 3, 3, 3, 0, 0],             # GoTo: rooms of 4..8
    [10, 9, 3, 3, 0, 0],
    [10, 8, 3, 3, 0, 2],             # doors_open 0 or 1
    [10, 8, 3, 3, 0, -1],
    [10, 3, 3, 3, 1, 0],             # FindObj: rooms of 4..8
    [10, 5, 2, 3, 1, 0],             # FindObj: a square grid
    [10, 5, 1, 1, 1, 0],             # FindObj: room (1, 1) must exist
    [10, 5, 3, 3, 1, 1],             # FindObj has no arg
    [10, 6, 3, 2, 2, 0],             # KeyCorridor: 3 columns
    [10, 6, 3, 3, 2, 1],             # KeyCorridor has no arg
    [10, 8, 3, 3, 3, 0],             # unknown level
    [10, 8, 3, 3, -1, 0],
    [10, 4, 4, 3, 0, 0],             # at most 9 rooms
    [11, 8, 3, 3, 0, 0],             # no variant 11
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
    for prm in ([10, 4, 1, 1, 0, 0], [10, 8, 3, 3, 0, 1], [10, 4, 2, 2, 1, 0], [10, 8, 3, 3, 1, 0], [10, 3, 2, 3, 2, 0]):
        assert _create(L, prm) in (0, -4), prm


# ---- the events the record is only worth something with ----
@pytest.mark.parametrize("env_id", IDS)
def test_oracle_runs_are_not_vacuous(env_id):
    """Counted on the oracle over the recorded scripted actions: successes on every id, doors added by connect_all,
    and on KeyCorridor a pickup pressed while carrying the key."""
    sc = REC["scripted"][env_id]["actions"]
    orc = MazeOracle(env_id, rec_mod.SCRIPT_ENVS)
    scripted_rollout(orc, rec_mod.SCRIPT_ENVS, rec_mod.SCRIPT_SEED, sc)
    assert orc.events["success"] > 0
    assert orc.events["connect_doors"] > 0
    if MAZE_SPECS[env_id][5][4] == KEYCORRIDOR:
        assert orc.events["pickup_while_carrying"] > 0
    if MAZE_SPECS[env_id][5][4] == FINDOBJ:
        assert orc.events["rejections"] == 0
