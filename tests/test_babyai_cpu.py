"""The single-room BabyAI GoTo levels without a GPU: the oracle (tests/babyai_oracle.py) against the reference's record
(tests/golden/ref_babyai_traces.json, written by oracle/ref_babyai.py), the device generator compiled by g++
(tests/host_emu) against the oracle, mg_create's parameter checks, and the events the record is only worth something
with (successes, a success on the truncating step, rejected levels, ...) counted on the oracle rather than assumed."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

import hash_support as hs
from oracle import ref_babyai
from oracle import ref_trace as rt
from babyai_oracle import BABYAI_SPECS, BabyAIOracle, hashed
from oracle.oracle import ENV_SPECS

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emu"))
from emu import EmuVecEnv  # noqa: E402

REC = ref_babyai.load_record()
IDS = list(BABYAI_SPECS)
MODES = ["next_step", "same_step"]
KINDS = ["empty", "doorkey", "crossing", "fourrooms", "lavagap", "distshift", "multiroom", "lockedroom", "playground",
         "gotodoor", "fetch", "redbluedoors", "gotoobject", "putnear", "memory", "dynobstacles", "roomgrid"]
COLORS = ["red", "green", "blue", "purple", "yellow", "grey"]
TYPES = ["key", "ball", "box"]


def test_ids_and_tables_agree():
    from minigrid_b200 import specs

    assert len(IDS) == 20
    assert set(specs.BABYAI_REGISTRY) == set(IDS) == set(REC["dims"])
    assert not set(specs.REGISTRY) & set(IDS) and not set(ENV_SPECS) & set(IDS)
    assert len(specs.REGISTRY) == 76
    for env_id, (kind, w, h, ms, st, prm) in BABYAI_SPECS.items():
        s = specs.get(env_id)
        assert (KINDS[s.kind], s.width, s.height, s.max_steps, s.see_through_walls) == (kind, w, h, ms, st), env_id
        assert list(s.params) == list(prm), env_id
        assert [w, h, ms, st] == REC["dims"][env_id], env_id


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_oracle_rollout_matches_reference(env_id, mode):
    orc = BabyAIOracle(env_id, ref_babyai.N_ENVS, autoreset=mode)
    got = rt.rollout(orc, ref_babyai.N_ENVS, ref_babyai.SEED, ref_babyai.ACT_SEED, ref_babyai.STEPS)
    assert got == REC["lockstep"][rt.key(env_id, mode)]


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_oracle_hash_rollout_matches_reference(env_id, mode):
    assert hs.hash_rollout(hashed(env_id, 6, autoreset=mode), 6) == REC["hash_rollout"][rt.key(env_id, mode)]


@pytest.mark.parametrize("env_id", IDS)
def test_oracle_hash_walk_matches_reference(env_id):
    assert hs.hash_walk(hashed(env_id, 6), 6) == REC["hash_walk"][env_id]


def _mission_pattern(mission):
    alt = {"article": "(the|a)", "color": "(" + "|".join(COLORS) + ")", "type": "(" + "|".join(TYPES) + ")"}
    return re.compile(re.sub(r"\\\{(\w+)\\\}", lambda m: alt[m.group(1)], re.escape(mission)) + r"\Z")


def test_recorded_missions_match_the_spec():
    """Constant missions are the recorded string after every reset; templates match every recorded string, and every
    alternative a template offers for the article shows up somewhere in the record."""
    from minigrid_b200 import specs

    articles = set()
    for env_id in IDS:
        mission, got = specs.get(env_id).mission, REC["missions"][env_id]
        assert len(got) == 50
        if "{" not in mission:
            assert set(got) == {mission}, env_id
            continue
        pat = _mission_pattern(mission)
        for m in got:
            assert pat.match(m), (env_id, m)
        if "{article}" in mission:
            articles |= {m.split()[2] for m in got}
    assert articles == {"the", "a"}


def test_dict_observation_indices_of_the_constant_missions():
    from minigrid_b200 import specs
    from minigrid_b200.wrappers import mission_to_indices

    assert set(REC["dict_missions"]) == {i for i in IDS if "{" not in specs.get(i).mission}
    for env_id, want in REC["dict_missions"].items():
        assert mission_to_indices(specs.get(env_id).mission) == want, env_id


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("layout", [0, 1], ids=["tiled", "window"])
def test_emu_generator_vs_oracle(env_id, layout):
    """The device's generator and fill (g++ build of the headers, tests/host_emu) against the oracle: a seeded reset,
    then unseeded resets that continue every env's stream through the rejection loops, comparing obs, direction,
    grid, agent record and RNG state each time. (That harness predates the BabyAI post-filter's front-cell input, so
    its steps are not compared here; K1's steps are, on the GPU, in tests/test_gpu_babyai.py.)"""
    n = 45
    emu = EmuVecEnv(BABYAI_SPECS[env_id], n, autoreset="next_step", layout=layout)
    orc = BabyAIOracle(env_id, n)
    for k in range(6):
        seed = 31 if k == 0 else None
        eo, ed = emu.reset(seed=seed)
        oo, od = orc.reset(seed=seed)
        np.testing.assert_array_equal(eo, oo, err_msg=f"obs, reset {k}")
        np.testing.assert_array_equal(ed, od, err_msg=f"dir, reset {k}")
        es, os_ = emu.get_state(), orc.get_state()
        for key in ("grid", "agent", "rng"):
            np.testing.assert_array_equal(es[key], os_[key], err_msg=f"{key}, reset {k}")


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
    [7, 8, 1, 1, 3],              # num_dists missing
    [7, 8, 1, 2, 3, 2],           # two rooms
    [7, 8, 2, 1, 3, 2],
    [7, 3, 1, 1, 1, 0],           # room_size 3: no cell for an object away from the agent
    [7, 8, 1, 1, 5, 2],           # unknown level
    [7, 8, 1, 1, -1, 2],
    [7, 8, 1, 1, 2, 2],           # GoToObj places exactly one object
    [7, 8, 1, 1, 3, 0],           # GoToLocal draws its target from the distractors
    [7, 8, 1, 1, 3, 9],           # more than 8 objects
    [7, 8, 1, 1, 0, 8],           # 1 + 8 objects
    [7, 4, 1, 1, 3, 2],           # a room of 4 has one cell away from the agent
    [7, 5, 1, 1, 3, 5],           # a room of 5: 4 cells in the worst case
    [7, 8, 1, 1, 1, -1],
    [8, 8, 1, 1, 3, 2],           # no variant 8
])
def test_create_refuses_malformed_babyai_params(params):
    from minigrid_b200 import _lib

    L = _lib.load()
    assert _create(L, params) == -1, params
    assert b"babyai" in L.mg_last_error() or b"roomgrid" in L.mg_last_error()


def test_create_accepts_the_registered_params_and_keeps_the_other_roomgrid_checks():
    """Valid parameters pass the checks (MG_OK on a GPU, MG_ERR_NO_DEVICE without one, never MG_ERR_INVALID_ARG); the
    ObstructedMaze and KeyCorridor checks are unchanged now that variant 7 exists."""
    from minigrid_b200 import _lib, specs

    L = _lib.load()
    ok = (0, -4)
    for env_id in IDS:
        s = specs.get(env_id)
        assert _create(L, list(s.params), s.width, s.height, s.max_steps) in ok, env_id
    for env_id in ["MiniGrid-ObstructedMaze-1Dlhb-v0", "MiniGrid-ObstructedMaze-Full-v1", "MiniGrid-KeyCorridorS3R1-v0",
                   "MiniGrid-KeyCorridorS6R3-v0", "MiniGrid-Unlock-v0", "MiniGrid-BlockedUnlockPickup-v0"]:
        s = specs.get(env_id)
        assert _create(L, list(s.params), s.width, s.height, s.max_steps) in ok, env_id
    assert _create(L, [5, 6, 3, 3, 1, 1, 0x11]) == -1 and b"obstructedmaze" in L.mg_last_error()  # num_quarters missing
    assert _create(L, [6, 6, 3, 3, 1, 1, 0x11, 5]) == -1  # 5 quarters
    assert _create(L, [4, 3, 1, 2, 1, 1, 0, 0]) == -1     # room_size 3
    assert _create(L, [3, 6, 3, 2]) == -1 and b"keycorridor" in L.mg_last_error()
    assert _create(L, [1, 6, 2, 2]) == -1 and b"1 x 2" in L.mg_last_error()


FAMILIES = {  # one id per generator, with what its level can produce
    "BabyAI-GoToRedBallGrey-v0": dict(rejects=True, multi=False, distractors=True),
    "BabyAI-GoToRedBall-v0": dict(rejects=True, multi=True, distractors=True),
    "BabyAI-GoToObj-v0": dict(rejects=False, multi=False, distractors=False),
    "BabyAI-GoToLocal-v0": dict(rejects=True, multi=True, distractors=True),
    "BabyAI-GoToRedBlueBall-v0": dict(rejects=True, multi=False, distractors=True),
}
DXY = [(1, 0), (0, 1), (-1, 0), (0, -1)]


@pytest.mark.parametrize("env_id", list(FAMILIES))
def test_oracle_runs_are_not_vacuous(env_id):
    """Over a seeded random-action run of the oracle (NEXT_STEP: a step's state is the one before its autoreset):
    successes occur; some step is terminated and truncated at once; RejectSampling threw levels away; with several
    objects matching the target, some success faces one that is not the first find_matching_objs lists; and some
    episode picked a distractor up and put it down before succeeding."""
    want = FAMILIES[env_id]
    n, steps = 256, 500
    orc = BabyAIOracle(env_id, n)
    orc.reset(seed=123)
    rng = np.random.default_rng(9)
    carried = np.zeros(n, bool)   # this episode picked something up
    dropped = np.zeros(n, bool)   # ... and later carried nothing again
    succ = both = later_match = after_drop = 0
    for _ in range(steps):
        _, _, r, te, tr = orc.step(rng.integers(0, 7, n).astype(np.int32))
        te, tr = np.asarray(te, bool).copy(), np.asarray(tr, bool).copy()
        st = orc.get_state()
        holding = st["agent"][:, 3] != -1
        dropped |= carried & ~holding
        carried |= holding
        win = te & (np.asarray(r) > 0)
        succ += int(win.sum())
        both += int((win & tr).sum())
        after_drop += int((win & dropped).sum())
        for i in np.nonzero(win)[0]:
            x, y, d = (int(v) for v in st["agent"][i, :3])
            fx, fy = x + DXY[d][0], y + DXY[d][1]
            cell = st["grid"][i, fx, fy]
            xs, ys = np.nonzero((st["grid"][i, :, :, 0] == cell[0]) & (st["grid"][i, :, :, 1] == cell[1]))
            if len(xs) >= 2 and (int(xs[0]), int(ys[0])) != (fx, fy):  # np.nonzero: x-major, as the reference scans
                later_match += 1
        done = te | tr
        carried &= ~done
        dropped &= ~done
    assert succ > 0 and both > 0
    assert (orc.rejections() > 0) == want["rejects"]
    assert (later_match > 0) == want["multi"]
    assert (after_drop > 0) == want["distractors"]
