"""The BabyAI Open and UnlockLocal levels on the GPU: K1 / K2 against the oracle (tests/babyai_open_oracle.py) at
N = 4133 (129 full tiles and a ragged one of 5 envs), the reference's record (tests/golden/ref_babyai_open_traces.json)
replayed on the device with its scripted rollouts, both HBM layouts with many tiles per warp, injected states (a target
door opened or closed again, a wrong door with and without strict, a locked door with and without its key, two-step
BeforeInstr / AfterInstr sequences played through, the second door first, the Debug failure on the first correct open),
hash(), the packed host path, reset_mask, the observation wrappers, and a 22 x 22 Open handle sharing the roomgrid K1
kernel with a smaller roomgrid handle."""
import numpy as np
import pytest
import torch

import hash_support as hs
import parity
from engine_adapter import EngineAdapter
from oracle import ref_babyai
from oracle import ref_babyai_open as rec_mod
from oracle import ref_trace as rt
from oracle.oracle import OracleVecEnv
from babyai_oracle import DIR_TO_VEC
from babyai_open_oracle import A_PICKUP, A_TOGGLE, OPEN_SPECS, OpenOracle, hashed, ordered, scripted_rollout

pytestmark = pytest.mark.gpu

REC = rec_mod.load_record()
IDS = list(OPEN_SPECS)
MODES = ["next_step", "same_step"]
N = 4133


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_lockstep_vs_oracle(env_id, mode):
    """obs, direction, reward bits, terminated and truncated after every step; grid, agent, RNG and pending flags
    every 40 steps and at the end (parity.check_lockstep_vs_oracle)."""
    eng = EngineAdapter(env_id, N, mode)
    orc = OpenOracle(env_id, N, autoreset=mode, n_threads=0)
    parity.check_lockstep_vs_oracle(eng, orc, 120, seed=17, check_state_every=40)
    assert orc.events["success"] > 0


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_reference_record_replayed_on_the_device(env_id, mode):
    eng = EngineAdapter(env_id, rec_mod.N_ENVS, mode)
    got = rt.rollout(eng, rec_mod.N_ENVS, rec_mod.SEED, rec_mod.ACT_SEED, rec_mod.STEPS)
    assert got == REC["lockstep"][rt.key(env_id, mode)]


@pytest.mark.parametrize("env_id", IDS)
def test_reference_scripted_rollout_replayed_on_the_device(env_id):
    """The scripted policy's recorded actions: successes, strict failures, sequences in and out of order, keys fetched."""
    sc = REC["scripted"][env_id]
    eng = EngineAdapter(env_id, rec_mod.SCRIPT_ENVS, "next_step")
    assert scripted_rollout(eng, rec_mod.SCRIPT_ENVS, rec_mod.SCRIPT_SEED, sc["actions"]) == sc["trace"]


@pytest.mark.parametrize("layout", ["0", "1"], ids=["tiled", "window"])
@pytest.mark.parametrize("env_id", ["BabyAI-OpenDoorsOrderN4Debug-v0", "BabyAI-UnlockLocalDist-v0"])
@pytest.mark.parametrize("mode", MODES)
def test_both_layouts_many_tiles_per_warp(env_id, layout, mode, monkeypatch):
    """Two CTAs of three tile warps share 130 tiles while episodes end all the time."""
    monkeypatch.setenv("MINIGRID_B200_LAYOUT", layout)
    monkeypatch.setenv("MINIGRID_B200_GRID", "2")
    monkeypatch.setenv("MINIGRID_B200_CFG", "3,0,0")
    eng = EngineAdapter(env_id, N, mode)
    orc = OpenOracle(env_id, N, autoreset=mode, n_threads=0)
    parity.check_lockstep_vs_oracle(eng, orc, 150, seed=5, check_state_every=50)


def _face(grid, cell):
    """An empty cell next to `cell` and the direction that faces `cell` from it, or None."""
    W, H = grid.shape[:2]
    for d, (dx, dy) in enumerate(DIR_TO_VEC):
        ax, ay = cell[0] - dx, cell[1] - dy
        if 0 < ax < W - 1 and 0 < ay < H - 1 and grid[ax, ay, 0] == 1:
            return (ax, ay), d
    return None


def _inject_and_step(env_id, layout, plan, monkeypatch, rounds=1, n=1000):
    """Resets the engine and the oracle alike; each round, plan(orc, i, grid, round) injects env i's state on the oracle
    and returns its action (or None: the env takes 'done', which does nothing here), the oracle's grid and agent records
    are copied into the engine (mg_set_state keeps the level's targets and the progress bit), both step once and every
    output is compared. Returns [(reward, terminated, planned)] per round."""
    monkeypatch.setenv("MINIGRID_B200_LAYOUT", layout)
    eng = EngineAdapter(env_id, n, "disabled")
    orc = OpenOracle(env_id, n, autoreset="disabled")
    eng.reset(seed=77)
    orc.reset(seed=77)
    out = []
    for k in range(rounds):
        acts = np.full(n, 6, np.int32)
        planned = np.zeros(n, bool)
        grid = orc.get_state()["grid"]
        for i in range(n):
            a = plan(orc, i, grid[i], k)
            if a is not None:
                acts[i], planned[i] = a, True
        st = orc.get_state()
        eng.set_state(grid=st["grid"], agent=st["agent"])
        e, o = eng.step(acts), orc.step(acts)
        np.testing.assert_array_equal(e[0], o[0])
        assert e[2].astype(np.float64).tobytes() == o[2].tobytes()
        np.testing.assert_array_equal(e[3], o[3])
        np.testing.assert_array_equal(e[4], o[4])
        for key in ("grid", "agent"):
            np.testing.assert_array_equal(eng.get_state()[key], orc.get_state()[key])
        out.append((o[2], o[3], planned))
    return out


LAYOUTS = pytest.mark.parametrize("layout", ["0", "1"], ids=["tiled", "window"])


def _toggle_at(orc, i, grid, door, state=None):
    """Env i's agent put in front of `door` (a cell), the door first set to `state` if given; returns toggle or None."""
    f = _face(grid, door)
    if f is None:
        return None
    orc.inject(i, pos=f[0], d=f[1], door_states=None if state is None else {door: state})
    return A_TOGGLE


@LAYOUTS
@pytest.mark.parametrize("env_id,case", [(e, c) for e in ["BabyAI-OpenRedDoor-v0", "BabyAI-OpenDoorColor-v0",
                                                          "BabyAI-OpenDoorLoc-v0", "BabyAI-OpenDoorDebug-v0",
                                                          "BabyAI-OpenDoorsOrderN4-v0"]
                                         for c in ("open", "close", "wrong") if (e, c) != ("BabyAI-OpenRedDoor-v0", "wrong")])
def test_injected_single_door(env_id, case, layout, monkeypatch):
    """A door of the first instruction's obj_set toggled open (success) or, injected open, toggled closed (nothing, or
    failure when strict), or a door outside obj_set toggled (nothing, or failure when strict)."""
    def plan(orc, i, grid, k):
        lv = orc.levels[i]
        first, second = ordered(lv.instrs)
        if case == "wrong":
            names = {id(d) for ins in (first, second) if ins for d in ins.desc.obj_set}
            others = [c for c, d in lv.doors.items() if id(d) not in names]
            return _toggle_at(orc, i, grid, others[0]) if others else None
        return _toggle_at(orc, i, grid, first.desc.obj_set[0].cur_pos, 0 if case == "close" else None)
    (r, te, planned), = _inject_and_step(env_id, layout, plan, monkeypatch)
    assert planned.sum() > 300
    strict = OPEN_SPECS[env_id][5][6]
    if case == "open":
        assert te[planned].any() and (r[planned & te] > 0).all()
        if env_id != "BabyAI-OpenDoorsOrderN4-v0":  # one instruction: every open succeeds
            assert te[planned].all() and (r[planned] > 0).all()
    else:
        assert (te[planned] == bool(strict)).all() and not r[planned].any()


@LAYOUTS
@pytest.mark.parametrize("env_id", ["BabyAI-UnlockLocal-v0", "BabyAI-UnlockLocalDist-v0"])
@pytest.mark.parametrize("key", [True, False], ids=["key", "no_key"])
def test_injected_locked_door(env_id, key, layout, monkeypatch):
    """UnlockLocal's locked door toggled with its key in hand (it opens: success) or without (nothing)."""
    def plan(orc, i, grid, k):
        lv = orc.levels[i]
        (cell, door), = lv.doors.items()
        f = _face(grid, cell)
        if f is None:
            return None
        orc.inject(i, pos=f[0], d=f[1], carry=door.color if key else None)
        return A_TOGGLE
    (r, te, planned), = _inject_and_step(env_id, layout, plan, monkeypatch)
    assert planned.sum() > 500
    assert (te[planned] == key).all() and ((r[planned] > 0) == key).all()


@LAYOUTS
@pytest.mark.parametrize("env_id", ["BabyAI-OpenTwoDoors-v0", "BabyAI-OpenRedBlueDoorsDebug-v0",
                                    "BabyAI-OpenDoorsOrderN4-v0", "BabyAI-OpenDoorsOrderN2Debug-v0"])
@pytest.mark.parametrize("order", ["in_order", "second_first"])
def test_injected_sequences(env_id, order, layout, monkeypatch):
    """BeforeInstr / AfterInstr played through by injection: the agent put in front of the first door, toggle, then in
    front of the second, toggle (in_order); or the second door first, then the first, then the second again (it closes),
    then once more (it opens). The device's progress bit must carry the sequence from one step to the next, and the Debug
    levels fail on the first correct open (the reference re-verifies the strict second instruction on that toggle)."""
    seqs = set()

    def plan(orc, i, grid, k):
        lv = orc.levels[i]
        first, second = ordered(lv.instrs)
        if second is None or (k > 0 and i not in seqs):
            return None
        d1, d2 = first.desc.obj_set[0].cur_pos, second.desc.obj_set[0].cur_pos
        steps = [d1, d2] if order == "in_order" else [d2, d1, d2, d2]
        a = _toggle_at(orc, i, grid, steps[k])
        if a is None:
            seqs.discard(i)
        elif k == 0:
            seqs.add(i)
        return a
    rounds = 2 if order == "in_order" else 4
    res = _inject_and_step(env_id, layout, plan, monkeypatch, rounds=rounds)
    planned = np.zeros(len(res[0][2]), bool)
    planned[sorted(seqs)] = True  # every round's toggle was injected
    assert planned.sum() > 100
    strict_first = env_id.endswith("Debug-v0")
    strict_second = env_id.endswith("N2Debug-v0")
    (r0, te0, _) = res[0]
    if order == "in_order":
        if strict_second:  # the first correct open re-verifies the strict second instruction: failure
            assert te0[planned].all() and not r0[planned].any()
        else:
            assert not te0[planned].any()
            assert res[1][1][planned].all() and (res[1][0][planned] > 0).all()
    elif strict_first:  # the second door first: a strict first instruction fails
        assert te0[planned].all() and not r0[planned].any()
    else:  # nothing until the second door, closed by the third toggle, is opened again
        assert not any(res[k][1][planned].any() for k in range(3))
        assert res[3][1][planned].all() and (res[3][0][planned] > 0).all()


@pytest.mark.parametrize("env_id", IDS)
def test_hash_reproduces_reference_record(env_id):
    from minigrid_b200 import MinigridVecEnv

    for mode in MODES:
        assert hs.hash_rollout(MinigridVecEnv(env_id, 6, autoreset_mode=mode), 6) == REC["hash_rollout"][rt.key(env_id, mode)]
    assert hs.hash_walk(MinigridVecEnv(env_id, 6), 6) == REC["hash_walk"][env_id]


@pytest.mark.parametrize("env_id", ["BabyAI-OpenRedDoor-v0", "BabyAI-OpenTwoDoors-v0", "BabyAI-UnlockLocalDist-v0"])
def test_hash_vs_oracle(env_id):
    """9 x 5, 16 x 16 and 22 x 22 are geometries K4 meets first here."""
    from minigrid_b200 import MinigridVecEnv

    env, orc = MinigridVecEnv(env_id, N), hashed(env_id, N)
    env.reset(seed=21)
    orc.reset(seed=21)
    rng = np.random.default_rng(8)
    for _ in range(10):
        a = np.where(rng.random(N) < 0.5, 2, rng.integers(0, 7, N)).astype(np.int32)
        env.step(torch.as_tensor(a, device=env.device))
        orc.step(a)
    assert env.hash(64) == orc.hash(64)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("env_id", ["BabyAI-OpenDoorsOrderN2-v0", "BabyAI-UnlockLocal-v0"])
def test_packed_host_path(env_id, mode):
    n = 1000 + 13
    eng = EngineAdapter(env_id, n, mode, host=True, host_format="packed", host_threads=2)
    orc = OpenOracle(env_id, n, autoreset=mode, n_threads=0)
    parity.check_lockstep_vs_oracle(eng, orc, 150, seed=21)


@pytest.mark.parametrize("env_id", ["BabyAI-OpenTwoDoors-v0", "BabyAI-OpenDoorDebug-v0"])
def test_partial_reset_mask(env_id):
    n = 1000
    eng = EngineAdapter(env_id, n, "next_step")
    orc = OpenOracle(env_id, n, autoreset="next_step")
    parity.check_lockstep_vs_oracle(eng, orc, 30, seed=3)
    rng = np.random.default_rng(8)
    for seed in (None, 5000, rng.integers(0, 2**62, n).astype(np.uint64)):
        mask = rng.random(n) < 0.3
        eo, ed = eng.reset(seed=seed, mask=mask)
        oo, od = orc.reset(seed=seed, mask=mask)
        np.testing.assert_array_equal(eo, oo)
        np.testing.assert_array_equal(ed, od)
        for t in range(25):
            a = np.where(rng.random(n) < 0.5, A_TOGGLE, rng.integers(0, 7, n)).astype(np.int32)
            e, o = eng.step(a), orc.step(a)
            np.testing.assert_array_equal(e[0], o[0], err_msg=f"obs t={t}")
            assert e[2].tobytes() == o[2].tobytes()
            np.testing.assert_array_equal(e[3], o[3], err_msg=f"terminated t={t}")
        es, os_ = eng.get_state(), orc.get_state()
        for k in ("grid", "agent", "rng", "pending"):
            np.testing.assert_array_equal(es[k], os_[k], err_msg=k)


@pytest.mark.parametrize("env_id", rec_mod.OBS_WRAPPER_IDS)
def test_observation_wrappers_reproduce_reference_record(env_id):
    """FullyObsWrapper, RGBImgPartialObsWrapper, RGBImgObsWrapper and, on the constant missions, FlatObsWrapper."""
    import minigrid_b200 as mb

    flat = env_id in rec_mod.CONSTANT_MISSION_IDS

    class Side:
        def __init__(self):
            self.env = mb.MinigridVecEnv(env_id, rec_mod.N_ENVS)
            self.obs = None

        def reset(self, seed):
            self.obs, _ = self.env.reset(seed=seed)

        def step(self, a):
            self.obs = self.env.step(torch.as_tensor(np.asarray(a, np.int32), device=self.env.device))[0]

    def views(s):
        out = [mb.FullyObsWrapper(s.env).observation(s.obs)["image"].cpu().numpy(),
               mb.RGBImgPartialObsWrapper(s.env).observation(s.obs)["image"].cpu().numpy(),
               mb.RGBImgObsWrapper(s.env).observation(s.obs)["image"].cpu().numpy()]
        return out + ([mb.FlatObsWrapper(s.env).observation(s.obs).cpu().numpy().astype(np.float32)] if flat else [])

    assert ref_babyai.observation_wrappers(Side(), rec_mod.N_ENVS, views) == REC["obs_wrappers"][env_id]


def test_dict_wrapper_and_mission_refusals():
    import minigrid_b200 as mb

    for env_id in IDS:
        env = mb.MinigridVecEnv(env_id, 4)
        if env_id in rec_mod.CONSTANT_MISSION_IDS:
            obs, _ = mb.DictObservationSpaceWrapper(env).reset(seed=0)
            assert obs["mission"] == REC["dict_missions"][env_id]
        else:
            with pytest.raises(ValueError):
                mb.DictObservationSpaceWrapper(env)
            with pytest.raises(ValueError):
                mb.FlatObsWrapper(env)


@pytest.mark.parametrize("small", ["MiniGrid-KeyCorridorS3R1-v0", "BabyAI-OneRoomS8-v0"])
@pytest.mark.parametrize("open_first", [True, False], ids=["open_first", "small_first"])
def test_22x22_handle_shares_the_roomgrid_kernel(small, open_first):
    """22 x 22 is the largest roomgrid geometry; a smaller roomgrid handle created before or after it must not lower
    the shared K1 kernel's shared-memory limit below the larger plan. Both are stepped interleaved against oracles."""
    from babyai_pickup_oracle import PickupOracle

    big = "BabyAI-UnlockLocalDist-v0"
    n = 2085
    mk_orc = {big: lambda: OpenOracle(big, n, n_threads=0),
              "MiniGrid-KeyCorridorS3R1-v0": lambda: OracleVecEnv("MiniGrid-KeyCorridorS3R1-v0", n),
              "BabyAI-OneRoomS8-v0": lambda: PickupOracle("BabyAI-OneRoomS8-v0", n, n_threads=0)}
    order = [big, small] if open_first else [small, big]
    pairs = [(EngineAdapter(e, n, "next_step"), mk_orc[e]()) for e in order]
    for k, (eng, orc) in enumerate(pairs):
        eo, _ = eng.reset(seed=10 + k)
        oo, _ = orc.reset(seed=10 + k)
        np.testing.assert_array_equal(eo, oo)
    rng = np.random.default_rng(3)
    for t in range(60):
        for name, (eng, orc) in zip(order, pairs):
            a = np.where(rng.random(n) < 0.4, A_TOGGLE if name == big else A_PICKUP, rng.integers(0, 7, n)).astype(np.int32)
            e, o = eng.step(a), orc.step(a)
            np.testing.assert_array_equal(e[0], o[0], err_msg=f"{name} obs t={t}")
            assert np.asarray(e[2], np.float64).tobytes() == o[2].tobytes(), f"{name} reward t={t}"
            np.testing.assert_array_equal(e[3], o[3], err_msg=f"{name} terminated t={t}")
            np.testing.assert_array_equal(e[4], o[4], err_msg=f"{name} truncated t={t}")
    for eng, orc in pairs:
        for key in ("grid", "agent", "rng", "pending"):
            np.testing.assert_array_equal(eng.get_state()[key], orc.get_state()[key], err_msg=key)
