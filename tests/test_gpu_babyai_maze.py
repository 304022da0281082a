"""The BabyAI maze levels (GoToObjMaze*, FindObjS*, KeyCorridor*) on the GPU: K1 / K2 against the oracle
(tests/babyai_maze_oracle.py) at N = 4133 (129 full tiles and a ragged one of 5 envs), the reference's record
(tests/golden/ref_babyai_maze_traces.json) replayed on the device with its scripted rollouts, both HBM layouts with many
tiles per warp, injected GoTo and Pickup successes and a pickup while carrying, hash(), full_obs, the packed host path,
reset_mask, missions=True codes and the observation wrappers, a 22 x 22 and a 7 x 7 maze handle sharing the roomgrid K1
kernel, and BabyAI-KeyCorridorS6R3 stepped next to MiniGrid-KeyCorridorS6R3."""
import numpy as np
import pytest
import torch

import hash_support as hs
import parity
from engine_adapter import EngineAdapter
from oracle import ref_babyai_maze as rec_mod
from oracle import ref_trace as rt
from babyai_maze_oracle import A_PICKUP, MAZE_SPECS, MazeOracle, hashed
from babyai_oracle import DIR_TO_VEC
from babyai_pickup_oracle import scripted_rollout

pytestmark = pytest.mark.gpu

REC = rec_mod.load_record()
IDS = list(MAZE_SPECS)
MODES = ["next_step", "same_step"]
N = 4133


def _biased(rng, n):
    """forward half the time, pickup / toggle often: enough to cross doors and end episodes"""
    u = rng.random(n)
    return np.where(u < 0.5, 2, np.where(u < 0.65, 5, np.where(u < 0.75, A_PICKUP, rng.integers(0, 7, n)))).astype(np.int32)


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_lockstep_vs_oracle(env_id, mode):
    """obs, direction, reward bits, terminated and truncated after every step; grid, agent, RNG and pending flags
    every 40 steps and at the end (parity.check_lockstep_vs_oracle)."""
    eng = EngineAdapter(env_id, N, mode)
    orc = MazeOracle(env_id, N, autoreset=mode, n_threads=0)
    parity.check_lockstep_vs_oracle(eng, orc, 120, seed=17, check_state_every=40)


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_reference_record_replayed_on_the_device(env_id, mode):
    eng = EngineAdapter(env_id, rec_mod.N_ENVS, mode)
    got = rt.rollout(eng, rec_mod.N_ENVS, rec_mod.SEED, rec_mod.ACT_SEED, rec_mod.STEPS)
    assert got == REC["lockstep"][rt.key(env_id, mode)]


@pytest.mark.parametrize("env_id", IDS)
def test_reference_scripted_rollout_replayed_on_the_device(env_id):
    """The scripted policy's recorded actions: doors toggled on the way, targets reached, keys fetched and dropped."""
    sc = REC["scripted"][env_id]
    eng = EngineAdapter(env_id, rec_mod.SCRIPT_ENVS, "next_step")
    assert scripted_rollout(eng, rec_mod.SCRIPT_ENVS, rec_mod.SCRIPT_SEED, sc["actions"]) == sc["trace"]


@pytest.mark.parametrize("layout", ["0", "1"], ids=["tiled", "window"])
@pytest.mark.parametrize("env_id", ["BabyAI-GoToObjMazeS4-v0", "BabyAI-GoToObjMaze-v0", "BabyAI-FindObjS7-v0",
                                    "BabyAI-KeyCorridorS3R3-v0"])
@pytest.mark.parametrize("mode", MODES)
def test_both_layouts_many_tiles_per_warp(env_id, layout, mode, monkeypatch):
    """Two CTAs of three tile warps share 130 tiles while episodes end all the time."""
    monkeypatch.setenv("MINIGRID_B200_LAYOUT", layout)
    monkeypatch.setenv("MINIGRID_B200_GRID", "2")
    monkeypatch.setenv("MINIGRID_B200_CFG", "3,0,0")
    eng = EngineAdapter(env_id, N, mode)
    orc = MazeOracle(env_id, N, autoreset=mode, n_threads=0)
    parity.check_lockstep_vs_oracle(eng, orc, 150, seed=5, check_state_every=50)


def _face(grid, cell):
    """An empty cell next to `cell` and the direction that faces `cell` from it, or None."""
    W, H = grid.shape[:2]
    for d, (dx, dy) in enumerate(DIR_TO_VEC):
        ax, ay = cell[0] - dx, cell[1] - dy
        if 0 < ax < W - 1 and 0 < ay < H - 1 and grid[ax, ay, 0] == 1:
            return (ax, ay), d
    return None


@pytest.mark.parametrize("layout", ["0", "1"], ids=["tiled", "window"])
@pytest.mark.parametrize("env_id,case", [("BabyAI-GoToObjMaze-v0", "goto"), ("BabyAI-GoToObjMazeOpen-v0", "goto"),
                                         ("BabyAI-GoToObjMazeS4R2-v0", "goto"), ("BabyAI-FindObjS5-v0", "pickup"),
                                         ("BabyAI-KeyCorridorS4R3-v0", "pickup"), ("BabyAI-KeyCorridorS4R3-v0", "carrying")])
def test_injected_successes(env_id, case, layout, monkeypatch):
    """The agent put next to the target: a left turn that faces it (GoTo: success on that step), a pickup facing it
    (success), or, on KeyCorridor, a pickup facing the ball while carrying the key (nothing: the ball stays, no reward)."""
    monkeypatch.setenv("MINIGRID_B200_LAYOUT", layout)
    n = 1000
    eng = EngineAdapter(env_id, n, "disabled")
    orc = MazeOracle(env_id, n, autoreset="disabled")
    eng.reset(seed=77)
    orc.reset(seed=77)
    grid = orc.get_state()["grid"]
    acts = np.full(n, 6, np.int32)
    planned = np.zeros(n, bool)
    for i in range(n):
        lv = orc.levels[i]
        tgt = lv.obj_set[0].cur_pos
        f = _face(grid[i], tgt)
        if f is None:
            continue
        if case == "carrying":
            key = next(p for p, o in lv.world.items() if o.type == "key")
            orc.inject(i, pos=f[0], d=f[1], carry=key)
        elif case == "goto":  # one turn right of facing it: the left turn faces the target
            orc.inject(i, pos=f[0], d=(f[1] + 1) % 4)
        else:
            orc.inject(i, pos=f[0], d=f[1])
        acts[i], planned[i] = (0 if case == "goto" else A_PICKUP), True
    st = orc.get_state()
    eng.set_state(grid=st["grid"], agent=st["agent"])
    assert planned.sum() > 300
    e, o = eng.step(acts), orc.step(acts)
    np.testing.assert_array_equal(e[0], o[0])
    assert np.asarray(e[2], np.float64).tobytes() == o[2].tobytes()
    np.testing.assert_array_equal(e[3], o[3])
    for key in ("grid", "agent"):
        np.testing.assert_array_equal(eng.get_state()[key], orc.get_state()[key])
    r, te = o[2], o[3]
    if case == "carrying":
        assert not te[planned].any() and not r[planned].any()
        assert orc.events["pickup_while_carrying"] >= planned.sum()
    else:
        assert te[planned].all() and (r[planned] > 0).all()


@pytest.mark.parametrize("env_id", IDS)
def test_hash_reproduces_reference_record(env_id):
    from minigrid_b200 import MinigridVecEnv

    for mode in MODES:
        assert hs.hash_rollout(MinigridVecEnv(env_id, 6, autoreset_mode=mode), 6) == REC["hash_rollout"][rt.key(env_id, mode)]
    assert hs.hash_walk(MinigridVecEnv(env_id, 6), 6) == REC["hash_walk"][env_id]


@pytest.mark.parametrize("env_id", ["BabyAI-GoToObjMaze-v0", "BabyAI-GoToObjMazeS4R2-v0", "BabyAI-FindObjS6-v0"])
def test_hash_and_full_obs_vs_oracle(env_id):
    from minigrid_b200 import MinigridVecEnv

    env, orc = MinigridVecEnv(env_id, N), hashed(env_id, N)
    env.reset(seed=21)
    orc.reset(seed=21)
    rng = np.random.default_rng(8)
    for _ in range(10):
        a = _biased(rng, N)
        env.step(torch.as_tensor(a, device=env.device))
        orc.step(a)
    assert env.hash(64) == orc.hash(64)
    eng, o2 = EngineAdapter(env_id, 1000, "next_step"), MazeOracle(env_id, 1000)
    parity.check_lockstep_vs_oracle(eng, o2, 20, seed=4)
    np.testing.assert_array_equal(eng.full_obs(), o2.full_obs())


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("env_id", ["BabyAI-GoToObjMazeOpen-v0", "BabyAI-KeyCorridor-v0"])
def test_packed_host_path(env_id, mode):
    n = 1000 + 13
    eng = EngineAdapter(env_id, n, mode, host=True, host_format="packed", host_threads=2)
    orc = MazeOracle(env_id, n, autoreset=mode, n_threads=0)
    parity.check_lockstep_vs_oracle(eng, orc, 150, seed=21)


@pytest.mark.parametrize("env_id", ["BabyAI-GoToObjMazeS4-v0", "BabyAI-FindObjS5-v0"])
def test_partial_reset_mask(env_id):
    n = 1000
    eng = EngineAdapter(env_id, n, "next_step")
    orc = MazeOracle(env_id, n, autoreset="next_step")
    parity.check_lockstep_vs_oracle(eng, orc, 30, seed=3)
    rng = np.random.default_rng(8)
    for seed in (None, 5000, rng.integers(0, 2**62, n).astype(np.uint64)):
        mask = rng.random(n) < 0.3
        eo, ed = eng.reset(seed=seed, mask=mask)
        oo, od = orc.reset(seed=seed, mask=mask)
        np.testing.assert_array_equal(eo, oo)
        np.testing.assert_array_equal(ed, od)
        for t in range(25):
            a = _biased(rng, n)
            e, o = eng.step(a), orc.step(a)
            np.testing.assert_array_equal(e[0], o[0], err_msg=f"obs t={t}")
            assert e[2].tobytes() == o[2].tobytes()
            np.testing.assert_array_equal(e[3], o[3], err_msg=f"terminated t={t}")
        es, os_ = eng.get_state(), orc.get_state()
        for k in ("grid", "agent", "rng", "pending"):
            np.testing.assert_array_equal(es[k], os_[k], err_msg=k)


def _codes(env):
    return env.mission_codes.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_mission_codes_follow_the_oracle(env_id, mode):
    """missions=True: the codes after every step against the oracle's, the strings every 20 steps, the outputs
    bit-identical to a missions=False handle; the recorded missions after seeded resets."""
    import minigrid_b200 as mb

    n = 1000
    on, off = mb.MinigridVecEnv(env_id, n, autoreset_mode=mode, missions=True), mb.MinigridVecEnv(env_id, n, autoreset_mode=mode)
    orc = MazeOracle(env_id, n, autoreset=mode, n_threads=0)
    on.reset(seed=5)
    off.reset(seed=5)
    orc.reset(seed=5)
    np.testing.assert_array_equal(_codes(on), orc.mission_codes())
    rng = np.random.default_rng(6)
    for t in range(60):
        a = _biased(rng, n)
        r1, r2 = on.step(torch.as_tensor(a, device="cuda")), off.step(torch.as_tensor(a, device="cuda"))
        orc.step(a)
        for x, y in zip(r1[:4], r2[:4]):
            x, y = (x["image"], y["image"]) if isinstance(x, dict) else (x, y)
            assert x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes(), t
        np.testing.assert_array_equal(_codes(on), orc.mission_codes(), err_msg=f"t={t}")
        if t % 20 == 19:
            assert on.missions() == orc.missions(), t
    m = mb.MinigridVecEnv(env_id, len(rec_mod.MISSION_SEEDS), missions=True)
    m.reset(seed=[int(s) for s in rec_mod.MISSION_SEEDS])
    assert m.missions() == REC["missions"][env_id]


@pytest.mark.parametrize("env_id", IDS)
def test_dict_and_flat_wrappers_accept_the_maze_missions(env_id):
    import minigrid_b200 as mb
    from minigrid_b200.wrappers import mission_to_indices

    n = len(rec_mod.MISSION_SEEDS)
    env = mb.MinigridVecEnv(env_id, n, missions=True)
    obs, _ = mb.DictObservationSpaceWrapper(env).reset(seed=[int(s) for s in rec_mod.MISSION_SEEDS])
    want = [mission_to_indices(m) for m in REC["missions"][env_id]]
    got = obs["mission"].cpu().tolist()
    assert [row[:len(w)] for row, w in zip(got, want)] == want
    flat = mb.FlatObsWrapper(mb.MinigridVecEnv(env_id, 4, missions=True))
    assert flat.observation(flat.env.reset(seed=0)[0]).shape[0] == 4


@pytest.mark.parametrize("big_first", [True, False], ids=["big_first", "small_first"])
def test_22x22_and_7x7_maze_handles_share_the_roomgrid_kernel(big_first):
    big, small, n = "BabyAI-GoToObjMaze-v0", "BabyAI-GoToObjMazeS4R2-v0", 2085
    order = [big, small] if big_first else [small, big]
    pairs = [(EngineAdapter(e, n, "next_step"), MazeOracle(e, n, n_threads=0)) for e in order]
    for k, (eng, orc) in enumerate(pairs):
        eo, _ = eng.reset(seed=10 + k)
        oo, _ = orc.reset(seed=10 + k)
        np.testing.assert_array_equal(eo, oo)
    rng = np.random.default_rng(3)
    for t in range(60):
        for name, (eng, orc) in zip(order, pairs):
            a = _biased(rng, n)
            e, o = eng.step(a), orc.step(a)
            np.testing.assert_array_equal(e[0], o[0], err_msg=f"{name} obs t={t}")
            assert np.asarray(e[2], np.float64).tobytes() == o[2].tobytes(), f"{name} reward t={t}"
            np.testing.assert_array_equal(e[3], o[3], err_msg=f"{name} terminated t={t}")
    for eng, orc in pairs:
        for key in ("grid", "agent", "rng", "pending"):
            np.testing.assert_array_equal(eng.get_state()[key], orc.get_state()[key], err_msg=key)


@pytest.mark.parametrize("mode", MODES)
def test_babyai_keycorridor_steps_like_minigrid_keycorridor(mode):
    """Same seeds and actions: identical obs, reward, terminated and truncated after every step and the same hash every
    100 steps, past the 1080-step limit so that every env autoresets at least once."""
    from minigrid_b200 import MinigridVecEnv

    n = 4133
    b = MinigridVecEnv("BabyAI-KeyCorridorS6R3-v0", n, autoreset_mode=mode)
    m = MinigridVecEnv("MiniGrid-KeyCorridorS6R3-v0", n, autoreset_mode=mode)
    ob, _ = b.reset(seed=11)
    om, _ = m.reset(seed=11)
    assert torch.equal(ob["image"], om["image"])
    rng = np.random.default_rng(12)
    ends = 0
    for t in range(1100):
        a = torch.as_tensor(_biased(rng, n), device="cuda")
        rb, rm = b.step(a), m.step(a)
        assert torch.equal(rb[0]["image"], rm[0]["image"]), t
        for x, y in zip(rb[1:4], rm[1:4]):
            assert torch.equal(x, y), t
        ends += int((rb[2] | rb[3]).sum())
        if t % 100 == 99:
            assert b.hash(64) == m.hash(64), t
    assert ends >= n
