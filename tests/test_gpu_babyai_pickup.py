"""The single-room BabyAI Pickup and PutNext levels on the GPU: K1 / K2 against the oracle (tests/babyai_pickup_oracle.py)
at N = 4133 (129 full tiles and a ragged one of 5 envs), the reference's record (tests/golden/ref_babyai_pickup_traces.json)
replayed on the device with its scripted rollouts, both HBM layouts with many tiles per warp, injected states that end
in a success, a diagonal near-miss or a strict failure, hash(), the packed host path, reset_mask and the observation
wrappers."""
import numpy as np
import pytest
import torch

import hash_support as hs
import parity
from engine_adapter import EngineAdapter
from oracle import ref_babyai
from oracle import ref_babyai_pickup as rec_mod
from oracle import ref_trace as rt
from babyai_oracle import DIR_TO_VEC
from babyai_pickup_oracle import A_DROP, A_PICKUP, PICKUP_SPECS, PickupOracle, hashed, scripted_rollout

pytestmark = pytest.mark.gpu

REC = rec_mod.load_record()
IDS = list(PICKUP_SPECS)
MODES = ["next_step", "same_step"]
N = 4133


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_lockstep_vs_oracle(env_id, mode):
    """obs, direction, reward bits, terminated and truncated after every step; grid, agent, RNG and pending flags
    every 40 steps and at the end (parity.check_lockstep_vs_oracle)."""
    eng = EngineAdapter(env_id, N, mode)
    orc = PickupOracle(env_id, N, autoreset=mode, n_threads=0)
    parity.check_lockstep_vs_oracle(eng, orc, 120, seed=17, check_state_every=40)


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_reference_record_replayed_on_the_device(env_id, mode):
    eng = EngineAdapter(env_id, rec_mod.N_ENVS, mode)
    got = rt.rollout(eng, rec_mod.N_ENVS, rec_mod.SEED, rec_mod.ACT_SEED, rec_mod.STEPS)
    assert got == REC["lockstep"][rt.key(env_id, mode)]


@pytest.mark.parametrize("env_id", IDS)
def test_reference_scripted_rollout_replayed_on_the_device(env_id):
    """The scripted policy's recorded actions: successes, and on PutNext a fixed object moved before the success."""
    sc = REC["scripted"][env_id]
    eng = EngineAdapter(env_id, rec_mod.N_ENVS, "next_step")
    assert scripted_rollout(eng, rec_mod.N_ENVS, rec_mod.SCRIPT_SEED, sc["actions"]) == sc["trace"]


@pytest.mark.parametrize("layout", ["0", "1"], ids=["tiled", "window"])
@pytest.mark.parametrize("env_id", ["BabyAI-PutNextLocal-v0", "BabyAI-OneRoomS12-v0"])
@pytest.mark.parametrize("mode", MODES)
def test_both_layouts_many_tiles_per_warp(env_id, layout, mode, monkeypatch):
    """Two CTAs of three tile warps share 130 tiles while episodes end all the time."""
    monkeypatch.setenv("MINIGRID_B200_LAYOUT", layout)
    monkeypatch.setenv("MINIGRID_B200_GRID", "2")
    monkeypatch.setenv("MINIGRID_B200_CFG", "3,0,0")
    eng = EngineAdapter(env_id, N, mode)
    orc = PickupOracle(env_id, N, autoreset=mode, n_threads=0)
    parity.check_lockstep_vs_oracle(eng, orc, 150, seed=5, check_state_every=50)


def _face(grid, cell):
    """An empty interior cell next to `cell` and the direction that faces `cell` from it, or None."""
    W, H = grid.shape[:2]
    for d, (dx, dy) in enumerate(DIR_TO_VEC):
        ax, ay = cell[0] - dx, cell[1] - dy
        if 0 < ax < W - 1 and 0 < ay < H - 1 and grid[ax, ay, 0] == 1:
            return (ax, ay), d
    return None


def _inject_and_step(env_id, layout, plan, monkeypatch, n=1000):
    """Resets the engine and the oracle alike, lets plan(orc, i, grid) inject env i's state on the oracle and return its
    action (or None: the env takes 'done', which does nothing here), copies the oracle's grid and agent records into
    the engine (mg_set_state keeps the drawn targets), steps both once and compares every output. Returns (reward,
    terminated, planned)."""
    monkeypatch.setenv("MINIGRID_B200_LAYOUT", layout)
    eng = EngineAdapter(env_id, n, "next_step")
    orc = PickupOracle(env_id, n)
    eng.reset(seed=77)
    orc.reset(seed=77)
    acts = np.full(n, 6, np.int32)
    planned = np.zeros(n, bool)
    grid = orc.get_state()["grid"]  # env i's cells change only through its own injection
    for i in range(n):
        a = plan(orc, i, grid[i])
        if a is not None:
            acts[i], planned[i] = a, True
    st = orc.get_state()
    eng.set_state(grid=st["grid"], agent=st["agent"])
    e, o = eng.step(acts), orc.step(acts)
    np.testing.assert_array_equal(e[0], o[0])
    assert e[2].astype(np.float64).tobytes() == o[2].tobytes()
    np.testing.assert_array_equal(e[3], o[3])
    np.testing.assert_array_equal(e[4], o[4])
    for k in ("grid", "agent"):
        np.testing.assert_array_equal(eng.get_state()[k], orc.get_state()[k])
    return o[2], o[3], planned


LAYOUTS = pytest.mark.parametrize("layout", ["0", "1"], ids=["tiled", "window"])


@LAYOUTS
@pytest.mark.parametrize("env_id", ["BabyAI-OneRoomS8-v0", "BabyAI-OneRoomS20-v0", "BabyAI-PickupDist-v0",
                                    "BabyAI-PickupDistDebug-v0"])
def test_injected_pickups(env_id, layout, monkeypatch):
    """The agent put in front of an object: the target (even envs) or one that does not match (odd envs, PickupDist),
    then pickup: success, nothing (non-strict) or failure (strict)."""
    def plan(orc, i, grid):
        lv = orc.levels[i]
        others = [o for o in lv.world.values() if not any(o is t for t in lv.obj_set)]
        pick = lv.obj_set[0] if i % 2 == 0 or not others else others[0]
        f = _face(grid, pick.cur_pos)
        if f is None:
            return None
        orc.inject(i, pos=f[0], d=f[1])
        return A_PICKUP
    r, te, planned = _inject_and_step(env_id, layout, plan, monkeypatch)
    even = (np.arange(len(r)) % 2 == 0) & planned
    assert even.sum() > 100 and te[even].all() and (r[even] > 0).all()
    odd = (np.arange(len(r)) % 2 == 1) & planned
    if env_id.startswith("BabyAI-PickupDist"):
        strict = env_id.endswith("Debug-v0")
        mismatched = odd & ~(r > 0)
        assert mismatched.sum() > 100 and (te[mismatched] == strict).all()


@LAYOUTS
@pytest.mark.parametrize("target", [True, False], ids=["target", "other"])
def test_injected_strict_pickup_while_carrying(target, layout, monkeypatch):
    """PickupDistDebug with the target (or another object) injected into the agent's hands: pickup fails."""
    def plan(orc, i, grid):
        lv = orc.levels[i]
        others = [o for o in lv.world.values() if not any(o is t for t in lv.obj_set)]
        if not target and not others:
            return None
        orc.inject(i, carry=(lv.obj_set[0] if target else others[0]).cur_pos)
        return A_PICKUP
    r, te, planned = _inject_and_step("BabyAI-PickupDistDebug-v0", layout, plan, monkeypatch)
    assert planned.sum() > 500 and te[planned].all() and not r[planned].any()


@LAYOUTS
@pytest.mark.parametrize("env_id", ["BabyAI-PutNextLocal-v0", "BabyAI-PutNextLocalS5N3-v0"])
@pytest.mark.parametrize("where", ["next", "diagonal"])
def test_injected_putnext_drops(env_id, where, layout, monkeypatch):
    """The agent carrying the move object, facing an empty cell next to the fixed object (success) or diagonal to it
    (nothing), then drop."""
    def plan(orc, i, grid):
        lv = orc.levels[i]
        fx, fy = lv.fixed_set[0].cur_pos
        offs = [(1, 0), (-1, 0), (0, 1), (0, -1)] if where == "next" else [(1, 1), (-1, 1), (1, -1), (-1, -1)]
        mv = lv.move_set[0].cur_pos
        g = grid.copy()
        g[mv] = (1, 0, 0)  # the move object leaves its cell
        for dx, dy in offs:
            c = (fx + dx, fy + dy)
            if not (0 < c[0] < g.shape[0] - 1 and 0 < c[1] < g.shape[1] - 1) or g[c][0] != 1:
                continue
            f = _face(g, c)
            if f is not None:
                orc.inject(i, carry=mv)
                orc.inject(i, pos=f[0], d=f[1])
                return A_DROP
        return None
    r, te, planned = _inject_and_step(env_id, layout, plan, monkeypatch)
    assert planned.sum() > 300
    if where == "next":
        assert te[planned].all() and (r[planned] > 0).all()
    else:
        assert not te[planned].any()


@pytest.mark.parametrize("env_id", IDS)
def test_hash_reproduces_reference_record(env_id):
    from minigrid_b200 import MinigridVecEnv

    for mode in MODES:
        assert hs.hash_rollout(MinigridVecEnv(env_id, 6, autoreset_mode=mode), 6) == REC["hash_rollout"][rt.key(env_id, mode)]
    assert hs.hash_walk(MinigridVecEnv(env_id, 6), 6) == REC["hash_walk"][env_id]


@pytest.mark.parametrize("env_id", ["BabyAI-OneRoomS12-v0", "BabyAI-OneRoomS20-v0", "BabyAI-PutNextLocal-v0"])
def test_hash_vs_oracle(env_id):
    """12 x 12 and 20 x 20 are square geometries K4 meets first here."""
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
@pytest.mark.parametrize("env_id", ["BabyAI-PutNextLocal-v0", "BabyAI-OneRoomS16-v0"])
def test_packed_host_path(env_id, mode):
    n = 1000 + 13
    eng = EngineAdapter(env_id, n, mode, host=True, host_format="packed", host_threads=2)
    orc = PickupOracle(env_id, n, autoreset=mode, n_threads=0)
    parity.check_lockstep_vs_oracle(eng, orc, 150, seed=21)


@pytest.mark.parametrize("env_id", ["BabyAI-PutNextLocalS5N3-v0", "BabyAI-PickupDistDebug-v0"])
def test_partial_reset_mask(env_id):
    n = 1000
    eng = EngineAdapter(env_id, n, "next_step")
    orc = PickupOracle(env_id, n, autoreset="next_step")
    parity.check_lockstep_vs_oracle(eng, orc, 30, seed=3)
    rng = np.random.default_rng(8)
    for seed in (None, 5000, rng.integers(0, 2**62, n).astype(np.uint64)):
        mask = rng.random(n) < 0.3
        eo, ed = eng.reset(seed=seed, mask=mask)
        oo, od = orc.reset(seed=seed, mask=mask)
        np.testing.assert_array_equal(eo, oo)
        np.testing.assert_array_equal(ed, od)
        for t in range(25):
            a = rng.integers(0, 7, n).astype(np.int32)
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
