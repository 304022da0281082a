"""K1 stages only the grid lines a step can read (mg_step_kernel.cuh: stage_lines): never the ring lines, and on the
walled kinds (mg_common.cuh: kind_walled) not the border lines either, while no grid has been injected. These tests run
that path against the oracle: the walled ids in lockstep through every output path and both tiled plans, a walled
handle given grids whose border is not a wall (mg_set_state: the handle falls back to staging the border) and brought
back by a full reset, and agent records injected onto the border lines, which are then never staged."""
import numpy as np
import pytest

import parity
from engine_adapter import EngineAdapter
from oracle.oracle import OracleVecEnv

pytestmark = pytest.mark.gpu

WALLED_TILED = ["MiniGrid-DoorKey-5x5-v0", "MiniGrid-DoorKey-8x8-v0", "MiniGrid-Empty-8x8-v0", "MiniGrid-LavaCrossingS9N1-v0"]


def _compare_step(e, o, t):
    for x, y, name in zip(e, o, ["obs", "dir", "reward", "terminated", "truncated"]):
        x, y = np.asarray(x), np.asarray(y)
        if name == "reward":
            assert x.astype(np.float64).tobytes() == y.tobytes(), f"reward bits t={t}"
        else:
            np.testing.assert_array_equal(x.astype(y.dtype), y, err_msg=f"{name} t={t}")


@pytest.mark.parametrize("path", ["device", "host-full", "host-packed"])
@pytest.mark.parametrize("env_id", WALLED_TILED)
@pytest.mark.parametrize("mode", ["next_step", "same_step"])
def test_walled_ids_lockstep(env_id, mode, path):
    n = 4096 + 37  # full tiles (bulk-copied obs blocks) and a ragged last tile
    if path == "device":
        eng = EngineAdapter(env_id, n, mode)
    else:
        eng = EngineAdapter(env_id, n, mode, host=True, host_format=path.split("-")[1])
    orc = OracleVecEnv(env_id, n, autoreset=mode, n_threads=0)
    parity.check_lockstep_vs_oracle(eng, orc, 150, seed=321, check_state_every=75)


@pytest.mark.parametrize("env_id", ["MiniGrid-DoorKey-8x8-v0", "MiniGrid-LavaCrossingS9N1-v0"])
def test_walled_ids_two_buffer_plan(env_id, monkeypatch):
    """the two-buffer kernel stages the next tile's lines while it works on the current one; few CTAs give every warp
    many tiles"""
    monkeypatch.setenv("MINIGRID_B200_CFG", "10,2,2")
    monkeypatch.setenv("MINIGRID_B200_GRID", "7")
    n = 4096 + 37
    eng = EngineAdapter(env_id, n, "next_step")
    orc = OracleVecEnv(env_id, n, autoreset="next_step", n_threads=0)
    parity.check_lockstep_vs_oracle(eng, orc, 120, seed=77, check_state_every=60)


def _open_border(grid, rng, frac=0.5):
    """replace about `frac` of the border cells of every grid [n][W][H][3] with lava or a goal: cells the view sees
    through, and that end the episode of an agent that walks onto them (so no agent stands on the border facing out)"""
    g = grid.copy()
    n, W, H, _ = g.shape
    border = np.zeros((W, H), bool)
    border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = True
    pick = border[None] & (rng.random((n, W, H)) < frac)
    lava = rng.random((n, W, H)) < 0.5
    g[pick & lava] = (9, 0, 0)
    g[pick & ~lava] = (8, 1, 0)
    return g


@pytest.mark.parametrize("env_id", ["MiniGrid-DoorKey-8x8-v0", "MiniGrid-Empty-8x8-v0", "MiniGrid-LavaCrossingS9N1-v0"])
@pytest.mark.parametrize("mode", ["next_step", "same_step"])
def test_injected_grid_with_open_border(env_id, mode):
    n = 2048 + 5
    eng = EngineAdapter(env_id, n, mode)
    orc = OracleVecEnv(env_id, n, autoreset=mode, n_threads=0)
    eng.reset(seed=3)
    orc.reset(seed=3)
    rng = np.random.default_rng(11)
    st = orc.get_state()
    grid = _open_border(st["grid"], rng)
    eng.set_state(grid=grid)
    orc.set_state(grid=grid)
    eo, ed = eng.gen_obs()
    oo, od = orc.gen_obs()
    np.testing.assert_array_equal(eo, oo)
    np.testing.assert_array_equal(ed, od)
    for t in range(120):
        a = rng.integers(0, 7, n).astype(np.int32)
        _compare_step(eng.step(a), orc.step(a), t)
    es, os_ = eng.get_state(), orc.get_state()
    for k in ("grid", "agent", "rng", "pending"):
        np.testing.assert_array_equal(es[k], os_[k], err_msg=k)
    # a full reset regenerates every grid: the border is a wall again and the handle skips it again
    parity.check_lockstep_vs_oracle(eng, orc, 120, seed=4, check_state_every=60)


@pytest.mark.parametrize("env_id", ["MiniGrid-DoorKey-8x8-v0", "MiniGrid-Empty-8x8-v0", "MiniGrid-LavaCrossingS9N1-v0"])
def test_agent_injected_onto_the_border(env_id):
    """agent records on a border line (allowed by mg_set_state) of a walled handle whose grids were not injected: the
    agent's own line is not staged, and reads as the wall it is. The agents face along the border or inwards and take
    no turns (a front cell outside the grid has no meaning in the reference)."""
    n = 2048 + 5
    eng = EngineAdapter(env_id, n, "next_step")
    orc = OracleVecEnv(env_id, n, autoreset="next_step", n_threads=0)
    eng.reset(seed=8)
    orc.reset(seed=8)
    W, H = orc.width, orc.height
    rng = np.random.default_rng(9)
    agent = orc.get_state()["agent"].copy()
    side = rng.integers(0, 4, n)  # 0 left column, 1 right column, 2 top row, 3 bottom row
    along = rng.integers(1, np.where(side < 2, H - 1, W - 1))
    agent[:, 0] = np.select([side == 0, side == 1], [0, W - 1], along)
    agent[:, 1] = np.select([side == 2, side == 3], [0, H - 1], along)
    outward = np.array([2, 0, 3, 1])[side]  # the direction that would face out of the grid
    turn = rng.integers(1, 4, n)
    agent[:, 2] = (outward + turn) % 4
    agent[:, 3] = -1
    agent[:, 4] = 0
    eng.set_state(agent=agent)
    orc.set_state(agent=agent)
    eo, ed = eng.gen_obs()
    oo, od = orc.gen_obs()
    np.testing.assert_array_equal(eo, oo)
    np.testing.assert_array_equal(ed, od)
    for t in range(3):
        a = rng.integers(2, 7, n).astype(np.int32)  # forward, pickup, drop, toggle, done: no turn
        _compare_step(eng.step(a), orc.step(a), t)
    es, os_ = eng.get_state(), orc.get_state()
    for k in ("grid", "agent"):
        np.testing.assert_array_equal(es[k], os_[k], err_msg=k)
