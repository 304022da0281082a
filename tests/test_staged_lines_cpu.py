"""CPU checks behind K1's line staging (mg_step_kernel.cuh: stage_lines), no GPU needed.

- The tiled gather on a tile of which only lines [edge, n - 1 - edge] were staged, every other row poisoned, equals the
  gather on the whole tile with its ring lines, for every position, direction, carry and visibility form of every
  tiled geometry the registered ids use (tests/host_emu/staged_gather.cpp: mg_obs.cuh compiled by g++).
- Every grid the generators of the walled kinds (mg_common.cuh: kind_walled) produce, through reset and autoreset
  streams, has a grey wall on every border cell: what lets K1 skip the border lines of those kinds."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from minigrid_b200 import specs
from oracle.oracle import OracleVecEnv

HERE = os.path.dirname(os.path.abspath(__file__))
KIND_NAMES = ["empty", "doorkey", "crossing", "fourrooms", "lavagap", "distshift", "multiroom", "lockedroom", "playground",
              "gotodoor", "fetch", "redbluedoors", "gotoobject", "putnear", "memory", "dynobstacles", "roomgrid"]
WALLED_KINDS = (specs.KIND_EMPTY, specs.KIND_DOORKEY, specs.KIND_CROSSING, specs.KIND_LAVAGAP, specs.KIND_DISTSHIFT)


def all_specs():
    out = dict(specs.REGISTRY)
    for reg in (specs.BABYAI_REGISTRY, specs.BABYAI_PICKUP_PUTNEXT_REGISTRY, specs.BABYAI_OPEN_REGISTRY, specs.BABYAI_MAZE_REGISTRY):
        out.update(reg)
    return out


def tiled(s):
    """mg_create's layout choice: whole tiles while an env's words (both arrays with one ring line) fit in 512 bytes"""
    wpe = (s.height + 2) * ((s.width + 3) // 4) + (s.width + 2) * ((s.height + 3) // 4)
    return wpe * 4 <= 512 or s.kind == specs.KIND_DYNOBS


TILED_SIZES = sorted({(s.width, s.height) for s in all_specs().values() if tiled(s)})
WALLED_IDS = sorted(i for i, s in specs.REGISTRY.items() if s.kind in WALLED_KINDS)


@pytest.fixture(scope="module")
def staged_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("staged") / "libstaged_gather.so")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so,
                           os.path.join(HERE, "host_emu", "staged_gather.cpp")])
    lib = C.CDLL(so)
    lib.check_staged_gather.restype = C.c_long
    lib.check_staged_gather.argtypes = [C.c_int, C.c_int, C.c_int, C.c_uint64]
    return lib


def test_the_registered_ids_cover_small_and_walled_tiled_geometries():
    assert (8, 8) in TILED_SIZES and (5, 5) in TILED_SIZES and (9, 9) in TILED_SIZES
    assert {"MiniGrid-DoorKey-8x8-v0", "MiniGrid-Empty-8x8-v0", "MiniGrid-LavaCrossingS9N1-v0",
            "MiniGrid-LavaGapS7-v0", "MiniGrid-DistShift1-v0"} <= set(WALLED_IDS)


@pytest.mark.parametrize("edge", [0, 1], ids=["ring-skipped", "border-skipped"])
@pytest.mark.parametrize("W,H", TILED_SIZES, ids=[f"{w}x{h}" for w, h in TILED_SIZES])
def test_staged_gather_equals_whole_tile_gather(staged_lib, W, H, edge):
    for seed in range(3):
        assert staged_lib.check_staged_gather(W, H, edge, seed) == 0, f"{W}x{H} edge {edge} seed {seed}"


def _assert_border_walls(grid, what):
    """grid [n][W][H][3] as the oracle encodes it: every border cell (type 2 wall, colour 5 grey)"""
    border = np.concatenate([grid[:, 0, :], grid[:, -1, :], grid[:, :, 0], grid[:, :, -1]], axis=1)
    bad = np.argwhere(~((border[..., 0] == 2) & (border[..., 1] == 5)).all(axis=1))
    assert bad.size == 0, f"{what}: envs {bad[:5, 0].tolist()} have a non-wall border cell"


@pytest.mark.parametrize("env_id", WALLED_IDS)
def test_walled_kinds_generate_wall_borders(env_id):
    s = specs.REGISTRY[env_id]
    spec = (KIND_NAMES[s.kind], s.width, s.height, s.max_steps, s.see_through_walls, list(s.params))
    n, rounds = 2048, 4
    for mode in ("next_step", "same_step"):
        orc = OracleVecEnv(None, n, spec=spec, autoreset=mode, n_threads=0)
        orc.reset(seed=17)
        _assert_border_walls(orc.get_state()["grid"], f"{mode} reset")
        rng = np.random.default_rng(5)
        for r in range(rounds):
            # a few random steps, then every episode truncated: the autoreset draws the next grid of each env's stream
            for t in range(3):
                orc.step(rng.integers(0, 7, n).astype(np.int32))
                _assert_border_walls(orc.get_state()["grid"], f"{mode} round {r} step {t}")
            agent = orc.get_state()["agent"]
            agent[:, 5] = s.max_steps - 1
            orc.set_state(agent=agent)
            orc.step(rng.integers(0, 7, n).astype(np.int32))
            if mode == "next_step":
                orc.step(rng.integers(0, 7, n).astype(np.int32))
            _assert_border_walls(orc.get_state()["grid"], f"{mode} autoreset {r}")
