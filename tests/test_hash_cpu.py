"""MiniGridEnv.hash (minigrid_env.py:159-170) without a GPU: the oracle's hash (tests/hash_support.py) against the
reference's record (tests/golden/ref_hash_traces.json), and the device's per-lane code (minigrid_b200/csrc/mg_hash.cuh)
compiled by g++ (tests/host_emu/hash_emu.cpp) against hashlib and the oracle."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

import hash_support as hs
from minigrid_b200 import specs

REC = hs.load_record()
IDS = list(specs.REGISTRY)
MODES = ["next_step", "same_step"]

_HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emu")
_CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "minigrid_b200", "csrc")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src, so = os.path.join(_HERE, "hash_emu.cpp"), os.path.join(_HERE, "libmg_hash_emu.so")
        deps = [src] + [os.path.join(_CSRC, f) for f in os.listdir(_CSRC)]
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
            subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-o", so, src])
        L = C.CDLL(so)
        p = C.c_void_p
        L.hash_emu_sha256.argtypes = [p, C.c_int64, p]
        L.hash_emu_batch.argtypes = [C.c_int] * 4 + [p] * 4
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def emu_hashes(W, H, layout, grid, agent, forms):
    n = len(forms)
    out = np.zeros((n, 32), np.uint8)
    g, a, f = (np.ascontiguousarray(grid, np.uint8), np.ascontiguousarray(agent, np.int32), np.ascontiguousarray(forms, np.int32))
    lib().hash_emu_batch(W, H, layout, n, _ptr(g), _ptr(a), _ptr(f), _ptr(out))
    return [bytes(r).hex() for r in out]


def test_record_covers_every_registered_id():
    assert set(REC["walk"]) == set(IDS)
    assert set(REC["rollout"]) == {f"{i}|{m}" for i in IDS for m in MODES}


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_oracle_hash_rollout_matches_reference(env_id, mode):
    assert hs.hash_rollout(hs.HashedOracle(env_id, 6, autoreset=mode), 6) == REC["rollout"][f"{env_id}|{mode}"]


@pytest.mark.parametrize("env_id", IDS)
def test_oracle_hash_walk_matches_reference(env_id):
    assert hs.hash_walk(hs.HashedOracle(env_id, 6), 6) == REC["walk"][env_id]


@pytest.mark.parametrize("env_id", ["MiniGrid-Empty-8x8-v0", "MiniGrid-Empty-16x16-v0"])
def test_same_state_after_walking_back_hashes_differently(env_id):
    """Back at the start, facing the same way, with the same grid: agent_pos is now a tuple of numpy ints."""
    orc = hs.HashedOracle(env_id, 4)
    orc.reset(seed=5)
    s0, h0 = orc.get_state(), orc.hash(64)
    for a in hs.HASH_WALK:
        orc.step(np.full(4, a))
    s1, h1 = orc.get_state(), orc.hash(64)
    assert np.array_equal(s0["grid"], s1["grid"]) and np.array_equal(s0["agent"][:, :3], s1["agent"][:, :3])
    assert all(a != b for a, b in zip(h0, h1))


def test_sha256_every_length_mod_64():
    rng = np.random.default_rng(3)
    for n in list(range(0, 200)) + [1000, 6925 + 29]:
        msg = rng.integers(0, 256, max(n, 1), dtype=np.uint8)
        out = np.zeros(32, np.uint8)
        lib().hash_emu_sha256(_ptr(msg), n, _ptr(out))
        assert bytes(out) == hashlib.sha256(msg[:n].tobytes()).digest(), n


def _ref_tail(x, y, form):
    if form == 0:
        return str((x, y))
    if form == 1:
        return str((np.int64(x), np.int64(y)))
    return str(np.array((x, y)))


@pytest.mark.parametrize("W,H", [(5, 5), (8, 8), (7, 3), (19, 19), (25, 25), (26, 26), (9, 7), (16, 8)])
@pytest.mark.parametrize("layout", [0, 1], ids=["tiled", "window"])
def test_synthetic_grids_every_tail_form(W, H, layout):
    """The template walk and the three tail forms with one- and two-digit coordinates on random grids: every
    (L + tail) mod 64 that a geometry and its coordinates give, including the endings that need a second block."""
    rng = np.random.default_rng(W * 100 + H)
    coords = [(0, 0), (1, 1), (W - 1, H - 1), (min(10, W - 1), 3), (3, min(10, H - 1)), (W - 1, 0)]
    cases = [(x, y, d, f) for x, y in coords for d in range(4) for f in range(3)]
    n = len(cases)
    t = rng.integers(1, 10, (n, W, H))
    grid = np.stack([t, np.where(t == 1, 0, rng.integers(0, 6, (n, W, H))), np.where(t == 4, rng.integers(0, 3, (n, W, H)), 0)], -1)
    grid[..., 1] = np.where(grid[..., 0] == 2, 5, grid[..., 1])  # walls are grey
    agent = np.zeros((n, 6), np.int32)
    agent[:, :3] = [(x, y, d) for x, y, d, _ in cases]
    got = emu_hashes(W, H, layout, grid, agent, [f for *_, f in cases])
    for i, (x, y, d, f) in enumerate(cases):
        want = hashlib.sha256((str(grid[i].tolist()) + _ref_tail(x, y, f) + str(d)).encode()).hexdigest()
        assert got[i] == want, (x, y, d, f)


EMU_IDS = ["MiniGrid-Empty-8x8-v0", "MiniGrid-DoorKey-8x8-v0", "MiniGrid-LavaCrossingS9N1-v0", "MiniGrid-FourRooms-v0",
           "MiniGrid-MemoryS7-v0", "MiniGrid-Dynamic-Obstacles-6x6-v0", "MiniGrid-DistShift1-v0", "MiniGrid-MultiRoom-N6-v0",
           "MiniGrid-ObstructedMaze-Full-v1"]


@pytest.mark.parametrize("env_id", EMU_IDS)
@pytest.mark.parametrize("layout", [0, 1], ids=["tiled", "window"])
@pytest.mark.parametrize("mode", MODES)
def test_per_lane_hash_matches_oracle_in_lockstep(env_id, layout, mode):
    """k_hash's staging and walk on the oracle's states (37 envs: a ragged second tile), with the form the oracle's
    tracking gives, against the oracle's Python hash after every step."""
    n = 37
    orc = hs.HashedOracle(env_id, n, autoreset=mode)
    W, H = orc.o.width, orc.o.height
    orc.reset(seed=9)
    rng = np.random.default_rng(4)
    for t in range(41):
        st = orc.get_state()
        assert emu_hashes(W, H, layout, st["grid"], st["agent"], orc.forms()) == orc.hash(64), t
        orc.step(np.where(rng.random(n) < 0.5, 2, rng.integers(0, 7, n)).astype(np.int32))
