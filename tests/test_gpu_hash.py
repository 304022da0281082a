"""MinigridVecEnv.hash / hash_digest (k_hash, minigrid_b200/csrc/mg_hash.cu) on the GPU against the C oracle's Python
hash (tests/hash_support.py: the reference's own str() + hashlib) and against the reference's record (tests/golden/ref_hash_traces.json)."""
import hashlib

import numpy as np
import pytest
import torch

from minigrid_b200 import specs
from minigrid_b200.vector_env import MinigridVecEnv, make_sharded
import hash_support as hs

pytestmark = pytest.mark.gpu

REC = hs.load_record()
MODES = ["next_step", "same_step"]
IDS = list(specs.REGISTRY)
N = 4133  # 129 full tiles and a ragged one of 5 envs
SAMPLE = np.r_[0:40, N - 40:N]


def _actions(rng, n):
    return np.where(rng.random(n) < 0.5, 2, rng.integers(0, 7, n)).astype(np.int32)


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_hash_lockstep_vs_oracle(env_id, mode):
    """Every registered id: the first and last tiles after the reset and after every step, every env at the end."""
    env = MinigridVecEnv(env_id, N, autoreset_mode=mode)
    orc = hs.HashedOracle(env_id, N, autoreset=mode)
    env.reset(seed=21)
    orc.reset(seed=21)
    rng = np.random.default_rng(8)
    # the oracle's Python hash costs ~0.1 ms per env: the first and last tiles at every step, every env at the end
    for t in range(7):
        got = env.hash(64)
        assert [got[i] for i in SAMPLE] == orc.hash(64, SAMPLE), t
        a = _actions(rng, N)
        env.step(torch.as_tensor(a, device=env.device))
        orc.step(a)
    assert env.hash(64) == orc.hash(64)


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_hash_rollout_reproduces_reference_record(env_id, mode):
    env = MinigridVecEnv(env_id, 6, autoreset_mode=mode)
    assert hs.hash_rollout(env, 6) == REC["rollout"][f"{env_id}|{mode}"]


@pytest.mark.parametrize("env_id", IDS)
def test_hash_walk_reproduces_reference_record(env_id):
    assert hs.hash_walk(MinigridVecEnv(env_id, 6), 6) == REC["walk"][env_id]


@pytest.mark.parametrize("layout", ["0", "1"], ids=["tiled", "window"])
@pytest.mark.parametrize("env_id", ["MiniGrid-DoorKey-8x8-v0", "MiniGrid-FourRooms-v0", "MiniGrid-LavaCrossingS9N1-v0",
                                    "MiniGrid-MultiRoom-N6-v0"])
def test_hash_both_layouts_many_tiles_per_warp(env_id, layout, monkeypatch):
    monkeypatch.setenv("MINIGRID_B200_LAYOUT", layout)
    monkeypatch.setenv("MINIGRID_B200_GRID", "3")  # 12 warps for 130 tiles
    env = MinigridVecEnv(env_id, N)
    orc = hs.HashedOracle(env_id, N)
    env.reset(seed=4)
    orc.reset(seed=4)
    rng = np.random.default_rng(2)
    for _ in range(12):
        a = _actions(rng, N)
        env.step(torch.as_tensor(a, device=env.device))
        orc.step(a)
    assert env.hash(64) == orc.hash(64)


def test_two_shards_equal_the_whole_batch():
    env_id, n = "MiniGrid-DoorKey-8x8-v0", 1000
    whole = MinigridVecEnv(env_id, n)
    shards = [make_sharded(env_id, n, r, 2) for r in range(2)]
    rng = np.random.default_rng(6)
    whole.reset()
    for s in shards:
        s.reset()
    for _ in range(10):
        a = _actions(rng, n)
        whole.step(torch.as_tensor(a, device=whole.device))
        shards[0].step(torch.as_tensor(a[:shards[0].num_envs], device=whole.device))
        shards[1].step(torch.as_tensor(a[shards[0].num_envs:], device=whole.device))
    assert torch.equal(whole.hash_digest(), torch.cat([s.hash_digest() for s in shards]))


@pytest.mark.parametrize("env_id", ["MiniGrid-Empty-8x8-v0", "MiniGrid-LavaGapS7-v0", "MiniGrid-DoorKey-8x8-v0"])
def test_injected_state_hashes_as_numpy_ints(env_id):
    """mg_set_state with agent records: agent_pos counts as a tuple of numpy ints, whatever the kind's reset form."""
    n = 64
    env, orc = MinigridVecEnv(env_id, n), hs.HashedOracle(env_id, n)
    env.reset(seed=3)
    orc.reset(seed=3)
    st = orc.get_state()
    env.set_state(agent=st["agent"])
    orc.set_state(agent=st["agent"])
    got = env.hash(64)
    assert got == orc.hash(64)
    grid, a = st["grid"][0], st["agent"][0]
    ref = hashlib.sha256((str(grid.tolist()) + str((np.int64(a[0]), np.int64(a[1]))) + str(int(a[2]))).encode()).hexdigest()
    assert got[0] == ref


def test_hash_digest_on_a_side_stream_sees_the_step():
    env_id, n = "MiniGrid-FourRooms-v0", 50000
    env, orc = MinigridVecEnv(env_id, n), hs.HashedOracle(env_id, n)
    env.reset(seed=1)
    orc.reset(seed=1)
    a = np.full(n, 2, np.int32)
    orc.step(a)
    s = torch.cuda.Stream(device=env.device)
    act = torch.as_tensor(a, device=env.device)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        env.step(act)
        d = env.hash_digest()
    s.synchronize()
    idx = list(range(0, n, 997))
    got = d.cpu().numpy()
    assert [bytes(got[i]).hex() for i in idx] == orc.hash(64, idx)


def test_hash_sizes_and_digest_key():
    env = MinigridVecEnv("MiniGrid-DoorKey-8x8-v0", 100)
    env.reset(seed=0)
    full = env.hash(64)
    assert all(len(h) == 64 for h in full)
    for size in (1, 16, 64):
        assert env.hash(size) == [h[:size] for h in full]
    d = env.hash_digest()
    assert d.shape == (100, 32) and d.dtype == torch.uint8
    assert [bytes(r).hex() for r in d.cpu().numpy()] == full
    key = d[:, :8].contiguous().view(torch.int64)
    assert key.shape == (100, 1)
    with pytest.raises(ValueError):
        env.hash(0)
    with pytest.raises(ValueError):
        env.hash(65)
