"""The single-room BabyAI GoTo levels on the GPU: K1 / K2 against the C oracle at N = 4133 (129 full tiles and a ragged
one of 5 envs), the reference's record (tests/golden/ref_babyai_traces.json) replayed on the device, both HBM layouts
with many tiles per warp, hash(), the packed host path, reset_mask and the observation wrappers."""
import numpy as np
import pytest
import torch

import hash_support as hs
import parity
from engine_adapter import EngineAdapter
from oracle import ref_babyai
from oracle import ref_trace as rt
from babyai_oracle import BABYAI_SPECS, BabyAIOracle, hashed

pytestmark = pytest.mark.gpu

REC = ref_babyai.load_record()
IDS = list(BABYAI_SPECS)
MODES = ["next_step", "same_step"]
N = 4133


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_lockstep_vs_oracle(env_id, mode):
    """obs, direction, reward bits, terminated and truncated after every step; grid, agent, RNG and pending flags
    every 40 steps and at the end (parity.check_lockstep_vs_oracle)."""
    eng = EngineAdapter(env_id, N, mode)
    orc = BabyAIOracle(env_id, N, autoreset=mode, n_threads=0)
    parity.check_lockstep_vs_oracle(eng, orc, 120, seed=17, check_state_every=40)


@pytest.mark.parametrize("env_id", IDS)
@pytest.mark.parametrize("mode", MODES)
def test_reference_record_replayed_on_the_device(env_id, mode):
    eng = EngineAdapter(env_id, ref_babyai.N_ENVS, mode)
    got = rt.rollout(eng, ref_babyai.N_ENVS, ref_babyai.SEED, ref_babyai.ACT_SEED, ref_babyai.STEPS)
    assert got == REC["lockstep"][rt.key(env_id, mode)]


@pytest.mark.parametrize("layout", ["0", "1"], ids=["tiled", "window"])
@pytest.mark.parametrize("env_id", ["BabyAI-GoToLocal-v0", "BabyAI-GoToRedBlueBall-v0"])
@pytest.mark.parametrize("mode", MODES)
def test_both_layouts_many_tiles_per_warp(env_id, layout, mode, monkeypatch):
    """Two CTAs of three tile warps share 130 tiles while episodes end all the time (64-step episodes, random walks)."""
    monkeypatch.setenv("MINIGRID_B200_LAYOUT", layout)
    monkeypatch.setenv("MINIGRID_B200_GRID", "2")
    monkeypatch.setenv("MINIGRID_B200_CFG", "3,0,0")
    eng = EngineAdapter(env_id, N, mode)
    orc = BabyAIOracle(env_id, N, autoreset=mode, n_threads=0)
    parity.check_lockstep_vs_oracle(eng, orc, 150, seed=5, check_state_every=50)


@pytest.mark.parametrize("env_id", IDS)
def test_hash_reproduces_reference_record(env_id):
    from minigrid_b200 import MinigridVecEnv

    for mode in MODES:
        assert hs.hash_rollout(MinigridVecEnv(env_id, 6, autoreset_mode=mode), 6) == REC["hash_rollout"][rt.key(env_id, mode)]
    assert hs.hash_walk(MinigridVecEnv(env_id, 6), 6) == REC["hash_walk"][env_id]


@pytest.mark.parametrize("env_id", ["BabyAI-GoToLocal-v0", "BabyAI-GoToObjS4-v0", "BabyAI-GoToRedBallGrey-v0"])
def test_hash_vs_oracle(env_id):
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
def test_packed_host_path(mode):
    env_id, n = "BabyAI-GoToLocal-v0", 1000 + 13
    eng = EngineAdapter(env_id, n, mode, host=True, host_format="packed", host_threads=2)
    orc = BabyAIOracle(env_id, n, autoreset=mode, n_threads=0)
    parity.check_lockstep_vs_oracle(eng, orc, 150, seed=21)


@pytest.mark.parametrize("env_id", ["BabyAI-GoToLocal-v0", "BabyAI-GoToRedBlueBall-v0"])
def test_partial_reset_mask(env_id):
    n = 1000
    eng = EngineAdapter(env_id, n, "next_step")
    orc = BabyAIOracle(env_id, n, autoreset="next_step")
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
        es, os_ = eng.get_state(), orc.get_state()
        for k in ("grid", "agent", "rng", "pending"):
            np.testing.assert_array_equal(es[k], os_[k], err_msg=k)


@pytest.mark.parametrize("env_id", ref_babyai.OBS_WRAPPER_IDS)
def test_observation_wrappers_reproduce_reference_record(env_id):
    """FullyObsWrapper, RGBImgPartialObsWrapper, RGBImgObsWrapper and, on the constant missions, FlatObsWrapper."""
    import minigrid_b200 as mb

    flat = env_id in ref_babyai.CONSTANT_MISSION_IDS

    class Side:
        def __init__(self):
            self.env = mb.MinigridVecEnv(env_id, ref_babyai.N_ENVS)
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

    assert ref_babyai.observation_wrappers(Side(), ref_babyai.N_ENVS, views) == REC["obs_wrappers"][env_id]


def test_dict_wrapper_and_mission_refusals():
    import minigrid_b200 as mb

    for env_id in IDS:
        env = mb.MinigridVecEnv(env_id, 4)
        if env_id in ref_babyai.CONSTANT_MISSION_IDS:
            obs, _ = mb.DictObservationSpaceWrapper(env).reset(seed=0)
            assert obs["mission"] == REC["dict_missions"][env_id]
        else:
            with pytest.raises(ValueError):
                mb.DictObservationSpaceWrapper(env)
            with pytest.raises(ValueError):
                mb.FlatObsWrapper(env)
