"""Per-episode missions of the 43 BabyAI ids on the GPU (MinigridVecEnv(..., missions=True)): the device's codes against
the oracles' (tests/babyai_mission_oracle.py) after every step at N = 4133 in both autoreset modes, with a missions=False
handle stepped alongside to show that the option changes no output; the reference's record
(tests/golden/ref_babyai_mission_traces.json) replayed on the device; both layouts with many tiles per warp; reset_mask;
the packed host path; a 22 x 22 handle with missions sharing the roomgrid K1 with a smaller one without; the text,
DictObservationSpaceWrapper and FlatObsWrapper outputs against the record; and what mg_enable_missions refuses."""
import numpy as np
import pytest
import torch

import babyai_mission_oracle as mo
from oracle import ref_babyai_missions as rec_mod
from oracle import ref_trace as rt
from oracle.ref_babyai import observation_wrappers

pytestmark = pytest.mark.gpu

REC = rec_mod.load_record()
MODES = ["next_step", "same_step"]
N = 4133


def _env(env_id, n, mode="next_step", missions=True):
    import minigrid_b200 as mb

    return mb.MinigridVecEnv(env_id, n, autoreset_mode=mode, missions=missions)


def _codes(env):
    return env.mission_codes.cpu().numpy().view(np.uint32)


def _outs(o, r, te, tr):
    return o["image"].cpu().numpy(), o["direction"].cpu().numpy(), r.cpu().numpy(), te.cpu().numpy(), tr.cpu().numpy()


@pytest.mark.parametrize("env_id", mo.IDS)
@pytest.mark.parametrize("mode", MODES)
def test_codes_follow_the_oracle(env_id, mode):
    """Codes after every step, strings every 20 steps; obs, direction, reward, terminated and truncated bit-identical to a
    missions=False handle stepped alongside."""
    on, off = _env(env_id, N, mode), _env(env_id, N, mode, missions=False)
    orc = mo.make(env_id, N, autoreset=mode)
    o1, _ = on.reset(seed=5)
    o2, _ = off.reset(seed=5)
    orc.reset(seed=5)
    np.testing.assert_array_equal(o1["image"].cpu().numpy(), o2["image"].cpu().numpy())
    np.testing.assert_array_equal(_codes(on), orc.mission_codes())
    acts = mo.record_actions(env_id, N, 60, 8)
    changed = 0
    for t in range(60):
        a = torch.as_tensor(acts[t].astype(np.int32), device="cuda")
        r1, r2 = _outs(*on.step(a)[:4]), _outs(*off.step(a)[:4])
        orc.step(acts[t])
        for x, y in zip(r1, r2):
            assert x.tobytes() == y.tobytes(), t
        c = _codes(on)
        want = orc.mission_codes()
        np.testing.assert_array_equal(c, want, err_msg=f"t={t}")
        if t % 20 == 19:
            assert on.missions() == orc.missions(), t
        changed += int((r1[3] | r1[4]).sum())
    assert changed > 0  # autoresets happened


@pytest.mark.parametrize("env_id", mo.IDS)
@pytest.mark.parametrize("mode", MODES)
def test_reference_record_replayed_on_the_device(env_id, mode):
    r = REC["missions"][rt.key(env_id, mode)]
    env = _env(env_id, rec_mod.N_ENVS, mode)
    acts = mo.record_actions(env_id, rec_mod.N_ENVS, rec_mod.MAX_STEPS, rec_mod.ACT_SEED)
    env.reset(seed=rec_mod.SEED)
    want = list(r["initial"])
    assert env.missions() == want
    changes = {}
    for t, i, m in r["changes"]:
        changes.setdefault(t, []).append((i, m))
    for t in range(r["steps"]):
        env.step(acts[t])
        if t in changes:
            for i, m in changes[t]:
                want[i] = m
            assert env.missions() == want, t
    assert env.missions() == want


@pytest.mark.parametrize("layout", ["0", "1"], ids=["tiled", "window"])
@pytest.mark.parametrize("env_id", ["BabyAI-GoToLocal-v0", "BabyAI-PickupDist-v0", "BabyAI-OpenDoorsOrderN4-v0",
                                    "BabyAI-OpenDoorLoc-v0"])
@pytest.mark.parametrize("mode", MODES)
def test_both_layouts_many_tiles_per_warp(env_id, layout, mode, monkeypatch):
    monkeypatch.setenv("MINIGRID_B200_LAYOUT", layout)
    monkeypatch.setenv("MINIGRID_B200_GRID", "2")
    monkeypatch.setenv("MINIGRID_B200_CFG", "3,0,0")
    n = 2085
    env, orc = _env(env_id, n, mode), mo.make(env_id, n, autoreset=mode)
    env.reset(seed=2)
    orc.reset(seed=2)
    acts = mo.record_actions(env_id, n, 80, 4)
    for t in range(80):
        env.step(acts[t])
        orc.step(acts[t])
        np.testing.assert_array_equal(_codes(env), orc.mission_codes(), err_msg=f"t={t}")


@pytest.mark.parametrize("env_id", ["BabyAI-GoToRedBall-v0", "BabyAI-PutNextLocal-v0", "BabyAI-OpenTwoDoors-v0"])
def test_reset_mask_resets_only_the_selected_missions(env_id):
    n = 1000
    env, orc = _env(env_id, n), mo.make(env_id, n)
    env.reset(seed=0)
    orc.reset(seed=0)
    before = _codes(env).copy()
    mask = np.random.default_rng(1).random(n) < 0.3
    env.reset(seed=777, options={"reset_mask": mask})
    orc.reset(seed=777, mask=mask)
    after = _codes(env)
    np.testing.assert_array_equal(after, orc.mission_codes())
    np.testing.assert_array_equal(after[~mask], before[~mask])
    assert (after[mask] != before[mask]).any()


def test_step_host_packed_leaves_correct_codes():
    env_id, n = "BabyAI-OpenDoor-v0", 3000
    env, orc = _env(env_id, n), mo.make(env_id, n)
    env.set_host_format("packed")
    env.reset_host(seed=9)
    orc.reset(seed=9)
    acts = mo.record_actions(env_id, n, 50, 2)
    for t in range(50):
        env.step_host(acts[t].astype(np.int32))
        orc.step(acts[t])
        np.testing.assert_array_equal(_codes(env), orc.mission_codes(), err_msg=f"t={t}")


@pytest.mark.parametrize("big_first", [True, False], ids=["big_first", "small_first"])
def test_22x22_with_missions_shares_the_roomgrid_kernel(big_first):
    big, small, n = "BabyAI-UnlockLocalDist-v0", "BabyAI-GoToLocal-v0", 2085
    make = {big: lambda: _env(big, n), small: lambda: _env(small, n, missions=False)}
    order = [big, small] if big_first else [small, big]
    envs = {k: make[k]() for k in order}
    orc = mo.make(big, n)
    for k, e in envs.items():
        e.reset(seed=3)
    orc.reset(seed=3)
    acts = mo.record_actions(big, n, 60, 5)
    for t in range(60):
        for k in order:
            envs[k].step(acts[t])
        orc.step(acts[t])
        np.testing.assert_array_equal(_codes(envs[big]), orc.mission_codes(), err_msg=f"t={t}")


@pytest.mark.parametrize("env_id", sorted(set(mo.IDS) - {"BabyAI-PutNextLocal-v0", "BabyAI-PutNextLocalS5N3-v0",
                                                      "BabyAI-PutNextLocalS6N4-v0", "BabyAI-OpenDoor-v0",
                                                      "BabyAI-OpenDoorDebug-v0", "BabyAI-OpenDoorLoc-v0"}
                                     - {f"BabyAI-OpenDoorsOrderN{n}{d}-v0" for n in (2, 4) for d in ("", "Debug")}))
def test_dict_wrapper_indices_and_text_match_the_reference(env_id):
    import minigrid_b200 as mb

    rows = REC["dict"][env_id]
    env = _env(env_id, len(rows))
    w = mb.DictObservationSpaceWrapper(env)
    obs, _ = w.reset(seed=list(rec_mod.DICT_SEEDS))
    assert obs["mission"].dtype == torch.int64 and obs["mission"].device.type == "cuda"
    assert obs["mission"].cpu().tolist() == [ix for _, ix in rows]
    assert env.missions() == [m for m, _ in rows]


def test_dict_wrapper_refuses_the_grammars_outside_the_vocabulary():
    import minigrid_b200 as mb

    refused = [i for i in mo.IDS if i not in REC["dict"]]
    assert len(refused) == 10
    for env_id in refused:
        with pytest.raises(ValueError, match="vocabulary"):
            mb.DictObservationSpaceWrapper(_env(env_id, 4))


@pytest.mark.parametrize("env_id", rec_mod.FLAT_IDS)
def test_flat_wrapper_rows_match_the_reference(env_id):
    import minigrid_b200 as mb

    n = rec_mod.N_ENVS
    env = _env(env_id, n)
    flat = mb.FlatObsWrapper(env)

    def views(e):
        return [flat.observation(e._obs()).cpu().numpy().astype(np.float32)]
    assert observation_wrappers(env, n, views) == REC["flat"][env_id]


def test_enable_missions_refusals_and_constant_missions():
    import minigrid_b200 as mb
    from minigrid_b200 import _lib

    L = _lib.load()
    env = _env("BabyAI-GoToLocal-v0", 8, missions=False)
    env.reset(seed=0)
    assert L.mg_enable_missions(env._h) == -1 and b"first seed, reset or step" in L.mg_last_error()
    with pytest.raises(ValueError):
        env.mission_codes
    with pytest.raises(_lib.MinigridB200Error, match="BabyAI"):
        _env("MiniGrid-KeyCorridorS3R1-v0", 8)
    with pytest.raises(_lib.MinigridB200Error, match="BabyAI"):
        _env("MiniGrid-Fetch-5x5-N2-v0", 8)
    dk = _env("MiniGrid-DoorKey-8x8-v0", 40)  # a constant mission: a no-op, every code 0
    dk.reset(seed=1)
    dk.step(np.zeros(40, np.int32))
    assert not _codes(dk).any()
    assert dk.missions() == ["use the key to open the door and then get to the goal"] * 40
    assert L.mg_mission_text(dk._h, dk._p(torch.empty((40, 96), dtype=torch.uint8, device="cuda")), None) == -1
    # the default handle and its wrappers are unchanged
    with pytest.raises(ValueError):
        mb.FlatObsWrapper(_env("BabyAI-GoToLocal-v0", 4, missions=False))
    with pytest.raises(ValueError):
        mb.DictObservationSpaceWrapper(_env("BabyAI-GoToLocal-v0", 4, missions=False))
    # obs["mission"] stays the spec's string with missions on
    e = _env("BabyAI-GoToLocal-v0", 4)
    obs, _ = e.reset(seed=0)
    assert obs["mission"] == e.level_spec.mission
