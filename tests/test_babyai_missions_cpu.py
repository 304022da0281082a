"""Per-episode missions of the 43 BabyAI ids, without a GPU: the oracles against the reference's record, the g++ build of
the device's generators and renderer (tests/host_emu/mission_emu.cpp) against the oracles, and the vocabulary split of
DictObservationSpaceWrapper."""
from __future__ import annotations

import collections
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import babyai_mission_oracle as mo
from oracle import ref_babyai_missions as rec_mod
from oracle import ref_trace as rt
from oracle.ref_babyai import observation_wrappers
from babyai_oracle import Level
from babyai_open_oracle import OpenLevel
from babyai_pickup_oracle import PickupLevel

HERE = os.path.dirname(os.path.abspath(__file__))
REC = rec_mod.load_record()
MODES = ["next_step", "same_step"]
_LIB = os.path.join(HERE, "host_emu", "libmg_mission_emu.so")
_emu = None


def emu():
    global _emu
    if _emu is None:
        src = os.path.join(HERE, "host_emu", "mission_emu.cpp")
        csrc = os.path.join(os.path.dirname(HERE), "minigrid_b200", "csrc")
        deps = [src] + [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_LIB) or any(os.path.getmtime(d) > os.path.getmtime(_LIB) for d in deps):
            subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-Wno-unknown-pragmas", "-ffp-contract=off",
                                   "-o", _LIB, src])
        L = C.CDLL(_LIB)
        p = C.c_void_p
        L.mis_draw.argtypes = [C.c_int, C.c_int, p, C.c_int, C.c_int, p, C.c_int, p]
        L.mis_text.argtypes = [p, C.c_int, p]
        L.mis_indices.argtypes = [p, C.c_int, C.c_int, p]
        L.mis_onehot.argtypes = [p, C.c_int, p]
        _emu = L
    return _emu


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def render(codes):
    codes = np.ascontiguousarray(codes, np.uint32)
    out = np.zeros((len(codes), 96), np.uint8)
    emu().mis_text(_p(codes), len(codes), _p(out))
    return [bytes(r).rstrip(b"\0").decode() for r in out]


def indices(codes, max_words=50):
    codes = np.ascontiguousarray(codes, np.uint32)
    out = np.zeros((len(codes), max_words), np.int64)
    emu().mis_indices(_p(codes), len(codes), max_words, _p(out))
    return out


def onehot(codes):
    codes = np.ascontiguousarray(codes, np.uint32)
    out = np.zeros((len(codes), 96 * 28), np.uint8)
    emu().mis_onehot(_p(codes), len(codes), _p(out))
    return out


def replay(env_id, mode):
    """The oracle stepped as the record's reference was; yields (step, oracle) after the reset (step -1) and every step."""
    r = REC["missions"][rt.key(env_id, mode)]
    orc = mo.make(env_id, rec_mod.N_ENVS, autoreset=mode)
    acts = mo.record_actions(env_id, rec_mod.N_ENVS, rec_mod.MAX_STEPS, rec_mod.ACT_SEED)
    orc.reset(seed=rec_mod.SEED)
    yield -1, orc
    for t in range(r["steps"]):
        orc.step(acts[t])
        yield t, orc


def test_ids_and_record_agree():
    from minigrid_b200 import specs

    assert len(mo.IDS) == 43 == len(rec_mod.babyai_ids())
    assert set(mo.IDS) == set(rec_mod.babyai_ids())
    assert set(REC["missions"]) == {rt.key(i, m) for i in mo.IDS for m in MODES}
    for env_id, (kind, w, h, ms, st, prm) in mo.ALL_SPECS.items():
        s = specs.get(env_id)
        assert specs.is_babyai(s) and list(s.params) == list(prm), env_id
    assert not any(specs.is_babyai(s) for s in specs.REGISTRY.values())


@pytest.mark.parametrize("env_id", mo.IDS)
@pytest.mark.parametrize("mode", MODES)
def test_oracle_missions_replay_the_record(env_id, mode):
    """Every env's mission after the seeded reset and after every step, through both autoresets; each code the oracle
    builds renders (g++ build of mission_words) to its mission."""
    r = REC["missions"][rt.key(env_id, mode)]
    assert min(r["ends"]) >= rec_mod.ENDS, "the record must see every env through two autoresets"
    changes = collections.defaultdict(list)
    for t, i, m in r["changes"]:
        changes[t].append((i, m))
    want = list(r["initial"])
    pairs = {}
    for t, orc in replay(env_id, mode):
        for i, m in changes.get(t, []):
            want[i] = m
        got = orc.missions()
        assert got == want, (t, got, want)
        for c, m in zip(orc.mission_codes().tolist(), got):
            pairs[c] = m
    codes = sorted(pairs)
    assert render(codes) == [pairs[c] for c in codes]
    assert [mo.surface(c) for c in codes] == [pairs[c] for c in codes]


def test_renderer_on_every_code_of_the_grammar():
    codes = mo.all_codes()
    assert len(codes) > 500
    assert render(codes) == [mo.surface(c) for c in codes]
    assert render([0]) == [""]  # MIS_CONST: the spec's constant string is the host's


def _oracle_level(env_id, seed):
    spec = mo.ALL_SPECS[env_id]
    g = np.random.default_rng(seed)
    if env_id in mo.BABYAI_SPECS:
        return mo.goto_code(Level(spec, g))
    if env_id in mo.PICKUP_SPECS:
        return mo.pickup_code(PickupLevel(spec, g))
    return mo.open_code(OpenLevel(spec, g))


@pytest.mark.parametrize("env_id", mo.IDS)
@pytest.mark.parametrize("layout", [0, 1])
def test_emu_generator_writes_the_oracle_code(env_id, layout):
    """draw_level (g++ build) leaves the oracle's mission code for 200 seeds, in both grid layouts."""
    _, W, H, _, _, prm = mo.ALL_SPECS[env_id]
    seeds = np.arange(500, 700, dtype=np.uint64)
    out = np.zeros(len(seeds), np.uint32)
    params = np.asarray(prm, np.int32)
    emu().mis_draw(W, H, _p(params), len(params), layout, _p(seeds), len(seeds), _p(out))
    want = [_oracle_level(env_id, int(s)) for s in seeds]
    assert out.tolist() == want


REFUSED = {"BabyAI-PutNextLocal-v0", "BabyAI-PutNextLocalS5N3-v0", "BabyAI-PutNextLocalS6N4-v0", "BabyAI-OpenDoor-v0",
           "BabyAI-OpenDoorDebug-v0", "BabyAI-OpenDoorLoc-v0", "BabyAI-OpenDoorsOrderN2-v0", "BabyAI-OpenDoorsOrderN4-v0",
           "BabyAI-OpenDoorsOrderN2Debug-v0", "BabyAI-OpenDoorsOrderN4Debug-v0"}


def test_dict_vocabulary_split():
    """The grammar-derived split: 33 ids whose missions stay in the Minigrid vocabulary, 10 that the reference's
    DictObservationSpaceWrapper would fail on ("Unknown word": next, after, on, your, left, right, in, front, behind)."""
    from minigrid_b200 import specs
    from minigrid_b200.wrappers import MINIGRID_WORDS

    accepted = set(rec_mod.dict_ids())
    assert accepted == set(mo.IDS) - REFUSED and len(accepted) == 33
    assert set(REC["dict"]) == accepted
    outside = set()
    for env_id in REFUSED:
        outside |= specs.babyai_mission_words(specs.get(env_id)) - set(MINIGRID_WORDS)
    assert outside == {"next", "after", "on", "your", "left", "right", "in", "front", "behind"}
    # every recorded mission of a refused id that uses such a word really is in the grammar
    for key, r in REC["missions"].items():
        env_id = key.split("|")[0]
        words = specs.babyai_mission_words(specs.get(env_id))
        for m in r["initial"] + [c[2] for c in r["changes"]]:
            assert set(m.replace(",", " , ").split()) <= words, (env_id, m)


@pytest.mark.parametrize("env_id", sorted(set(mo.IDS) - REFUSED))
def test_dict_indices_match_the_reference(env_id):
    from minigrid_b200.wrappers import mission_to_indices

    rows = REC["dict"][env_id]
    codes = [_oracle_level(env_id, s) for s in rec_mod.DICT_SEEDS]
    assert render(codes) == [m for m, _ in rows]
    assert indices(codes).tolist() == [ix for _, ix in rows]
    assert [mission_to_indices(m) for m, _ in rows] == [ix for _, ix in rows]


@pytest.mark.parametrize("env_id", rec_mod.FLAT_IDS)
def test_flat_rows_match_the_reference(env_id):
    """FlatObsWrapper rows: the oracle's image followed by the g++ one-hot of the oracle's codes."""
    n = rec_mod.N_ENVS

    def views(orc):
        img, _ = orc.gen_obs()
        return [np.concatenate([np.asarray(img).reshape(n, -1), onehot(orc.mission_codes())], 1).astype(np.float32)]
    assert observation_wrappers(mo.make(env_id, n), n, views) == REC["flat"][env_id]


def test_record_events():
    """Both articles, every location phrase and both sequence forms occur in the record."""
    text = [m for r in REC["missions"].values() for m in r["initial"] + [c[2] for c in r["changes"]]]
    ev = collections.Counter()
    for m in text:
        ev["a"] += " a " in m
        ev["the"] += " the " in m
        ev["object"] += "object" in m
        for loc in ("on your left", "on your right", "in front of you", "behind you"):
            ev[loc] += loc in m
        ev["then"] += ", then " in m
        ev["after"] += " after you " in m
        ev["putnext"] += " next to " in m
    assert all(ev[k] > 0 for k in ["a", "the", "object", "on your left", "on your right", "in front of you", "behind you",
                                   "then", "after", "putnext"]), ev
    ends = [sum(r["ends"]) for r in REC["missions"].values()]
    assert min(ends) >= rec_mod.N_ENVS * rec_mod.ENDS


def test_enable_missions_refuses_a_null_handle():
    from minigrid_b200 import _lib

    L = _lib.load()
    assert L.mg_enable_missions(None) == -1
    assert L.mg_mission_text(None, None, None) == -1
