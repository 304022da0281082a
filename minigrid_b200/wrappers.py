"""Batched equivalents of the reference's observation wrappers (minigrid/wrappers.py), computed on the device.

ImgObsWrapper            :187-214  the observation is obs["image"].
FullyObsWrapper          :383-426  obs["image"] = grid.encode() with the agent cell set to (OBJECT_TO_IDX["agent"],
                                   COLOR_TO_IDX["red"], agent_dir); shape (W, H, 3) per env.
ViewSizeWrapper          :629-673  obs["image"] regenerated with another odd agent_view_size (3..15).
OneHotPartialObsWrapper  :217-284  obs["image"] -> (V, V, 20) one-hot of (type, colour, state).
FlatObsWrapper           :557-626  uint8[V*V*3 + 28*96]: the image followed by the one-hot mission characters: the
                                   constant mission string, or each env's own mission on a BabyAI level created with
                                   missions=True.
SymbolicObsWrapper       :729-782  obs["image"] = int64 (W, H, 3): (x, y, type or -1), agent cell = 10.
RGBImgPartialObsWrapper  :334-380  obs["image"] = the agent's view rendered with 8 x 8 tiles, (56, 56, 3).
RGBImgObsWrapper         :287-331  obs["image"] = the whole grid rendered, the agent's view highlighted, (8 H, 8 W, 3).
The two RGB wrappers copy tiles that the reference's own Grid.render_tile drew (data/tile_atlas.npz).

DictObservationSpaceWrapper :428-554 obs["mission"] = the mission's words as indices into the Minigrid vocabulary, padded to
                                   max_words_in_mission: a host list for a constant mission string, an int64[n, max_words]
                                   device tensor on a BabyAI level created with missions=True whose grammar stays inside
                                   that vocabulary.

Reward wrappers (they act inside the engine's step kernel, because NoDeath decides whether an episode ends):
NoDeath                  :809-882  a terminated step into / on a death cell continues with reward + death_cost.
ActionBonus              :68-125   reward += 1 / sqrt(visits of (agent_pos, agent_dir, action)), per env.
PositionBonus            :128-184  reward += 1 / sqrt(visits of agent_pos), per env.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np
import torch

from . import _lib, specs


class _VecWrapper:
    def __init__(self, env):
        self.env = env

    def __getattr__(self, name):
        if name.startswith("_") or name == "env":
            raise AttributeError(name)
        return getattr(self.env, name)

    @property
    def unwrapped(self):
        return getattr(self.env, "unwrapped", self.env)

    def observation(self, obs):
        raise NotImplementedError

    def reset(self, *, seed=None, options=None):
        obs, info = self.env.reset(seed=seed, options=options)
        return self.observation(obs), info

    def step(self, actions):
        obs, r, te, tr, info = self.env.step(actions)
        return self.observation(obs), r, te, tr, info

    def close(self):
        return self.env.close()


class _RewardWrapper(_VecWrapper):
    """The wrapper is a setting of the batch's step kernel; the object only scopes it (close() / remove() take it off)."""

    def observation(self, obs):
        return obs

    def remove(self):
        raise NotImplementedError

    def close(self):
        self.remove()
        return self.env.close()


class NoDeath(_RewardWrapper):
    def __init__(self, env, no_death_types, death_cost: float = -1.0):
        super().__init__(env)
        self.no_death_types, self.death_cost = tuple(no_death_types), float(death_cost)
        self.unwrapped.set_no_death(self.no_death_types, self.death_cost)

    def remove(self):
        self.unwrapped.set_no_death(())


class ActionBonus(_RewardWrapper):
    def __init__(self, env):
        super().__init__(env)
        self.unwrapped.set_bonus("action")

    def remove(self):
        self.unwrapped.set_bonus(None)


class PositionBonus(_RewardWrapper):
    def __init__(self, env, scale=1):
        super().__init__(env)
        self.scale = 1  # as the reference: the argument is ignored (wrappers.py:157)
        self.unwrapped.set_bonus("position")

    def remove(self):
        self.unwrapped.set_bonus(None)


class ImgObsWrapper(_VecWrapper):
    def observation(self, obs):
        return obs["image"]


class FullyObsWrapper(_VecWrapper):
    def __init__(self, env):
        super().__init__(env)
        base = self.unwrapped
        self._full = torch.empty((base.num_envs, base.width, base.height, 3), dtype=torch.uint8, device=base.device)

    def observation(self, obs):
        self.unwrapped.full_obs(out=self._full)
        return {**obs, "image": self._full}


class _DeviceObsWrapper(_VecWrapper):
    """Shared plumbing: the wrapped vector env's handle, stream and a reused output tensor."""

    def _base(self):
        return self.unwrapped

    def _call(self, fn, *args):
        b = self._base()
        with torch.cuda.device(b.device):
            _lib.check(fn(b._h, *args, C.c_void_p(torch.cuda.current_stream(b.device).cuda_stream)))

    @staticmethod
    def _p(t):
        return C.c_void_p(t.data_ptr())


class ViewSizeWrapper(_DeviceObsWrapper):
    def __init__(self, env, agent_view_size=7):
        super().__init__(env)
        if agent_view_size % 2 != 1 or agent_view_size < 3:
            raise ValueError("agent_view_size must be odd and >= 3 (wrappers.py:650-651)")
        if agent_view_size > 15:
            raise ValueError("agent_view_size above 15 is not supported")
        b = self._base()
        self.agent_view_size = agent_view_size
        self._out = torch.empty((b.num_envs, agent_view_size, agent_view_size, 3), dtype=torch.uint8, device=b.device)

    def observation(self, obs):
        self._call(_lib.load().mg_obs_view, self.agent_view_size, self._p(self._out))
        return {**obs, "image": self._out}


class OneHotPartialObsWrapper(_DeviceObsWrapper):
    def __init__(self, env, tile_size=8):
        super().__init__(env)
        self.tile_size = tile_size
        self._out = None

    def observation(self, obs):
        img = obs["image"]
        if self._out is None or self._out.shape[:3] != img.shape[:3]:
            self._out = torch.empty(tuple(img.shape[:3]) + (20,), dtype=torch.uint8, device=img.device)
        self._call(_lib.load().mg_obs_onehot, self._p(img.contiguous()), int(img.shape[1]), self._p(self._out))
        return {**obs, "image": self._out}


def _per_env_missions(b) -> bool:
    """The wrapped env is a BabyAI level whose handle records each env's mission (MinigridVecEnv(..., missions=True))."""
    return bool(getattr(b, "missions_enabled", False)) and specs.is_babyai(b.level_spec)


class FlatObsWrapper(_DeviceObsWrapper):
    def __init__(self, env, maxStrLen=96):
        super().__init__(env)
        b = self._base()
        mission = b.mission
        self._per_env = _per_env_missions(b)
        if self._per_env:  # each env's own mission, one-hot encoded on the device (mg_obs_flat_missions)
            if maxStrLen != 96:
                raise ValueError("per-env missions are encoded with maxStrLen = 96 (the wrapper's default)")
            self.maxStrLen, self._out = maxStrLen, None
            return
        if "{" in mission:
            raise ValueError(f"FlatObsWrapper needs a constant mission string; {b.env_id} draws its mission per episode")
        if len(mission) > maxStrLen:
            raise ValueError(f"mission string too long ({len(mission)} chars)")
        arr = np.zeros((maxStrLen, 28), np.uint8)  # wrappers.py:597-621
        for idx, ch in enumerate(mission.lower()):
            if "a" <= ch <= "z":
                no = ord(ch) - ord("a")
            elif ch == " ":
                no = 26
            elif ch == ",":
                no = 27
            else:
                raise ValueError(f"Character {ch} is not available in mission string.")
            arr[idx, no] = 1
        self._mission = torch.as_tensor(arr.reshape(-1), device=b.device)
        self._out = None

    def observation(self, obs):
        img = obs["image"].contiguous()
        nb = int(np.prod(img.shape[1:]))
        if self._per_env:
            if self._out is None or self._out.shape[1] != nb + 28 * 96:
                self._out = torch.empty((img.shape[0], nb + 28 * 96), dtype=torch.uint8, device=img.device)
            self._call(_lib.load().mg_obs_flat_missions, self._p(img), nb, self._p(self._out))
            return self._out
        if self._out is None or self._out.shape[1] != nb + self._mission.numel():
            self._out = torch.empty((img.shape[0], nb + self._mission.numel()), dtype=torch.uint8, device=img.device)
        self._call(_lib.load().mg_obs_flat, self._p(img), nb, self._p(self._mission), int(self._mission.numel()), self._p(self._out))
        return self._out


MINIGRID_WORDS = (["red", "green", "blue", "yellow", "purple", "grey"]                                         # wrappers.py:475-531
                  + ["unseen", "empty", "wall", "floor", "box", "key", "ball", "door", "goal", "agent", "lava"]
                  + ["pick", "avoid", "get", "find", "put", "use", "open", "go", "fetch", "reach", "unlock", "traverse"]
                  + ["up", "the", "a", "at", ",", "square", "and", "then", "to", "of", "rooms", "near", "opening", "must", "you",
                     "matching", "end", "hallway", "object", "from", "room", "maze"])


def mission_to_indices(mission: str, max_words_in_mission: int = 50, word_dict=None, offset: int = 1):
    """DictObservationSpaceWrapper.string_to_indices + observation (wrappers.py:535-554): word indices + 1, zero padded."""
    wd = word_dict if word_dict is not None else {w: i for i, w in enumerate(MINIGRID_WORDS)}
    idx = []
    for word in mission.replace(",", " , ").split():
        if word not in wd:
            raise ValueError(f"Unknown word: {word}")
        idx.append(wd[word] + offset)
    assert len(idx) < max_words_in_mission
    return idx + [0] * (max_words_in_mission - len(idx))


class DictObservationSpaceWrapper(_DeviceObsWrapper):
    """obs["mission"] as a fixed-length list of vocabulary indices: the same list for every env of the batch when the
    mission string is constant; on a BabyAI level created with missions=True, an int64[n, max_words_in_mission] device
    tensor with each env's own mission. Refused: ids that draw their mission without missions=True, and BabyAI levels
    whose grammar has words outside the vocabulary (the reference raises "Unknown word" on those episodes)."""

    def __init__(self, env, max_words_in_mission=50, word_dict=None):
        super().__init__(env)
        b = self.unwrapped
        self._per_env = _per_env_missions(b)
        if self._per_env:
            unknown = sorted(specs.babyai_mission_words(b.level_spec) - set(MINIGRID_WORDS))
            if unknown:
                raise ValueError(f"{b.env_id}: its missions can contain words outside the Minigrid vocabulary ({', '.join(unknown)})")
            if word_dict is not None:
                raise ValueError("per-env missions are encoded with the Minigrid vocabulary (word_dict=None)")
            if max_words_in_mission <= specs.BABYAI_MISSION_MAX_WORDS:
                raise ValueError(f"max_words_in_mission must exceed {specs.BABYAI_MISSION_MAX_WORDS}, the longest BabyAI mission")
            self.max_words_in_mission = max_words_in_mission
            self.word_dict = {w: i for i, w in enumerate(MINIGRID_WORDS)}
            self._out = torch.empty((b.num_envs, max_words_in_mission), dtype=torch.int64, device=b.device)
            return
        if "{" in b.mission:
            raise ValueError(f"DictObservationSpaceWrapper needs a constant mission string; {b.env_id} draws its mission per episode")
        self.max_words_in_mission = max_words_in_mission
        self.word_dict = word_dict if word_dict is not None else {w: i for i, w in enumerate(MINIGRID_WORDS)}
        self._mission = mission_to_indices(b.mission, max_words_in_mission, self.word_dict)

    def observation(self, obs):
        if self._per_env:
            self._call(_lib.load().mg_mission_indices, self.max_words_in_mission, self._p(self._out))
            return {**obs, "mission": self._out}
        return {**obs, "mission": list(self._mission)}


class SymbolicObsWrapper(_DeviceObsWrapper):
    def __init__(self, env):
        super().__init__(env)
        b = self._base()
        self._out = torch.empty((b.num_envs, b.width, b.height, 3), dtype=torch.int64, device=b.device)

    def observation(self, obs):
        self._call(_lib.load().mg_obs_symbolic, self._p(self._out))
        return {**obs, "image": self._out}


_ATLAS = {}


def _atlas(device):
    """(tiles uint8[T, 8, 8, 3], index uint16 -> int16 storage [128, 5, 2]) on `device`."""
    key = str(device)
    if key not in _ATLAS:
        d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "tile_atlas.npz"))
        tiles = torch.as_tensor(np.ascontiguousarray(d["tiles"]), device=device)
        index = torch.as_tensor(np.ascontiguousarray(d["index"]).view(np.int16), device=device)
        _ATLAS[key] = (tiles, index)
    return _ATLAS[key]


class RGBImgPartialObsWrapper(_DeviceObsWrapper):
    def __init__(self, env, tile_size=8):
        super().__init__(env)
        if tile_size != 8:
            raise ValueError("only tile_size = 8 (TILE_PIXELS / 4 ... the wrapper's default) is baked into the tile atlas")
        b = self._base()
        self.tile_size = tile_size
        self._tiles, self._index = _atlas(b.device)
        self._out = torch.empty((b.num_envs, 56, 56, 3), dtype=torch.uint8, device=b.device)

    def observation(self, obs):
        img = obs["image"]
        if tuple(img.shape[1:]) != (7, 7, 3):
            raise ValueError("RGBImgPartialObsWrapper renders the 7 x 7 view")
        self._call(_lib.load().mg_obs_rgb_partial, self._p(img.contiguous()), self._p(self._tiles), self._p(self._index), self._p(self._out))
        return {**obs, "image": self._out}


class RGBImgObsWrapper(_DeviceObsWrapper):
    def __init__(self, env, tile_size=8):
        super().__init__(env)
        if tile_size != 8:
            raise ValueError("only tile_size = 8 is baked into the tile atlas")
        b = self._base()
        self.tile_size = tile_size
        self._tiles, self._index = _atlas(b.device)
        self._out = torch.empty((b.num_envs, b.height * 8, b.width * 8, 3), dtype=torch.uint8, device=b.device)

    def observation(self, obs):
        img = obs["image"]
        if tuple(img.shape[1:]) != (7, 7, 3):
            raise ValueError("RGBImgObsWrapper takes its highlight from the 7 x 7 view: apply it to the base env")
        self._call(_lib.load().mg_obs_rgb_full, self._p(img.contiguous()), self._p(self._tiles), self._p(self._index), self._p(self._out))
        return {**obs, "image": self._out}
