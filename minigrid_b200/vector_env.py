"""gymnasium.vector.VectorEnv-shaped surface over the C-ABI (include/minigrid_b200.h).

Replaces, for a whole batch, what `gymnasium.vector.SyncVectorEnv([lambda: gym.make(id)] * n)` does with n
reference `MiniGridEnv` objects (tests/test_envs.py:328-340 of the reference): reset / step with autoreset,
observations {"image": uint8[n,7,7,3], "direction": int32[n], "mission": str} (minigrid_env.py:72-84),
reward float64[n], terminated / truncated bool[n], info {}. Tensors live on the GPU and are reused between
calls (SyncVectorEnv's copy=False convention). `direction` is int32 (gymnasium's Discrete samples int64).
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib, specs

AUTORESET = {"next_step": 0, "same_step": 1, "disabled": 2}
_ACT_DTYPES = {torch.int32: 0, torch.int64: 1, torch.uint8: 2}


def _spaces():
    try:  # a real gymnasium wins when it exists
        from gymnasium import spaces as gs

        return gs.Discrete, gs.MultiDiscrete, gs.Box, gs.Dict, None
    except Exception:
        from . import spaces as s

        return s.Discrete, s.MultiDiscrete, s.Box, s.Dict, s.Text


try:  # subclass the real base class when gymnasium exists (it is not in this image: SURVEY 8c)
    from gymnasium.vector import VectorEnv as _VectorEnvBase
except Exception:  # noqa: BLE001
    _VectorEnvBase = object


class MinigridVecEnv(_VectorEnvBase):
    """Batched MiniGridEnv on one GPU. `seed_offset` is this shard's first global env index (multi-GPU): without an
    explicit seed, env i starts from seed `seed_offset + i`."""

    def __init__(self, env_id: str | None = None, num_envs: int = 1, *, spec: specs.EnvSpec | None = None,
                 device: int | str | torch.device | None = None, autoreset_mode: str = "next_step",
                 seed_offset: int = 0):
        if not torch.cuda.is_available():
            raise _lib.MinigridB200Error("minigrid_b200 needs a CUDA device (H100, sm_90a); there is no CPU path")
        self.level_spec = spec if spec is not None else specs.get(env_id)
        self.env_id = env_id
        self.num_envs = int(num_envs)
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if dev.type != "cuda":
            raise ValueError("device must be a CUDA device")
        self.device = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        self.autoreset_mode = autoreset_mode
        self.metadata = {"autoreset_mode": autoreset_mode}
        self.seed_offset = int(seed_offset)
        self._L = _lib.load()
        prm = (C.c_int32 * max(1, len(self.level_spec.params)))(*self.level_spec.params)
        h = C.c_void_p()
        _lib.check(self._L.mg_create(self.level_spec.kind, self.level_spec.width, self.level_spec.height, self.level_spec.max_steps,
                                     int(self.level_spec.see_through_walls), prm, len(self.level_spec.params), self.num_envs,
                                     AUTORESET[autoreset_mode], self.device.index, C.byref(h)))
        self._h = h
        if self.seed_offset:  # mg_create seeds env i with i: shards of one batch must not hold identical envs
            _lib.check(self._L.mg_seed_base(self._h, C.c_uint64(self.seed_offset), self._stream()))
        n, d = self.num_envs, self.device
        self._image = torch.zeros((n, 7, 7, 3), dtype=torch.uint8, device=d)
        self._direction = torch.zeros(n, dtype=torch.int32, device=d)
        self._reward = torch.zeros(n, dtype=torch.float64, device=d)
        self._terminated = torch.zeros(n, dtype=torch.bool, device=d)
        self._truncated = torch.zeros(n, dtype=torch.bool, device=d)
        self._host = None
        self.host_format = "full"
        self._act_shape = (n,)
        self._mg_step = self._L.mg_step
        self._out_ptrs = tuple(C.c_void_p(t.data_ptr()) for t in
                               (self._image, self._direction, self._reward, self._terminated, self._truncated))
        self._info = {}
        Discrete, MultiDiscrete, Box, Dict, Text = _spaces()
        self.single_action_space = Discrete(7)  # core/actions.py:7-20
        self.action_space = MultiDiscrete([7] * n) if n <= 1 << 16 else MultiDiscrete(np.full(n, 7))
        img = Box(0, 255, (7, 7, 3), np.uint8)
        mission = Text(self.level_spec.mission) if Text is not None else None
        single = {"image": img, "direction": Discrete(4)}
        batched = {"image": Box(0, 255, (n, 7, 7, 3), np.uint8), "direction": MultiDiscrete(np.full(n, 4))}
        if mission is not None:
            single["mission"] = mission
            batched["mission"] = mission
        self.single_observation_space = Dict(single)
        self.observation_space = Dict(batched)
        self.mission = self.level_spec.mission
        self._obs_dict = {"image": self._image, "direction": self._direction, "mission": self.mission}
        self.width, self.height, self.max_steps = self.level_spec.width, self.level_spec.height, self.level_spec.max_steps

    # ---- plumbing ----
    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    @staticmethod
    def _p(t):
        return None if t is None else C.c_void_p(t.data_ptr())

    def _obs(self):
        return {"image": self._image, "direction": self._direction, "mission": self.mission}

    def _as_actions(self, actions):
        if isinstance(actions, torch.Tensor):
            a = actions
            if a.device != self.device:
                a = a.to(self.device, non_blocking=True)
            if a.dtype not in _ACT_DTYPES:
                a = a.to(torch.int32)
        else:
            a = torch.as_tensor(np.ascontiguousarray(actions, dtype=np.int32), device=self.device)
        a = a.contiguous()
        if a.shape != (self.num_envs,):
            raise ValueError(f"actions must have shape ({self.num_envs},), got {tuple(a.shape)}")
        return a

    # ---- VectorEnv API ----
    def _mask(self, mask):
        m = torch.as_tensor(mask)
        if m.shape != (self.num_envs,):
            raise ValueError(f"reset_mask must have shape ({self.num_envs},)")
        return (m != 0).to(device=self.device, dtype=torch.uint8).contiguous()

    def seed(self, seed, mask=None):
        """seed: int -> env i gets seed + seed_offset + i (SyncVectorEnv convention); sequence -> one per env.
        mask (bool[n], optional): only those envs are re-seeded."""
        m = None if mask is None else (mask if isinstance(mask, torch.Tensor) and mask.dtype == torch.uint8 and mask.device == self.device else self._mask(mask))
        if np.isscalar(seed):
            base = C.c_uint64(int(seed) + self.seed_offset)
            if m is None:
                _lib.check(self._L.mg_seed_base(self._h, base, self._stream()))
            else:
                _lib.check(self._L.mg_seed_masked(self._h, self._p(m), None, base, self._stream()))
        else:
            s = np.ascontiguousarray([0 if v is None else v for v in seed] if isinstance(seed, (list, tuple)) else seed,
                                     dtype=np.uint64)
            if s.shape != (self.num_envs,):
                raise ValueError("seed sequence must have one entry per env")
            if m is None:
                _lib.check(self._L.mg_seed(self._h, s.ctypes.data_as(C.c_void_p), self._stream()))
            else:
                _lib.check(self._L.mg_seed_masked(self._h, self._p(m), s.ctypes.data_as(C.c_void_p), C.c_uint64(0), self._stream()))

    def reset(self, *, seed=None, options=None):
        """VectorEnv.reset. options={"reset_mask": bool[n]} (gymnasium >= 1.1 SyncVectorEnv.reset) resets, and seeds,
        only the selected envs; the others keep their state and their slots of the returned buffers."""
        mask = None if not options else options.get("reset_mask")
        with torch.cuda.device(self.device):
            m = None if mask is None else self._mask(mask)
            if seed is not None:
                self.seed(seed, m)
            if m is None:
                _lib.check(self._L.mg_reset(self._h, self._p(self._image), self._p(self._direction), self._stream()))
            else:
                _lib.check(self._L.mg_reset_masked(self._h, self._p(m), self._p(self._image), self._p(self._direction), self._stream()))
                torch.cuda.current_stream(self.device).synchronize()  # m may be a temporary
        return self._obs(), {}

    def step(self, actions):
        # hot path: keep the Python work per call to a few microseconds (the kernel itself takes ~20 us for 262144
        # envs). The C-ABI selects the device itself; output pointers are cached.
        if not (isinstance(actions, torch.Tensor) and actions.device == self.device and actions.dtype in _ACT_DTYPES
                and actions.is_contiguous() and actions.shape == self._act_shape):
            actions = self._as_actions(actions)
        rc = self._mg_step(self._h, actions.data_ptr(), _ACT_DTYPES[actions.dtype], *self._out_ptrs,
                           torch.cuda.current_stream(self.device).cuda_stream)
        if rc:
            _lib.check(rc)
        return self._obs_dict, self._reward, self._terminated, self._truncated, self._info

    def gen_obs(self):
        """MiniGridEnv.gen_obs() for every env (no transition)."""
        with torch.cuda.device(self.device):
            _lib.check(self._L.mg_gen_obs(self._h, self._p(self._image), self._p(self._direction), self._stream()))
        return self._obs()

    def check_actions(self):
        """Synchronises and raises ValueError if any step since the last check saw an action outside 0..6
        (the reference raises at once, minigrid_env.py:584-585; kernels can only set a flag)."""
        _lib.check(self._L.mg_check_error(self._h, self._stream()))

    def close(self):
        if getattr(self, "_h", None):
            self._L.mg_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- host-buffer (end-to-end) path: pinned numpy views in, pinned numpy views out ----
    def _host_buffers(self):
        if self._host is None:
            n = self.num_envs
            pin = lambda shape, dt: torch.zeros(shape, dtype=dt).pin_memory()  # noqa: E731
            self._host = {
                "actions": pin((n,), torch.int32), "image": pin((n, 7, 7, 3), torch.uint8),
                "direction": pin((n,), torch.int32), "reward": pin((n,), torch.float64),
                "terminated": pin((n,), torch.bool), "truncated": pin((n,), torch.bool),
            }
        return self._host

    def set_host_format(self, fmt: str, threads: int = 0):
        """How step_host / reset_host move the results to the host: "full" copies the arrays as they are (161 B per
        env-step over PCIe); "packed" copies 52 B per env-step (cell codes + flags + reward index) and expands them on
        `threads` host threads (0 = all usable) into the same arrays, bit-identical."""
        if fmt not in ("full", "packed"):
            raise ValueError("host format must be 'full' or 'packed'")
        with torch.cuda.device(self.device):
            _lib.check(self._L.mg_set_host_format(self._h, 1 if fmt == "packed" else 0, int(threads)))
        self.host_format = fmt

    @property
    def host_d2h_bytes_per_step(self) -> int:
        return int(self._L.mg_host_d2h_bytes(self._h))

    @property
    def host_threads(self) -> int:
        return int(self._L.mg_host_threads(self._h))

    def reset_host(self, *, seed=None):
        hb = self._host_buffers()
        with torch.cuda.device(self.device):
            if seed is not None:
                self.seed(seed)
                torch.cuda.current_stream(self.device).synchronize()
            _lib.check(self._L.mg_reset_host(self._h, self._p(hb["image"]), self._p(hb["direction"])))
        return {"image": hb["image"], "direction": hb["direction"], "mission": self.mission}, {}

    def step_host(self, actions):
        """actions: host int32 array/tensor [n]. Returns host (pinned) tensors; H2D and D2H are inside."""
        hb = self._host_buffers()
        if isinstance(actions, torch.Tensor) and actions.dtype == torch.int32 and actions.is_pinned():
            src = actions
        else:
            hb["actions"].copy_(torch.as_tensor(np.asarray(actions), dtype=torch.int32))
            src = hb["actions"]
        with torch.cuda.device(self.device):
            _lib.check(self._L.mg_step_host(self._h, self._p(src), self._p(hb["image"]), self._p(hb["direction"]),
                                            self._p(hb["reward"]), self._p(hb["terminated"]), self._p(hb["truncated"])))
        obs = {"image": hb["image"], "direction": hb["direction"], "mission": self.mission}
        return obs, hb["reward"], hb["terminated"], hb["truncated"], {}

    # ---- wrappers' data and state exchange ----
    def full_obs(self, out: torch.Tensor | None = None):
        """FullyObsWrapper.observation (wrappers.py:419-426): uint8[n, W, H, 3]."""
        if out is None:
            out = torch.empty((self.num_envs, self.width, self.height, 3), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(self._L.mg_full_obs(self._h, self._p(out), self._stream()))
        return out

    def hash_digest(self, out: torch.Tensor | None = None):
        """MiniGridEnv.hash (minigrid_env.py:159-170) of every env as the raw SHA-256 digest: uint8[n, 32] on the device,
        enqueued on the current stream. The first 8 bytes viewed as int64 make a state key for counting bonuses."""
        if out is None:
            out = torch.empty((self.num_envs, 32), dtype=torch.uint8, device=self.device)
        elif out.shape != (self.num_envs, 32) or out.dtype != torch.uint8 or out.device != self.device or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous uint8 tensor of shape ({self.num_envs}, 32) on {self.device}")
        with torch.cuda.device(self.device):
            _lib.check(self._L.mg_hash(self._h, self._p(out), self._stream()))
        return out

    def hash(self, size: int = 16):
        """[env.hash(size) for every env]: the reference's hex strings, 1 <= size <= 64 (synchronises)."""
        if not 1 <= int(size) <= 64:
            raise ValueError("size must be in 1..64 (a SHA-256 hex digest has 64 digits)")
        d = self.hash_digest().cpu().numpy()
        hexd = np.frombuffer(b"0123456789abcdef", np.uint8)
        txt = np.empty((self.num_envs, 64), np.uint8)
        txt[:, 0::2] = hexd[d >> 4]
        txt[:, 1::2] = hexd[d & 15]
        return np.ascontiguousarray(txt[:, :int(size)]).view(f"S{int(size)}").ravel().astype(str).tolist()

    def get_state(self):
        n, d = self.num_envs, self.device
        st = {
            "grid": torch.empty((n, self.width, self.height, 3), dtype=torch.uint8, device=d),
            "agent": torch.empty((n, 6), dtype=torch.int32, device=d),
            "rng": torch.empty((n, 6), dtype=torch.int64, device=d),
            "pending": torch.empty(n, dtype=torch.uint8, device=d),
        }
        with torch.cuda.device(self.device):
            _lib.check(self._L.mg_get_state(self._h, self._p(st["grid"]), self._p(st["agent"]), self._p(st["rng"]),
                                            self._p(st["pending"]), self._stream()))
        return st

    def set_state(self, grid=None, agent=None, rng=None, pending=None):
        def dev(x, dt):
            if x is None:
                return None
            if isinstance(x, np.ndarray) and x.dtype == np.uint64:
                x = x.view(np.int64)
            return torch.as_tensor(x).to(device=self.device, dtype=dt).contiguous()

        g, a, r, p = dev(grid, torch.uint8), dev(agent, torch.int32), dev(rng, torch.int64), dev(pending, torch.uint8)
        with torch.cuda.device(self.device):
            _lib.check(self._L.mg_set_state(self._h, self._p(g), self._p(a), self._p(r), self._p(p), self._stream()))
            torch.cuda.current_stream(self.device).synchronize()  # g/a/r/p may be temporaries

    # ---- the reference's reward wrappers (they change `terminated`, so they live inside the step: wrappers.py) ----
    OBJECT_TO_IDX = {"unseen": 0, "empty": 1, "wall": 2, "floor": 3, "door": 4, "key": 5, "ball": 6, "box": 7, "goal": 8, "lava": 9, "agent": 10}

    def set_no_death(self, no_death_types=(), death_cost: float = -1.0):
        """NoDeath(env, no_death_types, death_cost) around every env (wrappers.py:809-882); () removes it."""
        assert "goal" not in no_death_types, "goal cannot be a death cell"
        mask = 0
        for t in no_death_types:
            mask |= 1 << self.OBJECT_TO_IDX[t]
        _lib.check(self._L.mg_set_no_death(self._h, mask, float(death_cost)))

    def set_bonus(self, kind):
        """kind: None, "action" (ActionBonus, wrappers.py:68-125) or "position" (PositionBonus, :128-184): a fresh wrapper
        (zeroed per-env counts) around every env, outside NoDeath."""
        with torch.cuda.device(self.device):
            _lib.check(self._L.mg_set_bonus(self._h, {None: 0, "action": 1, "position": 2}[kind]))

    def profile_kernels(self, enable: bool):
        """Bracket every step+obs kernel launch with CUDA events on the launching stream (measurement aid)."""
        _lib.check(self._L.mg_profile(self._h, int(bool(enable))))

    def kernel_time_ms(self):
        """(summed K1 kernel milliseconds, launches) since the last call; synchronises."""
        ms, cnt = C.c_double(0.0), C.c_int64(0)
        _lib.check(self._L.mg_profile_read(self._h, C.byref(ms), C.byref(cnt)))
        return float(ms.value), int(cnt.value)

    @property
    def launch_count(self) -> int:
        return int(self._L.mg_launch_count(self._h))


def shard_range(total_envs: int, rank: int, world_size: int):
    """Contiguous block of the global batch owned by `rank` (SURVEY.md 8e): (first index, count)."""
    base, rem = divmod(total_envs, world_size)
    count = base + (1 if rank < rem else 0)
    first = rank * base + min(rank, rem)
    return first, count


def make_sharded(env_id: str, total_envs: int, rank: int, world_size: int, *, device=None, **kw):
    """One process per GPU: this rank's shard of a `total_envs` batch. Seeds are global-index based, so the
    environments are the same whatever the number of GPUs. No collective is involved."""
    first, count = shard_range(total_envs, rank, world_size)
    return MinigridVecEnv(env_id, count, device=device, seed_offset=first, **kw)
