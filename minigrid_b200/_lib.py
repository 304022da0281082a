"""ctypes binding of the C-ABI in include/minigrid_b200.h. Fails loudly when the CUDA extension is missing:
the engine has no CPU path."""
from __future__ import annotations

import ctypes as C
import os

from . import _build

MG_OK = 0
MG_ERR_INVALID_ACTION = -3

_lib = None

EXPORTS = [
    "mg_create", "mg_destroy", "mg_last_error", "mg_num_envs", "mg_launch_count", "mg_seed", "mg_seed_base",
    "mg_reset", "mg_seed_masked", "mg_reset_masked", "mg_step", "mg_gen_obs", "mg_reset_host", "mg_step_host", "mg_full_obs", "mg_get_state", "mg_set_state",
    "mg_check_error", "mg_profile", "mg_profile_read", "mg_set_host_format", "mg_host_d2h_bytes", "mg_host_threads", "mg_expand_packed", "mg_expand_packed_mt", "mg_obs_view", "mg_obs_onehot", "mg_obs_flat", "mg_obs_symbolic",
    "mg_obs_rgb_partial", "mg_obs_rgb_full", "mg_hash",
    "mg_enable_missions", "mg_get_mission_codes", "mg_mission_text", "mg_mission_indices", "mg_obs_flat_missions",
]


class MinigridB200Error(RuntimeError):
    pass


def load(build_if_missing: bool = True):
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("MINIGRID_B200_LIB") or _build.LIB_PATH  # override: A/B runs of two builds on one box
    if not os.path.exists(path):
        if not build_if_missing:
            raise MinigridB200Error(f"{path} is missing: run `python -m minigrid_b200._build` (needs nvcc)")
        _build.build()
    elif build_if_missing and path == _build.LIB_PATH:
        try:
            _build.build()  # no-op unless a source under csrc/ or the header is newer than the library
        except Exception as exc:  # noqa: BLE001  (no nvcc on this machine: keep the library that is there, loudly)
            import warnings

            warnings.warn(f"minigrid_b200: {path} is older than its sources and could not be rebuilt ({exc})")
    L = C.CDLL(path)
    p, i32, i64, u64 = C.c_void_p, C.c_int, C.c_int64, C.c_uint64
    L.mg_create.argtypes = [i32, i32, i32, i32, i32, p, i32, i64, i32, i32, C.POINTER(p)]
    L.mg_destroy.argtypes = [p]
    L.mg_last_error.restype = C.c_char_p
    L.mg_num_envs.restype = i64
    L.mg_num_envs.argtypes = [p]
    L.mg_launch_count.restype = i64
    L.mg_launch_count.argtypes = [p]
    L.mg_seed.argtypes = [p, p, p]
    L.mg_seed_base.argtypes = [p, u64, p]
    L.mg_reset.argtypes = [p, p, p, p]
    L.mg_seed_masked.argtypes = [p, p, p, u64, p]
    L.mg_reset_masked.argtypes = [p, p, p, p, p]
    L.mg_step.argtypes = [p, p, i32, p, p, p, p, p, p]
    L.mg_step.restype = i32
    L.mg_gen_obs.argtypes = [p, p, p, p]
    L.mg_reset_host.argtypes = [p, p, p]
    L.mg_step_host.argtypes = [p] * 7
    L.mg_full_obs.argtypes = [p, p, p]
    L.mg_hash.argtypes = [p, p, p]
    L.mg_set_host_format.argtypes = [p, i32, i32]
    L.mg_host_d2h_bytes.restype = i64
    L.mg_host_d2h_bytes.argtypes = [p]
    L.mg_host_threads.argtypes = [p]
    L.mg_obs_view.argtypes = [p, i32, p, p]
    L.mg_obs_onehot.argtypes = [p, p, i32, p, p]
    L.mg_obs_flat.argtypes = [p, p, i32, p, i32, p, p]
    L.mg_obs_symbolic.argtypes = [p, p, p]
    L.mg_obs_rgb_partial.argtypes = [p, p, p, p, p, p]
    L.mg_obs_rgb_full.argtypes = [p, p, p, p, p, p]
    L.mg_expand_packed.argtypes = [p, i64, i32, p, p, p, p, p]
    L.mg_expand_packed_mt.argtypes = [p, i64, i32, p, p, p, p, p, i32]
    L.mg_enable_missions.argtypes = [p]
    L.mg_get_mission_codes.argtypes = [p, p, p]
    L.mg_mission_text.argtypes = [p, p, p]
    L.mg_mission_indices.argtypes = [p, i32, p, p]
    L.mg_obs_flat_missions.argtypes = [p, p, i32, p, p]
    L.mg_get_state.argtypes = [p] * 6
    L.mg_set_state.argtypes = [p] * 6
    L.mg_check_error.argtypes = [p, p]
    try:
        L.mg_set_no_death.argtypes = [p, i32, C.c_double]
        L.mg_set_bonus.argtypes = [p, i32]
    except AttributeError:  # an older build loaded through MINIGRID_B200_LIB for an A/B run
        pass
    L.mg_profile.argtypes = [p, i32]
    L.mg_profile_read.argtypes = [p, C.POINTER(C.c_double), C.POINTER(i64)]
    for name in EXPORTS:
        getattr(L, name)  # AttributeError here means the .so does not match include/minigrid_b200.h
    _lib = L
    return L


def check(rc: int):
    if rc == MG_OK:
        return
    msg = load().mg_last_error().decode()
    if rc == MG_ERR_INVALID_ACTION:
        raise ValueError(msg)  # the reference raises ValueError (minigrid_env.py:584-585)
    raise MinigridB200Error(f"minigrid_b200 C-ABI error {rc}: {msg}")
