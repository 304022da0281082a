/*
 * minigrid_b200.h — C-ABI of the H100-native (sm_90a) lockstep-batched Minigrid engine.
 *
 * The reference (Farama-Foundation/Minigrid, pure Python) has no FFI layer; the boundary it implements is
 * the Gymnasium API (MiniGridEnv(gym.Env), minigrid/minigrid_env.py:24) and, batched, gymnasium.vector's
 * VectorEnv as used in tests/test_envs.py:328-340. Each entry point below cites the reference interface
 * it replaces for a whole batch of environments. All file:line citations are relative to
 * /root/reference/minigrid/.
 *
 * Conventions
 *  - plain C types only; every function returns MG_OK (0) or a negative MG_ERR_* code and records a
 *    message retrievable with mg_last_error() (thread-local).
 *  - `*_dev` pointers are device memory on the handle's GPU, owned by the caller (torch tensors in the
 *    Python host layer); `*_host` pointers are host memory. The library owns only its state arena.
 *  - device work is enqueued on the caller's `stream` (a cudaStream_t passed as void*) and is
 *    asynchronous; the *_host entry points run on a private stream of the handle, which is first ordered after
 *    the work already enqueued on the last caller stream that touched the handle, and synchronise before
 *    returning. mg_seed (host seed array) and mg_set_state with agent records (range validation) also synchronise.
 *  - a handle is bound to one device; one host thread per handle. Distinct handles may run concurrently.
 *    Every entry point selects the handle's device and restores the calling thread's current device on return.
 *  - device kernels cannot raise: an action outside 0..6 (ValueError at minigrid_env.py:584-585) sets a
 *    sticky device error word, reported by mg_check_error() / the *_host calls.
 */
#ifndef MINIGRID_B200_H
#define MINIGRID_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MG_OK 0
#define MG_ERR_INVALID_ARG (-1)
#define MG_ERR_CUDA (-2)
#define MG_ERR_INVALID_ACTION (-3)
#define MG_ERR_NO_DEVICE (-4)

/* generators (envs/empty.py, doorkey.py, crossing.py, fourrooms.py; round-1 widening: lavagap.py, distshift.py) */
#define MG_KIND_EMPTY 0
#define MG_KIND_DOORKEY 1
#define MG_KIND_CROSSING 2
#define MG_KIND_FOURROOMS 3
#define MG_KIND_LAVAGAP 4   /* envs/lavagap.py */
#define MG_KIND_DISTSHIFT 5 /* envs/distshift.py */
#define MG_KIND_MULTIROOM 6 /* envs/multiroom.py (up to 6 rooms) */
#define MG_KIND_LOCKEDROOM 7 /* envs/lockedroom.py (square, 13 <= size <= 26) */
#define MG_KIND_PLAYGROUND 8 /* envs/playground.py (19 x 19) */
/* generator + step post-filter */
#define MG_KIND_GOTODOOR 9      /* envs/gotodoor.py */
#define MG_KIND_FETCH 10        /* envs/fetch.py: params {numObjs} */
#define MG_KIND_REDBLUEDOORS 11 /* envs/redbluedoors.py: width = 2 * height */
#define MG_KIND_GOTOOBJECT 12   /* envs/gotoobject.py: params {numObjs} */
#define MG_KIND_PUTNEAR 13      /* envs/putnear.py: params {numObjs} */
#define MG_KIND_MEMORY 14       /* envs/memory.py: params {random_length}; odd height */
/* RNG draws inside step */
#define MG_KIND_ROOMGRID 16     /* core/roomgrid.py + envs/unlock.py, unlockpickup.py, blockedunlockpickup.py, keycorridor.py:
                                   obstructedmaze.py, obstructedmaze_v1.py: params {variant (0 Unlock, 1 UnlockPickup,
                                   2 BlockedUnlockPickup, 3 KeyCorridor, 4 ObstructedMaze_1Dlhb, 5 ObstructedMaze_Full,
                                   6 ObstructedMaze_Full_V1), room_size, num_rows, num_cols[, key_in_box, blocked,
                                   agent_room_i | agent_room_j << 4, num_quarters]};
                                   envs/babyai/goto.py, the one-room GoTo levels: {7, room_size 4..8, 1, 1, level
                                   (0 GoToRedBallGrey, 1 GoToRedBall, 2 GoToObj, 3 GoToLocal, 4 GoToRedBlueBall), num_dists}
                                   with at most 8 objects that the room can hold away from the agent; max_steps is
                                   room_size^2 for the registered ids;
                                   envs/babyai/other.py (OneRoomS*), pickup.py (PickupDist), putnext.py (PutNextLocal):
                                   {8, room_size, 1, 1, level (0 OneRoom, 1 PickupDist, 2 PutNextLocal), num_objs, strict}
                                   with room_size 4..20 for OneRoom and 4..8 otherwise, num_objs 1 for OneRoom and >= 2 for
                                   PutNextLocal, the same object capacity as GoTo, and strict (PickupInstr's) only on
                                   PickupDist; max_steps is room_size^2 (OneRoom, PickupDist) or 2 room_size^2 (PutNextLocal)
                                   for the registered ids */
#define MG_KIND_DYNOBS 15       /* envs/dynamicobstacles.py: params {n_obstacles, random_start, start_x, start_y, start_dir} */

/* gymnasium.vector.AutoresetMode */
#define MG_AUTORESET_NEXT_STEP 0
#define MG_AUTORESET_SAME_STEP 1
#define MG_AUTORESET_DISABLED 2

/* dtype of the action buffer handed to mg_step */
#define MG_ACT_I32 0
#define MG_ACT_I64 1
#define MG_ACT_U8 2

#define MG_VIEW 7                 /* agent_view_size (minigrid_env.py:42) */
#define MG_OBS_BYTES (7 * 7 * 3)  /* one "image" (minigrid_env.py:72-77) */

typedef struct mg_env mg_env;

/* Replaces: constructing n_envs MiniGridEnv objects (minigrid_env.py:34-117) of one registered id
 * (minigrid/__init__.py). kind/width/height/max_steps/see_through_walls are the constructor arguments;
 * params: EMPTY {random_start, start_x, start_y, start_dir}; CROSSING {num_crossings, obstacle_type
 * (9 lava | 2 wall)}; LAVAGAP {obstacle_type}; DISTSHIFT {strip2_row, start_x, start_y, start_dir};
 * MULTIROOM {minNumRooms, maxNumRooms, maxRoomSize}; others (DOORKEY, FOURROOMS, LOCKEDROOM, PLAYGROUND) none.
 * device < 0 selects the current CUDA device. */
int mg_create(int kind, int width, int height, int max_steps, int see_through_walls,
              const int32_t *params, int n_params, int64_t n_envs, int autoreset_mode, int device,
              mg_env **out);
int mg_destroy(mg_env *env);
const char *mg_last_error(void);

int64_t mg_num_envs(const mg_env *env);
/* total kernels this handle has launched so far (bench.py's gpu_launches) */
int64_t mg_launch_count(const mg_env *env);

/* Replaces: gym.Env.reset(seed=s) -> np_random = Generator(PCG64(SeedSequence(s))) (minigrid_env.py:125,
 * gymnasium.utils.seeding.np_random). SeedSequence hashing runs on the device. seeds_host: uint64[n]. */
int mg_seed(mg_env *env, const uint64_t *seeds_host, void *stream);
/* env i gets seed base_seed + i (gymnasium.vector seed convention: reset(seed=int)) */
int mg_seed_base(mg_env *env, uint64_t base_seed, void *stream);

/* Replaces: MiniGridEnv.reset() for every env (minigrid_env.py:119-157): _gen_grid, carrying=None,
 * step_count=0, gen_obs. RNG streams continue unless mg_seed* was called first.
 * obs_dev: uint8[n][7][7][3]; dir_dev: int32[n]. Either may be NULL. */
int mg_reset(mg_env *env, uint8_t *obs_dev, int32_t *dir_dev, void *stream);

/* Replaces: gymnasium >= 1.1 VectorEnv.reset(seed=..., options={"reset_mask": mask}) (SyncVectorEnv.reset): only the
 * envs with mask_dev[i] != 0 (uint8[n]) are re-seeded / reset; the others keep their state, their NEXT_STEP autoreset
 * flag and their slots of obs_dev / dir_dev. mg_seed_masked: seeds_host uint64[n] (entries of unselected envs are
 * ignored) or NULL for base_seed + i. */
int mg_seed_masked(mg_env *env, const uint8_t *mask_dev, const uint64_t *seeds_host, uint64_t base_seed, void *stream);
int mg_reset_masked(mg_env *env, const uint8_t *mask_dev, uint8_t *obs_dev, int32_t *dir_dev, void *stream);

/* Replaces: MiniGridEnv.step(action) (minigrid_env.py:525-595) + gen_obs (:597-650) for every env, with
 * gymnasium.vector.SyncVectorEnv autoreset semantics (mode given at mg_create).
 * actions_dev: n actions of dtype action_dtype; obs_dev uint8[n][7][7][3]; dir_dev int32[n];
 * reward_dev float64[n]; terminated_dev / truncated_dev uint8[n] (0/1). The output pointers need no alignment beyond
 * their element type's: obs_dev may start at any byte (e.g. step t of a rollout buffer, rollout_obs + t * n * 147); a
 * 16-byte aligned obs_dev lets full tiles leave through one bulk store, any other goes through a byte copy. */
int mg_step(mg_env *env, const void *actions_dev, int action_dtype, uint8_t *obs_dev, int32_t *dir_dev,
            double *reward_dev, uint8_t *terminated_dev, uint8_t *truncated_dev, void *stream);

/* Replaces: MiniGridEnv.gen_obs() (minigrid_env.py:634-650) for every env: the observation of the current
 * state, no transition, state untouched. */
int mg_gen_obs(mg_env *env, uint8_t *obs_dev, int32_t *dir_dev, void *stream);

/* Same two calls with HOST buffers (the end-to-end path: H2D of actions and D2H of every output happen
 * inside the call, through pinned staging owned by the handle; returns after the results are on the host).
 * actions_host: int32[n]. Returns MG_ERR_INVALID_ACTION if any action was outside 0..6. */
int mg_reset_host(mg_env *env, uint8_t *obs_host, int32_t *dir_host);
int mg_step_host(mg_env *env, const int32_t *actions_host, uint8_t *obs_host, int32_t *dir_host,
                 double *reward_host, uint8_t *terminated_host, uint8_t *truncated_host);

/* How the *_host calls bring the results to the host. MG_HOST_FULL: the arrays cross PCIe as they are
 * (161 B per env-step). MG_HOST_PACKED: 52 B per env-step cross (49 one-byte cell codes of the view, one byte
 * direction | terminated | truncated | goal, the step count the reward is a function of) and are expanded by
 * n_threads host threads (0 = all the process may use) into the same arrays, bit-identical: the (type, colour, state)
 * table and the reward table `1 - 0.9 * (step_count / max_steps)` (minigrid_env.py:240-245) are host-computed in
 * both formats. mg_host_d2h_bytes: device-to-host bytes of one mg_step_host call in the current format. */
#define MG_HOST_FULL 0
#define MG_HOST_PACKED 1
int mg_set_host_format(mg_env *env, int format, int n_threads);
/* The host-side expansion itself (host code, no device work), for callers that move the packed records themselves:
 * packed uint8[n][52] -> obs uint8[n][7][7][3], dir int32[n], reward float64[n], terminated / truncated uint8[n]
 * (any output may be NULL). Single-threaded: split n over threads by offsetting the pointers. */
int mg_expand_packed(const uint8_t *packed, int64_t n_envs, int32_t max_steps, uint8_t *obs, int32_t *dir,
                     double *reward, uint8_t *terminated, uint8_t *truncated);
/* the same on n_threads host threads (0 = all the process may use); one call at a time per process */
int mg_expand_packed_mt(const uint8_t *packed, int64_t n_envs, int32_t max_steps, uint8_t *obs, int32_t *dir,
                        double *reward, uint8_t *terminated, uint8_t *truncated, int n_threads);
int64_t mg_host_d2h_bytes(const mg_env *env);
int mg_host_threads(const mg_env *env);

/* Replaces: FullyObsWrapper.observation (wrappers.py:419-426): grid.encode() with the agent cell set to
 * (10, 0, agent_dir). out_dev: uint8[n][W][H][3]. */
int mg_full_obs(mg_env *env, uint8_t *out_dev, void *stream);

/* Replaces: MiniGridEnv.hash (minigrid_env.py:159-170) for every env, before its truncation to `size` hex digits:
 * digest_dev uint8[n][32] = SHA-256(str(grid.encode().tolist()) + str(agent_pos) + str(agent_dir)). Reads the grid and
 * the agent records only; ordered on `stream` like every other entry point.
 * str(agent_pos) depends on how the reference last assigned agent_pos, and the engine reproduces that rule:
 *  - after a forward move that succeeded since the last reset (minigrid_env.py:553, tuple(agent_pos + dir_vec)), and
 *    after mg_set_state with agent records: a tuple of numpy ints, "(np.int64(3), np.int64(12))";
 *  - otherwise the form the kind's generator leaves: a tuple of ints "(1, 1)" for the fixed starts (empty.py:109,
 *    distshift.py:115, dynamicobstacles.py:123), numpy's str(ndarray) "[ 3 10]" for crossing.py:141, lavagap.py:110
 *    and memory.py:129, and a tuple of numpy ints for every generator that calls place_agent / place_obj
 *    (minigrid_env.py:347-350, 383-395).
 * The "moved" state is not part of mg_get_state's output. */
int mg_hash(mg_env *env, uint8_t *digest_dev, void *stream);

/* The reference's observation wrappers (minigrid/wrappers.py) for the whole batch, on the device. `image_dev` is the
 * observation image the last mg_step / mg_reset / mg_gen_obs wrote (uint8[n][V][V][3]).
 *  mg_obs_view         ViewSizeWrapper.observation (:663-673): gen_obs with agent_view_size = view_size (odd, 3..15);
 *                      out_dev uint8[n][V][V][3]
 *  mg_obs_onehot       OneHotPartialObsWrapper.observation (:268-284): out_dev uint8[n][V][V][20]
 *  mg_obs_flat         FlatObsWrapper.observation (:589-626): out_dev uint8[n][image_bytes + mission_bytes], the image
 *                      followed by the one-hot mission characters (mission_dev: uint8[mission_bytes], the same for
 *                      every env: only ids with a constant mission string)
 *  mg_obs_symbolic     SymbolicObsWrapper.observation (:762-782): out_dev int64[n][W][H][3] = (x, y, type | -1), the
 *                      agent's cell carries OBJECT_TO_IDX["agent"]
 *  mg_obs_rgb_partial  RGBImgPartialObsWrapper.observation (:371-380), tile_size 8: out_dev uint8[n][56][56][3]
 *  mg_obs_rgb_full     RGBImgObsWrapper.observation (:325-331), tile_size 8: out_dev uint8[n][8 H][8 W][3]; image_dev
 *                      supplies the highlight (the visible cells of the agent's view)
 * tiles_dev uint8[T][8][8][3] and index_dev uint16[128][5][2] (cell code, 0 no agent | 1 + agent_dir, highlight) are the
 * tile atlas rendered once by the reference's Grid.render_tile (grid.py:145-198; minigrid_b200/data/tile_atlas.npz). */
int mg_obs_view(mg_env *env, int view_size, uint8_t *out_dev, void *stream);
int mg_obs_onehot(mg_env *env, const uint8_t *image_dev, int view_size, uint8_t *out_dev, void *stream);
int mg_obs_flat(mg_env *env, const uint8_t *image_dev, int image_bytes, const uint8_t *mission_dev, int mission_bytes,
                uint8_t *out_dev, void *stream);
int mg_obs_symbolic(mg_env *env, int64_t *out_dev, void *stream);
int mg_obs_rgb_partial(mg_env *env, const uint8_t *image_dev, const uint8_t *tiles_dev, const uint16_t *index_dev,
                       uint8_t *out_dev, void *stream);
int mg_obs_rgb_full(mg_env *env, const uint8_t *image_dev, const uint8_t *tiles_dev, const uint16_t *index_dev,
                    uint8_t *out_dev, void *stream);

/* Replaces: pickling / inspecting env objects (tests/test_envs.py:185-195) and lets tests inject states.
 * grid_dev: Grid.encode() uint8[n][W][H][3]; agent_dev: int32[n][6] {x, y, dir, carry_type (-1 none),
 * carry_color, step_count}; rng_dev: uint64[n][6] {state_hi, state_lo, inc_hi, inc_lo, has_uint32,
 * uinteger} (numpy PCG64 bit-generator state); pending_dev: uint8[n] NEXT_STEP autoreset flags.
 * Any pointer may be NULL. mg_set_state validates agent records (0 <= x < W, 0 <= y < H, 0 <= dir <= 3,
 * carry_type in {-1, 5 key, 6 ball, 7 box}, carry_color 0..5, step_count >= 0): records that fail are left
 * unchanged and the call returns MG_ERR_INVALID_ARG. */
int mg_get_state(mg_env *env, uint8_t *grid_dev, int32_t *agent_dev, uint64_t *rng_dev,
                 uint8_t *pending_dev, void *stream);
int mg_set_state(mg_env *env, const uint8_t *grid_dev, const int32_t *agent_dev, const uint64_t *rng_dev,
                 const uint8_t *pending_dev, void *stream);

/* The reference's reward wrappers, as a SyncVectorEnv of wrapped envs applies them (they change `terminated`, so they
 * live inside the step and its autoreset, not behind it). Order: the bonus wrapper is the outermost.
 *   mg_set_no_death  NoDeath(env, no_death_types, death_cost) (wrappers.py:809-882): type_mask bit t set = the
 *                    OBJECT_TO_IDX type t (constants.py:25-37: 2 wall, 4 door, 5 key, 6 ball, 7 box, 9 lava ...) is a
 *                    death cell; a step that terminated while moving into / standing on such a cell returns
 *                    terminated = False and reward + death_cost, and the episode goes on. Bit 8 (goal) is refused
 *                    (the wrapper's assert, :845). type_mask 0 removes the wrapper.
 *   mg_set_bonus     mode 1: ActionBonus(env) (wrappers.py:68-125), reward += 1 / sqrt(count[(agent_pos, agent_dir,
 *                    action)]); mode 2: PositionBonus(env) (:128-184), reward += 1 / sqrt(count[agent_pos]) (its scale is
 *                    the constant 1, :157); counts are per environment, start at zero when the call is made and live as
 *                    long as the wrapper (they are not cleared by resets, like the wrappers' dicts); mode 0 removes it.
 * Both are incompatible with MG_HOST_PACKED (the packed record carries no reward value). */
int mg_set_no_death(mg_env *env, int type_mask, double death_cost);
int mg_set_bonus(mg_env *env, int mode);

/* Measurement aid (no reference counterpart): while enabled, every K1 (step+obs) launch is bracketed by CUDA
 * events on the launching stream; mg_profile_read synchronises them, returns the summed kernel milliseconds
 * and the number of launches since the last read, and clears the list. */
int mg_profile(mg_env *env, int enable);
int mg_profile_read(mg_env *env, double *total_ms, int64_t *n_launches);

/* Synchronises `stream`, returns MG_ERR_INVALID_ACTION if a kernel saw an action outside 0..6 since the
 * last check (and clears the flag), else MG_OK. */
int mg_check_error(mg_env *env, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* MINIGRID_B200_H */
