// mg_common.cuh — device data layout shared by every kernel of the engine.
//
// The reference's per-env object graph (Grid = list[WorldObj|None], minigrid/core/grid.py:35; WorldObj with
// type/color/is_open/is_locked, core/world_object.py:27-43,171-176) becomes:
//
//   cell code (1 byte)   bits 0-3  t4     = OBJECT_TO_IDX type (core/constants.py:25-37) with the door state
//                                           folded in: 4 door open, 11 door closed, 12 door locked
//                        bits 4-6  colour = COLOR_TO_IDX (core/constants.py:20)
//                        bit  7    opaque = !see_behind() (world_object.py:57,164,181), kept redundantly so
//                                           that Grid.process_vis's transparency test is one bit
//   grid tile            32 consecutive envs ("one warp-lane per environment"), word-interleaved:
//                        tile[w][lane] uint32, w < wpe. Lane L's w-th word sits in shared-memory bank L, so
//                        per-lane gathers at lane-specific offsets are conflict-free, and a tile is one
//                        contiguous block that a single TMA bulk copy (cp.async.bulk) stages.
//   per env words        array R: lines y = -ring..H+ring-1 (row-major x bytes, ring lines are grey wall), then
//                        array C: lines x = -ring..W+ring-1 (column-major y bytes): every 7-cell run of the
//                        egocentric view (Grid.slice + rotate_left, grid.py:110-143) is 7 consecutive
//                        bytes of one line of R (facing +-x) or C (facing +-y).
//   agent record         uint4 {x | y<<8, dir | flags<<8, carry code (0 none), step_count}
//   rng record           numpy PCG64 bit-generator state (state, inc, has_uint32, uinteger)
#pragma once
#include <stdint.h>
#ifdef __CUDACC__
#include <cuda_runtime.h>
#define MG_HD __host__ __device__ __forceinline__
#define MG_D __device__ __forceinline__
#else
// Host build of the per-lane logic (tests/host_emu only: a CPU check of the device arithmetic before GPU time
// is spent; never part of the product library). The shim supplies uint4 and the few intrinsics used below.
#include "mg_host_shim.h"
#define MG_HD inline
#define MG_D inline
#endif

namespace mg {

constexpr int VIEW = 7;
constexpr int OBS_BYTES = 147;
constexpr int TILE = 32;                    // envs per tile == lanes per warp
constexpr int OBS_TILE_BYTES = OBS_BYTES * TILE;  // 4704, a multiple of 16
constexpr int OBS_WORDS = 37;               // ceil(147 / 4)
constexpr int MAX_DIM = 26;                 // W, H <= 26 (the OOB bit mask is built in 32 bits)

// core/constants.py:25-37
enum : uint32_t { T_UNSEEN = 0, T_EMPTY = 1, T_WALL = 2, T_FLOOR = 3, T_DOOR = 4, T_KEY = 5, T_BALL = 6,
                  T_BOX = 7, T_GOAL = 8, T_LAVA = 9, T_AGENT = 10, T4_DOOR_CLOSED = 11, T4_DOOR_LOCKED = 12,
                  // Box.contains (world_object.py:273-293) is None everywhere except ObstructedMaze, whose grey boxes hide
                  // the key of a door: t4 = 13 is "a grey box with a key inside", the colour field is the KEY's colour
                  T4_BOX_WITH_KEY = 13 };
enum : uint32_t { C_RED = 0, C_GREEN = 1, C_BLUE = 2, C_PURPLE = 3, C_YELLOW = 4, C_GREY = 5 };
// core/actions.py:7-20
enum : int { A_LEFT = 0, A_RIGHT = 1, A_FORWARD = 2, A_PICKUP = 3, A_DROP = 4, A_TOGGLE = 5, A_DONE = 6 };

constexpr uint32_t OPAQUE_BIT = 0x80u;
constexpr uint32_t CODE_EMPTY = T_EMPTY;
constexpr uint32_t CODE_WALL = T_WALL | (C_GREY << 4) | OPAQUE_BIT;  // 0xD2, Wall() (world_object.py:160-162)
constexpr uint32_t CODE_WALL4 = CODE_WALL * 0x01010101u;
constexpr uint32_t CODE_GOAL = T_GOAL | (C_GREEN << 4);
constexpr uint32_t CODE_LAVA = T_LAVA | (C_RED << 4);

// agent flags (second word of the agent record, bits 8..)
constexpr uint32_t FLAG_PENDING = 2u;  // episode ended last step (SyncVectorEnv._autoreset_envs[i], NEXT_STEP)
// a forward move succeeded since the last reset, or the agent record was injected (mg_set_state): agent_pos is then a
// tuple of numpy ints (minigrid_env.py:553), which MiniGridEnv.hash() prints differently (mg_hash.cuh)
constexpr uint32_t FLAG_MOVED = 1u;

enum : int { KIND_EMPTY = 0, KIND_DOORKEY = 1, KIND_CROSSING = 2, KIND_FOURROOMS = 3, KIND_LAVAGAP = 4, KIND_DISTSHIFT = 5,
             KIND_MULTIROOM = 6,
             // SURVEY 8(f-1) and 8(f-2), next: the generators (mg_levels.cuh) and step post-filters (mg_postfilter.cuh) of
             // the kinds below exist and are checked against the oracle on the CPU (tests/test_oracle_next.py); K1 / K2
             // are not instantiated for them yet and mg_create rejects them (KIND_COUNT)
             KIND_LOCKEDROOM = 7, KIND_PLAYGROUND = 8,
             KIND_GOTODOOR = 9, KIND_FETCH = 10, KIND_REDBLUEDOORS = 11, KIND_GOTOOBJECT = 12, KIND_PUTNEAR = 13,
             KIND_MEMORY = 14,
             // SURVEY 8(f-4): RNG draws inside step (envs/dynamicobstacles.py)
             KIND_DYNOBS = 15,
             // SURVEY 8(f-2), second half: core/roomgrid.py with unlock.py, unlockpickup.py, blockedunlockpickup.py, keycorridor.py
             KIND_ROOMGRID = 16 };
constexpr int KIND_COUNT = 17;
// Kinds whose grids keep grey walls on the whole border: the generator starts with wall_rect(0, 0, W, H) and places
// nothing on the border, there is no step post-filter and no draw inside step (Dynamic-Obstacles re-places its
// obstacles anywhere), and no action changes a wall. K1 then does not stage the border lines of their tiles
// (mg_step_kernel.cuh: stage_lines) while no grid has been injected (mg_set_state).
MG_HD constexpr bool kind_walled(int kind) {
  return kind == KIND_EMPTY || kind == KIND_DOORKEY || kind == KIND_CROSSING || kind == KIND_LAVAGAP || kind == KIND_DISTSHIFT;
}
// kp[0] of KIND_ROOMGRID; the ObstructedMaze variants (envs/obstructedmaze.py, obstructedmaze_v1.py) also read
// kp[4] key_in_box, kp[5] blocked, kp[6] agent room i | j << 4, kp[7] num_quarters
enum : int { RG_UNLOCK = 0, RG_UNLOCKPICKUP = 1, RG_BLOCKEDUNLOCKPICKUP = 2, RG_KEYCORRIDOR = 3, RG_OBSTRUCTED_1D = 4,
             RG_OBSTRUCTED_FULL = 5, RG_OBSTRUCTED_FULL_V1 = 6,
             // the single-room BabyAI GoTo levels (envs/babyai/goto.py): kp = {7, room_size, 1, 1, level, num_dists}
             RG_BABYAI_GOTO = 7,
             // the single-room BabyAI Pickup and PutNext levels (envs/babyai/other.py, pickup.py, putnext.py):
             // kp = {8, room_size, 1, 1, level, num_objs, strict}
             RG_BABYAI_PICKUP_PUTNEXT = 8,
             // the BabyAI Open and UnlockLocal levels (envs/babyai/open.py, unlock.py):
             // kp = {9, room_size, num_rows, num_cols, level, arg, strict}
             RG_BABYAI_OPEN = 9,
             // the BabyAI levels that span a maze of rooms joined by connect_all (envs/babyai/goto.py GoTo with one
             // object, other.py FindObjS5 and KeyCorridor): kp = {10, room_size, num_rows, num_cols, level, arg}
             RG_BABYAI_MAZE = 10 };  // kinds mg_create accepts: the kernels are instantiated for the kinds below this
MG_HD bool rg_obstructed(int variant) { return variant >= RG_OBSTRUCTED_1D && variant <= RG_OBSTRUCTED_FULL_V1; }
// kp[4] of RG_BABYAI_GOTO: GoToRedBallGrey, GoToRedBall(NoDists), GoToObj, GoToLocal, GoToRedBlueBall
enum : int { BABYAI_REDBALL_GREY = 0, BABYAI_REDBALL = 1, BABYAI_OBJ = 2, BABYAI_LOCAL = 3, BABYAI_REDBLUEBALL = 4 };
// kp[4] of RG_BABYAI_PICKUP_PUTNEXT: OneRoomS*, PickupDist(Debug), PutNextLocal*
enum : int { BABYAI_ONEROOM = 0, BABYAI_PICKUPDIST = 1, BABYAI_PUTNEXTLOCAL = 2 };
// level_aux of a Pickup level: which parts of ObjDesc(type, colour) are set, and PickupInstr's strict flag
enum : uint32_t { PICK_TYPE = 1u, PICK_COLOR = 2u, PICK_STRICT = 4u };
// kp[4] of RG_BABYAI_OPEN; kp[5] is OpenDoor's select_by (0 colour, 1 loc, 2 drawn), OpenTwoDoors' fixed red / blue
// colours (0 or 1), OpenDoorsOrder's num_doors (2..4) or UnlockLocal's distractors (0 or 1); kp[6] strict / debug
enum : int { BABYAI_OPENREDDOOR = 0, BABYAI_OPENDOOR = 1, BABYAI_OPENTWODOORS = 2, BABYAI_OPENDOORSORDER = 3,
             BABYAI_UNLOCKLOCAL = 4 };
// level_aux of an Open level. level_tx / level_ty are the doors the first / second OpenInstr's obj_set holds, as a mask
// of door colours (every door of these levels has a colour of its own); OPEN_SEQ: two OpenInstrs in sequence (an
// AfterInstr is stored with its two instructions swapped), OPEN_STRICT1 / 2: their strict flags; OPEN_DONE: the first
// has succeeded (BeforeInstr.a_done / AfterInstr.b_done), the one bit K1 changes during an episode
enum : uint32_t { OPEN_SEQ = 1u, OPEN_STRICT1 = 2u, OPEN_STRICT2 = 4u, OPEN_DONE = 8u };
// kp[4] of RG_BABYAI_MAZE: GoToObjMaze* (kp[5] = doors_open), FindObjS*, KeyCorridor* (MiniGrid KeyCorridor's generator)
enum : int { BABYAI_MAZE_GOTO = 0, BABYAI_FINDOBJ = 1, BABYAI_MAZE_KEYCORRIDOR = 2 };
// KeyCorridor's generator: the MiniGrid level, or the BabyAI level that makes the same draws
MG_HD bool rg_keycorridor(const int *kp) {
  return kp[0] == RG_KEYCORRIDOR || (kp[0] == RG_BABYAI_MAZE && kp[4] == BABYAI_MAZE_KEYCORRIDOR);
}
// Mission code of a BabyAI level (Params::mission, one word per env, written by every reset when the handle asked for
// missions): the instruction that RoomGridLevel._gen_grid turns into self.mission = self.instrs.surface(self)
// (babyai/core/roomgrid_level.py:142-144), rendered back into text by mission_words (mg_mission.cuh).
//   bits  0-2   form: MIS_CONST the spec's constant string (every id that is not a BabyAI level), MIS_GOTO "go to A",
//               MIS_PICKUP "pick up A", MIS_OPEN "open A", MIS_PUTNEXT "put A next to B", MIS_BEFORE "open A, then open B"
//               (BeforeInstr), MIS_AFTER "open A after you open B" (AfterInstr, in the reference's surface order:
//               instr_a first, although level_tx / level_ty hold it swapped)
//   bits  3-12  ObjDesc A, bits 13-22 ObjDesc B, 10 bits each (verifier.py:44-100):
//               type:3   0 none ("object"), 1 key, 2 ball, 3 box, 4 door
//               colour:3 0 none, 1 + COLOR_TO_IDX
//               loc:3    0 none, 1 left, 2 right, 3 front, 4 behind (LOC_NAMES order)
//               plural:1 len(obj_set) > 1 at reset: "a" instead of "the"
//   bits 23-31  zero (forms 7 and up and these bits are free for missions of other levels)
enum : uint32_t { MIS_CONST = 0, MIS_GOTO = 1, MIS_PICKUP = 2, MIS_OPEN = 3, MIS_PUTNEXT = 4, MIS_BEFORE = 5, MIS_AFTER = 6 };
enum : uint32_t { MIS_TYPE_NONE = 0, MIS_TYPE_KEY = 1, MIS_TYPE_BALL = 2, MIS_TYPE_BOX = 3, MIS_TYPE_DOOR = 4 };
enum : uint32_t { MIS_LOC_NONE = 0, MIS_LOC_LEFT = 1, MIS_LOC_RIGHT = 2, MIS_LOC_FRONT = 3, MIS_LOC_BEHIND = 4 };
// one ObjDesc: type MIS_TYPE_*, colour COLOR_TO_IDX or -1 for none, loc MIS_LOC_*
MG_HD uint32_t mission_desc(uint32_t type, int color, uint32_t loc, bool plural) {
  return type | ((color < 0 ? 0u : (uint32_t)color + 1u) << 3) | (loc << 6) | ((plural ? 1u : 0u) << 9);
}
MG_HD uint32_t mission_code(uint32_t form, uint32_t a, uint32_t b) { return form | (a << 3) | (b << 13); }
enum : int { AUTORESET_NEXT_STEP = 0, AUTORESET_SAME_STEP = 1, AUTORESET_DISABLED = 2 };
// bits of the sticky device error word (Params::err)
enum : int { ERR_BAD_ACTION = 1, ERR_BAD_STATE = 2, ERR_PACKED_RANGE = 4 };

// (type, colour, state) -> cell code. None/unseen/agent all mean "no object" (WorldObj.decode,
// world_object.py:77-78) and encode as (1,0,0) (grid.py:258-261).
MG_HD uint32_t encode_cell(uint32_t type, uint32_t color, uint32_t state) {
  if (type == T_EMPTY || type == T_UNSEEN || type >= T_AGENT) return CODE_EMPTY;
  uint32_t t4 = type, opaque = 0;
  if (type == T_DOOR) {
    t4 = state == 0 ? (uint32_t)T_DOOR : (state == 1 ? (uint32_t)T4_DOOR_CLOSED : (uint32_t)T4_DOOR_LOCKED);
    opaque = state != 0;
  } else if (type == T_WALL) {
    opaque = 1;
  }
  return t4 | ((color & 7u) << 4) | (opaque << 7);
}
// cell code -> type | colour << 8 | state << 16 (WorldObj.encode / Door.encode, world_object.py:65-67,196-212)
MG_HD uint32_t decode_cell(uint32_t code) {
  uint32_t t4 = code & 15u, color = (code >> 4) & 7u;
  if (t4 == T_UNSEEN) return 0;
  if (t4 == T_EMPTY) return T_EMPTY;
  if (t4 == T4_DOOR_CLOSED) return T_DOOR | (color << 8) | (1u << 16);
  if (t4 == T4_DOOR_LOCKED) return T_DOOR | (color << 8) | (2u << 16);
  if (t4 == T4_BOX_WITH_KEY) return T_BOX | (C_GREY << 8);  // what is inside does not show (Box.encode is WorldObj.encode)
  return t4 | (color << 8);
}

// Two HBM layouts of the per-env words (same words, same r_word / c_word indices):
//   LAYOUT_TILED   tile[w][lane] for 32 consecutive envs (small grids): one TMA bulk copy stages a whole tile and
//                  per-lane gathers are bank-conflict free.
//   LAYOUT_WINDOW  env-major, lines of ceil(W / 4) words, 3 ring lines (large grids): a step only touches the 7 lines of
//                  the egocentric view, contiguous in one array, which each lane gathers straight into registers;
//                  HBM traffic per env-step grows with the grid's side, not its area.
enum : int { LAYOUT_TILED = 0, LAYOUT_WINDOW = 1 };
constexpr int WIN_LANE_BYTES = 240; // (host emulation of the round-1 window staging only)

struct Geom {
  int W, H;
  int lswR, lswC;  // words per line of R / C
  int ring;        // wall lines stored before line 0 and after the last line of each array
  int offC;        // word offset of array C inside an env
  int wpe;         // words per env
  int layout;
};

MG_HD Geom make_geom(int W, int H, int layout) {
  Geom g;
  g.W = W; g.H = H; g.layout = layout;
  if (layout == LAYOUT_TILED) { g.lswR = (W + 3) >> 2; g.lswC = (H + 3) >> 2; g.ring = 1; }
  else { g.lswR = (W + 3) >> 2; g.lswC = (H + 3) >> 2; g.ring = 3; }  // lines as wide as the grid: a step's 7 lines are 7 * lsw words
  g.offC = (H + 2 * g.ring) * g.lswR;
  g.wpe = g.offC + (W + 2 * g.ring) * g.lswC;
  if (layout != LAYOUT_TILED) {  // both arrays of every env start on 16 bytes (K3 stages array C with bulk copies)
    g.offC = (g.offC + 3) & ~3;
    g.wpe = (g.offC + (W + 2 * g.ring) * g.lswC + 3) & ~3;
  }
  return g;
}
// index in the grid arena (in words) of word w of environment env
MG_HD size_t grid_word(const Geom &g, int env, int w) {
  return g.layout == LAYOUT_TILED ? ((size_t)(env >> 5) * g.wpe + w) * 32 + (env & 31) : (size_t)env * g.wpe + w;
}

struct RngRec {  // 48 bytes, 16-byte aligned
  uint64_t state_hi, state_lo, inc_hi, inc_lo;
  uint32_t has_uint32, uinteger;
  uint64_t pad;
};

struct Params {
  Geom g;
  int n_envs, n_tiles;
  int max_steps, see_through, mode, kind;
  int kp[8];                // generator parameters (see include/minigrid_b200.h)
  uint32_t *grid;           // n_tiles * 32 * wpe words, see grid_word()
  uint4 *agent;             // [n_tiles * 32]
  // [n_tiles * 32] KIND_DYNOBS: the obstacles in list order, 16 bits each (x | y << 8); KIND_ROOMGRID: the mission codes
  // (mission_codes()), null unless mg_enable_missions. One slot for both: Params is every kernel's by-value argument,
  // and a field of its own would move the parameters of every kernel
  uint4 *extra;
  RngRec *rng;              // [n_tiles * 32]
  const double *reward_lut; // [max_steps + 1], 1 - 0.9 * (k / max_steps) computed on the host in IEEE double
  const uint32_t *cell_lut; // [256] decode_cell()
  const uint16_t *vis_tbl;  // [128 * 128] process_vis row table (mg_obs.cuh: build_vis_table)
  const uint32_t *tmpl;     // [wpe] level template: the words of a blank draw (mg_levels.cuh)
  int *err;                 // sticky error word
  int hot_first;            // visit the tiles flagged in tile_hot right after a CTA's first round (MINIGRID_B200_HOTFIRST=0 turns it off)
  uint8_t *tile_hot;        // [n_tiles] 1 = an env of the tile ended in the last step (K1's scheduling hint, never semantics)
  int win_prefetch;         // LAYOUT_WINDOW: L2-prefetch the next tile's view lines (MINIGRID_B200_WINPREF=0 turns it off)
  // the reference's reward wrappers around every env (wrappers.py:68-184, 809-882), 0 = absent
  int no_death_mask;        // NoDeath: bit t = OBJECT_TO_IDX type t is a death cell
  int bonus_mode;           // 1 ActionBonus, 2 PositionBonus
  double death_cost;        // NoDeath.death_cost
  uint32_t *counts;         // [n_envs][W * H * 28] (ActionBonus) or [n_envs][W * H] (PositionBonus): the wrappers' self.counts
};

// KIND_ROOMGRID: one mission code (MIS_*) per env, written by every reset; null unless the handle asked for missions
MG_HD uint32_t *mission_codes(const Params &p) { return reinterpret_cast<uint32_t *>(p.extra); }

struct StepPlan {  // launch shape of K1, chosen once per handle (mg_step.cu: configure_step)
  int warps, vis, nbuf, mode, ctas_per_sm, grid;
  size_t smem;
};

// word index of byte (line, pos) and helpers for the interleaved tile
MG_HD int r_word(const Geom &g, int x, int y) { return (y + g.ring) * g.lswR + (x >> 2); }
MG_HD int c_word(const Geom &g, int x, int y) { return g.offC + (x + g.ring) * g.lswC + (y >> 2); }
// byte offsets in the grid arena of cell (x, y) in the two arrays
MG_HD size_t cell_byte_R(const Geom &g, int env, int x, int y) { return grid_word(g, env, r_word(g, x, y)) * 4 + (x & 3); }
MG_HD size_t cell_byte_C(const Geom &g, int env, int x, int y) { return grid_word(g, env, c_word(g, x, y)) * 4 + (y & 3); }

// PTX prmt.b32 (generic mode): selector nibble bits 0-2 pick one of the 8 source bytes, bit 3 replicates that
// byte's sign bit instead. CUDA's __byte_perm() only honours the low 3 bits, hence the inline PTX.
MG_D uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
#ifdef __CUDA_ARCH__
  uint32_t d;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
  return d;
#else
  return __byte_perm(a, b, sel);
#endif
}
MG_HD int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
// bit i (i < 4) -> bit 8i
MG_HD uint32_t spread4(uint32_t b) { return (b * 0x00204081u) & 0x01010101u; }

#ifdef __CUDACC__
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
#endif

}  // namespace mg
