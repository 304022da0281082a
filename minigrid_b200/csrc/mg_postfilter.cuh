// mg_postfilter.cuh — SURVEY 8(f-2): the environments that wrap MiniGridEnv.step in a few integer predicates
// ("super().step(action)", then terminate / reward on a target). Pure register logic, like mg_transition.cuh:
//   pre_filter   what the subclass does to the action before super().step
//   post_filter  what it does to (reward, terminated) afterwards
// The comparison targets are drawn at reset (mg_levels.cuh: level_target) and live in the spare bits of the
// agent record. Called by K1 (mg_step_kernel.cuh) for the kinds has_post_filter() names; also replayed by the host
// emulation (tests/host_emu) against the oracle.
#pragma once
#include "mg_common.cuh"
#include "mg_pcg64.cuh"

namespace mg {

// memory.py:152-154: pickup is replaced with toggle
template <int KIND>
MG_HD int pre_filter(int action) {
  if (KIND == KIND_MEMORY && action == A_PICKUP) return A_TOGGLE;
  return action;
}

struct PostIn {
  int action;                   // after pre_filter
  int ax, ay, dir;              // agent after the transition
  uint32_t carry_before, carry; // carried cell code (0 none) before / after the transition
  int tx, ty;                   // level_tx, level_ty
  uint32_t aux;                 // level_aux
  // redbluedoors only: is_open of the two doors before and after the transition
  bool red_before, blue_before, red_after, blue_after;
  // roomgrid only: kp[0], and whether the cell at (tx, ty) is an open door after the transition (Unlock's self.door.is_open)
  int variant;
  bool door_open;
  // roomgrid BabyAI GoTo only: the code of the cell in front of the agent after the transition (0 = not read)
  uint32_t front = 0;
  // roomgrid BabyAI Pickup / PutNext only: kp[4], and on a drop the codes of the three cells next to the front cell other
  // than the agent's, one per byte, after the transition (0 = not read)
  int level = 0;
  uint32_t next_to = 0;
};
enum : int { POST_KEEP = 0, POST_REWARD = 1, POST_ZERO = 2 };  // what becomes of the step's reward
struct PostOut { uint32_t terminated; int reward; };

template <int KIND>
MG_HD PostOut post_filter(const PostIn &in, uint32_t terminated) {
  PostOut o = {terminated, POST_KEEP};
  if (KIND == KIND_GOTODOOR || KIND == KIND_GOTOOBJECT) {  // gotodoor.py:130-149, gotoobject.py:141-160
    if (in.action == A_TOGGLE) o.terminated = 1u;
    if (in.action == A_DONE) {
      const int dx = in.ax - in.tx, dy = in.ay - in.ty;
      if ((dx == 0 && (dy == 1 || dy == -1)) || (dy == 0 && (dx == 1 || dx == -1))) o.reward = POST_REWARD;
      o.terminated = 1u;
    }
  } else if (KIND == KIND_FETCH) {  // fetch.py:162-175: anything carried ends the episode
    if (in.carry != 0u) {
      o.reward = ((int)(in.carry & 15u) == in.tx && (int)((in.carry >> 4) & 7u) == in.ty) ? POST_REWARD : POST_ZERO;
      o.terminated = 1u;
    }
  } else if (KIND == KIND_PUTNEAR) {  // putnear.py:168-199; aux = the object to move as a cell code (type | colour << 4)
    const int ox = in.ax + (in.dir == 0) - (in.dir == 2), oy = in.ay + (in.dir == 1) - (in.dir == 3);
    if (in.action == A_PICKUP && in.carry != 0u && (in.carry & 0x7Fu) != in.aux) o.terminated = 1u;
    if (in.action == A_DROP && in.carry_before != 0u) {
      const int dx = ox - in.tx, dy = oy - in.ty;
      // "self.grid.get(ox, oy) is preCarrying": the drop took place, nothing is carried any more
      if (in.carry == 0u && dx >= -1 && dx <= 1 && dy >= -1 && dy <= 1) o.reward = POST_REWARD;
      o.terminated = 1u;
    }
  } else if (KIND == KIND_MEMORY) {  // memory.py:156-164; aux = failure_pos (x | y << 8)
    if (in.ax == in.tx && in.ay == in.ty) { o.reward = POST_REWARD; o.terminated = 1u; }
    if (in.ax == (int)(in.aux & 255u) && in.ay == (int)((in.aux >> 8) & 255u)) { o.reward = POST_ZERO; o.terminated = 1u; }
  } else if (KIND == KIND_ROOMGRID) {
    if (in.variant == RG_BABYAI_GOTO) {
      // RoomGridLevel.step (babyai/core/roomgrid_level.py:87-104) with GoToInstr.verify_action (verifier.py:290-316):
      // success when front_pos is one of the positions find_matching_objs recorded at reset. A matching object leaves
      // its cell only by being picked up, which needs the agent to face it first, and facing it already ended the
      // episode; so the test is "the front cell holds an object of the target's type and colour" (tx, ty).
      if ((int)(in.front & 15u) == in.tx && (int)((in.front >> 4) & 7u) == in.ty) { o.reward = POST_REWARD; o.terminated = 1u; }
    } else if (in.variant == RG_BABYAI_PICKUP_PUTNEXT) {
      // RoomGridLevel.step (babyai/core/roomgrid_level.py:87-104). The verifiers' preCarrying is what was carried after
      // the previous step: carry_before. No object appears or changes colour in these rooms (a box can only vanish, by
      // toggle), so "is one of obj_set" is "matches the descriptor", and an object is identified by its cell code.
      if (in.level == BABYAI_PUTNEXTLOCAL) {
        // PutNextInstr.verify_action (verifier.py:411-435) after update_objs_poss on a drop: success when preCarrying is
        // the move object and its cur_pos is 4-adjacent to where the fixed object (cell code aux) is now. A drop that
        // failed leaves cur_pos = (-1, -1) from the pickup; one that succeeded put it in the front cell, and the fixed
        // object next to that cell is in one of the three neighbours that are not the agent's cell.
        const uint32_t f = in.aux & 0xFFu, n = in.next_to;
        const bool moved = (int)(in.carry_before & 15u) == in.tx && (int)((in.carry_before >> 4) & 7u) == in.ty;
        if (in.action == A_DROP && in.carry == 0u && moved &&
            ((n & 0xFFu) == f || ((n >> 8) & 0xFFu) == f || ((n >> 16) & 0xFFu) == f)) {
          o.reward = POST_REWARD; o.terminated = 1u;
        }
      } else if (in.action == A_PICKUP) {
        // PickupInstr.verify_action (verifier.py:343-363): success when nothing was carried and the carried object
        // matches ObjDesc(type if PICK_TYPE, colour if PICK_COLOR); strict: any other pickup that leaves something
        // carried (the wrong object, or pressing pickup while carrying) fails
        const bool match = in.carry != 0u && (!(in.aux & PICK_TYPE) || (int)(in.carry & 15u) == in.tx) &&
                           (!(in.aux & PICK_COLOR) || (int)((in.carry >> 4) & 7u) == in.ty);
        if (in.carry_before == 0u && match) { o.reward = POST_REWARD; o.terminated = 1u; }
        else if ((in.aux & PICK_STRICT) && in.carry != 0u) { o.reward = POST_ZERO; o.terminated = 1u; }
      }
    } else if (in.variant == RG_UNLOCK) {  // unlock.py:88-96
      if (in.action == A_TOGGLE && in.door_open) { o.reward = POST_REWARD; o.terminated = 1u; }
    } else if (in.action == A_PICKUP && in.carry != 0u && (int)(in.carry & 15u) == in.tx && (int)((in.carry >> 4) & 7u) == in.ty) {
      // "self.carrying and self.carrying == self.obj" (unlockpickup.py:97-105, blockedunlockpickup.py:107-115,
      // keycorridor.py:128-136): an identity test; these generators make exactly one object of self.obj's type
      o.reward = POST_REWARD; o.terminated = 1u;
    }
  } else if (KIND == KIND_REDBLUEDOORS) {  // redbluedoors.py:105-126
    if (in.blue_after) {
      o.reward = in.red_before ? POST_REWARD : POST_ZERO;
      o.terminated = 1u;
    } else if (in.red_after && in.blue_before) {
      o.reward = POST_ZERO;
      o.terminated = 1u;
    }
  }
  return o;
}

// ---- SURVEY 8(f-4): DynamicObstaclesEnv.step (dynamicobstacles.py:135-167), the part that runs BEFORE super().step ----
// Every obstacle is re-placed inside the 3 x 3 box around its old position (place_obj(top=old - 1, size=(3, 3),
// max_tries=100): up to 101 attempts of two draws each, minigrid_env.py:313-372; a RecursionError leaves it where it
// is), then its old cell is cleared. The draws continue the env's own numpy stream, so the RNG record is on the step
// path for this kind. get(x, y) reads a cell code, put(x, y, code) writes one (both arrays); ex = Params::extra.
constexpr uint32_t CODE_OBSTACLE = T_BALL | (C_BLUE << 4);
template <class Get, class Put>
MG_D void dynobs_move(const Geom &g, Pcg &r, int n_obst, uint32_t (&ex)[4], int ax, int ay, Get &&get, Put &&put) {
  for (int i = 0; i < n_obst; ++i) {
    const uint32_t rec = (ex[i >> 1] >> (16 * (i & 1))) & 0xFFFFu;
    const int ox = (int)(rec & 0xFFu), oy = (int)(rec >> 8);
    const int tx = max(ox - 1, 0), ty = max(oy - 1, 0);
    const int hx = min(tx + 3, g.W), hy = min(ty + 3, g.H);
    for (int tries = 0; tries <= 100; ++tries) {
      const int x = rng_integers(r, tx, hx), y = rng_integers(r, ty, hy);
      if (get(x, y) != CODE_EMPTY) continue;   // the old position is still occupied: an obstacle never stays
      if (x == ax && y == ay) continue;
      put(x, y, CODE_OBSTACLE);
      put(ox, oy, CODE_EMPTY);
      const uint32_t nrec = (uint32_t)x | ((uint32_t)y << 8);
      ex[i >> 1] = (ex[i >> 1] & ~(0xFFFFu << (16 * (i & 1)))) | (nrec << (16 * (i & 1)));
      break;
    }
  }
}

template <int KIND>
MG_HD constexpr bool has_post_filter() {
  return KIND == KIND_GOTODOOR || KIND == KIND_GOTOOBJECT || KIND == KIND_FETCH || KIND == KIND_PUTNEAR ||
         KIND == KIND_MEMORY || KIND == KIND_REDBLUEDOORS || KIND == KIND_ROOMGRID;
}

}  // namespace mg
