// mg_transition.cuh — MiniGridEnv.step's state transition (minigrid_env.py:525-588) for one environment,
// on the byte-coded cell in front of the agent. Pure register logic: the caller reads the front cell and
// writes it back when `newc != fc`.
#pragma once
#include "mg_common.cuh"

namespace mg {

struct StepOut {
  uint32_t newc;        // front cell after the action (== fc when unchanged)
  uint32_t terminated;  // 0/1
  uint32_t goal;        // reached the goal: reward = _reward() (minigrid_env.py:240-245)
  uint32_t bad_action;  // action outside 0..6 (ValueError, :584-585)
};

// DIR_TO_VEC (core/constants.py:49-58)
MG_HD void front_pos(const Geom &g, int ax, int ay, int dir, int &fx, int &fy) {
  const int dx = (dir == 0) - (dir == 2), dy = (dir == 1) - (dir == 3);
  fx = clampi(ax + dx, 0, g.W - 1);
  fy = clampi(ay + dy, 0, g.H - 1);
}

// flags: the agent flags (mg_common.cuh), if given; a forward move that succeeds sets FLAG_MOVED in them.
// Straight-line (select-based) form: every lane runs the same instructions whatever its action, so a warp of
// 32 environments with 32 different actions does not diverge.
MG_HD StepOut transition(int action, uint32_t fc, int fx, int fy, int &ax, int &ay, int &dir, uint32_t &carry,
                         uint32_t *flags = nullptr) {
  StepOut o;
  const uint32_t t4 = fc & 15u, col = (fc >> 4) & 7u;
  const bool isF = action == A_FORWARD, isP = action == A_PICKUP, isD = action == A_DROP, isT = action == A_TOGGLE;
  // left / right: agent_dir = (dir -/+ 1) mod 4                                           :541-548
  dir = (dir + (action == A_LEFT ? 3 : 0) + (action == A_RIGHT ? 1 : 0)) & 3;
  // forward: can_overlap = None, Goal, Floor, Lava, open Door (world_object.py:45,113,128,141,177)   :551-558
  const bool mv = isF && ((0x031Au >> t4) & 1u);
  ax = mv ? fx : ax;
  ay = mv ? fy : ay;
  if (flags) *flags |= mv ? FLAG_MOVED : 0u;  // agent_pos = tuple(fwd_pos) (:553): MiniGridEnv.hash prints numpy ints from now on
  o.goal = (isF && t4 == T_GOAL) ? 1u : 0u;
  o.terminated = (isF && (t4 == T_GOAL || t4 == T_LAVA)) ? 1u : 0u;
  // pickup: can_pickup = Key, Ball, Box, and nothing carried                               :561-566
  const bool pick = isP && ((t4 >= T_KEY && t4 <= T_BOX) || t4 == T4_BOX_WITH_KEY) && carry == 0;
  // drop: front cell is None and something is carried                                      :569-573
  const bool drop = isD && t4 == T_EMPTY && carry != 0;
  // toggle: Door.toggle (world_object.py:184-194), Box.toggle with contains == None (:290-293)   :576-578
  const bool unlock = t4 == T4_DOOR_LOCKED && (carry & 15u) == T_KEY && ((carry >> 4) & 7u) == col;
  const bool opens = isT && (t4 == T4_DOOR_CLOSED || unlock);
  const bool closes = isT && t4 == T_DOOR;
  const bool unbox = isT && t4 == T_BOX;
  uint32_t newc = fc;
  newc = (pick || unbox) ? CODE_EMPTY : newc;
  newc = drop ? carry : newc;
  newc = opens ? (T_DOOR | (col << 4)) : newc;
  newc = closes ? (T4_DOOR_CLOSED | (col << 4) | OPAQUE_BIT) : newc;
  newc = (isT && t4 == T4_BOX_WITH_KEY) ? (T_KEY | (col << 4)) : newc;  // Box.toggle: the box is replaced by its contents
  carry = pick ? (fc & 0x7Fu) : (drop ? 0u : carry);
  o.newc = newc;
  o.bad_action = ((unsigned)action > (unsigned)A_DONE) ? 1u : 0u;  // ValueError, :584-585
  return o;
}

}  // namespace mg
