// mg_levels.cuh — the level generators (_gen_grid) as "draw the integers, then evaluate a cell function".
//   envs/empty.py:97-114, envs/doorkey.py:74-99, envs/crossing.py:131-188, envs/fourrooms.py:78-126,
//   envs/lavagap.py:100-135, envs/distshift.py:98-120, envs/multiroom.py:117-284; next (not instantiated in the
//   kernels yet): envs/lockedroom.py:108-173, envs/playground.py:33-90,
//   place_obj / place_agent rejection sampling: minigrid_env.py:313-397.
// A finished level is a pure function of a handful of drawn integers, so generation is two phases:
//   draw   the RNG calls in exactly the reference's order (rejection loops test the closed-form cell
//          function instead of reading a half-built grid);
//   fill   every word of the env's two arrays is computed from the cell function and stored once.
#pragma once
#include "mg_common.cuh"
#include "mg_pcg64.cuh"

namespace mg {

struct Level {
  int ax, ay, adir;
  int a, b, c, d, e, f;        // kind-specific drawn integers
  uint32_t rv, rh;             // crossing: river position bit masks (vertical = column x, horizontal = row y)
  // crossing: every river is crossed exactly once (crossing.py:170-188). 5-bit fields, one per river in
  // ascending position order: the open row y of each vertical river / the open column x of each horizontal river.
  unsigned long long ov, oh;
  // multiroom: up to 6 rooms in creation order, 32 bits each (rooms 0-3 in rm03, 4-5 in rm45):
  // top_x:5 top_y:5 size_x:4 size_y:4 entry_door_x:5 entry_door_y:5 door_colour:3; (e, f) = goal
  // playground: 12 objects in placement order, 15 bits each (objects 0-7 in rm03, 8-11 in rm45):
  // x:5 y:5 kind:2 (0 key, 1 ball, 2 box) colour:3; nrooms = objects placed so far
  // goto-object / fetch / put-near: the objects in placement order, same 15-bit records, nrooms = their number
  u128 rm03;
  unsigned long long rm45;
  int nrooms;
  u128 rmx;  // roomgrid: object records 8..15 (ObstructedMaze creates up to 16 before its target ball, which is (e, f))
  // kinds with a step post-filter (mg_postfilter.cuh): what the filter compares against is packed into `ov`
  // (tx | ty << 8 | aux << 16, see level_target) and from there into the spare bits of the agent record
  // (x | y << 8 | tx << 16 | ty << 24, dir | flags << 8 | aux << 16). The struct itself is unchanged: MultiRoom keeps
  // it in local memory and its code must not move while these kinds are CPU-checked only.
};
MG_D void level_target(Level &L, int tx, int ty, uint32_t aux) {
  L.ov = (unsigned long long)(uint32_t)tx | ((unsigned long long)(uint32_t)ty << 8) | ((unsigned long long)aux << 16);
}
MG_D int level_tx(const Level &L) { return (int)(L.ov & 0xFFull); }
MG_D int level_ty(const Level &L) { return (int)((L.ov >> 8) & 0xFFull); }
MG_D uint32_t level_aux(const Level &L) { return (uint32_t)((L.ov >> 16) & 0xFFFFull); }

MG_D uint32_t room_get(const Level &L, int i) {
  return i < 4 ? (uint32_t)(L.rm03 >> (32 * i)) : (uint32_t)(L.rm45 >> (32 * (i - 4)));
}
MG_D void room_set(Level &L, int i, uint32_t v) {
  if (i < 4) L.rm03 = (L.rm03 & ~((u128)0xFFFFFFFFu << (32 * i))) | ((u128)v << (32 * i));
  else L.rm45 = (L.rm45 & ~(0xFFFFFFFFull << (32 * (i - 4)))) | ((unsigned long long)v << (32 * (i - 4)));
}
struct Room { int tx, ty, sx, sy, dx, dy, col; };
MG_D Room room_unpack(uint32_t v) {
  Room r;
  r.tx = v & 31; r.ty = (v >> 5) & 31; r.sx = (v >> 10) & 15; r.sy = (v >> 14) & 15;
  r.dx = (v >> 18) & 31; r.dy = (v >> 23) & 31; r.col = (v >> 28) & 7;
  return r;
}
MG_D uint32_t room_pack(int tx, int ty, int sx, int sy, int dx, int dy, int col) {
  return (uint32_t)tx | ((uint32_t)ty << 5) | ((uint32_t)sx << 10) | ((uint32_t)sy << 14) | ((uint32_t)dx << 18) |
         ((uint32_t)dy << 23) | ((uint32_t)col << 28);
}

// ---- cell functions: the finished grid of each generator ----
MG_D bool on_border(const Geom &g, int x, int y) { return x == 0 || y == 0 || x == g.W - 1 || y == g.H - 1; }

// envs/empty.py:97-114
MG_D uint32_t cell_empty(const Geom &g, const Level &, int x, int y) {
  if (on_border(g, x, y)) return CODE_WALL;
  if (x == g.W - 2 && y == g.H - 2) return CODE_GOAL;
  return CODE_EMPTY;
}
// envs/doorkey.py:74-99: a = splitIdx, b = doorIdx, (c, d) = key position
MG_D uint32_t cell_doorkey(const Geom &g, const Level &L, int x, int y) {
  if (on_border(g, x, y)) return CODE_WALL;
  if (x == L.a) return y == L.b ? (T4_DOOR_LOCKED | (C_YELLOW << 4) | OPAQUE_BIT) : CODE_WALL;
  if (x == L.c && y == L.d) return T_KEY | (C_YELLOW << 4);
  if (x == g.W - 2 && y == g.H - 2) return CODE_GOAL;
  return CODE_EMPTY;
}
// envs/crossing.py:131-188
MG_D uint32_t cell_crossing(const Geom &g, const Level &L, int x, int y, uint32_t obstacle) {
  if (on_border(g, x, y)) return CODE_WALL;
  const bool on_v = (L.rv >> x) & 1u, on_h = (L.rh >> y) & 1u;
  if (on_v && (int)((L.ov >> (5 * __popc(L.rv & ((1u << x) - 1u)))) & 31u) == y) return CODE_EMPTY;
  if (on_h && (int)((L.oh >> (5 * __popc(L.rh & ((1u << y) - 1u)))) & 31u) == x) return CODE_EMPTY;
  if (on_v || on_h) return obstacle;
  if (x == g.W - 2 && y == g.H - 2) return CODE_GOAL;
  return CODE_EMPTY;
}
// envs/fourrooms.py:78-126: gaps (9,a) (b,9) (c,9) (9,d) for the 19x19 layout; (e, f) = goal
MG_D uint32_t cell_fourrooms_walls(const Geom &g, const Level &L, int x, int y) {
  if (on_border(g, x, y)) return CODE_WALL;
  const int xm = g.W / 2, ym = g.H / 2;
  if (x == xm && y < g.H - 1) return (y == L.a || y == L.d) ? CODE_EMPTY : CODE_WALL;
  if (y == ym && x < g.W - 1) return (x == L.b || x == L.c) ? CODE_EMPTY : CODE_WALL;
  return CODE_EMPTY;
}
MG_D uint32_t cell_fourrooms(const Geom &g, const Level &L, int x, int y) {
  if (x == L.e && y == L.f) return CODE_GOAL;
  return cell_fourrooms_walls(g, L, x, y);
}

// envs/lavagap.py:100-135: (a, b) = gap position; the obstacle column spans y = 1..H-2
MG_D uint32_t cell_lavagap(const Geom &g, const Level &L, int x, int y, uint32_t obstacle) {
  if (on_border(g, x, y)) return CODE_WALL;
  if (x == L.a) return y == L.b ? CODE_EMPTY : obstacle;
  if (x == g.W - 2 && y == g.H - 2) return CODE_GOAL;
  return CODE_EMPTY;
}
// envs/distshift.py:98-120: lava strips on rows 1 and strip2_row, x = 3..W-4; goal at (W-2, 1); no draws
MG_D uint32_t cell_distshift(const Geom &g, int strip2_row, int x, int y) {
  if (on_border(g, x, y)) return CODE_WALL;
  if (x == g.W - 2 && y == 1) return CODE_GOAL;
  if (x >= 3 && x < g.W - 3 && (y == 1 || y == strip2_row)) return CODE_LAVA;
  return CODE_EMPTY;
}

// envs/multiroom.py:149-193: rooms are drawn in creation order (walls, then the room's entry door), the goal last;
// everything outside the rooms stays None
MG_D uint32_t cell_multiroom(const Level &L, int x, int y) {
  uint32_t code = CODE_EMPTY;
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    if (i < L.nrooms) {
      const Room r = room_unpack(room_get(L, i));
      const bool inside = x >= r.tx && x < r.tx + r.sx && y >= r.ty && y < r.ty + r.sy;
      if (inside && (x == r.tx || x == r.tx + r.sx - 1 || y == r.ty || y == r.ty + r.sy - 1)) code = CODE_WALL;
      if (i > 0 && x == r.dx && y == r.dy) code = T4_DOOR_CLOSED | ((uint32_t)r.col << 4) | OPAQUE_BIT;  // Door(color): closed
    }
  }
  if (x == L.e && y == L.f) code = CODE_GOAL;
  return code;
}

// COLOR_NAMES = sorted(COLORS) (constants.py:17): blue green grey purple red yellow -> COLOR_TO_IDX, 3 bits each
MG_D uint32_t color_name_idx(int i) { return (0403512u >> (3 * i)) & 7u; }  // octal digits, last = blue: yellow 4, red 0, purple 3, grey 5, green 1, blue 2

// envs/lockedroom.py:108-173. Six rooms: room k is on the left (k even) or right of the corridor, in row band k / 2;
// a = locked room, (b, c) = goal, d = the rooms' colours (3 bits each), e = key room (not needed by the cells),
// (rv, rh) = key position. Doors sit at fixed cells: (lWall | rWall, band * (H / 3) + 3).
MG_D uint32_t cell_lockedroom(const Geom &g, const Level &L, int x, int y) {
  if (on_border(g, x, y)) return CODE_WALL;
  const int lw = g.W / 2 - 2, rw = g.W / 2 + 2, h3 = g.H / 3;
  if (x == lw || x == rw) {
    const int band = y / h3;
    if (band < 3 && y - band * h3 == 3) {
      const int k = 2 * band + (x == rw);
      const uint32_t col = ((uint32_t)L.d >> (3 * k)) & 7u;
      return (k == L.a ? T4_DOOR_LOCKED : T4_DOOR_CLOSED) | (col << 4) | OPAQUE_BIT;
    }
    return CODE_WALL;
  }
  if ((x < lw || x > rw) && y % h3 == 0 && y / h3 < 3) return CODE_WALL;
  if (x == L.b && y == L.c) return CODE_GOAL;
  if (x == (int)L.rv && y == (int)L.rh) return T_KEY | ((((uint32_t)L.d >> (3 * L.a)) & 7u) << 4);
  return CODE_EMPTY;
}

// envs/playground.py:33-90 (19 x 19: a 3 x 3 arrangement of 6 x 6 rooms). a = the 6 doors in the vertical walls
// (index 2 j + i for the wall right of room (i, j)), b = the 6 doors in the horizontal walls (index 3 j + i for the
// wall below room (i, j)); 5 bits each: offset:2 (door cell = first interior cell + offset) colour:3, colour 7 = no
// door (the blank template). Objects: see Level.
MG_D uint32_t play_obj(const Level &L, int k) {
  return k < 8 ? (uint32_t)(L.rm03 >> (15 * k)) & 0x7FFFu : (uint32_t)(L.rm45 >> (15 * (k - 8))) & 0x7FFFu;
}
MG_D uint32_t cell_playground(const Geom &g, const Level &L, int x, int y) {
  if (on_border(g, x, y)) return CODE_WALL;
  const int rw = g.W / 3, rh = g.H / 3;
  const int i = x / rw, j = y / rh, lx = x - i * rw, ly = y - j * rh;
  if (ly == 0 && j >= 1 && j <= 2 && i < 3) {  // the wall below room (i, j - 1): x = i rw .. i rw + rw - 1
    const uint32_t dsc = ((uint32_t)L.b >> (5 * (3 * (j - 1) + i))) & 31u;
    if (lx >= 1 && (dsc >> 2) != 7u && lx - 1 == (int)(dsc & 3u)) return T4_DOOR_CLOSED | ((dsc >> 2) << 4) | OPAQUE_BIT;
    return CODE_WALL;
  }
  if (lx == 0 && i >= 1 && i <= 2 && j < 3) {  // the wall right of room (i - 1, j): y = j rh .. j rh + rh - 1
    const uint32_t dsc = ((uint32_t)L.a >> (5 * (2 * j + (i - 1)))) & 31u;
    if (ly >= 1 && (dsc >> 2) != 7u && ly - 1 == (int)(dsc & 3u)) return T4_DOOR_CLOSED | ((dsc >> 2) << 4) | OPAQUE_BIT;
    return CODE_WALL;
  }
  for (int k = 0; k < 12; ++k) {
    if (k < L.nrooms) {
      const uint32_t o = play_obj(L, k);
      if ((int)(o & 31u) == x && (int)((o >> 5) & 31u) == y) return (T_KEY + ((o >> 10) & 3u)) | (((o >> 12) & 7u) << 4);
    }
  }
  return CODE_EMPTY;
}

// envs/gotoobject.py:92-139, fetch.py:118-160, putnear.py:99-166: border walls and the objects
MG_D uint32_t cell_objroom(const Geom &g, const Level &L, int x, int y) {
  if (on_border(g, x, y)) return CODE_WALL;
  for (int k = 0; k < 8; ++k) {
    if (k < L.nrooms) {
      const uint32_t o = play_obj(L, k);
      if ((int)(o & 31u) == x && (int)((o >> 5) & 31u) == y) return (T_KEY + ((o >> 10) & 3u)) | (((o >> 12) & 7u) << 4);
    }
  }
  return CODE_EMPTY;
}
// envs/gotodoor.py:88-128: a = room width | height << 8 (the room is the top-left corner of the grid, the rest stays
// None), b = door coordinates (5 bits each: x on the top wall, x on the bottom wall, y on the left, y on the right),
// c = their colours (3 bits each)
MG_D uint32_t cell_gotodoor(const Geom &, const Level &L, int x, int y) {
  const int rw = L.a & 255, rh = (L.a >> 8) & 255;
  if (x >= rw || y >= rh) return CODE_EMPTY;
  const uint32_t b = (uint32_t)L.b, c = (uint32_t)L.c;
  if (y == 0 && x == (int)(b & 31u)) return T4_DOOR_CLOSED | ((c & 7u) << 4) | OPAQUE_BIT;
  if (y == rh - 1 && x == (int)((b >> 5) & 31u)) return T4_DOOR_CLOSED | (((c >> 3) & 7u) << 4) | OPAQUE_BIT;
  if (x == 0 && y == (int)((b >> 10) & 31u)) return T4_DOOR_CLOSED | (((c >> 6) & 7u) << 4) | OPAQUE_BIT;
  if (x == rw - 1 && y == (int)((b >> 15) & 31u)) return T4_DOOR_CLOSED | (((c >> 9) & 7u) << 4) | OPAQUE_BIT;
  if (x == 0 || y == 0 || x == rw - 1 || y == rh - 1) return CODE_WALL;
  return CODE_EMPTY;
}
// envs/redbluedoors.py:78-103 (W = 2 H): a = row of the red door in column H / 2, b = row of the blue door in
// column H / 2 + H - 1; -1 = no door (the blank template)
MG_D uint32_t cell_redbluedoors(const Geom &g, const Level &L, int x, int y) {
  const int s = g.H, xl = s / 2, xr = s / 2 + s - 1;
  if (x == xl && y == L.a) return T4_DOOR_CLOSED | (C_RED << 4) | OPAQUE_BIT;
  if (x == xr && y == L.b) return T4_DOOR_CLOSED | (C_BLUE << 4) | OPAQUE_BIT;
  if (on_border(g, x, y) || x == xl || x == xr) return CODE_WALL;
  return CODE_EMPTY;
}
// envs/memory.py:90-150: a = hallway_end, b = type of the object in the start room, c = type of the upper object at
// the end of the hallway (the lower one is the other type); all three are green
MG_D uint32_t cell_memory(const Geom &g, const Level &L, int x, int y) {
  if (on_border(g, x, y)) return CODE_WALL;
  const int mid = g.H / 2, upper = mid - 2, lower = mid + 2, he = L.a;
  if (x >= 1 && x <= 4 && (y == upper || y == lower)) return CODE_WALL;
  if (x == 4 && (y == upper + 1 || y == lower - 1)) return CODE_WALL;
  if (x >= 5 && x < he && (y == upper + 1 || y == lower - 1)) return CODE_WALL;
  if ((x == he && y != mid) || x == he + 2) return CODE_WALL;
  if (x == 1 && y == mid - 1) return (uint32_t)L.b | (C_GREEN << 4);
  if (x == he + 1 && y == mid - 2) return (uint32_t)L.c | (C_GREEN << 4);
  if (x == he + 1 && y == mid + 2) return (uint32_t)(L.c == (int)T_BALL ? T_KEY : T_BALL) | (C_GREEN << 4);
  return CODE_EMPTY;
}

// core/roomgrid.py:123-177 (RoomGrid._gen_grid) and the envs on it. kp = {variant, room_size S, num_rows, num_cols}; rooms
// are S x S with shared walls on the lines x, y = k (S - 1). A door descriptor is 8 bits: off:3 (door cell = first
// interior cell + off, drawn for every wall between two rooms whether or not a door is put there) colour:3 locked:1
// exists:1. oh = the doors in the vertical walls (index j (cols - 1) + i for the wall right of room (i, j)), rm45 = those
// in the horizontal walls (index j cols + i for the wall below room (i, j)); the objects are records in rm03 like
// Playground's (x:5 y:5 kind:2 colour:3), nrooms = their number. KeyCorridor removes the walls between the rooms of
// the middle column (keycorridor.py:107-109).
// object record k (x:5 y:5 kind:2 colour:3; kind 0 key, 1 ball, 2 box, 3 grey box hiding a key of that colour)
MG_D uint32_t rg_obj(const Level &L, int k) {
  return k < 8 ? (uint32_t)(L.rm03 >> (15 * k)) & 0x7FFFu : (uint32_t)(L.rmx >> (15 * (k - 8))) & 0x7FFFu;
}
MG_D void rg_obj_append(Level &L, uint32_t o) {
  if (L.nrooms < 8) L.rm03 |= (u128)o << (15 * L.nrooms); else L.rmx |= (u128)o << (15 * (L.nrooms - 8));
  L.nrooms += 1;
}
MG_D uint32_t rg_vdoor(const Level &L, int idx) { return (uint32_t)(L.oh >> (8 * idx)) & 0xFFu; }
MG_D uint32_t rg_hdoor(const Level &L, int idx) { return (uint32_t)(L.rm45 >> (8 * idx)) & 0xFFu; }
MG_D uint32_t rg_door_code(uint32_t dsc) {
  return ((dsc & 0x40u) ? T4_DOOR_LOCKED : T4_DOOR_CLOSED) | (((dsc >> 3) & 7u) << 4) | OPAQUE_BIT;  // Door(color, is_locked)
}
MG_D uint32_t cell_roomgrid(const Geom &g, const int *kp, const Level &L, int x, int y) {
  const int S1 = kp[1] - 1, cols = kp[3];
  const int i = x / S1, j = y / S1, lx = x - i * S1, ly = y - j * S1;
  if (lx == 0 && ly == 0) return CODE_WALL;
  if (lx == 0) {  // the vertical wall left of room (i, j) = right of room (i - 1, j)
    if (i == 0 || x == g.W - 1) return CODE_WALL;
    const uint32_t dsc = rg_vdoor(L, j * (cols - 1) + (i - 1));
    return ((dsc & 0x80u) && ly - 1 == (int)(dsc & 7u)) ? rg_door_code(dsc) : CODE_WALL;
  }
  if (ly == 0) {  // the horizontal wall above room (i, j) = below room (i, j - 1)
    if (j == 0 || y == g.H - 1) return CODE_WALL;
    if (kp[0] == RG_KEYCORRIDOR && i == 1) return CODE_EMPTY;  // remove_wall(1, j, 3), j >= 1
    const uint32_t dsc = rg_hdoor(L, (j - 1) * cols + i);
    return ((dsc & 0x80u) && lx - 1 == (int)(dsc & 7u)) ? rg_door_code(dsc) : CODE_WALL;
  }
  if (rg_obstructed(kp[0]) && x == L.e && y == L.f) return T_BALL | (C_BLUE << 4);  // self.obj: COLOR_NAMES[0]
  // the objects in creation order; a later grid.set wins (ObstructedMaze v0 puts blocking balls over earlier keys)
  for (int k = 15; k >= 0; --k)
    if (k < L.nrooms) {
      const uint32_t o = rg_obj(L, k);
      if ((int)(o & 31u) == x && (int)((o >> 5) & 31u) == y) {
        const uint32_t kind = (o >> 10) & 3u, col = (o >> 12) & 7u;
        return kind == 3u ? (T4_BOX_WITH_KEY | (col << 4)) : ((T_KEY + kind) | (col << 4));
      }
    }
  return CODE_EMPTY;
}

// envs/dynamicobstacles.py:107-133: border walls, goal at (W - 2, H - 2), nrooms blue balls (Ball() defaults to blue)
// in the object records of rm03 (x:5 y:5 kind:2 colour:3, see play_obj)
MG_D uint32_t cell_dynobs(const Geom &g, const Level &L, int x, int y) {
  if (on_border(g, x, y)) return CODE_WALL;
  if (x == g.W - 2 && y == g.H - 2) return CODE_GOAL;
  return cell_objroom(g, L, x, y);
}
// the obstacle list as kept between steps (Params::extra): 8 x (x | y << 8)
MG_D void dynobs_pack(const Level &L, uint32_t (&ex)[4]) {
  ex[0] = ex[1] = ex[2] = ex[3] = 0;
  for (int k = 0; k < 8; ++k)
    if (k < L.nrooms) {
      const uint32_t o = play_obj(L, k);
      ex[k >> 1] |= ((o & 31u) | (((o >> 5) & 31u) << 8)) << (16 * (k & 1));
    }
}

template <int KIND>
MG_D uint32_t cell_of(const Params &p, const Level &L, int x, int y) {
  if (KIND == KIND_ROOMGRID) return cell_roomgrid(p.g, p.kp, L, x, y);
  if (KIND == KIND_DYNOBS) return cell_dynobs(p.g, L, x, y);
  if (KIND == KIND_GOTOOBJECT || KIND == KIND_FETCH || KIND == KIND_PUTNEAR) return cell_objroom(p.g, L, x, y);
  if (KIND == KIND_GOTODOOR) return cell_gotodoor(p.g, L, x, y);
  if (KIND == KIND_REDBLUEDOORS) return cell_redbluedoors(p.g, L, x, y);
  if (KIND == KIND_MEMORY) return cell_memory(p.g, L, x, y);
  if (KIND == KIND_LOCKEDROOM) return cell_lockedroom(p.g, L, x, y);
  if (KIND == KIND_PLAYGROUND) return cell_playground(p.g, L, x, y);
  if (KIND == KIND_MULTIROOM) return cell_multiroom(L, x, y);
  if (KIND == KIND_LAVAGAP) return cell_lavagap(p.g, L, x, y, (p.kp[0] == (int)T_WALL) ? CODE_WALL : CODE_LAVA);
  if (KIND == KIND_DISTSHIFT) return cell_distshift(p.g, p.kp[0], x, y);
  if (KIND == KIND_EMPTY) return cell_empty(p.g, L, x, y);
  if (KIND == KIND_DOORKEY) return cell_doorkey(p.g, L, x, y);
  if (KIND == KIND_CROSSING) {
    const uint32_t obstacle = (p.kp[1] == (int)T_LAVA) ? CODE_LAVA : CODE_WALL;
    return cell_crossing(p.g, L, x, y, obstacle);
  }
  return cell_fourrooms(p.g, L, x, y);
}

// ---- draw phase ----
template <int KIND>
MG_D void draw_level(const Params &p, Pcg &r, Level &L) {
  const Geom &g = p.g;
  const int W = g.W, H = g.H;
  L.a = L.b = L.c = L.d = L.e = L.f = -1;
  L.rv = L.rh = 0;
  L.ov = L.oh = 0;
  L.rm03 = 0; L.rm45 = 0; L.nrooms = 0; L.rmx = 0;
  if (KIND == KIND_MULTIROOM) {
    // MultiRoomEnv._gen_grid / _placeRoom (multiroom.py:117-284). _placeRoom returns True as soon as ONE next room
    // has been placed (or after 8 failed tries), so the recursion is a chain without backtracking: room k+1 is
    // tried up to 8 times against room k, and the list only grows.
    const int num_rooms = rng_integers(r, p.kp[0], p.kp[1] + 1);
    const int max_sz = p.kp[2];
    while (L.nrooms < num_rooms) {
      Level cur;
      cur.rm03 = 0; cur.rm45 = 0; cur.nrooms = 0;
      int ex = rng_integers(r, 0, W - 2);
      int ey = rng_integers(r, 0, W - 2);
      int entry_wall = 2;
      auto try_place = [&](int wall, int dx, int dy) -> bool {
        const int sx = rng_integers(r, 4, max_sz + 1), sy = rng_integers(r, 4, max_sz + 1);
        int tx, ty;
        if (cur.nrooms == 0) { tx = dx; ty = dy; }
        else if (wall == 0) { tx = dx - sx + 1; ty = rng_integers(r, dy - sy + 2, dy); }
        else if (wall == 1) { tx = rng_integers(r, dx - sx + 2, dx); ty = dy - sy + 1; }
        else if (wall == 2) { tx = dx; ty = rng_integers(r, dy - sy + 2, dy); }
        else { tx = rng_integers(r, dx - sx + 2, dx); ty = dy; }
        if (tx < 0 || ty < 0) return false;
        if (tx + sx > W || ty + sy >= H) return false;
        for (int k = 0; k < cur.nrooms - 1; ++k) {  // roomList[:-1]
          const Room o = room_unpack(room_get(cur, k));
          const bool non_overlap = tx + sx < o.tx || o.tx + o.sx <= tx || ty + sy < o.ty || o.ty + o.sy <= ty;
          if (!non_overlap) return false;
        }
        room_set(cur, cur.nrooms, room_pack(tx, ty, sx, sy, dx, dy, 0));
        cur.nrooms += 1;
        return true;
      };
      bool placed = try_place(entry_wall, ex, ey);
      while (placed && cur.nrooms < num_rooms) {
        placed = false;
        const Room last = room_unpack(room_get(cur, cur.nrooms - 1));
        for (int i = 0; i < 8; ++i) {
          int exit_wall = rng_integers(r, 0, 3);  // _rand_elem(sorted({0,1,2,3} - {entryDoorWall}))
          if (exit_wall >= entry_wall) exit_wall += 1;
          const int next_entry = (exit_wall + 2) & 3;
          int px, py;
          if (exit_wall == 0) { px = last.tx + last.sx - 1; py = last.ty + rng_integers(r, 1, last.sy - 1); }
          else if (exit_wall == 1) { px = last.tx + rng_integers(r, 1, last.sx - 1); py = last.ty + last.sy - 1; }
          else if (exit_wall == 2) { px = last.tx; py = last.ty + rng_integers(r, 1, last.sy - 1); }
          else { px = last.tx + rng_integers(r, 1, last.sx - 1); py = last.ty; }
          if (try_place(next_entry, px, py)) { placed = true; entry_wall = next_entry; break; }
        }
      }
      if (cur.nrooms > L.nrooms) { L.rm03 = cur.rm03; L.rm45 = cur.rm45; L.nrooms = cur.nrooms; }
    }
    // door colours: _rand_elem(sorted(COLOR_NAMES minus the previous door's colour)); sorted names are
    // blue green grey purple red yellow
    int prev = -1;
    for (int idx = 1; idx < L.nrooms; ++idx) {
      int pick = rng_integers(r, 0, prev < 0 ? 6 : 5), col = 0;
      for (int c = 0; c < 6; ++c) {
        const int cidx = (int)((0x403512u >> (4 * c)) & 15u);  // C_BLUE, C_GREEN, C_GREY, C_PURPLE, C_RED, C_YELLOW
        if (cidx == prev) continue;
        if (pick-- == 0) { col = cidx; break; }
      }
      room_set(L, idx, (room_get(L, idx) & 0x0FFFFFFFu) | ((uint32_t)col << 28));
      prev = col;
    }
    const Room first = room_unpack(room_get(L, 0)), lastr = room_unpack(room_get(L, L.nrooms - 1));
    for (;;) {  // place_agent(roomList[0].top, roomList[0].size)
      const int x = rng_integers(r, first.tx, min(first.tx + first.sx, W)), y = rng_integers(r, first.ty, min(first.ty + first.sy, H));
      if (cell_multiroom(L, x, y) != CODE_EMPTY) continue;
      L.ax = x; L.ay = y;
      break;
    }
    L.adir = rng_integers(r, 0, 4);
    for (;;) {  // place_obj(Goal(), roomList[-1].top, roomList[-1].size)
      const int x = rng_integers(r, lastr.tx, min(lastr.tx + lastr.sx, W)), y = rng_integers(r, lastr.ty, min(lastr.ty + lastr.sy, H));
      if (cell_multiroom(L, x, y) != CODE_EMPTY) continue;
      if (x == L.ax && y == L.ay) continue;
      L.e = x; L.f = y;
      break;
    }
  } else if (KIND == KIND_ROOMGRID) {
    // RoomGrid._gen_grid (roomgrid.py:123-177), then the env's own _gen_grid (unlock.py:72-84, unlockpickup.py:80-93,
    // blockedunlockpickup.py:87-103, keycorridor.py:104-126) with RoomGrid's helpers restated as lambdas
    const int variant = p.kp[0], S = p.kp[1], rows = p.kp[2], cols = p.kp[3], S1 = S - 1;
    for (int j = 0; j < rows; ++j)
      for (int i = 0; i < cols; ++i) {  // door_pos draws: right wall (y), then bottom wall (x)
        if (i < cols - 1) L.oh |= (unsigned long long)rng_integers(r, 0, S - 2) << (8 * (j * (cols - 1) + i));
        if (j < rows - 1) L.rm45 |= (unsigned long long)rng_integers(r, 0, S - 2) << (8 * (j * cols + i));
      }
    L.ax = (cols / 2) * S1 + S / 2; L.ay = (rows / 2) * S1 + S / 2; L.adir = 0;  // "the agent starts in the middle, facing right"
    unsigned long long conn = 0;  // Room.doors[k] is truthy: bit 4 q + k of room q = j cols + i (k: right, down, left, up)
    uint32_t locked_rooms = 0;    // Room.locked
    auto nbr = [&](int i, int j, int k, int &ni, int &nj) -> bool {
      ni = i + (k == 0) - (k == 2); nj = j + (k == 1) - (k == 3);
      return ni >= 0 && ni < cols && nj >= 0 && nj < rows;
    };
    // descriptor slot of the wall on side k of room (i, j): vertical walls in oh, horizontal walls in rm45
    auto add_door = [&](int i, int j, int k, int color, int lockd, int &px, int &py) -> int {  // roomgrid.py:226-273
      int ni, nj;
      if (k < 0)
        for (;;) {
          k = rng_integers(r, 0, 4);
          if (nbr(i, j, k, ni, nj) && !((conn >> (4 * (j * cols + i) + k)) & 1ull)) break;
        }
      if (color < 0) color = (int)color_name_idx(rng_integers(r, 0, 6));
      if (lockd < 0) lockd = rng_integers(r, 0, 2) == 0;
      if (lockd) locked_rooms |= 1u << (j * cols + i); else locked_rooms &= ~(1u << (j * cols + i));
      nbr(i, j, k, ni, nj);
      const bool vertical = (k == 0 || k == 2);
      const int wi = vertical ? (k == 0 ? i : i - 1) : i, wj = vertical ? j : (k == 1 ? j : j - 1);
      const int idx = vertical ? wj * (cols - 1) + wi : wj * cols + wi;
      const unsigned long long set = (unsigned long long)(0x80u | (lockd ? 0x40u : 0u) | ((uint32_t)color << 3)) << (8 * idx);
      if (vertical) { L.oh |= set; px = (wi + 1) * S1; py = wj * S1 + 1 + (int)(rg_vdoor(L, idx) & 7u); }
      else { L.rm45 |= set; px = wi * S1 + 1 + (int)(rg_hdoor(L, idx) & 7u); py = (wj + 1) * S1; }
      conn |= 1ull << (4 * (j * cols + i) + k);
      conn |= 1ull << (4 * (nj * cols + ni) + ((k + 2) & 3));
      return color;
    };
    auto place_in_room = [&](int i, int j, int &x, int &y) {  // roomgrid.py:179-194: place_obj(top, size, reject_fn=reject_next_to, max_tries=1000)
      for (;;) {
        x = rng_integers(r, i * S1, min(i * S1 + S, W)); y = rng_integers(r, j * S1, min(j * S1 + S, H));
        if (cell_roomgrid(g, p.kp, L, x, y) != CODE_EMPTY) continue;
        if (x == L.ax && y == L.ay) continue;
        const int ddx = L.ax - x, ddy = L.ay - y;
        if ((ddx < 0 ? -ddx : ddx) + (ddy < 0 ? -ddy : ddy) < 2) continue;
        return;
      }
    };
    auto add_object = [&](int i, int j, int kind, int color) -> uint32_t {  // roomgrid.py:196-224
      if (kind < 0) kind = rng_integers(r, 0, 3);  // _rand_elem(["key", "ball", "box"])
      if (color < 0) color = (int)color_name_idx(rng_integers(r, 0, 6));
      int x, y;
      place_in_room(i, j, x, y);
      const uint32_t o = (uint32_t)x | ((uint32_t)y << 5) | ((uint32_t)kind << 10) | ((uint32_t)color << 12);
      rg_obj_append(L, o);
      return o;
    };
    auto place_agent = [&](int i, int j) {  // roomgrid.py:313-335: until the front cell is None or a wall
      for (;;) {
        int x, y;
        for (;;) {  // MiniGridEnv.place_agent(room.top, room.size): agent_pos = (-1, -1) while placing
          x = rng_integers(r, i * S1, min(i * S1 + S, W)); y = rng_integers(r, j * S1, min(j * S1 + S, H));
          if (cell_roomgrid(g, p.kp, L, x, y) == CODE_EMPTY) break;
        }
        const int d = rng_integers(r, 0, 4);
        L.ax = x; L.ay = y; L.adir = d;
        const uint32_t front = cell_roomgrid(g, p.kp, L, x + (d == 0) - (d == 2), y + (d == 1) - (d == 3));
        if (front == CODE_EMPTY || front == CODE_WALL) break;
      }
    };
    // check_objs_reachable (roomgrid_level.py:250-302) on the BabyAI levels' one room: flood fill from the agent through
    // empty cells; an object cell is reached but stops the fill; false when an object is not reached. The one room is
    // the whole grid, <= 8 x 8 cells: bit y W + x of a 64-bit mask (border cells are walls, so no shift leaves the grid).
    auto objs_reachable = [&]() -> bool {
      unsigned long long objs = 0, free = 0;
      for (int y = 1; y < H - 1; ++y) free |= (((1ull << (W - 2)) - 1ull) << 1) << (y * W);
      for (int k = 0; k < L.nrooms; ++k) {
        const uint32_t o = rg_obj(L, k);
        objs |= 1ull << ((int)((o >> 5) & 31u) * W + (int)(o & 31u));
      }
      free &= ~objs;
      unsigned long long reach = 1ull << (L.ay * W + L.ax), prev = 0;
      while (reach != prev) {
        prev = reach;
        const unsigned long long from = reach & free;
        reach |= ((from << 1) | (from >> 1) | (from << W) | (from >> W)) & (free | objs);
      }
      return !(objs & ~reach);
    };
    int dpx = 0, dpy = 0;
    if (variant == RG_BABYAI_PICKUP_PUTNEXT) {
      // RoomGridLevel._gen_grid (babyai/core/roomgrid_level.py:119-177) with the gen_mission of OneRoomS* (other.py:329-332),
      // PickupDist (pickup.py:275-290) and PutNextLocal (putnext.py:71-80), then validate_instrs; RejectSampling starts
      // the next attempt from an empty room while the stream continues. As for GoTo, place_obj's RecursionError is not
      // modelled.
      const int level = p.kp[4], nobj = p.kp[5];
      uint32_t tx = 0, ty = 0, aux = 0;
      for (;;) {
        L.rm03 = 0; L.nrooms = 0;
        L.ax = S / 2; L.ay = S / 2; L.adir = 0;
        if (level == BABYAI_ONEROOM) {  // add_object(0, 0, kind="ball") draws the colour; PickupInstr(ObjDesc("ball"))
          const uint32_t o = add_object(0, 0, 1, -1);
          place_agent(0, 0);
          tx = T_KEY + ((o >> 10) & 3u); ty = (o >> 12) & 7u; aux = PICK_TYPE;
          break;
        }
        // PutNextLocal places the agent first; PickupDist's objects are placed around the default room centre
        if (level == BABYAI_PUTNEXTLOCAL) place_agent(0, 0);
        while (L.nrooms < nobj) {  // add_distractors(all_unique=True) (roomgrid.py:396-438): colour, then type
          const uint32_t col = color_name_idx(rng_integers(r, 0, 6));
          const uint32_t kind = (uint32_t)rng_integers(r, 0, 3);
          bool dup = false;
          for (int k = 0; k < L.nrooms; ++k) dup |= ((rg_obj(L, k) >> 10) & 31u) == (kind | (col << 2));
          if (!dup) add_object(0, 0, (int)kind, (int)col);
        }
        if (level == BABYAI_PICKUPDIST) {
          place_agent(0, 0);
          const uint32_t o = rg_obj(L, rng_integers(r, 0, L.nrooms));  // _rand_elem(objs)
          const int select_by = rng_integers(r, 0, 3);                // _rand_elem(["type", "color", "both"])
          tx = T_KEY + ((o >> 10) & 3u); ty = (o >> 12) & 7u;
          aux = (select_by == 1 ? 0u : PICK_TYPE) | (select_by == 0 ? 0u : PICK_COLOR) | (p.kp[6] ? PICK_STRICT : 0u);
          break;
        }
        if (!objs_reachable()) continue;  // RejectSampling("unreachable object at ...")
        // o1, o2 = _rand_subset(objs, 2): the second draw indexes the list without the first
        const int i1 = rng_integers(r, 0, L.nrooms), i2 = rng_integers(r, 0, L.nrooms - 1);
        const uint32_t mv = rg_obj(L, i1), fo = rg_obj(L, i2 < i1 ? i2 : i2 + 1);
        const int ddx = (int)(mv & 31u) - (int)(fo & 31u), ddy = (int)((mv >> 5) & 31u) - (int)((fo >> 5) & 31u);
        if ((ddx < 0 ? -ddx : ddx) + (ddy < 0 ? -ddy : ddy) == 1) continue;  // RejectSampling("objs already next to each other")
        // PutNextInstr(ObjDesc(move), ObjDesc(fixed)): the move object's type and colour, the fixed object's cell code
        tx = T_KEY + ((mv >> 10) & 3u); ty = (mv >> 12) & 7u;
        aux = (T_KEY + ((fo >> 10) & 3u)) | (((fo >> 12) & 7u) << 4);
        break;
      }
      level_target(L, (int)tx, (int)ty, aux);
    } else if (variant == RG_BABYAI_GOTO) {
      // RoomGridLevel._gen_grid (babyai/core/roomgrid_level.py:119-144): an attempt is RoomGrid._gen_grid (one room: no
      // door draws) and gen_mission (babyai/goto.py:67-78, 133-141, 192-193, 256-260, 333-338, 661-677); RejectSampling
      // starts the next attempt from an empty grid while the stream continues. The RecursionError of place_obj's 1000
      // tries is not modelled: the worst case, GoToObjS4, has 1 valid cell in the 16 drawn, (15/16)^1001 ~ 1e-28.
      const int level = p.kp[4], ndist = p.kp[5];
      uint32_t tgt;
      for (;;) {
        L.rm03 = 0; L.nrooms = 0;
        L.ax = S / 2; L.ay = S / 2; L.adir = 0;
        place_agent(0, 0);  // place_agent(): i = _rand_int(0, 1), j = _rand_int(0, 1) draw nothing
        tgt = 0;
        if (level == BABYAI_REDBALL_GREY || level == BABYAI_REDBALL) tgt = add_object(0, 0, 1, C_RED);
        bool red_or_blue_ball = false;
        for (int k = 0; k < ndist; ++k) {  // add_distractors (roomgrid.py:396-438): colour, then type; all_unique only
          const int col = (int)color_name_idx(rng_integers(r, 0, 6));  // matters for GoToObj, whose list starts empty
          const int kind = rng_integers(r, 0, 3);
          red_or_blue_ball |= kind == 1 && (col == (int)C_RED || col == (int)C_BLUE);
          // GoToRedBallGrey recolours its distractors after placing them; placement does not look at colours
          add_object(0, 0, kind, level == BABYAI_REDBALL_GREY ? (int)C_GREY : col);
        }
        if (level == BABYAI_OBJ) { tgt = rg_obj(L, 0); break; }  // no reachability check
        if (level == BABYAI_REDBLUEBALL) {
          if (red_or_blue_ball) continue;  // RejectSampling("can only have one blue or red ball")
          tgt = add_object(0, 0, 1, rng_integers(r, 0, 2) == 0 ? (int)C_RED : (int)C_BLUE);
        }
        if (!objs_reachable()) continue;  // RejectSampling("unreachable object at ...")
        if (level == BABYAI_LOCAL) tgt = rg_obj(L, rng_integers(r, 0, L.nrooms));  // _rand_elem(objs)
        break;
      }
      // GoToInstr(ObjDesc(type, colour)): the step post-filter compares the front cell with (type, colour)
      level_target(L, (int)(T_KEY + ((tgt >> 10) & 3u)), (int)((tgt >> 12) & 7u), 0u);
    } else if (rg_obstructed(variant)) {
      // ObstructedMazeEnv._gen_grid (obstructedmaze.py:112-126): door_colors = _rand_subset(COLOR_NAMES, 6), the ball to find
      // is COLOR_NAMES[0] (blue), blocking balls COLOR_NAMES[1] (green), boxes COLOR_NAMES[2] (grey)
      const int key_in_box = p.kp[4], blocked = p.kp[5];
      uint32_t left = 0403512u, colors = 0;  // sorted names as 3-bit colour indices, see color_name_idx
      for (int k = 0; k < 6; ++k) {
        const int pick = rng_integers(r, 0, 6 - k);
        colors |= ((left >> (3 * pick)) & 7u) << (3 * k);
        left = (left & ((1u << (3 * pick)) - 1u)) | ((left >> (3 * (pick + 1))) << (3 * pick));
      }
      auto door_color = [&](int k) { return (int)((colors >> (3 * ((k + 6) % 6))) & 7u); };
      auto add_locked_door = [&](int i, int j, int k, int color) {  // obstructedmaze_v1.py:77-85 / the door half of obstructedmaze.py:135-165
        int x, y;
        add_door(i, j, k, color, 1, x, y);
        if (blocked) rg_obj_append(L, (uint32_t)(x - ((k == 0) - (k == 2))) | ((uint32_t)(y - ((k == 1) - (k == 3))) << 5) | (1u << 10) | ((uint32_t)C_GREEN << 12));
      };
      auto add_key = [&](int i, int j, int color) {  // obstructedmaze_v1.py:87-99 / the key half: a key, or a grey box hiding it
        int x, y;
        place_in_room(i, j, x, y);
        rg_obj_append(L, (uint32_t)x | ((uint32_t)y << 5) | ((key_in_box ? 3u : 0u) << 10) | ((uint32_t)color << 12));
      };
      int bx, by;
      if (variant == RG_OBSTRUCTED_1D) {  // obstructedmaze.py:188-203
        add_locked_door(0, 0, 0, door_color(0));
        add_key(0, 0, door_color(0));
        place_in_room(1, 0, bx, by);
        L.e = bx; L.f = by;
        place_agent(0, 0);
      } else {  // obstructedmaze.py:229-262, obstructedmaze_v1.py:37-75
        const int nq = p.kp[7];
        for (int i = 0; i < nq; ++i) {
          const int si = i == 0 ? 2 : (i == 2 ? 0 : 1), sj = i == 1 ? 2 : (i == 3 ? 0 : 1);  // side_rooms = (2,1) (1,2) (0,1) (1,0)
          int x, y;
          add_door(1, 1, i, door_color(i), 0, x, y);
          if (variant == RG_OBSTRUCTED_FULL) {
            for (int k = -1; k <= 1; k += 2) {
              add_locked_door(si, sj, (i + k + 4) % 4, door_color(i + k));
              add_key(si, sj, door_color(i + k));
            }
          } else {
            for (int k = -1; k <= 1; k += 2) add_locked_door(si, sj, (i + k + 4) % 4, door_color(i + k));
            for (int k = -1; k <= 1; k += 2) add_key(si, sj, door_color(i + k));
          }
        }
        const int corner = rng_integers(r, 0, nq);  // corners = (2,0) (2,2) (0,2) (0,0)
        place_in_room(corner < 2 ? 2 : 0, (corner == 1 || corner == 2) ? 2 : 0, bx, by);
        L.e = bx; L.f = by;
        place_agent(p.kp[6] & 15, p.kp[6] >> 4);
      }
      level_target(L, (int)T_BALL, (int)C_BLUE, 0u);
    } else if (variant == RG_KEYCORRIDOR) {
      for (int j = 1; j < rows; ++j) {  // remove_wall(1, j, 3): the cells are handled by cell_roomgrid, the rooms become connected
        conn |= 1ull << (4 * (j * cols + 1) + 3);
        conn |= 1ull << (4 * ((j - 1) * cols + 1) + 1);
      }
      const int room_idx = rng_integers(r, 0, rows);
      const int door_color = add_door(2, room_idx, 2, -1, 1, dpx, dpy);
      const uint32_t obj = add_object(2, room_idx, 1, -1);  // kind = self.obj_type = "ball"
      const int key_row = rng_integers(r, 0, rows);
      add_object(0, key_row, 0, door_color);
      place_agent(1, rows / 2);
      // connect_all (roomgrid.py:337-393): random doors until every room is reachable from the agent's
      const int start = (L.ay / S1) * cols + (L.ax / S1);
      for (;;) {
        uint32_t reach = 0, stack = 1u << start;
        while (stack) {
          const int q = __ffs(stack) - 1;
          stack &= stack - 1;
          if ((reach >> q) & 1u) continue;
          reach |= 1u << q;
          for (int k = 0; k < 4; ++k) {
            int ni, nj;
            if (((conn >> (4 * q + k)) & 1ull) && nbr(q % cols, q / cols, k, ni, nj)) stack |= 1u << (nj * cols + ni);
          }
        }
        if (__popc(reach) == rows * cols) break;
        const int i = rng_integers(r, 0, cols), j = rng_integers(r, 0, rows), k = rng_integers(r, 0, 4);
        int ni, nj;
        if (!nbr(i, j, k, ni, nj) || ((conn >> (4 * (j * cols + i) + k)) & 1ull)) continue;  // no door_pos there, or already a door
        if (((locked_rooms >> (j * cols + i)) & 1u) || ((locked_rooms >> (nj * cols + ni)) & 1u)) continue;
        const int color = (int)color_name_idx(rng_integers(r, 0, 6));
        int qx, qy;
        add_door(i, j, k, color, 0, qx, qy);
      }
      level_target(L, (int)(T_KEY + ((obj >> 10) & 3u)), (int)((obj >> 12) & 7u), 0u);
    } else {
      uint32_t obj = 0;
      if (variant != RG_UNLOCK) obj = add_object(1, 0, 2, -1);  // a box in the room on the right
      const int door_color = add_door(0, 0, 0, -1, 1, dpx, dpy);
      if (variant == RG_BLOCKEDUNLOCKPICKUP) {  // a ball of a random colour in front of the door (grid.set, no placement draws)
        const uint32_t col = color_name_idx(rng_integers(r, 0, 6));
        rg_obj_append(L, (uint32_t)(dpx - 1) | ((uint32_t)dpy << 5) | (1u << 10) | (col << 12));
      }
      add_object(0, 0, 0, door_color);
      place_agent(0, 0);
      if (variant == RG_UNLOCK) level_target(L, dpx, dpy, 0u);
      else level_target(L, (int)(T_KEY + ((obj >> 10) & 3u)), (int)((obj >> 12) & 7u), 0u);
    }
  } else if (KIND == KIND_DYNOBS) {
    // dynamicobstacles.py:107-133. kp = {n_obstacles, random_start, start_x, start_y, start_dir}
    if (!p.kp[1]) { L.ax = p.kp[2]; L.ay = p.kp[3]; L.adir = p.kp[4]; }
    else {  // place_agent() over the whole grid
      for (;;) {
        const int x = rng_integers(r, 0, W), y = rng_integers(r, 0, H);
        if (cell_dynobs(g, L, x, y) != CODE_EMPTY) continue;
        L.ax = x; L.ay = y;
        break;
      }
      L.adir = rng_integers(r, 0, 4);
    }
    for (int k = 0; k < p.kp[0]; ++k)  // place_obj(Ball(), max_tries=100): 101 attempts, then RecursionError (not modelled: never seen)
      for (int tries = 0; tries <= 100; ++tries) {
        const int x = rng_integers(r, 0, W), y = rng_integers(r, 0, H);
        if (cell_dynobs(g, L, x, y) != CODE_EMPTY) continue;
        if (x == L.ax && y == L.ay) continue;
        L.rm03 |= (u128)((uint32_t)x | ((uint32_t)y << 5) | (1u << 10) | ((uint32_t)C_BLUE << 12)) << (15 * L.nrooms);
        L.nrooms += 1;
        break;
      }
  } else if (KIND == KIND_GOTOOBJECT || KIND == KIND_FETCH || KIND == KIND_PUTNEAR) {
    // gotoobject.py:100-139, fetch.py:127-160, putnear.py:108-166. kp[0] = numObjs.
    const int n_objs = p.kp[0];
    while (L.nrooms < n_objs) {
      const uint32_t kind = (uint32_t)rng_integers(r, 0, KIND == KIND_FETCH ? 2 : 3);  // fetch: key | ball only
      const uint32_t col = color_name_idx(rng_integers(r, 0, 6));
      if (KIND != KIND_FETCH) {  // `if (objType, objColor) in objs: continue`
        bool dup = false;
        for (int k = 0; k < 8; ++k)
          if (k < L.nrooms) dup |= ((play_obj(L, k) >> 10) & 31u) == (kind | (col << 2));
        if (dup) continue;
      }
      for (;;) {  // place_obj(obj[, reject_fn=near_obj]) over the whole grid; the agent is not placed yet
        const int x = rng_integers(r, 0, W), y = rng_integers(r, 0, H);
        if (cell_objroom(g, L, x, y) != CODE_EMPTY) continue;
        if (KIND == KIND_PUTNEAR) {
          bool near = false;
          for (int k = 0; k < 8; ++k)
            if (k < L.nrooms) {
              const uint32_t o = play_obj(L, k);
              const int dx = x - (int)(o & 31u), dy = y - (int)((o >> 5) & 31u);
              near |= dx >= -1 && dx <= 1 && dy >= -1 && dy <= 1;
            }
          if (near) continue;
        }
        L.rm03 |= (u128)((uint32_t)x | ((uint32_t)y << 5) | (kind << 10) | (col << 12)) << (15 * L.nrooms);
        L.nrooms += 1;
        break;
      }
    }
    for (;;) {  // place_agent()
      const int x = rng_integers(r, 0, W), y = rng_integers(r, 0, H);
      if (cell_objroom(g, L, x, y) != CODE_EMPTY) continue;
      L.ax = x; L.ay = y;
      break;
    }
    L.adir = rng_integers(r, 0, 4);
    const uint32_t first = play_obj(L, rng_integers(r, 0, n_objs));  // target (fetch, gotoobject) / object to move (putnear)
    if (KIND == KIND_FETCH) {
      level_target(L, (int)(T_KEY + ((first >> 10) & 3u)), (int)((first >> 12) & 7u), 0u);  // targetType, targetColor
      (void)rng_integers(r, 0, 5);  // the wording of the mission: drawn, not modelled
    } else if (KIND == KIND_GOTOOBJECT) {
      level_target(L, (int)(first & 31u), (int)((first >> 5) & 31u), 0u);  // target_pos
    } else {
      uint32_t target;
      do { target = play_obj(L, rng_integers(r, 0, n_objs)); } while (target == first);  // objects are distinct
      // target_pos; move_type, moveColor as a cell code
      level_target(L, (int)(target & 31u), (int)((target >> 5) & 31u), (T_KEY + ((first >> 10) & 3u)) | (((first >> 12) & 7u) << 4));
    }
  } else if (KIND == KIND_GOTODOOR) {
    const int rw = rng_integers(r, 5, W + 1), rh = rng_integers(r, 5, H + 1);
    L.a = rw | (rh << 8);
    const uint32_t d0 = (uint32_t)rng_integers(r, 2, rw - 2), d1 = (uint32_t)rng_integers(r, 2, rw - 2);
    const uint32_t d2 = (uint32_t)rng_integers(r, 2, rh - 2), d3 = (uint32_t)rng_integers(r, 2, rh - 2);
    L.b = (int)(d0 | (d1 << 5) | (d2 << 10) | (d3 << 15));
    uint32_t cols = 0;
    for (int n = 0; n < 4;) {  // distinct colours, redrawn on a repeat
      const uint32_t col = color_name_idx(rng_integers(r, 0, 6));
      bool dup = false;
      for (int k = 0; k < 4; ++k)
        if (k < n) dup |= ((cols >> (3 * k)) & 7u) == col;
      if (dup) continue;
      cols |= col << (3 * n);
      ++n;
    }
    L.c = (int)cols;
    for (;;) {  // place_agent(size=(width, height))
      const int x = rng_integers(r, 0, rw), y = rng_integers(r, 0, rh);
      if (cell_gotodoor(g, L, x, y) != CODE_EMPTY) continue;
      L.ax = x; L.ay = y;
      break;
    }
    L.adir = rng_integers(r, 0, 4);
    const int idx = rng_integers(r, 0, 4);
    level_target(L, idx == 0 ? (int)d0 : idx == 1 ? (int)d1 : idx == 2 ? 0 : rw - 1,
                 idx == 0 ? 0 : idx == 1 ? rh - 1 : idx == 2 ? (int)d2 : (int)d3, 0u);
  } else if (KIND == KIND_REDBLUEDOORS) {
    const int s = H;
    L.a = L.b = -1;  // the agent is placed before the doors exist
    for (;;) {  // place_agent(top=(size // 2, 0), size=(size, size))
      const int x = rng_integers(r, s / 2, s / 2 + s), y = rng_integers(r, 0, s);
      if (cell_redbluedoors(g, L, x, y) != CODE_EMPTY) continue;
      L.ax = x; L.ay = y;
      break;
    }
    L.adir = rng_integers(r, 0, 4);
    L.a = rng_integers(r, 1, s - 1);
    L.b = rng_integers(r, 1, s - 1);
    level_target(L, L.a, L.b, 0u);
  } else if (KIND == KIND_MEMORY) {
    const int mid = H / 2;
    L.a = p.kp[0] ? rng_integers(r, 4, W - 2) : W - 3;  // hallway_end
    L.ax = rng_integers(r, 1, L.a + 1); L.ay = mid; L.adir = 0;
    L.b = rng_integers(r, 0, 2) == 0 ? (int)T_KEY : (int)T_BALL;  // _rand_elem([Key, Ball])
    L.c = rng_integers(r, 0, 2) == 0 ? (int)T_BALL : (int)T_KEY;  // _rand_elem([[Ball, Key], [Key, Ball]])[0]
    const int x = L.a + 1;
    const bool upper_matches = L.b == L.c;
    level_target(L, x, upper_matches ? mid - 1 : mid + 1,                               // success_pos
                 (uint32_t)x | ((uint32_t)(upper_matches ? mid + 1 : mid - 1) << 8));  // failure_pos
  } else if (KIND == KIND_LOCKEDROOM) {
    const int lw = W / 2 - 2, rw = W / 2 + 2, h3 = H / 3;
    auto room_x = [&](int k) { return (k & 1) ? rw : 0; };   // LockedRoom.top; size = (lw + 1, h3 + 1)
    auto room_y = [&](int k) { return (k >> 1) * h3; };
    L.a = rng_integers(r, 0, 6);                              // lockedRoom = _rand_elem(self.rooms)
    L.b = rng_integers(r, room_x(L.a) + 1, room_x(L.a) + lw); // goalPos = lockedRoom.rand_pos(): x in [topX + 1, topX + sizeX - 1)
    L.c = rng_integers(r, room_y(L.a) + 1, room_y(L.a) + h3);
    uint32_t left = 0403512u, cols = 0;                       // sorted(colors) as 3-bit entries, room colours
    for (int k = 0; k < 6; ++k) {                             // color = _rand_elem(sorted(colors)); colors.remove(color)
      const int pick = rng_integers(r, 0, 6 - k);             // (the sixth pick has one candidate: numpy draws nothing)
      cols |= ((left >> (3 * pick)) & 7u) << (3 * k);
      left = (left & ((1u << (3 * pick)) - 1u)) | ((left >> (3 * (pick + 1))) << (3 * pick));
    }
    L.d = (int)cols;
    do { L.e = rng_integers(r, 0, 6); } while (L.e == L.a);   // keyRoom
    L.rv = (uint32_t)rng_integers(r, room_x(L.e) + 1, room_x(L.e) + lw);
    L.rh = (uint32_t)rng_integers(r, room_y(L.e) + 1, room_y(L.e) + h3);
    for (;;) {  // place_agent(top=(lWallIdx, 0), size=(rWallIdx - lWallIdx, height))
      const int x = rng_integers(r, lw, rw), y = rng_integers(r, 0, H);
      if (cell_lockedroom(g, L, x, y) != CODE_EMPTY) continue;
      L.ax = x; L.ay = y;
      break;
    }
    L.adir = rng_integers(r, 0, 4);
  } else if (KIND == KIND_PLAYGROUND) {
    const int rw = W / 3, rh = H / 3;
    uint32_t vd = 0, hd = 0;
    for (int j = 0; j < 3; ++j)
      for (int i = 0; i < 3; ++i) {
        if (i + 1 < 3) {  // pos = (xR, _rand_int(yT + 1, yB - 1)); color = _rand_elem(COLOR_NAMES)
          const uint32_t off = (uint32_t)rng_integers(r, 0, rh - 2);
          const uint32_t col = color_name_idx(rng_integers(r, 0, 6));
          vd |= (off | (col << 2)) << (5 * (2 * j + i));
        }
        if (j + 1 < 3) {
          const uint32_t off = (uint32_t)rng_integers(r, 0, rw - 2);
          const uint32_t col = color_name_idx(rng_integers(r, 0, 6));
          hd |= (off | (col << 2)) << (5 * (3 * j + i));
        }
      }
    // doors that do not exist keep colour 7 in the blank template; here all 12 exist
    L.a = (int)vd; L.b = (int)hd;
    L.nrooms = 0;
    for (;;) {  // place_agent()
      const int x = rng_integers(r, 0, W), y = rng_integers(r, 0, H);
      if (cell_playground(g, L, x, y) != CODE_EMPTY) continue;
      L.ax = x; L.ay = y;
      break;
    }
    L.adir = rng_integers(r, 0, 4);
    for (int k = 0; k < 12; ++k) {  // objType = _rand_elem(types); objColor = _rand_elem(COLOR_NAMES); place_obj(obj)
      const uint32_t kind = (uint32_t)rng_integers(r, 0, 3);
      const uint32_t col = color_name_idx(rng_integers(r, 0, 6));
      for (;;) {
        const int x = rng_integers(r, 0, W), y = rng_integers(r, 0, H);
        if (cell_playground(g, L, x, y) != CODE_EMPTY) continue;
        if (x == L.ax && y == L.ay) continue;
        const uint32_t o = (uint32_t)x | ((uint32_t)y << 5) | (kind << 10) | (col << 12);
        if (k < 8) L.rm03 |= (u128)o << (15 * k); else L.rm45 |= (unsigned long long)o << (15 * (k - 8));
        L.nrooms = k + 1;
        break;
      }
    }
  } else if (KIND == KIND_EMPTY) {
    if (!p.kp[0]) { L.ax = p.kp[1]; L.ay = p.kp[2]; L.adir = p.kp[3]; }
    else {  // place_agent(): minigrid_env.py:383-397 over the whole grid
      for (;;) {
        const int x = rng_integers(r, 0, W), y = rng_integers(r, 0, H);
        if (cell_empty(g, L, x, y) != CODE_EMPTY) continue;
        L.ax = x; L.ay = y;
        break;
      }
      L.adir = rng_integers(r, 0, 4);
    }
  } else if (KIND == KIND_LAVAGAP) {
    L.ax = 1; L.ay = 1; L.adir = 0;
    L.a = rng_integers(r, 2, W - 2);
    L.b = rng_integers(r, 1, H - 1);
  } else if (KIND == KIND_DISTSHIFT) {
    L.ax = p.kp[1]; L.ay = p.kp[2]; L.adir = p.kp[3];
  } else if (KIND == KIND_DOORKEY) {
    const int split = rng_integers(r, 2, W - 2);
    L.a = split;
    for (;;) {  // place_agent(size=(splitIdx, height)); door and key do not exist yet
      const int x = rng_integers(r, 0, split), y = rng_integers(r, 0, H);
      if (x == 0 || y == 0 || y == H - 1) continue;
      L.ax = x; L.ay = y;
      break;
    }
    L.adir = rng_integers(r, 0, 4);
    L.b = rng_integers(r, 1, H - 2);
    for (;;) {  // place_obj(Key, top=(0,0), size=(splitIdx, height)): empty cell that is not the agent's
      const int x = rng_integers(r, 0, split), y = rng_integers(r, 0, H);
      if (x == 0 || y == 0 || y == H - 1) continue;
      if (x == L.ax && y == L.ay) continue;
      L.c = x; L.d = y;
      break;
    }
  } else if (KIND == KIND_CROSSING) {
    L.ax = 1; L.ay = 1; L.adir = 0;
    // rivers = [(v, i) for i in range(2, H-2, 2)] + [(h, j) for j in range(2, W-2, 2)]. Kept in registers: up to 32
    // one-byte entries (pos | dir << 7) in two 128-bit words, so the rare path needs no local-memory arrays.
    u128 r_lo = 0, r_hi = 0;
    auto rget = [&](int i) -> uint32_t { return (uint32_t)(((i < 16) ? r_lo : r_hi) >> (8 * (i & 15))) & 0xFFu; };
    auto rset = [&](int i, uint32_t v) {
      const u128 m = (u128)0xFF << (8 * (i & 15)), val = (u128)v << (8 * (i & 15));
      if (i < 16) r_lo = (r_lo & ~m) | val; else r_hi = (r_hi & ~m) | val;
    };
    int n = 0;
    for (int i = 2; i < H - 2; i += 2) rset(n++, (uint32_t)i);
    for (int j = 2; j < W - 2; j += 2) rset(n++, (uint32_t)j | 128u);
    for (int i = n - 1; i >= 1; --i) {  // np_random.shuffle(list)
      const int j = (int)rng_interval(r, (uint32_t)i);
      const uint32_t a = rget(i), b = rget(j);
      rset(i, b); rset(j, a);
    }
    if (p.kp[0] < n) n = p.kp[0];
    int nv = 0, nh = 0;
    for (int k = 0; k < n; ++k) {
      const uint32_t e = rget(k);
      if (e & 128u) { L.rh |= 1u << (e & 127u); ++nh; } else { L.rv |= 1u << e; ++nv; }
    }
    // path = [h] * len(rivers_v) + [v] * len(rivers_h), shuffled; bit k of `path` set = h
    const int np_ = nv + nh;
    uint32_t path = (nv >= 32) ? 0xFFFFFFFFu : ((1u << nv) - 1u);
    for (int i = np_ - 1; i >= 1; --i) {
      const int j = (int)rng_interval(r, (uint32_t)i);
      const uint32_t bi = (path >> i) & 1u, bj = (path >> j) & 1u;
      path = (path & ~((1u << i) | (1u << j))) | (bj << i) | (bi << j);
    }
    // limits_v = [0] + sorted(rivers_v) + [H-1]: walk the sorted positions through the bit masks
    int lim_v_lo = 0, lim_h_lo = 0;  // limits_v[room_i], limits_h[room_j]
    int room_i = 0, room_j = 0;
    L.ov = 0; L.oh = 0;
    for (int k = 0; k < np_; ++k) {
      const uint32_t mv = L.rv & ~((2u << lim_v_lo) - 1u), mh = L.rh & ~((2u << lim_h_lo) - 1u);
      const int lim_v_hi = mv ? (__ffs(mv) - 1) : H - 1;  // limits_v[room_i + 1]
      const int lim_h_hi = mh ? (__ffs(mh) - 1) : W - 1;  // limits_h[room_j + 1]
      if ((path >> k) & 1u) {  // h: cross the next vertical river at a random row of the current room
        const int j = lim_h_lo + 1 + rng_integers(r, 0, lim_h_hi - lim_h_lo - 1);  // choice(range(lo+1, hi))
        L.ov |= (unsigned long long)j << (5 * room_i);
        lim_v_lo = lim_v_hi; ++room_i;
      } else {
        const int i = lim_v_lo + 1 + rng_integers(r, 0, lim_v_hi - lim_v_lo - 1);
        L.oh |= (unsigned long long)i << (5 * room_j);
        lim_h_lo = lim_h_hi; ++room_j;
      }
    }
  } else {  // FOURROOMS
    const int rw = W / 2, rh = H / 2;
    // loop order j (rows of rooms) then i: (0,0): vertical wall gap, horizontal wall gap; (1,0): horizontal;
    // (0,1): vertical; (1,1): nothing   -> fourrooms.py:93-110
    L.a = rng_integers(r, 1, rh);               // (xR=rw, y in [1, rh))
    L.b = rng_integers(r, 1, rw);               // (x in [1, rw), yB=rh)
    L.c = rng_integers(r, rw + 1, 2 * rw);      // (x in [rw+1, 2rw), yB=rh)
    L.d = rng_integers(r, rh + 1, 2 * rh);      // (xR=rw, y in [rh+1, 2rh))
    for (;;) {  // place_agent()
      const int x = rng_integers(r, 0, W), y = rng_integers(r, 0, H);
      if (cell_fourrooms_walls(g, L, x, y) != CODE_EMPTY) continue;
      L.ax = x; L.ay = y;
      break;
    }
    L.adir = rng_integers(r, 0, 4);
    for (;;) {  // place_obj(Goal())
      const int x = rng_integers(r, 0, W), y = rng_integers(r, 0, H);
      if (cell_fourrooms_walls(g, L, x, y) != CODE_EMPTY) continue;
      if (x == L.ax && y == L.ay) continue;
      L.e = x; L.f = y;
      break;
    }
  }
}

// fill phase. Word w of an env (w < wpe): 4 consecutive bytes of one line of array R (w < offC) or C.
template <int KIND>
MG_D uint32_t level_word(const Params &p, const Level &L, int w) {
  const Geom &g = p.g;
  const bool inC = w >= g.offC;
  const int lw = inC ? g.lswC : g.lswR;
  const int rel = inC ? w - g.offC : w;
  const int line = rel / lw - g.ring, wi = rel - (line + g.ring) * lw;
  const int nlines = inC ? g.W : g.H, plen = inC ? g.H : g.W;
  uint32_t word = 0;
#pragma unroll
  for (int b = 0; b < 4; ++b) {
    const int pos = 4 * wi + b;
    uint32_t c = CODE_WALL;
    if (line >= 0 && line < nlines && pos < plen) c = inC ? cell_of<KIND>(p, L, line, pos) : cell_of<KIND>(p, L, pos, line);
    word |= c << (8 * b);
  }
  return word;
}
// both arrays of one env
template <int KIND>
MG_D void fill_level(const Params &p, const Level &L, int env) {
  for (int w = 0; w < p.g.wpe; ++w) p.grid[grid_word(p.g, env, w)] = level_word<KIND>(p, L, w);
}

// ---- template + patch form of the fill (the in-step autoreset of K1) ----
// Most of a level never changes between episodes. The template is the level of a "blank" draw (no split wall,
// key, rivers, gaps or goal where those are drawn); a freshly drawn level differs from it only on a few lines,
// whose cells are re-evaluated with the same cell function and written as bytes.
MG_D Level blank_level() {
  Level L;
  L.ax = L.ay = 1; L.adir = 0;
  L.a = L.b = L.c = L.d = L.e = L.f = -1;
  L.rv = L.rh = 0;
  L.ov = L.oh = 0;
  L.rm03 = 0; L.rm45 = 0; L.nrooms = 0; L.rmx = 0;
  return L;
}
// calls put(x, y) for this lane's share of the cells that may differ from the template
template <int KIND, class Put>
MG_D void patch_level(const Params &p, const Level &L, int lane, Put &&put) {
  const Geom &g = p.g;
  if (KIND == KIND_MULTIROOM) {
    for (int i = 0; i < L.nrooms; ++i) {  // every room's perimeter (doors are on perimeters), then the goal
      const Room r = room_unpack(room_get(L, i));
      for (int k = lane; k < 2 * (r.sx + r.sy); k += 32) {
        if (k < r.sx) put(r.tx + k, r.ty);
        else if (k < 2 * r.sx) put(r.tx + k - r.sx, r.ty + r.sy - 1);
        else if (k < 2 * r.sx + r.sy) put(r.tx, r.ty + k - 2 * r.sx);
        else put(r.tx + r.sx - 1, r.ty + k - 2 * r.sx - r.sy);
      }
    }
    if (lane == 0) put(L.e, L.f);
  } else if (KIND == KIND_GOTOOBJECT || KIND == KIND_FETCH || KIND == KIND_PUTNEAR || KIND == KIND_DYNOBS) {
    if (lane < L.nrooms) { const uint32_t o = play_obj(L, lane); put((int)(o & 31u), (int)((o >> 5) & 31u)); }
  } else if (KIND == KIND_REDBLUEDOORS) {
    if (lane == 0) put(g.H / 2, L.a);
    if (lane == 1) put(g.H / 2 + g.H - 1, L.b);
  } else if (KIND == KIND_GOTODOOR || KIND == KIND_MEMORY || KIND == KIND_ROOMGRID) {
    // the walls themselves are drawn (room size / hallway length / where the doors are): every cell may differ from the template
    for (int c = lane; c < g.W * g.H; c += 32) put(c % g.W, c / g.W);
  } else if (KIND == KIND_LOCKEDROOM) {
    const int lw = g.W / 2 - 2, rw = g.W / 2 + 2, h3 = g.H / 3;
    if (lane < 6) put((lane & 1) ? rw : lw, (lane >> 1) * h3 + 3);  // the six doors (colours and the lock are drawn)
    if (lane == 6) put(L.b, L.c);                                    // goal
    if (lane == 7) put((int)L.rv, (int)L.rh);                        // key
  } else if (KIND == KIND_PLAYGROUND) {
    const int rw = g.W / 3, rh = g.H / 3;
    if (lane < 6) put((lane % 2 + 1) * rw, (lane / 2) * rh + 1 + (int)(((uint32_t)L.a >> (5 * lane)) & 3u));
    else if (lane < 12) put(((lane - 6) % 3) * rw + 1 + (int)(((uint32_t)L.b >> (5 * (lane - 6))) & 3u), ((lane - 6) / 3 + 1) * rh);
    else if (lane < 24) { const uint32_t o = play_obj(L, lane - 12); put((int)(o & 31u), (int)((o >> 5) & 31u)); }
  } else if (KIND == KIND_LAVAGAP) {
    if (lane >= 1 && lane <= g.H - 2) put(L.a, lane);  // the obstacle column (gap included)
  } else if (KIND == KIND_DOORKEY) {
    if (lane >= 1 && lane <= g.H - 2) put(L.a, lane);  // the split column (door included)
    if (lane == 31) put(L.c, L.d);                      // the key
  } else if (KIND == KIND_CROSSING) {
    for (uint32_t m = L.rv; m; m &= m - 1)              // river columns (openings lie on rivers)
      if (lane >= 1 && lane <= g.H - 2) put(__ffs(m) - 1, lane);
    for (uint32_t m = L.rh; m; m &= m - 1)              // river rows
      if (lane >= 1 && lane <= g.W - 2) put(lane, __ffs(m) - 1);
  } else if (KIND == KIND_FOURROOMS) {
    const int xm = g.W / 2, ym = g.H / 2;
    if (lane == 0) put(xm, L.a);
    if (lane == 1) put(L.b, ym);
    if (lane == 2) put(L.c, ym);
    if (lane == 3) put(xm, L.d);
    if (lane == 4) put(L.e, L.f);
  }
}

}  // namespace mg
