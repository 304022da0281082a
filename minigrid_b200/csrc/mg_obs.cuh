// mg_obs.cuh — the egocentric 7x7x3 observation (MiniGridEnv.gen_obs, minigrid_env.py:597-650) for one
// environment per lane, computed entirely in registers from the lane's interleaved grid tile.
//
// Reference pipeline                                   here
//   get_view_exts + Grid.slice   (:453-484, grid.py:124)   closed form: world = agent + d*(6-vy) + r*(vx-3)
//   (dir+1) x Grid.rotate_left   (grid.py:110-122)         -> a view column vx is 7 consecutive bytes of one
//                                                          line of array R (dir 0/2) or C (dir 1/3), read
//                                                          forwards or backwards: 3 word loads + 2 funnel
//                                                          shifts + 2 byte permutes per column
//   out of bounds -> Wall()      (grid.py:136-139)         per-column line mask + a per-step byte mask
//   Grid.process_vis             (grid.py:291-328)         49-bit boards (byte = view row, bit = view column):
//                                                          carry-chain fill rightwards, Kogge-Stone leftwards
//   carry overlay                (minigrid_env.py:623-630) one byte permute
//   Grid.encode(vis_mask)        (grid.py:244-268)         256-entry (type,colour,state) table + byte permutes
//                                                          straight into the 147-byte C-order [vx][vy][c] stream
#pragma once
#include "mg_common.cuh"

namespace mg {

// Word accessors: gen_obs_words asks for word w of the environment (w as in r_word / c_word).
// `edge`: only lines [edge, n - 1 - edge] of each array may be read (n = H lines of R, W lines of C). 0: every grid line,
// the ring lines never; 1 (K1 on a walled level, mg_step_kernel.cuh: stage_lines): not the border lines either. The
// gather reads every line outside that range as a grey wall, which is what those lines hold.
struct AccTiled {   // LAYOUT_TILED, lane column of a tile in shared (K1) or global (K2) memory: word w at base[w * 32]
  const uint32_t *base;
  bool smem;
  int edge = 0;
  MG_D uint32_t operator()(int w) const {
#ifdef __CUDA_ARCH__
    if (smem) {
      uint32_t v;
      asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(smem_u32(base) + (uint32_t)(w << 7)));
      return v;
    }
#endif
    return base[w << 5];
  }
};
struct AccFlat {    // LAYOUT_WINDOW: env-major words; `base` is shifted so that base[w] is word w (global memory in
  const uint32_t *base;  // K2; in K1 the lane's 7-line window in shared memory, shifted by its first word index)
  int edge = 0;
  MG_D uint32_t operator()(int w) const { return base[w]; }
};
// kept for the transition's single front-cell read out of a staged tile
template <bool SMEM>
MG_D uint32_t tile_word(const uint32_t *base, int w) {
  AccTiled a = {base, SMEM};
  return a(w);
}
// The cell at position `pos` of the agent's own line: line ay of array R when it faces +-x (dir 0 / 2), line ax of array
// C when it faces +-y. That line is readable for every agent that stands inside the readable lines; a line outside them
// (an agent record injected onto the border of a walled level) or a position outside the grid reads as a grey wall.
template <class Acc>
MG_D uint32_t own_line_cell(const Geom &g, const Acc &acc, int ax, int ay, int dir, int pos) {
  const bool useC = dir & 1;
  const int l = useC ? ax : ay, nlines = useC ? g.W : g.H, plen = useC ? g.H : g.W;
  if ((unsigned)(l - acc.edge) >= (unsigned)(nlines - 2 * acc.edge) || (unsigned)pos >= (unsigned)plen) return CODE_WALL;
  const int w = (useC ? g.offC : 0) + (l + g.ring) * (useC ? g.lswC : g.lswR) + (pos >> 2);
  return (acc(w) >> (8 * (pos & 3))) & 0xFFu;
}

// One row of Grid.process_vis (grid.py:291-328) on 7-bit masks (bit i = view column i): m = cells of this row
// already visible, p = transparent cells (see_behind). Returns the row's final visibility v2 and the mask `up`
// it lights in the row above.
MG_HD void vis_row(uint32_t m, uint32_t p, uint32_t &v2, uint32_t &up) {
  // first sweep, i = 0..5 ascending: a visible transparent cell lights i+1 (and i, i+1 of the row above).
  // That recurrence is the carry chain of g + p with generate g = m & p, propagate p.
  const uint32_t g = m & p;
  const uint32_t c = (g + p) ^ g ^ p;
  const uint32_t v1 = (m | c) & 0x7Fu;
  const uint32_t a1 = v1 & p & 0x3Fu;
  // second sweep, i = 6..1 descending: prefix fill towards bit 0 (Kogge-Stone, 3 rounds cover 7 bits)
  uint32_t f = v1 & p, q = p;
  f |= q & (f >> 1); q &= q >> 1;
  f |= q & (f >> 2); q &= q >> 2;
  f |= q & (f >> 4);
  v2 = v1 | (f >> 1);
  const uint32_t a2 = f & 0x7Eu;  // == v2 & p on i = 1..6
  up = (a1 | (a1 << 1) | a2 | (a2 >> 1)) & 0x7Fu;  // the `if j > 0` writes into row j-1
}

// Grid.process_vis on bit boards. op*: opaque cells, v*: visible cells; byte j of (lo, hi) is view row vy = j
// (hi holds rows 4..6), bit i is view column vx = i. The agent is at (3, 6).
MG_D void process_vis(uint32_t oplo, uint32_t ophi, uint32_t &vlo, uint32_t &vhi) {
  uint32_t m = 1u << 3;
  vlo = 0; vhi = 0;
#pragma unroll
  for (int j = VIEW - 1; j >= 0; --j) {
    const uint32_t op = ((j < 4) ? (oplo >> (8 * j)) : (ophi >> (8 * (j - 4)))) & 0x7Fu;
    uint32_t v2, up;
    vis_row(m, op ^ 0x7Fu, v2, up);
    if (j < 4) vlo |= v2 << (8 * j); else vhi |= v2 << (8 * (j - 4));
    m = up;
  }
}

// Table-driven form: vis_row for all 128 x 128 (m, p) pairs, 2 bytes each = 32 KB that K1 keeps in shared
// memory. Entry at byte offset 2m + 256p: low byte v2, high byte up << 1 (i.e. the next row's 2m), so a row
// costs a shift, an and-or, one 16-bit shared load, a shift and a byte insert.
constexpr int VIS_TBL_BYTES = 128 * 128 * 2;
inline void build_vis_table(uint16_t *tbl) {
  for (uint32_t p = 0; p < 128; ++p)
    for (uint32_t m = 0; m < 128; ++m) {
      uint32_t v2, up;
      vis_row(m, p, v2, up);
      tbl[m + 128 * p] = (uint16_t)(v2 | (up << 9));
    }
}
MG_D void process_vis_tbl(const uint16_t *tbl, uint32_t oplo, uint32_t ophi, uint32_t &vlo, uint32_t &vhi) {
  const uint32_t plo = ~oplo & 0x7F7F7F7Fu, phi = ~ophi & 0x007F7F7Fu;
  const uint8_t *t8 = reinterpret_cast<const uint8_t *>(tbl);
  uint32_t m2 = (1u << 3) << 1;
  vlo = 0; vhi = 0;
#pragma unroll
  for (int j = VIEW - 1; j >= 0; --j) {
    const uint32_t pj8 = (j < 4) ? ((j == 0 ? plo << 8 : plo >> (8 * j - 8)) & 0x7F00u)
                                 : ((j == 4 ? phi << 8 : phi >> (8 * (j - 4) - 8)) & 0x7F00u);
    const uint32_t e = *reinterpret_cast<const uint16_t *>(t8 + (m2 | pj8));
    if (j < 4) vlo = prmt(vlo, e, 0x3210u ^ (0x4u << (4 * j)) ^ ((uint32_t)j << (4 * j)));
    else vhi = prmt(vhi, e, 0x3210u ^ (0x4u << (4 * (j - 4))) ^ ((uint32_t)(j - 4) << (4 * (j - 4))));
    m2 = e >> 8;
  }
}

// gen_obs up to and including the carry overlay: the 49 cell CODES of the view (0 = unseen), column vx in
// (clo[vx], chi[vx]): byte j of clo = view row vy = j, byte j of chi = view row 4 + j (its top byte is zero).
//   acc    word accessor (AccTiled / AccFlat)
//   VIS    VIS_NONE: see_through_walls (minigrid_env.py:616-621); VIS_ALU: bit tricks; VIS_TBL: vis_tbl lookups
constexpr int VIS_NONE = 0, VIS_ALU = 1, VIS_TBL = 2;
template <int VIS, class Acc>
MG_D void gather_view(const Geom &g, const Acc &acc, const uint16_t *vis_tbl, int ax, int ay, int dir, uint32_t carry,
                      uint32_t (&clo)[VIEW], uint32_t (&chi)[VIEW]) {
  const bool useC = dir & 1;
  const bool rev = dir < 2;
  const int lc = useC ? ax : ay;       // line coordinate of the agent in the chosen array
  const int pc = useC ? ay : ax;       // position inside a line
  const int lstep = (dir == 0 || dir == 3) ? 1 : -1;
  const int nlines = useC ? g.W : g.H;
  const int plen = useC ? g.H : g.W;
  const int lsw = useC ? g.lswC : g.lswR;
  const int abase = useC ? g.offC : 0;
  const int p0 = rev ? pc : pc - 6;    // first byte position of every 7-byte run
  const int wi0 = p0 >> 2;
  const uint32_t sh = (uint32_t)(p0 & 3) * 8u;
  const int k0 = clampi(wi0, 0, lsw - 1), k1 = clampi(wi0 + 1, 0, lsw - 1), k2 = clampi(wi0 + 2, 0, lsw - 1);
  // bytes whose position falls outside [0, plen) read as grey wall (Grid.slice, grid.py:136-139)
  uint32_t valid7 = ((((1u << plen) - 1u) << 6) >> (p0 + 6)) & 0x7Fu;
  if (rev) valid7 = __brev(valid7) >> 25;
  const uint32_t mlo = spread4(valid7 & 0xFu) * 0xFFu;
  const uint32_t mhi = spread4(valid7 >> 4) * 0xFFu;
  const uint32_t selLo = rev ? 0x3456u : 0x3210u;
  const uint32_t selHi = rev ? 0x7012u : 0x7654u;

  uint32_t oplo = 0, ophi = 0;
#pragma unroll
  for (int vx = 0; vx < VIEW; ++vx) {
    // a view column on a line the accessor may not read is a wall line: past the grid (Grid.slice) or a walled border
    const int lv = lc + lstep * (vx - 3);
    const int l = clampi(lv, acc.edge, nlines - 1 - acc.edge);
    const int rw = abase + (l + g.ring) * lsw;
    const uint32_t w0 = acc(rw + k0);
    const uint32_t w1 = acc(rw + k1);
    const uint32_t w2 = acc(rw + k2);
    const uint32_t a = __funnelshift_r(w0, w1, sh);
    const uint32_t b = __funnelshift_r(w1, w2, sh);
    uint32_t lo = prmt(a, b, selLo);
    uint32_t hi = prmt(a, b, selHi);
    const uint32_t ml = l == lv ? mlo : 0u, mh = l == lv ? mhi : 0u;
    lo = (lo & ml) | (CODE_WALL4 & ~ml);
    hi = (hi & mh) | ((CODE_WALL4 & 0x00FFFFFFu) & ~mh);
    clo[vx] = lo; chi[vx] = hi;
    if (VIS != VIS_NONE) {
      oplo |= ((lo >> 7) & 0x01010101u) << vx;
      ophi |= ((hi >> 7) & 0x01010101u) << vx;
    }
  }
  if (VIS != VIS_NONE) {
    uint32_t vlo, vhi;
    if (VIS == VIS_TBL) process_vis_tbl(vis_tbl, oplo, ophi, vlo, vhi);
    else process_vis(oplo, ophi, vlo, vhi);
#pragma unroll
    for (int vx = 0; vx < VIEW; ++vx) {
      // bit vx of every row byte -> bit 7, then prmt's sign-replicate mode turns it into a 0x00/0xFF byte mask
      clo[vx] &= prmt(vlo << (7 - vx), 0u, 0xBA98u);  // unseen -> code 0 -> (0,0,0)
      chi[vx] &= prmt(vhi << (7 - vx), 0u, 0xBA98u);
    }
  }
  // the agent's own view cell (3,6) shows what it carries, else empty (minigrid_env.py:623-630)
  chi[3] = prmt(chi[3], carry ? carry : CODE_EMPTY, 0x3410u);
}

// ---- LAYOUT_WINDOW (large grids): the view's words are loaded straight into registers, geometry applied later ----
// Which 7 lines the view needs is known BEFORE the transition (a turn depends on the action alone and a forward move
// never changes the line coordinate of the array the agent faces along); only the position inside the lines can still
// shift by one byte (forward move). So each lane loads, per line, the 3 words that cover the 8 bytes of both cases —
// 21 independent 4-byte loads, 7 sectors, ONE memory round trip per step — and the transition reads its front cell out
// of the same words (the cell in front is view cell (3, 5) unless the agent turns, in which case it is not needed).
struct ViewWords {
  uint32_t w[VIEW][3];
  int ws;       // index of w[.][0] inside a line (may be negative: clamped words only ever supply masked bytes)
};
// first byte position the loaded words must cover, for an agent at (ax, ay) that will face `dirn` after the action
MG_D int view_first_pos(int ax, int ay, int dirn) {
  const int pc = (dirn & 1) ? ay : ax;
  return (dirn < 2) ? pc : pc - 7;  // facing +: run starts at pc (pc + 1 after a move); facing -: pc - 6 (pc - 7 after a move)
}
template <class Load>
MG_D void load_view_words(const Geom &g, int ax, int ay, int dirn, ViewWords &vw, Load &&load) {
  const bool useC = dirn & 1;
  const int lc = useC ? ax : ay;
  const int lstep = (dirn == 0 || dirn == 3) ? 1 : -1;
  const int abase = useC ? g.offC : 0;
  const int ws = view_first_pos(ax, ay, dirn) >> 2;
  const int lsw = useC ? g.lswC : g.lswR;  // words per line of the array the agent faces along
  const int k0 = clampi(ws, 0, lsw - 1), k1 = clampi(ws + 1, 0, lsw - 1), k2 = clampi(ws + 2, 0, lsw - 1);
  vw.ws = ws;
#pragma unroll
  for (int vx = 0; vx < VIEW; ++vx) {
    const int rw = abase + (lc + lstep * (vx - 3) + g.ring) * lsw;  // ring = 3 lines: lc +- 3 always exists
    vw.w[vx][0] = load(rw + k0);
    vw.w[vx][1] = load(rw + k1);
    vw.w[vx][2] = load(rw + k2);
  }
}
// the byte at position `pos` of the agent's own line (view column 3); pos must lie in the 12 bytes loaded
MG_D uint32_t view_words_byte(const ViewWords &vw, int pos) {
  const int o = pos - 4 * vw.ws;
  const uint32_t w = o < 4 ? vw.w[3][0] : (o < 8 ? vw.w[3][1] : vw.w[3][2]);
  return (w >> (8 * (o & 3))) & 0xFFu;
}
MG_D void view_words_set_byte(ViewWords &vw, int pos, uint32_t code) {
  const int o = pos - 4 * vw.ws;
  const uint32_t sh = 8u * (uint32_t)(o & 3), m = 0xFFu << sh, v = (code & 0xFFu) << sh;
  if (o < 4) vw.w[3][0] = (vw.w[3][0] & ~m) | v;
  else if (o < 8) vw.w[3][1] = (vw.w[3][1] & ~m) | v;
  else vw.w[3][2] = (vw.w[3][2] & ~m) | v;
}
// gather_view on preloaded words: (ax, ay, dir) is the state AFTER the transition; the words were loaded for this
// direction and cover its run of 7 bytes
template <int VIS>
MG_D void gather_from_words(const Geom &g, const ViewWords &vw, const uint16_t *vis_tbl, int ax, int ay, int dir, uint32_t carry,
                            uint32_t (&clo)[VIEW], uint32_t (&chi)[VIEW]) {
  const bool useC = dir & 1;
  const bool rev = dir < 2;
  const int pc = useC ? ay : ax;
  const int plen = useC ? g.H : g.W;
  const int p0 = rev ? pc : pc - 6;
  const uint32_t sh = (uint32_t)(p0 - 4 * vw.ws) * 8u;  // 0..32: the clamping funnel shift returns the upper word at 32
  uint32_t valid7 = ((((1u << plen) - 1u) << 6) >> (p0 + 6)) & 0x7Fu;
  if (rev) valid7 = __brev(valid7) >> 25;
  const uint32_t mlo = spread4(valid7 & 0xFu) * 0xFFu;
  const uint32_t mhi = spread4(valid7 >> 4) * 0xFFu;
  const uint32_t selLo = rev ? 0x3456u : 0x3210u;
  const uint32_t selHi = rev ? 0x7012u : 0x7654u;
  uint32_t oplo = 0, ophi = 0;
#pragma unroll
  for (int vx = 0; vx < VIEW; ++vx) {
    const uint32_t a = __funnelshift_rc(vw.w[vx][0], vw.w[vx][1], sh);
    const uint32_t b = __funnelshift_rc(vw.w[vx][1], vw.w[vx][2], sh);
    uint32_t lo = prmt(a, b, selLo);
    uint32_t hi = prmt(a, b, selHi);
    lo = (lo & mlo) | (CODE_WALL4 & ~mlo);
    hi = (hi & mhi) | ((CODE_WALL4 & 0x00FFFFFFu) & ~mhi);
    clo[vx] = lo; chi[vx] = hi;
    if (VIS != VIS_NONE) {
      oplo |= ((lo >> 7) & 0x01010101u) << vx;
      ophi |= ((hi >> 7) & 0x01010101u) << vx;
    }
  }
  if (VIS != VIS_NONE) {
    uint32_t vlo, vhi;
    if (VIS == VIS_TBL) process_vis_tbl(vis_tbl, oplo, ophi, vlo, vhi);
    else process_vis(oplo, ophi, vlo, vhi);
#pragma unroll
    for (int vx = 0; vx < VIEW; ++vx) {
      clo[vx] &= prmt(vlo << (7 - vx), 0u, 0xBA98u);
      chi[vx] &= prmt(vhi << (7 - vx), 0u, 0xBA98u);
    }
  }
  chi[3] = prmt(chi[3], carry ? carry : CODE_EMPTY, 0x3410u);
}

// Grid.encode on the gathered codes: the 147-byte image of one env as 37 little-endian words S (byte 147 is zero).
// image[vx][vy][c], i.e. triple q = 7*vx + vy occupies stream bytes 3q..3q+2; lut: 256-entry decode table.
MG_D void encode_stream(const uint32_t *lut, const uint32_t (&clo)[VIEW], const uint32_t (&chi)[VIEW], uint32_t (&S)[OBS_WORDS]) {
  uint32_t T[VIEW * VIEW + 1];
#pragma unroll
  for (int vx = 0; vx < VIEW; ++vx) {
#pragma unroll
    for (int vy = 0; vy < VIEW; ++vy) {
      const uint32_t word = (vy < 4) ? clo[vx] : chi[vx];
      const uint32_t code = (word >> (8 * (vy & 3))) & 0xFFu;
      T[vx * VIEW + vy] = lut[code];
    }
  }
  T[VIEW * VIEW] = 0;
#pragma unroll
  for (int j = 0; j < OBS_WORDS; ++j) {
    const int a = (4 * j) / 3, r = 4 * j - 3 * a;
    S[j] = prmt(T[a], T[a + 1], r == 0 ? 0x4210u : (r == 1 ? 0x5421u : 0x6542u));
  }
}

template <int VIS, class Acc>
MG_D void gen_obs_words(const Geom &g, const Acc &acc, const uint32_t *lut, const uint16_t *vis_tbl,
                        int ax, int ay, int dir, uint32_t carry, uint32_t (&S)[OBS_WORDS]) {
  uint32_t clo[VIEW], chi[VIEW];
  gather_view<VIS>(g, acc, vis_tbl, ax, ay, dir, carry, clo, chi);
  encode_stream(lut, clo, chi, S);
}

// The packed record of the host path (MG_HOST_PACKED, include/minigrid_b200.h): 52 bytes = 13 words per env.
//   bytes 0..48  the view's cell codes in image order (q = 7*vx + vy), i.e. the image before Grid.encode's table
//   byte  49     dir | terminated << 2 | truncated << 3 | rewarded << 4 | (step_count >> 16) << 5
//   bytes 50-51  step_count & 0xFFFF (the reward is the host-side table entry of this step count when `rewarded`)
constexpr int PACKED_WORDS = 13, PACKED_BYTES = 52, PACKED_TILE_BYTES = PACKED_BYTES * TILE;  // 1664, a multiple of 16
constexpr uint32_t PACKED_MAX_STEPS = (1u << 19) - 1u;
MG_D void pack_codes(const uint32_t (&clo)[VIEW], const uint32_t (&chi)[VIEW], uint32_t tail, uint32_t (&P)[PACKED_WORDS]) {
#pragma unroll
  for (int j = 0; j < PACKED_WORDS; ++j) {
    // output byte b = 4j + k comes from column b / 7, row b % 7: at most two source words per output word
    uint32_t sel = 0, src[2] = {0u, 0u};
    int nsrc = 0, id[2] = {-1, -1};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int b = 4 * j + k;
      if (b >= VIEW * VIEW) { sel |= 0x8u << (4 * k); continue; }  // filled from `tail` below
      const int vx = b / VIEW, vy = b % VIEW;
      const int wid = 2 * vx + (vy >= 4);
      int slot = (id[0] == wid) ? 0 : ((id[1] == wid) ? 1 : -1);
      if (slot < 0) { slot = nsrc++; id[slot] = wid; src[slot] = (vy < 4) ? clo[vx] : chi[vx]; }
      sel |= (uint32_t)(4 * slot + (vy & 3)) << (4 * k);
    }
    if (j < PACKED_WORDS - 1) P[j] = prmt(src[0], src[1], sel);
    else P[j] = ((chi[VIEW - 1] >> 16) & 0xFFu) | (tail << 8);  // byte 48 = cell (6, 6), then the three tail bytes
  }
}
MG_HD uint32_t packed_tail(int dir, uint32_t terminated, uint32_t truncated, uint32_t rewarded, uint32_t steps) {
  return (uint32_t)dir | (terminated << 2) | (truncated << 3) | (rewarded << 4) | (((steps >> 16) & 7u) << 5) | ((steps & 0xFFFFu) << 8);
}

// Stage one warp's 32 images into shared memory exactly as they lie in the [n][7][7][3] output
// (147-byte stride, so lane L starts at byte 147 L = word (147 L) / 4 plus (L & 3) bytes). Lane L skips its
// first (L & 3) bytes; they travel in the last word written by lane L-1.
// n0 is word 0 of lane L+1's stream (a warp shuffle on the device).
MG_D void emit_obs_staged(uint32_t *stage, int lane, const uint32_t (&S)[OBS_WORDS], uint32_t n0) {
  const uint32_t o8 = (uint32_t)(lane & 3) * 8u;
  uint32_t *dst = stage + ((OBS_BYTES * lane + 3) >> 2);
#pragma unroll
  for (int i = 0; i < OBS_WORDS - 1; ++i) dst[i] = __funnelshift_r(S[i], S[i + 1], o8);
  const uint32_t s36 = prmt(S[OBS_WORDS - 1], n0, 0x4210u);  // own bytes 144..146, then the next lane's byte 0
  if ((lane & 3) != 3) dst[OBS_WORDS - 1] = __funnelshift_r(s36, n0 >> 8, o8);
}

// Slow emitter for the rare paths (reset kernel, partial tiles): plain byte stores.
MG_D void emit_obs_bytes(uint8_t *dst, const uint32_t (&S)[OBS_WORDS]) {
#pragma unroll
  for (int w = 0; w < OBS_WORDS; ++w) {
#pragma unroll
    for (int b = 0; b < 4; ++b)
      if (4 * w + b < OBS_BYTES) dst[4 * w + b] = (uint8_t)(S[w] >> (8 * b));
  }
}

}  // namespace mg
