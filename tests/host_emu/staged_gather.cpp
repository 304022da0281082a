// staged_gather.cpp — TEST BUILD ONLY. The tiled gather of K1 as it runs on a tile staged by stage_lines (only lines
// [edge, n - 1 - edge] of each array copied in, the other rows of the buffer holding whatever was there before),
// compared with the gather on the whole tile, the ring lines included. mg_obs.cuh compiled by g++ through
// mg_host_shim.h (tests/test_staged_gather_cpu.py).
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../minigrid_b200/csrc/mg_common.cuh"
#include "../../minigrid_b200/csrc/mg_obs.cuh"

using namespace mg;

static uint32_t xs(uint64_t &s) {  // xorshift64*
  s ^= s >> 12; s ^= s << 25; s ^= s >> 27;
  return (uint32_t)((s * 0x2545F4914F6CDD1DULL) >> 32);
}

template <int VIS>
static long compare_all(const Geom &g, const uint32_t *whole, const uint32_t *staged, int edge, const uint16_t *tbl) {
  long bad = 0;
  const AccTiled aw = {whole, false, -g.ring};  // every line of the whole tile readable: the ring lines are read
  const AccTiled as = {staged, false, edge};
  const uint32_t carries[2] = {0u, 0x15u};  // nothing, a red key
  for (int ax = 0; ax < g.W; ++ax)
    for (int ay = 0; ay < g.H; ++ay)
      for (int dir = 0; dir < 4; ++dir)
        for (uint32_t carry : carries) {
          uint32_t clo0[VIEW], chi0[VIEW], clo1[VIEW], chi1[VIEW];
          gather_view<VIS>(g, aw, tbl, ax, ay, dir, carry, clo0, chi0);
          gather_view<VIS>(g, as, tbl, ax, ay, dir, carry, clo1, chi1);
          if (memcmp(clo0, clo1, sizeof clo0) || memcmp(chi0, chi1, sizeof chi0)) ++bad;
          // the single-cell reads of K1: the agent's own cell and every position of its line, against the whole tile
          const bool useC = dir & 1;
          const int plen = useC ? g.H : g.W;
          for (int pos = -1; pos <= plen; ++pos) {
            const int x = useC ? ax : pos, y = useC ? pos : ay;
            uint32_t want = CODE_WALL;
            if (pos >= 0 && pos < plen) want = (tile_word<false>(whole, r_word(g, x, y)) >> (8 * (x & 3))) & 0xFFu;
            if (own_line_cell(g, as, ax, ay, dir, pos) != want) ++bad;
          }
        }
  return bad;
}

// W x H tiled geometry, edge 0 (ring lines unstaged) or 1 (border lines unstaged too, which then hold walls).
// Returns the number of mismatching (position, direction, carry, visibility form) cases.
extern "C" long check_staged_gather(int W, int H, int edge, uint64_t seed) {
  const Geom g = make_geom(W, H, LAYOUT_TILED);
  std::vector<uint32_t> whole((size_t)g.wpe * 32), staged((size_t)g.wpe * 32);
  uint64_t s = seed * 2654435761u + 1u;
  // the grid: random cell codes (any type, colour, opacity), the ring lines grey walls, and on a walled handle the border
  std::vector<uint8_t> cells((size_t)W * H);
  for (int lane = 0; lane < 32; ++lane) {
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        const bool border = x == 0 || y == 0 || x == W - 1 || y == H - 1;
        uint32_t c = (edge && border) ? CODE_WALL : (xs(s) & 0xFFu);
        if ((c & 15u) == T_UNSEEN) c |= T_EMPTY;  // a stored cell is never "unseen"
        cells[(size_t)y * W + x] = (uint8_t)c;
      }
    for (int w = 0; w < g.wpe; ++w) whole[(size_t)w * 32 + lane] = CODE_WALL4;  // ring lines and line padding
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        const uint32_t c = cells[(size_t)y * W + x];
        uint8_t *wb = reinterpret_cast<uint8_t *>(whole.data());
        wb[((size_t)r_word(g, x, y) * 32 + lane) * 4 + (x & 3)] = (uint8_t)c;
        wb[((size_t)c_word(g, x, y) * 32 + lane) * 4 + (y & 3)] = (uint8_t)c;
      }
  }
  // what stage_lines copies: rows r_word(0, edge) .. r_word(0, H - edge) and c_word(edge, 0) .. c_word(W - edge, 0);
  // every other row is poison (an open door of a colour beyond the palette: no gather result can contain it)
  const uint32_t POISON = 0x74747474u;
  for (auto &v : staged) v = POISON;
  const int r0 = r_word(g, 0, edge), r1 = r_word(g, 0, H - edge), c0 = c_word(g, edge, 0), c1 = c_word(g, W - edge, 0);
  for (int w = r0; w < r1; ++w) memcpy(&staged[(size_t)w * 32], &whole[(size_t)w * 32], 128);
  for (int w = c0; w < c1; ++w) memcpy(&staged[(size_t)w * 32], &whole[(size_t)w * 32], 128);
  std::vector<uint16_t> tbl(VIS_TBL_BYTES / 2);
  build_vis_table(tbl.data());
  long bad = 0;
  for (int lane = 0; lane < 32; lane += 7) {
    bad += compare_all<VIS_NONE>(g, whole.data() + lane, staged.data() + lane, edge, tbl.data());
    bad += compare_all<VIS_ALU>(g, whole.data() + lane, staged.data() + lane, edge, tbl.data());
    bad += compare_all<VIS_TBL>(g, whole.data() + lane, staged.data() + lane, edge, tbl.data());
  }
  return bad;
}

