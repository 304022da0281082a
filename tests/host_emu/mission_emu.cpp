// mission_emu.cpp — TEST BUILD ONLY. The engine's mission code path compiled for the CPU with g++: the roomgrid generator
// (mg_levels.cuh: draw_level, which leaves the mission code in the Level) and the renderer every mission kernel calls
// (mg_mission.cuh), so tests/test_babyai_missions_cpu.py checks them against the oracles without a GPU. Not part of
// the product: minigrid_b200/ never builds or loads it.
#include <cstring>

#include "../../minigrid_b200/csrc/mg_common.cuh"
#include "../../minigrid_b200/csrc/mg_levels.cuh"
#include "../../minigrid_b200/csrc/mg_mission.cuh"
#include "../../minigrid_b200/csrc/mg_pcg64.cuh"

using namespace mg;

extern "C" {

// the mission code K2 / K1 store for each seed (np_random = Generator(PCG64(SeedSequence(seed))), then one reset)
void mis_draw(int W, int H, const int32_t *params, int n_params, int layout, const uint64_t *seeds, int n, uint32_t *out) {
  Params p;
  memset(&p, 0, sizeof(p));
  p.g = make_geom(W, H, layout);
  p.kind = KIND_ROOMGRID;
  for (int i = 0; i < 8; ++i) p.kp[i] = i < n_params ? params[i] : 0;
  for (int k = 0; k < n; ++k) {
    Pcg r = seed_pcg64(seeds[k]);
    Level L = blank_level();
    draw_level<KIND_ROOMGRID>(p, r, L);
    out[k] = level_mission(L);
  }
}

// k_mission_text, k_mission_indices and k_flat_missions' text, one code at a time
void mis_text(const uint32_t *codes, int n, uint8_t *out) {
  for (int k = 0; k < n; ++k) mission_text(codes[k], out + (size_t)k * MISSION_TEXT_BYTES);
}
void mis_indices(const uint32_t *codes, int n, int max_words, int64_t *out) {
  for (int k = 0; k < n; ++k) mission_indices(codes[k], max_words, reinterpret_cast<long long *>(out) + (size_t)k * max_words);
}
void mis_onehot(const uint32_t *codes, int n, uint8_t *out) {  // the 96 x 28 mission part of a FlatObsWrapper row
  for (int k = 0; k < n; ++k) {
    uint8_t t[MISSION_TEXT_BYTES];
    mission_text(codes[k], t);
    uint8_t *o = out + (size_t)k * MISSION_TEXT_BYTES * MISSION_CHAR_CODES;
    memset(o, 0, MISSION_TEXT_BYTES * MISSION_CHAR_CODES);
    for (int j = 0; j < MISSION_TEXT_BYTES && t[j]; ++j) o[j * MISSION_CHAR_CODES + mission_char_code(t[j])] = 1;
  }
}

}  // extern "C"
