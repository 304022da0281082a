// hash_emu.cpp — TEST BUILD ONLY. mg_hash.cuh (the per-lane SHA-256 and the template walk of k_hash) compiled by g++
// through mg_host_shim.h, with k_hash's staging replayed tile by tile on the CPU, so that tests/test_hash_cpu.py can
// check it against hashlib and the oracle WITHOUT a GPU. Not part of the product.
#include <cstring>
#include <vector>

#include "../../minigrid_b200/csrc/mg_common.cuh"
#include "../../minigrid_b200/csrc/mg_hash.cuh"

using namespace mg;

namespace {
struct Tmpl {
  const uint4 *t;
  uint4 operator()(int i) const { return t[i]; }
};
struct Stage {
  const uint8_t *base;
  uint32_t operator()(uint32_t off) const { return base[off]; }
};
void digit_table(uint8_t *dig) {  // k_hash's [3][256] digit table
  for (int i = 0; i < 3 * 256; ++i) dig[i] = (uint8_t)('0' + ((decode_cell((uint32_t)(i & 255)) >> (8 * (i >> 8))) & 0xFFu));
}
void store_digest(const uint32_t (&st)[8], uint8_t *out) {
  for (int i = 0; i < 32; ++i) out[i] = (uint8_t)(st[i >> 2] >> (24 - 8 * (i & 3)));
}
}  // namespace

extern "C" {

// SHA-256 of an arbitrary message through sha256_compress and sha256_pad
void hash_emu_sha256(const uint8_t *msg, int64_t len, uint8_t *out) {
  uint32_t st[8], w[16];
  sha256_init(st);
  int64_t off = 0;
  for (; off + 64 <= len; off += 64) {
    sha256_block_words(msg + off, w);
    sha256_compress(st, w);
  }
  alignas(4) uint8_t buf[128];
  const int rem = (int)(len - off);
  if (rem) memcpy(buf, msg + off, (size_t)rem);
  const int nb = sha256_pad(buf, rem, (uint64_t)len);
  for (int b = 0; b < nb; ++b) {
    sha256_block_words(buf + 64 * b, w);
    sha256_compress(st, w);
  }
  store_digest(st, out);
}

// k_hash on n envs given as Grid.encode() arrays (uint8[n][W][H][3]), agent records (int32[n][6]: x, y, dir, ...) and
// forms (int32[n], FORM_*): the grid arena is built in `layout`, each tile's array C staged [word][lane] as k_hash
// stages it, one hash_lane per lane. out: uint8[n][32].
void hash_emu_batch(int W, int H, int layout, int n, const uint8_t *grid, const int32_t *agent, const int32_t *forms, uint8_t *out) {
  const Geom g = make_geom(W, H, layout);
  const int n_tiles = (n + TILE - 1) / TILE;
  std::vector<uint32_t> arena((size_t)n_tiles * g.wpe * 32, CODE_WALL4);
  uint8_t *ab = reinterpret_cast<uint8_t *>(arena.data());
  for (int env = 0; env < n; ++env)
    for (int x = 0; x < W; ++x)
      for (int y = 0; y < H; ++y) {
        const uint8_t *c = grid + (((size_t)env * W + x) * H + y) * 3;
        ab[cell_byte_C(g, env, x, y)] = (uint8_t)encode_cell(c[0], c[1], c[2]);
      }
  const HashShape hs = hash_shape(W, H);
  std::vector<uint4> tmpl(hs.nwords);
  build_hash_template(W, H, g.lswC, tmpl.data());
  uint8_t dig[3 * 256];
  digit_table(dig);
  const int sw = W * g.lswC, first = g.offC + g.ring * g.lswC;
  std::vector<uint32_t> stage((size_t)sw * 32);
  alignas(4) uint8_t scratch[HASH_SCRATCH_BYTES];
  for (int tile = 0; tile < n_tiles; ++tile) {
    for (int lane = 0; lane < 32; ++lane)
      for (int w = 0; w < sw; ++w) stage[(size_t)w * 32 + lane] = arena[grid_word(g, tile * TILE + lane, first + w)];
    for (int lane = 0; lane < 32; ++lane) {
      const int env = tile * TILE + lane;
      if (env >= n) continue;
      const int32_t *a = agent + (size_t)env * 6;
      uint32_t st[8];
      hash_lane(hs, Tmpl{tmpl.data()}, Stage{reinterpret_cast<const uint8_t *>(stage.data()) + lane * 4}, dig, scratch, a[0], a[1], a[2],
                forms[env], st);
      store_digest(st, out + (size_t)env * 32);
    }
  }
}

}  // extern "C"
