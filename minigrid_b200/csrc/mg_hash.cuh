// mg_hash.cuh — MiniGridEnv.hash() (minigrid_env.py:159-170) for one environment per lane: SHA-256 of
//   str(grid.encode().tolist()) + str(agent_pos) + str(agent_dir)
// Per-lane code only (the kernel is mg_hash.cu); g++ compiles it too for tests/host_emu.
//
// The grid part has a fixed length for a geometry: every value of Grid.encode() is one digit (types 1..9, colours
// 0..5, states 0..2; the grid never holds the agent), so each cell prints as "[t, c, s]" and the prefix is
// L = 11 W H + 2 W bytes, in x-major order (array C's line order). Only its 3 W H digits vary between envs. A table
// built once per geometry (build_hash_template) gives, for every 4-byte word of the prefix, the literal bytes and up
// to two digit slots (a digit never follows another within 3 bytes). The tail str(agent_pos) + str(agent_dir) is 6 to
// 29 bytes and depends on how the reference last assigned agent_pos (see hash_form below).
#pragma once
#include "mg_common.cuh"

namespace mg {

// str(agent_pos) forms. A: tuple of Python ints "(1, 1)"; B: tuple of numpy ints "(np.int64(3), np.int64(12))";
// C: numpy's str(ndarray), elements right-aligned to a common width "[ 3 10]".
// A lane's form is FORM_NPINT when FLAG_MOVED is set in its agent record, else the kind's hash_initial_form.
enum : int { FORM_TUPLE = 0, FORM_NPINT = 1, FORM_ARRAY = 2 };

// The form right after a reset, per kind (kp as in Params::kp):
//   A  agent_pos = self.agent_start_pos: empty.py:109, distshift.py:115, dynamicobstacles.py:123 (fixed starts)
//   C  agent_pos = np.array(...): crossing.py:141, lavagap.py:110, memory.py:129
//   B  place_agent / place_obj (minigrid_env.py:347-350, 383-395) everywhere else, and after every successful forward
//      move (minigrid_env.py:553, tuple(agent_pos + dir_vec)), whatever the kind
MG_HD int hash_initial_form(int kind, const int *kp) {
  if ((kind == KIND_EMPTY && !kp[0]) || kind == KIND_DISTSHIFT || (kind == KIND_DYNOBS && !kp[1])) return FORM_TUPLE;
  if (kind == KIND_CROSSING || kind == KIND_LAVAGAP || kind == KIND_MEMORY) return FORM_ARRAY;
  return FORM_NPINT;
}

struct HashShape {
  int L;       // prefix bytes
  int nwords;  // template words: ceil(L / 4)
  int nfull;   // whole prefix blocks: floor(L / 64)
  int rem;     // prefix bytes in the last, lane-specific blocks: L mod 64
};
MG_HD HashShape hash_shape(int W, int H) {
  HashShape s;
  s.L = 11 * W * H + 2 * W;
  s.nwords = (s.L + 3) >> 2;
  s.nfull = s.L >> 6;
  s.rem = s.L & 63;
  return s;
}

// Digit slot of a template word: bit 31 valid, bits 24-28 shift of the byte in the big-endian word, bits 16-17 the
// component (type, colour, state), bits 0-15 the cell's byte offset in a lane's stage (hash_stage_offset).
// The stage holds lines x = 0..W-1 of array C as [word][lane] (32-bit words, lane-interleaved).
MG_HD uint32_t hash_stage_offset(int lswC, int x, int y) { return (uint32_t)((x * lswC + (y >> 2)) * 128 + (y & 3)); }
inline void build_hash_template(int W, int H, int lswC, uint4 *tmpl) {
  const HashShape s = hash_shape(W, H);
  for (int i = 0; i < s.nwords; ++i) tmpl[i] = make_uint4(0, 0, 0, 0);
  int pos = 0;
  auto lit = [&](char c) {
    uint4 &t = tmpl[pos >> 2];
    t.x |= (uint32_t)(uint8_t)c << (24 - 8 * (pos & 3));
    ++pos;
  };
  auto digit = [&](int x, int y, int comp) {
    uint4 &t = tmpl[pos >> 2];
    const uint32_t slot = 0x80000000u | ((uint32_t)(24 - 8 * (pos & 3)) << 24) | ((uint32_t)comp << 16) | hash_stage_offset(lswC, x, y);
    if (t.y == 0) t.y = slot; else t.z = slot;
    ++pos;
  };
  lit('[');
  for (int x = 0; x < W; ++x) {
    if (x) { lit(','); lit(' '); }
    lit('[');
    for (int y = 0; y < H; ++y) {
      if (y) { lit(','); lit(' '); }
      lit('['); digit(x, y, 0); lit(','); lit(' '); digit(x, y, 1); lit(','); lit(' '); digit(x, y, 2); lit(']');
    }
    lit(']');
  }
  lit(']');
}

// One template word for a lane. stage: the lane's stage bytes (byte at a slot offset); dig: [3][256] ASCII digit of
// component j of cell code c (decode_cell).
template <class Stage>
MG_HD uint32_t hash_tmpl_word(const uint4 &t, const Stage &stage, const uint8_t *dig) {
  uint32_t w = t.x;
  if (t.y) w |= (uint32_t)dig[((t.y >> 8) & 0x300u) | stage(t.y & 0xFFFFu)] << ((t.y >> 24) & 31u);
  if (t.z) w |= (uint32_t)dig[((t.z >> 8) & 0x300u) | stage(t.z & 0xFFFFu)] << ((t.z >> 24) & 31u);
  return w;
}

MG_HD uint32_t rotr32(uint32_t x, int n) {
#ifdef __CUDA_ARCH__
  return __funnelshift_r(x, x, (uint32_t)n);
#else
  return (x >> n) | (x << (32 - n));
#endif
}
MG_HD uint32_t bswap32(uint32_t x) {
#ifdef __CUDA_ARCH__
  return __byte_perm(x, 0u, 0x0123u);
#else
  return __builtin_bswap32(x);
#endif
}

MG_HD void sha256_init(uint32_t (&st)[8]) {
  st[0] = 0x6a09e667u; st[1] = 0xbb67ae85u; st[2] = 0x3c6ef372u; st[3] = 0xa54ff53au;
  st[4] = 0x510e527fu; st[5] = 0x9b05688cu; st[6] = 0x1f83d9abu; st[7] = 0x5be0cd19u;
}

// FIPS 180-4 section 6.2.2 on one 64-byte block of big-endian words; the schedule is kept in w (16 words, rolling).
MG_HD void sha256_compress(uint32_t (&st)[8], uint32_t (&w)[16]) {
  const uint32_t K[64] = {
      0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u,
      0xd807aa98u, 0x12835b01u, 0x243185beu, 0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u,
      0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau, 0x5cb0a9dcu, 0x76f988dau,
      0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u,
      0x27b70a85u, 0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u,
      0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u, 0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u,
      0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu, 0x682e6ff3u,
      0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};
  uint32_t a = st[0], b = st[1], c = st[2], d = st[3], e = st[4], f = st[5], g = st[6], h = st[7];
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    if (i >= 16) {
      const uint32_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
      const uint32_t s0 = rotr32(w15, 7) ^ rotr32(w15, 18) ^ (w15 >> 3);
      const uint32_t s1 = rotr32(w2, 17) ^ rotr32(w2, 19) ^ (w2 >> 10);
      w[i & 15] += s0 + w[(i - 7) & 15] + s1;
    }
    const uint32_t S1 = rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25);
    const uint32_t ch = (e & f) ^ (~e & g);
    const uint32_t t1 = h + S1 + ch + K[i] + w[i & 15];
    const uint32_t S0 = rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22);
    const uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
    h = g; g = f; f = e; e = d + t1;
    d = c; c = b; b = a; a = t1 + S0 + mj;
  }
  st[0] += a; st[1] += b; st[2] += c; st[3] += d; st[4] += e; st[5] += f; st[6] += g; st[7] += h;
}

// SHA-256 padding of the message's last `rem` bytes (rem < 64), which buf already holds at 0..rem-1 (buf: 128
// bytes, 4-aligned): 0x80, zeros, the 64-bit big-endian bit length of the whole `len`-byte message. Returns the
// number of blocks to compress from buf: 1, or 2 when rem > 55.
MG_HD int sha256_pad(uint8_t *buf, int rem, uint64_t len) {
  const int nb = rem + 9 > 64 ? 2 : 1;
  buf[rem] = 0x80;
  for (int i = rem + 1; i < 64 * nb - 8; ++i) buf[i] = 0;
  const uint64_t bits = len * 8u;
  for (int i = 0; i < 8; ++i) buf[64 * nb - 1 - i] = (uint8_t)(bits >> (8 * i));
  return nb;
}
MG_HD void sha256_block_words(const uint8_t *blk, uint32_t (&w)[16]) {
#pragma unroll
  for (int i = 0; i < 16; ++i) w[i] = bswap32(*reinterpret_cast<const uint32_t *>(blk + 4 * i));
}

// str(v) of a coordinate (0 <= v < 100) right-aligned in `width` characters
MG_HD int put_coord(uint8_t *d, int n, int v, int width) {
  if (width == 2) d[n++] = v >= 10 ? (uint8_t)('0' + v / 10) : (uint8_t)' ';
  d[n++] = (uint8_t)('0' + v % 10);
  return n;
}
MG_HD int put_npint_open(uint8_t *d, int n) {  // "np.int64("
  d[n] = 'n'; d[n + 1] = 'p'; d[n + 2] = '.'; d[n + 3] = 'i'; d[n + 4] = 'n'; d[n + 5] = 't'; d[n + 6] = '6'; d[n + 7] = '4';
  d[n + 8] = '(';
  return n + 9;
}
// str(agent_pos) + str(agent_dir) in the given form, then the 0x80 padding byte. Returns the tail's length (without it).
MG_HD int hash_tail(uint8_t *d, int x, int y, int dir, int form) {
  const int lx = x >= 10 ? 2 : 1, ly = y >= 10 ? 2 : 1;
  int n = 0;
  if (form == FORM_ARRAY) {  // numpy pads every element to the widest one
    const int wd = lx > ly ? lx : ly;
    d[n++] = '[';
    n = put_coord(d, n, x, wd);
    d[n++] = ' ';
    n = put_coord(d, n, y, wd);
    d[n++] = ']';
  } else {
    const bool np = form == FORM_NPINT;
    d[n++] = '(';
    if (np) n = put_npint_open(d, n);
    n = put_coord(d, n, x, lx);
    if (np) d[n++] = ')';
    d[n++] = ','; d[n++] = ' ';
    if (np) n = put_npint_open(d, n);
    n = put_coord(d, n, y, ly);
    if (np) d[n++] = ')';
    d[n++] = ')';
  }
  d[n++] = (uint8_t)('0' + (dir & 3));
  d[n] = 0x80;
  return n;
}

constexpr int HASH_SCRATCH_BYTES = 36;  // a lane's tail: up to 3 alignment bytes + 29 + 0x80; 9 words (odd: no bank conflicts)

// The whole hash of one lane's env. tmpl(i): template word i (the same for every lane: a broadcast); stage(off):
// the lane's stage byte at a slot offset; scratch: HASH_SCRATCH_BYTES of the lane's own, 4-aligned. The prefix
// blocks run in lockstep across lanes; only the last one or two blocks (prefix remainder + tail + padding) differ.
template <class Tmpl, class Stage>
MG_HD void hash_lane(const HashShape &hs, const Tmpl &tmpl, const Stage &stage, const uint8_t *dig, uint8_t *scratch,
                     int x, int y, int dir, int form, uint32_t (&st)[8]) {
  sha256_init(st);
  for (int b = 0; b < hs.nfull; ++b) {
    uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) w[i] = hash_tmpl_word(tmpl(16 * b + i), stage, dig);
    sha256_compress(st, w);
  }
  // the last blocks: prefix bytes 0..rem-1 from the template, the tail at rem.., 0x80, zeros, the bit length
  uint32_t *sw = reinterpret_cast<uint32_t *>(scratch);
#pragma unroll
  for (int k = 0; k < HASH_SCRATCH_BYTES / 4; ++k) sw[k] = 0;
  const int r = hs.rem, r4 = r >> 2;
  const int t = hash_tail(scratch + (r & 3), x, y, dir, form);
  const uint64_t bits = (uint64_t)(hs.L + t) * 8u;
  const bool two = r + t + 9 > 64;
  const int rw = (r + 3) >> 2;  // template words that hold prefix bytes
#pragma unroll 1
  for (int blk = 0; blk < 2; ++blk) {
    uint32_t w[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int wi = 16 * blk + i;
      uint32_t v = wi < rw ? hash_tmpl_word(tmpl(16 * hs.nfull + wi), stage, dig) : 0u;
      const int k = wi - r4;
      if (k >= 0 && k < HASH_SCRATCH_BYTES / 4) v |= bswap32(sw[k]);
      if (blk == (two ? 1 : 0) && i >= 14) v = i == 14 ? (uint32_t)(bits >> 32) : (uint32_t)bits;
      w[i] = v;
    }
    if (blk == 0 || two) sha256_compress(st, w);
  }
}

}  // namespace mg
