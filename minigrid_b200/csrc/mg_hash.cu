// mg_hash.cu — K4: MiniGridEnv.hash() (minigrid_env.py:159-170) of every env, as the 32-byte SHA-256 digest.
// One warp per tile of 32 envs, one lane per env (mg_hash.cuh: hash_lane). Compute-bound: a prefix block is a few
// template broadcasts, up to 32 digit lookups and one SHA-256 compression per lane.
#include <cstdlib>

#include "mg_common.cuh"
#include "mg_hash.cuh"

namespace mg {

constexpr int HASH_WARPS = 4;

// Shared memory of a CTA: the template (uint4 per prefix word), the [3][256] digit table, then per warp the stage
// (lines x = 0..W-1 of array C as [word][lane]) and the lanes' tail scratch.
__host__ __device__ inline uint32_t hash_stage_bytes(const Geom &g) { return (uint32_t)(g.W * g.lswC) * 128u; }
__host__ __device__ inline size_t hash_smem_bytes(const Geom &g) {
  return (size_t)hash_shape(g.W, g.H).nwords * 16 + 3 * 256 + (size_t)HASH_WARPS * (hash_stage_bytes(g) + TILE * HASH_SCRATCH_BYTES);
}

struct HashTmplSmem {
  const uint4 *t;
  __device__ __forceinline__ uint4 operator()(int i) const { return t[i]; }
};
struct HashStageSmem {  // the lane's column of the [word][lane] stage
  const uint8_t *base;
  __device__ __forceinline__ uint32_t operator()(uint32_t off) const { return base[off]; }
};

__global__ void __launch_bounds__(HASH_WARPS * 32, 1)  // (the bare bound makes ptxas spill at 56 registers)
k_hash(const __grid_constant__ Params p, const uint4 *__restrict__ tmpl, int form0, uint8_t *__restrict__ digest) {
  extern __shared__ __align__(16) uint8_t hs_raw[];
  const Geom &g = p.g;
  const HashShape hs = hash_shape(g.W, g.H);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint4 *s_tmpl = reinterpret_cast<uint4 *>(hs_raw);
  uint8_t *s_dig = hs_raw + (size_t)hs.nwords * 16;
  const uint32_t stage_bytes = hash_stage_bytes(g);
  uint8_t *wbase = s_dig + 3 * 256 + (size_t)warp * (stage_bytes + TILE * HASH_SCRATCH_BYTES);
  uint32_t *stage = reinterpret_cast<uint32_t *>(wbase);
  uint8_t *scratch = wbase + stage_bytes + lane * HASH_SCRATCH_BYTES;
  for (int i = threadIdx.x; i < hs.nwords; i += blockDim.x) s_tmpl[i] = tmpl[i];
  for (int i = threadIdx.x; i < 3 * 256; i += blockDim.x) s_dig[i] = (uint8_t)('0' + ((p.cell_lut[i & 255] >> (8 * (i >> 8))) & 0xFFu));
  __syncthreads();
  // This stage is not K3's: K3 stages array C env-major in the window layout (TMA bulk copies need a 16-byte stride),
  // where lanes reading the same cell would hit the same bank (FourRooms: a 512-byte stride, 32-way). Every slot read
  // here is one byte per lane at the same offset, so both layouts are staged [word][lane], with plain loads.
  const int sw = g.W * g.lswC;  // staged words per env
  const int first = g.offC + g.ring * g.lswC;
  const bool tiled = g.layout == LAYOUT_TILED;
  const HashTmplSmem tacc = {s_tmpl};
  const HashStageSmem sacc = {reinterpret_cast<const uint8_t *>(stage) + lane * 4};
  for (int tile = blockIdx.x * HASH_WARPS + warp; tile < p.n_tiles; tile += gridDim.x * HASH_WARPS) {
    __syncwarp();  // every lane is done with the previous tile's stage
    if (tiled) {
      const uint32_t *src = p.grid + ((size_t)tile * g.wpe + first) * 32;
      for (int i = lane; i < sw * 32; i += 32) stage[i] = src[i];
    } else {
      const uint32_t *src = p.grid + (size_t)(tile * TILE + lane) * g.wpe + first;
      for (int w = 0; w < sw; ++w) stage[w * 32 + lane] = src[w];
    }
    __syncwarp();
    const int env = tile * TILE + lane;
    const uint4 rec = p.agent[env];  // padded lanes of the last tile hold a parked agent: harmless, not written
    const int form = ((rec.y >> 8) & FLAG_MOVED) ? FORM_NPINT : form0;
    uint32_t st[8];
    hash_lane(hs, tacc, sacc, s_dig, scratch, (int)(rec.x & 0xFFu), (int)((rec.x >> 8) & 0xFFu), (int)(rec.y & 3u), form, st);
    if (env < p.n_envs) {
      uint8_t *o = digest + (size_t)env * 32;
      if ((reinterpret_cast<uintptr_t>(digest) & 15u) == 0) {
        reinterpret_cast<uint4 *>(o)[0] = make_uint4(bswap32(st[0]), bswap32(st[1]), bswap32(st[2]), bswap32(st[3]));
        reinterpret_cast<uint4 *>(o)[1] = make_uint4(bswap32(st[4]), bswap32(st[5]), bswap32(st[6]), bswap32(st[7]));
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i) o[i] = (uint8_t)(st[i >> 2] >> (24 - 8 * (i & 3)));
      }
    }
  }
}

// Launch shape, once per handle (on its device): as many CTAs as fit, capped by the tile count.
cudaError_t configure_hash(const Params &p, int *grid_out) {
  const size_t smem = hash_smem_bytes(p.g);
  int dev = 0, sms = 0, ctas = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  // the attribute belongs to the kernel, not the handle (as K1's, configure_step): the largest geometry's need, so no
  // handle lowers it for another
  const size_t smem_max = hash_smem_bytes(make_geom(MAX_DIM, MAX_DIM, LAYOUT_TILED));
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_hash, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_max);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas, k_hash, HASH_WARPS * 32, smem);
  if (e != cudaSuccess) return e;
  long long grid = (long long)sms * (ctas > 0 ? ctas : 1);
  const long long want = ((long long)p.n_tiles + HASH_WARPS - 1) / HASH_WARPS;
  if (grid > want) grid = want;
  // test knob shared with K1: a small grid makes every warp walk many tiles
  if (const char *s = getenv("MINIGRID_B200_GRID")) { const long long cap = atoll(s); if (cap >= 1 && cap < grid) grid = cap; }
  *grid_out = (int)(grid < 1 ? 1 : grid);
  return cudaSuccess;
}

cudaError_t launch_hash(const Params &p, int grid, const uint4 *tmpl, int form0, uint8_t *digest, cudaStream_t stream) {
  k_hash<<<(unsigned)grid, HASH_WARPS * 32, hash_smem_bytes(p.g), stream>>>(p, tmpl, form0, digest);
  return cudaGetLastError();
}

}  // namespace mg
