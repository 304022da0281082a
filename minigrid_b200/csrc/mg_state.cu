// mg_state.cu — K3 (FullyObsWrapper.observation, wrappers.py:419-426) and the state exchange kernels
// behind mg_get_state / mg_set_state (the checkpoint / parity-injection boundary).
#include "mg_common.cuh"

namespace mg {

__device__ __forceinline__ uint32_t load_code(const Params &p, int env, int x, int y) {
  return reinterpret_cast<const uint8_t *>(p.grid)[cell_byte_C(p.g, env, x, y)];
}

// K3. out[n][W][H][3] = grid.encode(), agent cell = (OBJECT_TO_IDX["agent"], COLOR_TO_IDX["red"], agent_dir).
// One CTA per tile of 32 environments, whose output block (32 x 3WH bytes) is contiguous. The tile's array C (lines x,
// column-major: ordered like the output) is staged in shared memory by TMA bulk copies — one for a tiled block, one per
// env in the window layout — so that every HBM read of the CTA is in flight at once instead of behind the per-cell
// dependency chain (offset lookup -> byte load -> table lookup -> store) of the previous version. Four consecutive
// cells are twelve output bytes = three aligned words: a thread takes a GROUP of four cells of the tile's flat cell
// sequence (a group may straddle two envs): four code bytes out of the stage, four (type, colour, state) lookups, three
// byte permutes like K1's image stream, three word stores. HBM-bound: array C + the agent record in, 3*W*H out.
__device__ __forceinline__ uint32_t k3_smem(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__host__ __device__ inline uint32_t k3_env_bytes(const Geom &g) { return (uint32_t)(g.wpe - g.offC) * 4u; }  // array C of one env (window layout: a multiple of 16)
__host__ __device__ inline size_t k3_smem_bytes(const Geom &g) {
  return (size_t)TILE * k3_env_bytes(g) + 256 * 4 + TILE * 4 + (MAX_DIM * MAX_DIM + 2) * 2 + 16;
}
__global__ void __launch_bounds__(256)
k_full_obs(const __grid_constant__ Params p, uint8_t *__restrict__ out, int with_agent) {
  extern __shared__ __align__(128) uint8_t k3_raw[];
  const Geom &g = p.g;
  const uint32_t cbytes = k3_env_bytes(g), stage_bytes = TILE * cbytes;
  uint8_t *stage = k3_raw;                                               // tiled: [word][lane] words of array C; window: [env][cbytes]
  uint32_t *s_lut = reinterpret_cast<uint32_t *>(k3_raw + stage_bytes);
  uint32_t *s_agent = s_lut + 256;                  // agent cell index x * H + y | dir << 16 (no agent: never matches)
  uint16_t *s_off = reinterpret_cast<uint16_t *>(s_agent + TILE);  // cell c = x * H + y -> byte offset of the cell inside an env's part of the stage
  uint64_t *bar = reinterpret_cast<uint64_t *>(k3_raw + ((stage_bytes + 256 * 4 + TILE * 4 + (MAX_DIM * MAX_DIM + 2) * 2 + 7) & ~7u));
  const int WH = g.W * g.H, env_bytes = 3 * WH;
  const int tile = blockIdx.x;
  const int nvalid = min(TILE, p.n_envs - tile * TILE);
  const bool tiled = g.layout == LAYOUT_TILED;
  const uint32_t bar_s = k3_smem(bar);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar_s), "r"(1));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0)
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_s), "r"(stage_bytes) : "memory");
  __syncwarp();  // the byte count is armed before any lane of warp 0 issues its copy
  const uint8_t *tb = reinterpret_cast<const uint8_t *>(p.grid) + (size_t)tile * g.wpe * 128;  // both layouts: 32 envs x wpe words
  if (tiled) {
    if (threadIdx.x == 0)  // words offC .. wpe - 1 of all 32 lanes: one contiguous block
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(k3_smem(stage)),
                   "l"(tb + (size_t)g.offC * 128), "r"(stage_bytes), "r"(bar_s) : "memory");
  } else if (threadIdx.x < TILE) {  // env-major: array C of env e is cbytes contiguous bytes
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(k3_smem(stage + threadIdx.x * cbytes)),
                 "l"(tb + (size_t)threadIdx.x * g.wpe * 4 + (size_t)g.offC * 4), "r"(cbytes), "r"(bar_s) : "memory");
  }
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_lut[i] = decode_cell((uint32_t)i);
  if (threadIdx.x < TILE) {
    const uint4 rec = p.agent[tile * TILE + threadIdx.x];
    s_agent[threadIdx.x] = with_agent ? ((rec.x & 0xFFu) * (uint32_t)g.H + ((rec.x >> 8) & 0xFFu)) | ((rec.y & 3u) << 16) : 0xFFFFu;
  }
  const float inv_h = 1.0f / (float)g.H;
  for (int c = threadIdx.x; c < WH; c += blockDim.x) {
    const int x = (int)(((float)c + 0.5f) * inv_h), y = c - x * g.H;  // exact: (c + 0.5) / H is never within rounding of an integer
    const int cw = c_word(g, x, y) - g.offC;  // word of the cell inside array C
    s_off[c] = (uint16_t)(tiled ? cw * 128 + (y & 3) : cw * 4 + (y & 3));
  }
  if (threadIdx.x == 0) {  // the stage has landed: one thread watches the barrier, the CTA barrier passes it on
    asm volatile(
        "{\n.reg .pred p;\nK3W_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra K3D_%=;\nbra K3W_%=;\nK3D_%=:\n}\n" ::"r"(bar_s), "r"(0) : "memory");
  }
  __syncthreads();
  const uint32_t estride = tiled ? 4u : cbytes;
  const float inv_wh = 1.0f / (float)WH;
  auto triple = [&](int e, int c) -> uint32_t {  // type | colour << 8 | state << 16 of cell c of env e
    const uint32_t ag = s_agent[e];
    const uint32_t t = s_lut[stage[(uint32_t)e * estride + s_off[c]]];
    return (ag & 0xFFFFu) == (uint32_t)c ? (T_AGENT | (C_RED << 8) | (ag & 0x30000u)) : t;
  };
  uint8_t *dst = out + (size_t)tile * TILE * env_bytes;
  const int n_cells = nvalid * WH;
  if ((reinterpret_cast<uintptr_t>(dst) & 3u) == 0) {
    uint32_t *d32 = reinterpret_cast<uint32_t *>(dst);
    for (int gq = threadIdx.x; gq < n_cells / 4; gq += blockDim.x) {
      const int f0 = 4 * gq;
      int e = (int)(((float)f0 + 0.5f) * inv_wh), c = f0 - e * WH;  // exact small-integer division
      uint32_t t[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        t[k] = triple(e, c);
        if (++c == WH) { c = 0; ++e; }
      }
      d32[3 * gq] = prmt(t[0], t[1], 0x4210u);
      d32[3 * gq + 1] = prmt(t[1], t[2], 0x5421u);
      d32[3 * gq + 2] = prmt(t[2], t[3], 0x6542u);
    }
    for (int f = (n_cells & ~3) + threadIdx.x; f < n_cells; f += blockDim.x) {  // ragged last tile: up to 3 cells left
      const int e = f / WH, c = f - e * WH;
      const uint32_t t = triple(e, c);
      dst[3 * f] = (uint8_t)t; dst[3 * f + 1] = (uint8_t)(t >> 8); dst[3 * f + 2] = (uint8_t)(t >> 16);
    }
  } else {
    for (int f = threadIdx.x; f < n_cells; f += blockDim.x) {
      const int e = f / WH, c = f - e * WH;
      const uint32_t t = triple(e, c);
      dst[3 * f] = (uint8_t)t; dst[3 * f + 1] = (uint8_t)(t >> 8); dst[3 * f + 2] = (uint8_t)(t >> 16);
    }
  }
}

__global__ void k_get_agent(Params p, int32_t *__restrict__ agent, uint64_t *__restrict__ rng, uint8_t *__restrict__ pending) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= p.n_envs) return;
  const uint4 rec = p.agent[env];
  if (agent) {
    int32_t *a = agent + (size_t)env * 6;
    a[0] = rec.x & 0xFF; a[1] = (rec.x >> 8) & 0xFF; a[2] = rec.y & 3;
    const bool boxed = (rec.z & 15u) == T4_BOX_WITH_KEY;  // carrying.encode(): a grey box, whatever is inside
    a[3] = rec.z ? (boxed ? (int32_t)T_BOX : (int32_t)(rec.z & 15u)) : -1;
    a[4] = rec.z ? (boxed ? (int32_t)C_GREY : (int32_t)((rec.z >> 4) & 7u)) : 0; a[5] = (int32_t)rec.w;
  }
  if (rng) {
    const RngRec r = p.rng[env];
    uint64_t *o = rng + (size_t)env * 6;
    o[0] = r.state_hi; o[1] = r.state_lo; o[2] = r.inc_hi; o[3] = r.inc_lo; o[4] = r.has_uint32; o[5] = r.uinteger;
  }
  if (pending) pending[env] = ((rec.y >> 8) & FLAG_PENDING) ? 1 : 0;
}

// grid[n][W][H][3] -> both arrays of every env. One thread per (env, cell): two byte stores.
__global__ void k_set_grid(Params p, const uint8_t *__restrict__ grid) {
  const int cells = p.g.W * p.g.H;
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= (long long)p.n_envs * cells) return;
  const int env = (int)(gid / cells), c = (int)(gid % cells);
  const int x = c / p.g.H, y = c % p.g.H;
  const uint8_t *in = grid + gid * 3;
  const uint8_t code = (uint8_t)encode_cell(in[0], in[1], in[2]);
  uint8_t *gb = reinterpret_cast<uint8_t *>(p.grid);
  gb[cell_byte_R(p.g, env, x, y)] = code;
  gb[cell_byte_C(p.g, env, x, y)] = code;
}

__global__ void k_set_agent(Params p, const int32_t *__restrict__ agent, const uint64_t *__restrict__ rng,
                            const uint8_t *__restrict__ pending) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= p.n_envs) return;
  uint4 rec = p.agent[env];
  if (agent) {
    const int32_t *a = agent + (size_t)env * 6;
    // K1 derives window offsets and bit-mask shifts from the record without further checks: refuse what the
    // reference could never hold (agent_pos inside the grid, dir 0..3, carrying in {None, Key, Ball, Box})
    const bool ok = a[0] >= 0 && a[0] < p.g.W && a[1] >= 0 && a[1] < p.g.H && a[2] >= 0 && a[2] <= 3 &&
                    (a[3] < 0 || ((a[3] >= (int)T_KEY && a[3] <= (int)T_BOX) && a[4] >= 0 && a[4] <= (int)C_GREY)) && a[5] >= 0;
    if (!ok) {
      atomicOr(p.err, ERR_BAD_STATE);
      return;  // record, rng and pending flag of this env stay as they were
    }
    rec.x = (rec.x & 0xFFFF0000u) | (uint32_t)(a[0] & 0xFF) | ((uint32_t)(a[1] & 0xFF) << 8);  // keeps the post-filter targets
    rec.y = (rec.y & ~3u) | (uint32_t)(a[2] & 3) | (FLAG_MOVED << 8);  // an injected position hashes as a tuple of numpy ints
    rec.z = a[3] >= 0 ? ((uint32_t)(a[3] & 15) | ((uint32_t)(a[4] & 7) << 4)) : 0u;
    rec.w = (uint32_t)a[5];
  }
  if (pending) {
    uint32_t flags = (rec.y >> 8) & ~FLAG_PENDING;
    if (pending[env]) flags |= FLAG_PENDING;
    rec.y = (rec.y & 0xFFu) | (flags << 8);
  }
  p.agent[env] = rec;
  if (rng) {
    const uint64_t *i = rng + (size_t)env * 6;
    RngRec r;
    r.state_hi = i[0]; r.state_lo = i[1]; r.inc_hi = i[2]; r.inc_lo = i[3];
    r.has_uint32 = (uint32_t)i[4]; r.uinteger = (uint32_t)i[5]; r.pad = 0;
    p.rng[env] = r;
  }
}

// arena initialisation: every byte a grey wall (ring lines and line padding stay that way), agents parked
// at (1,1) facing right so that padded lanes of a partial tile compute something harmless.
__global__ void k_init(Params p) {
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long words = (long long)p.n_tiles * p.g.wpe * 32;
  if (gid < words) p.grid[gid] = CODE_WALL4;
  if (gid < (long long)p.n_tiles * 32) {
    p.agent[gid] = make_uint4(1u | (1u << 8), 0u, 0u, 0u);
    RngRec r;
    r.state_hi = r.state_lo = r.inc_hi = 0; r.inc_lo = 1; r.has_uint32 = r.uinteger = 0; r.pad = 0;
    p.rng[gid] = r;
  }
}

cudaError_t launch_full_obs(const Params &p, uint8_t *out, int with_agent, cudaStream_t stream) {
  k_full_obs<<<(unsigned)p.n_tiles, 256, k3_smem_bytes(p.g), stream>>>(p, out, with_agent);  // <= 35 KB: under the 48 KB default
  return cudaGetLastError();
}
cudaError_t launch_get_state(const Params &p, uint8_t *grid, int32_t *agent, uint64_t *rng, uint8_t *pending, cudaStream_t stream) {
  if (grid) {
    cudaError_t e = launch_full_obs(p, grid, 0, stream);
    if (e != cudaSuccess) return e;
  }
  if (agent || rng || pending) k_get_agent<<<(p.n_envs + 127) / 128, 128, 0, stream>>>(p, agent, rng, pending);
  return cudaGetLastError();
}
cudaError_t launch_set_state(const Params &p, const uint8_t *grid, const int32_t *agent, const uint64_t *rng,
                             const uint8_t *pending, cudaStream_t stream) {
  if (grid) {
    const long long total = (long long)p.n_envs * p.g.W * p.g.H;
    k_set_grid<<<(unsigned)((total + 255) / 256), 256, 0, stream>>>(p, grid);
  }
  if (agent || rng || pending) k_set_agent<<<(p.n_envs + 127) / 128, 128, 0, stream>>>(p, agent, rng, pending);
  return cudaGetLastError();
}
__global__ void k_clear_err(int *err, int bits) { atomicAnd(err, ~bits); }
cudaError_t launch_clear_err(const Params &p, int bits, cudaStream_t stream) {
  k_clear_err<<<1, 1, 0, stream>>>(p.err, bits);
  return cudaGetLastError();
}
cudaError_t launch_init(const Params &p, cudaStream_t stream) {
  const long long words = (long long)p.n_tiles * p.g.wpe * 32;
  k_init<<<(unsigned)((words + 255) / 256), 256, 0, stream>>>(p);
  return cudaGetLastError();
}

}  // namespace mg
