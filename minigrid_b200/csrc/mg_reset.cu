// mg_reset.cu — K2: MiniGridEnv.reset (minigrid_env.py:119-157) = per-kind _gen_grid with numpy-exact RNG for
// EVERY environment (the explicit VectorEnv.reset()), one lane per environment; autoreset of individual
// environments happens inside K1 (mg_step.cu). Also the seeding kernel (SeedSequence -> PCG64).
// The generators themselves live in mg_levels.cuh.
#include "mg_common.cuh"
#include "mg_obs.cuh"
#include "mg_pcg64.cuh"
#include "mg_levels.cuh"
#include "mg_postfilter.cuh"

namespace mg {

// gen_obs straight out of HBM (rare paths), either layout
__device__ void gen_obs_global(const Params &p, int env, int ax, int ay, int dir, uint32_t carry, uint32_t (&S)[OBS_WORDS]) {
  const uint32_t *base = p.grid + grid_word(p.g, env, 0);
  if (p.g.layout == LAYOUT_TILED) {
    const AccTiled acc = {base, false};
    if (p.see_through) gen_obs_words<VIS_NONE>(p.g, acc, p.cell_lut, p.vis_tbl, ax, ay, dir, carry, S);
    else gen_obs_words<VIS_ALU>(p.g, acc, p.cell_lut, p.vis_tbl, ax, ay, dir, carry, S);
  } else {
    const AccFlat acc = {base};
    if (p.see_through) gen_obs_words<VIS_NONE>(p.g, acc, p.cell_lut, p.vis_tbl, ax, ay, dir, carry, S);
    else gen_obs_words<VIS_ALU>(p.g, acc, p.cell_lut, p.vis_tbl, ax, ay, dir, carry, S);
  }
}

template <int KIND>
__global__ void __launch_bounds__(128)
k_reset(Params p, const uint8_t *__restrict__ mask, uint8_t *__restrict__ obs, int32_t *__restrict__ dir_out) {
  for (int env = blockIdx.x * blockDim.x + threadIdx.x; env < p.n_envs; env += gridDim.x * blockDim.x) {
    // partial reset (gymnasium >= 1.1 VectorEnv.reset(options={"reset_mask": mask})): the other envs keep their
    // state, their pending flag and their slots of the output buffers
    if (mask && !mask[env]) continue;
    Pcg r = load_rng(p.rng + env);
    Level L;
    draw_level<KIND>(p, r, L);
    store_rng(p.rng + env, r);
    fill_level<KIND>(p, L, env);
    uint4 rec;
    rec.x = (uint32_t)L.ax | ((uint32_t)L.ay << 8);
    rec.y = (uint32_t)L.adir;  // flags cleared: SyncVectorEnv.reset() clears _autoreset_envs; FLAG_MOVED: the generator placed the agent
    if (has_post_filter<KIND>()) {  // post-filter targets in the spare bits (mg_postfilter.cuh)
      rec.x |= ((uint32_t)level_tx(L) << 16) | ((uint32_t)level_ty(L) << 24);
      rec.y |= level_aux(L) << 16;
    }
    if (KIND == KIND_DYNOBS) {
      uint32_t ex[4];
      dynobs_pack(L, ex);
      p.extra[env] = make_uint4(ex[0], ex[1], ex[2], ex[3]);
    }
    rec.z = 0;  // carrying = None
    rec.w = 0;  // step_count = 0
    p.agent[env] = rec;
    if (dir_out) dir_out[env] = L.adir;
    if (obs) {
      uint32_t S[OBS_WORDS];
      gen_obs_global(p, env, L.ax, L.ay, L.adir, 0u, S);
      emit_obs_bytes(obs + (size_t)env * OBS_BYTES, S);
    }
  }
}

cudaError_t launch_reset(const Params &p, const uint8_t *mask, uint8_t *obs, int32_t *dir, cudaStream_t stream) {
  const int threads = 128;
  const int blocks = (p.n_envs + threads - 1) / threads;
  switch (p.kind) {
    case KIND_EMPTY: k_reset<KIND_EMPTY><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_DOORKEY: k_reset<KIND_DOORKEY><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_CROSSING: k_reset<KIND_CROSSING><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_LAVAGAP: k_reset<KIND_LAVAGAP><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_DISTSHIFT: k_reset<KIND_DISTSHIFT><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_MULTIROOM: k_reset<KIND_MULTIROOM><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_LOCKEDROOM: k_reset<KIND_LOCKEDROOM><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_PLAYGROUND: k_reset<KIND_PLAYGROUND><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_GOTODOOR: k_reset<KIND_GOTODOOR><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_FETCH: k_reset<KIND_FETCH><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_REDBLUEDOORS: k_reset<KIND_REDBLUEDOORS><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_GOTOOBJECT: k_reset<KIND_GOTOOBJECT><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_PUTNEAR: k_reset<KIND_PUTNEAR><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_MEMORY: k_reset<KIND_MEMORY><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_DYNOBS: k_reset<KIND_DYNOBS><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    case KIND_ROOMGRID: k_reset<KIND_ROOMGRID><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
    default: k_reset<KIND_FOURROOMS><<<blocks, threads, 0, stream>>>(p, mask, obs, dir); break;
  }
  return cudaGetLastError();
}

// the level template (words of a blank draw), once per handle
template <int KIND>
__global__ void k_template(Params p, uint32_t *tmpl) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= p.g.wpe) return;
  const Level L = blank_level();
  tmpl[w] = level_word<KIND>(p, L, w);
}
cudaError_t launch_template(const Params &p, uint32_t *tmpl, cudaStream_t stream) {
  const int blocks = (p.g.wpe + 63) / 64;
  switch (p.kind) {
    case KIND_EMPTY: k_template<KIND_EMPTY><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_DOORKEY: k_template<KIND_DOORKEY><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_CROSSING: k_template<KIND_CROSSING><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_LAVAGAP: k_template<KIND_LAVAGAP><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_DISTSHIFT: k_template<KIND_DISTSHIFT><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_MULTIROOM: k_template<KIND_MULTIROOM><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_LOCKEDROOM: k_template<KIND_LOCKEDROOM><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_PLAYGROUND: k_template<KIND_PLAYGROUND><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_GOTODOOR: k_template<KIND_GOTODOOR><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_FETCH: k_template<KIND_FETCH><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_REDBLUEDOORS: k_template<KIND_REDBLUEDOORS><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_GOTOOBJECT: k_template<KIND_GOTOOBJECT><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_PUTNEAR: k_template<KIND_PUTNEAR><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_MEMORY: k_template<KIND_MEMORY><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_DYNOBS: k_template<KIND_DYNOBS><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    case KIND_ROOMGRID: k_template<KIND_ROOMGRID><<<blocks, 64, 0, stream>>>(p, tmpl); break;
    default: k_template<KIND_FOURROOMS><<<blocks, 64, 0, stream>>>(p, tmpl); break;
  }
  return cudaGetLastError();
}

// np_random = Generator(PCG64(SeedSequence(seed)))
__global__ void k_seed(Params p, const uint8_t *__restrict__ mask, const uint64_t *__restrict__ seeds, uint64_t base) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= p.n_envs) return;
  if (mask && !mask[env]) return;  // SyncVectorEnv.reset seeds only the envs its reset_mask selects
  const uint64_t s = seeds ? seeds[env] : base + (uint64_t)env;
  const Pcg r = seed_pcg64(s);
  store_rng(p.rng + env, r);
}

cudaError_t launch_seed(const Params &p, const uint8_t *mask, const uint64_t *seeds_dev, uint64_t base, cudaStream_t stream) {
  k_seed<<<(p.n_envs + 127) / 128, 128, 0, stream>>>(p, mask, seeds_dev, base);
  return cudaGetLastError();
}

}  // namespace mg
