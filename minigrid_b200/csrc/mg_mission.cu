// mg_mission.cu — the per-env missions of the BabyAI levels (Params::mission, one code per env) as the three forms a
// training loop consumes, one pass over all envs each:
//   k_mission_text      uint8[n, 96]              MiniGridEnv.mission, zero padded
//   k_mission_indices   int64[n, max_words]       DictObservationSpaceWrapper.observation (wrappers.py:535-554)
//   k_flat_missions     uint8[n, img + 28 * 96]   FlatObsWrapper.observation (wrappers.py:591-626)
// All three render through mission_words (mg_mission.cuh). They read the codes and their output only, never the grid.
#include "mg_common.cuh"
#include "mg_mission.cuh"

namespace mg {

// one thread per env; the row is built in registers and stored as six 16-byte words
__global__ void __launch_bounds__(128) k_mission_text(const uint32_t *__restrict__ codes, uint8_t *__restrict__ out, int n) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= n) return;
  union { uint8_t b[MISSION_TEXT_BYTES]; uint4 v[MISSION_TEXT_BYTES / 16]; } t;
  mission_text(codes[env], t.b);
  uint4 *o = reinterpret_cast<uint4 *>(out + (size_t)env * MISSION_TEXT_BYTES);
#pragma unroll
  for (int k = 0; k < MISSION_TEXT_BYTES / 16; ++k) o[k] = t.v[k];
}

__global__ void __launch_bounds__(128) k_mission_indices(const uint32_t *__restrict__ codes, long long *__restrict__ out, int max_words, int n) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= n) return;
  mission_indices(codes[env], max_words, out + (size_t)env * max_words);
}

// FlatObsWrapper rows: the image bytes, then 96 x 28 one-hot characters. FLAT_ENVS envs per block: their texts are
// rendered into shared memory (one thread each), then the whole block writes the rows byte by byte, coalesced.
constexpr int FLAT_ENVS = 32, FLAT_THREADS = 256;
__global__ void __launch_bounds__(FLAT_THREADS) k_flat_missions(const uint8_t *__restrict__ img, int img_bytes, const uint32_t *__restrict__ codes,
                                                                 uint8_t *__restrict__ out, int n) {
  __shared__ uint8_t text[FLAT_ENVS][MISSION_TEXT_BYTES];
  const int e0 = blockIdx.x * FLAT_ENVS;
  const int ne = min(FLAT_ENVS, n - e0);
  if ((int)threadIdx.x < ne) mission_text(codes[e0 + threadIdx.x], text[threadIdx.x]);
  __syncthreads();
  const int row = img_bytes + MISSION_TEXT_BYTES * MISSION_CHAR_CODES;
  const long long total = (long long)ne * row;
  uint8_t *o = out + (size_t)e0 * row;
  const uint8_t *im = img + (size_t)e0 * img_bytes;
  for (long long i = threadIdx.x; i < total; i += FLAT_THREADS) {
    const int e = (int)(i / row), j = (int)(i - (long long)e * row);
    uint8_t v;
    if (j < img_bytes) v = im[(size_t)e * img_bytes + j];
    else {
      const int q = j - img_bytes, pos = q / MISSION_CHAR_CODES, ch = q - pos * MISSION_CHAR_CODES;
      const uint8_t c = text[e][pos];
      v = c != 0 && mission_char_code(c) == ch;
    }
    o[i] = v;
  }
}

cudaError_t launch_mission_text(const uint32_t *codes, uint8_t *out, int n, cudaStream_t s) {
  k_mission_text<<<(n + 127) / 128, 128, 0, s>>>(codes, out, n);
  return cudaGetLastError();
}
cudaError_t launch_mission_indices(const uint32_t *codes, long long *out, int max_words, int n, cudaStream_t s) {
  k_mission_indices<<<(n + 127) / 128, 128, 0, s>>>(codes, out, max_words, n);
  return cudaGetLastError();
}
cudaError_t launch_flat_missions(const uint8_t *img, int img_bytes, const uint32_t *codes, uint8_t *out, int n, cudaStream_t s) {
  k_flat_missions<<<(n + FLAT_ENVS - 1) / FLAT_ENVS, FLAT_THREADS, 0, s>>>(img, img_bytes, codes, out, n);
  return cudaGetLastError();
}

}  // namespace mg
