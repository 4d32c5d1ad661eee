// Host-side helpers shared by the engine (engine.cu) and the operator hooks (ops.cu); internal to
// libmsd_b200.so.  No device code.
#pragma once

#include <stdint.h>
#include <stdlib.h>

#include <vector>

#include "common.cuh"
#include "kernels.h"

namespace msd {

// Device scratch of one call, freed when it goes out of scope
struct TempBufs {
  std::vector<void*> p;
  ~TempBufs() { for (void* q : p) cudaFree(q); }
  template <typename T> int get(T** out, size_t n) {
    void* q = nullptr;
    MSD_CUDA_CHECK(cudaMalloc(&q, (n ? n : 1) * sizeof(T)));
    p.push_back(q);
    *out = reinterpret_cast<T*>(q);
    return 0;
  }
};

// jax.random keys: Threefry-2x32, 20 rounds (host twin of the device function in elementwise.cu)
inline void threefry2x32_host(uint32_t k0, uint32_t k1, uint32_t x0, uint32_t x1, uint32_t* out) {
  const uint32_t ks[3] = {k0, k1, k0 ^ k1 ^ 0x1BD11BDAu};
  static const int rot[2][4] = {{13, 15, 26, 6}, {17, 29, 16, 24}};
  x0 += ks[0];
  x1 += ks[1];
  for (int g = 0; g < 5; ++g) {
    for (int j = 0; j < 4; ++j) {
      x0 += x1;
      x1 = ((x1 << rot[g & 1][j]) | (x1 >> (32 - rot[g & 1][j]))) ^ x0;
    }
    x0 += ks[(g + 1) % 3];
    x1 += ks[(g + 2) % 3] + static_cast<uint32_t>(g + 1);
  }
  out[0] = x0;
  out[1] = x1;
}
// PRNGKey(seed): the seed's high and low words
inline void prng_key(unsigned long long seed, uint32_t* key) {
  key[0] = static_cast<uint32_t>(seed >> 32);
  key[1] = static_cast<uint32_t>(seed);
}
// fold_in(PRNGKey(seed), step)
inline void fold_in(unsigned long long seed, uint32_t step, uint32_t* key) {
  uint32_t k[2];
  prng_key(seed, k);
  threefry2x32_host(k[0], k[1], 0u, step, key);
}
// The [steps + 1][2] key table the sampler reads (SamplerArgs::rng_keys): PRNGKey(seed), then
// fold_in(PRNGKey(seed), i) for every scan index i
inline void step_keys(unsigned long long seed, int steps, uint32_t* out) {
  prng_key(seed, out);
  for (int i = 0; i < steps; ++i) fold_in(seed, static_cast<uint32_t>(i), out + 2 * (i + 1));
}

// Tuning / test switches of the attention launches, 0 when unset: MSD_ATTN_SPLITS forces a split
// count, MSD_ATTN_TAIL a tail of that many key blocks.  Read per launch: the tests change them.
struct AttnSwitches { int splits, tail; };
inline AttnSwitches attn_switches() {
  const char* s = getenv("MSD_ATTN_SPLITS");
  const char* t = getenv("MSD_ATTN_TAIL");
  return {s ? atoi(s) : 0, t ? atoi(t) : 0};
}

// One attention launch, as AttnArgs (bf16) or AttnF32Args (f32) describe it.  Q / K / V are
// (buffer, element offset, leading dimension) views of bf16 or (f32) fp32 elements; O is the
// first output column, ldo the output row stride (f32: the width of each third of the
// [hi | lo | hi] rows).  The workspace part_o / part_ml holds max_splits splits.  tail and
// kv_static apply to the bf16 kernel only.  Build it as `AttnView v = {};`.
struct AttnView {
  bool f32;
  const void* Q; size_t q_off; int ldq;
  const void* K; size_t k_off; int ldk;
  const void* V; size_t v_off; int ldv;
  bf16* O; int ldo;
  int nbatch, heads, Lq, Lk;
  const uint32_t* mask_bits; int mask_stride_words;
  float* part_o; float* part_ml; int max_splits;
  int splits, tail, kv_static, kv_batch_rows, kv_row0;
};
int launch_attention_view(const AttnView& v, cudaStream_t stream);

}  // namespace msd
