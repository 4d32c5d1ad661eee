// Fused attention O = softmax(Q K^T + keymask) V on the Hopper tensor cores, head_dim 64,
// NO 1/sqrt(d) scaling (msd/layers.py:158-181, note at 254-258), key-padding mask as in
// msd/layers.py:341-348 (0 / -1e10 bias == masked keys get exactly zero weight in fp32), and
// rows with no attendable key produce 0 (msd/layers.py:882-902 zero_activations_if_masked).
//
// One CTA per (128-query tile, head, batch row [, key split]), three warpgroups:
//   warpgroup 0 (one lane)  TMA producer: the Q tile once, then K/V BKV-key tiles into a ring; its
//                           register allowance goes to the consumers (setmaxnreg)
//   warpgroups 1, 2         64 queries each: S = Q K^T with wgmma (m64 x nBKV x k16, both operands
//                           K-major from shared memory) into a register fragment, online softmax on
//                           the fragment in fp32 (row max / sum over the quad of lanes that shares a
//                           row), P repacked in registers as the bf16 A operand of
//                           O += P V (m64 x n64 x k16, V MN-major straight from its [key,64] tile).
//                           The two warpgroups run independently, so one's softmax overlaps the
//                           other's MMAs.
// Key blocks whose mask bits are all zero are skipped by every role.  With splits > 1 every split
// writes an unnormalised partial (O fp32, running max m, sum l) that the combine kernel merges.
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace msd {

namespace {

constexpr int BQ = 128;   // queries per CTA
constexpr int HD = 64;    // head dim
constexpr int Q_BYTES = BQ * HD * 2;         // 16 KB
constexpr int ATTN_THREADS = 384;  // warps 0-3 producer group (warp 0 loads), 4-7 / 8-11 consumers
constexpr float LOG2E = 1.4426950408889634f;

// Two instances, by keys per block (MSD_ATTN_BKV selects; 128 by default: half the barrier round
// trips per key).
template <int BKV>
struct ACfg {
  static constexpr int KV_TILE_BYTES = BKV * HD * 2;   // 16 / 8 KB
  static constexpr int KV_STAGES = BKV == 128 ? 3 : 4;
  static constexpr int WPB = BKV / 32;                 // mask words per key block
  static constexpr int SMEM = Q_BYTES + KV_STAGES * 2 * KV_TILE_BYTES + 256 + 1024 /*align*/;
};

struct AttnDev {
  bf16* O;
  int ldo;
  int heads, Lq, Lk;
  const uint32_t* mask_bits;
  int mask_stride_words;
  // split-KV: blockIdx.z = batch * splits + split; each split covers nkb / splits key blocks
  // tail > 0 (splits == 2): an uneven split, split 1 covers the last `tail` key blocks
  int splits, tail;
  float* part_o;   // [rows * heads * splits][64]
  float* part_ml;  // [rows * heads * splits][2]
  int kv_static;    // K, V and mask_bits are not produced by the preceding kernels (see TMA warp)
  int kv_batch_rows, kv_row0;  // K/V row of (batch b, key block j) = b*kv_batch_rows + kv_row0 + j*BKV
};

// Bit j = key block j has at least one attendable key.  One coalesced pass by a whole warp.
template <int WPB>
__device__ __forceinline__ uint64_t active_blocks(const uint32_t* mrow, int nkb_all, int lane) {
  if (mrow == nullptr) return ~0ull;
  uint32_t word[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int j = h * 32 + lane;
    bool a = false;
    if (j < nkb_all) {
      if (WPB == 4) {
        const uint4 w = *reinterpret_cast<const uint4*>(mrow + j * 4);
        a = (w.x | w.y | w.z | w.w) != 0u;
      } else {
        const uint2 w = *reinterpret_cast<const uint2*>(mrow + j * 2);
        a = (w.x | w.y) != 0u;
      }
    }
    word[h] = __ballot_sync(0xffffffffu, a);
  }
  return static_cast<uint64_t>(word[0]) | (static_cast<uint64_t>(word[1]) << 32);
}
__device__ __forceinline__ bool block_active(uint64_t act, int blk) { return (act >> blk) & 1ull; }
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int BKV>
__global__ void __launch_bounds__(ATTN_THREADS, 1)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_q,
                       const __grid_constant__ CUtensorMap tmap_k,
                       const __grid_constant__ CUtensorMap tmap_v, const AttnDev p) {
  using Cfg = ACfg<BKV>;
  constexpr int KV_STAGES = Cfg::KV_STAGES;
  constexpr int KV_TILE_BYTES = Cfg::KV_TILE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;                                   // [16 KB]
  uint8_t* sK = sQ + Q_BYTES;                           // [KV_STAGES][KV tile]
  uint8_t* sV = sK + KV_STAGES * KV_TILE_BYTES;         // [KV_STAGES][KV tile]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + KV_STAGES * KV_TILE_BYTES);
  uint64_t* q_full = bars;                  // 1
  uint64_t* kv_full = bars + 1;             // [KV_STAGES]
  uint64_t* kv_empty = kv_full + KV_STAGES; // [KV_STAGES] (one arrival per consumer warpgroup)

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int head = blockIdx.y;
  const int b = static_cast<int>(blockIdx.z) / p.splits;
  const int split = static_cast<int>(blockIdx.z) - b * p.splits;
  const int q0 = blockIdx.x * BQ;                     // first query row of this CTA
  const int nkb_all = p.Lk / BKV;
  // this CTA's key blocks [kb0, nkb)
  const int kb0 = p.tail > 0 ? (split ? nkb_all - p.tail : 0) : split * nkb_all / p.splits;
  const int nkb = p.tail > 0 ? (split ? nkb_all : nkb_all - p.tail) : (split + 1) * nkb_all / p.splits;
  const uint32_t* mrow =
      p.mask_bits ? p.mask_bits + static_cast<size_t>(b) * p.mask_stride_words : nullptr;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    mbar_init(q_full, 1);
    for (int s = 0; s < KV_STAGES; ++s) {
      mbar_init(&kv_full[s], 1);
      mbar_init(&kv_empty[s], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  griddep_launch_dependents();
  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp != 0) return;
    // kv_static: K, V and the key mask were written long before the preceding kernel (the
    // cross-attention cache of a diffusion step), so the first ring-full of K/V tiles is
    // requested ahead of the dependency wait; only Q comes from the preceding kernel.
    if (!p.kv_static) griddep_wait();
    const uint64_t act = active_blocks<Cfg::WPB>(mrow, nkb_all, lane);
    if (lane == 0) {
      int it = 0, j = kb0;
      auto load_kv = [&](int jb) {
        const int s = it % KV_STAGES;
        const uint32_t ph = (it / KV_STAGES) & 1;
        mbar_wait(&kv_empty[s], ph ^ 1u);
        mbar_arrive_expect_tx(&kv_full[s], 2 * KV_TILE_BYTES);
        const int krow = b * p.kv_batch_rows + p.kv_row0 + jb * BKV;
        tma_load_2d(sK + s * KV_TILE_BYTES, &tmap_k, &kv_full[s], head * HD, krow);
        tma_load_2d(sV + s * KV_TILE_BYTES, &tmap_v, &kv_full[s], head * HD, krow);
        ++it;
      };
      if (p.kv_static) {
        for (; j < nkb && it < KV_STAGES; ++j)
          if (block_active(act, j)) load_kv(j);
        griddep_wait();
      }
      // the consumers wait for Q at their first active key block: with none in [kb0, nkb) nobody
      // would, and the CTA could exit with the copy still in flight
      bool any = false;
      for (int jj = kb0; jj < nkb; ++jj) any = any || block_active(act, jj);
      if (any) {
        mbar_arrive_expect_tx(q_full, Q_BYTES);
        tma_load_2d(sQ, &tmap_q, q_full, head * HD, b * p.Lq + q0);
      }
      for (; j < nkb; ++j)
        if (block_active(act, j)) load_kv(j);
    }
    return;
  }

  // ------------------------- softmax / output warpgroups -------------------------
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  griddep_wait();  // mask words may come from the previous kernel; O is written by these warps
  const uint64_t act = active_blocks<Cfg::WPB>(mrow, nkb_all, lane);
  const int wg = (warp >> 2) - 1;
  const int tid = threadIdx.x & 127;
  const int q = lane & 3;
  const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's rows: r0 and r0 + 8
  const uint64_t dq = make_smem_desc_sw128(smem_u32(sQ) + wg * 64 * 128);
  const uint64_t dk0 = make_smem_desc_sw128(smem_u32(sK));
  const uint64_t dv0 = make_smem_desc_sw128(smem_u32(sV));
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};  // running max (natural units), partial sums
  int it = 0;
  for (int j = kb0; j < nkb; ++j) {
    if (!block_active(act, j)) continue;
    uint32_t mw[Cfg::WPB];
    bool all_on = true;
#pragma unroll
    for (int c = 0; c < Cfg::WPB; ++c) {
      mw[c] = mrow != nullptr ? mrow[j * Cfg::WPB + c] : 0xffffffffu;
      all_on = all_on && mw[c] == 0xffffffffu;
    }
    const int s = it % KV_STAGES;
    if (it == 0) mbar_wait(q_full, 0);
    mbar_wait(&kv_full[s], (it / KV_STAGES) & 1);
    // S = Q K^T : 4 k-steps of 16 along head_dim (32 bytes each inside the swizzle atom)
    float sc[BKV / 2];
    const uint64_t dk = dk0 + static_cast<uint64_t>(s * (KV_TILE_BYTES >> 4));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / 16; ++k) WgmmaSS<BKV>::mma(sc, dq + k * 2, dk + k * 2, k != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    if (!all_on) {
      // fragment column of sc[4 jj + 2 h + e] is 8 jj + 2 q + e
#pragma unroll
      for (int jj = 0; jj < BKV / 8; ++jj) {
        const uint32_t bits = mw[jj >> 2] >> ((jj & 3) * 8 + 2 * q);
#pragma unroll
        for (int e = 0; e < 2; ++e)
          if (!((bits >> e) & 1u)) { sc[4 * jj + e] = -INFINITY; sc[4 * jj + 2 + e] = -INFINITY; }
      }
    }
    // row max over attendable keys (finite: an active block has >= 1 attendable key)
    float alpha[2], nmb[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < BKV / 8; ++jj) mx = fmaxf(mx, fmaxf(sc[4 * jj + 2 * h], sc[4 * jj + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[h], mx);
      alpha[h] = ex2_approx((m[h] - m_new) * LOG2E);  // first block: exp2(-inf) = 0
      m[h] = m_new;
      nmb[h] = -m_new * LOG2E;
    }
    // p = exp(s - m): row sums in fp32, P packed as the A fragments of the PV MMAs
    uint32_t pa[BKV / 16][4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float sum = 0.f;
#pragma unroll
      for (int jj = 0; jj < BKV / 8; ++jj) {
        const float e0 = ex2_approx(fmaf(sc[4 * jj + 2 * h], LOG2E, nmb[h]));
        const float e1 = ex2_approx(fmaf(sc[4 * jj + 2 * h + 1], LOG2E, nmb[h]));
        sum += e0 + e1;
        pa[jj >> 1][(jj & 1) * 2 + h] = pack_bf16(e0, e1);
      }
      l[h] = fmaf(l[h], alpha[h], sum);
    }
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      o[4 * jj + 0] *= alpha[0]; o[4 * jj + 1] *= alpha[0];
      o[4 * jj + 2] *= alpha[1]; o[4 * jj + 3] *= alpha[1];
    }
    // O += P V : BKV/16 k-steps of 16 keys; V (MN-major): 16 keys = 16 rows of 128 B -> +2048 B
    const uint64_t dv = dv0 + static_cast<uint64_t>(s * (KV_TILE_BYTES >> 4));
    wgmma_fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BKV / 16; ++k) wgmma_rs_n64_tb(o, pa[k], dv + k * (2048 >> 4), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    if (tid == 0) mbar_arrive(&kv_empty[s]);  // K/V of this block are dead for this warpgroup
    ++it;
  }
  // ---- output: the row sums are completed over the quad, then O / l (or the unnormalised partial)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float lt = l[h];
    lt += __shfl_xor_sync(0xffffffffu, lt, 1);
    lt += __shfl_xor_sync(0xffffffffu, lt, 2);
    const size_t grow = static_cast<size_t>(b) * p.Lq + q0 + r0 + 8 * h;
    if (p.splits > 1) {
      const size_t prow = (grow * p.heads + head) * p.splits + split;
      float* po = p.part_o + prow * HD;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<float2*>(po + 8 * jj + 2 * q) = make_float2(o[4 * jj + 2 * h], o[4 * jj + 2 * h + 1]);
      if (q == 0) *reinterpret_cast<float2*>(p.part_ml + prow * 2) = make_float2(m[h], lt);
    } else {
      const float inv = lt > 0.f ? 1.0f / lt : 0.f;
      bf16* orow = p.O + grow * p.ldo + head * HD;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(orow + 8 * jj + 2 * q) =
            pack_bf16(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
    }
  }
}

// Merge the split-KV partials of every (row, head): out = sum_s w_s O_s / sum_s w_s l_s with
// w_s = exp(m_s - max_s m_s); a split with no attendable key has m = -inf, l = 0 (weight 0).
__global__ void __launch_bounds__(256)
attention_combine_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml,
                         bf16* __restrict__ O, int ldo, int heads, int splits, long long n_rh) {
  griddep_launch_dependents();
  const long long gid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long rh = gid >> 4;  // (row, head) pair; 16 threads x 4 columns each
  const int c4 = static_cast<int>(gid & 15);
  if (rh >= n_rh) return;
  griddep_wait();
  float mmax = -INFINITY;
  for (int s = 0; s < splits; ++s) mmax = fmaxf(mmax, part_ml[(rh * splits + s) * 2]);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  float lt = 0.f;
  for (int s = 0; s < splits; ++s) {
    const float2 ml = *reinterpret_cast<const float2*>(part_ml + (rh * splits + s) * 2);
    const float w = (ml.x == -INFINITY) ? 0.f : __expf(ml.x - mmax);
    const float4 v = *reinterpret_cast<const float4*>(part_o + (rh * splits + s) * HD + c4 * 4);
    acc.x += w * v.x; acc.y += w * v.y; acc.z += w * v.z; acc.w += w * v.w;
    lt += w * ml.y;
  }
  const float inv = lt > 0.f ? 1.0f / lt : 0.f;
  const long long row = rh / heads;
  const int head = static_cast<int>(rh - row * heads);
  uint2 u;
  u.x = pack_bf16(acc.x * inv, acc.y * inv);
  u.y = pack_bf16(acc.z * inv, acc.w * inv);
  *reinterpret_cast<uint2*>(O + row * ldo + head * HD + c4 * 4) = u;
}

}  // namespace

// Which instance runs: 128-key blocks unless MSD_ATTN_BKV=64 asks for the small one.
static int attention_bkv(int Lk) {
  const char* e = getenv("MSD_ATTN_BKV");  // read per launch: the tests switch instances
  const int forced = e ? atoi(e) : 0;
  return (forced == 64 && Lk % 64 == 0) ? 64 : 128;
}

// Split-KV pays when the unsplit grid would leave more than half of the SMs idle (one segment at
// batch 1: 12-24 CTAs): the largest split count that keeps >= 3 key blocks of 128 per CTA and at
// most two CTAs per SM in the launch.
int attention_pick_splits(int nbatch, int heads, int Lq, int Lk) {
  const int ctas = ((Lq + BQ - 1) / BQ) * heads * nbatch;
  const int nkb = Lk / 128;
  const int sms = device_sm_count();
  if (ctas >= sms / 2 || nkb < 6) return 1;
  int best = 1;
  for (int s = 2; s <= 8; ++s) {
    if (nkb % s != 0 || nkb / s < 3) continue;
    if (ctas * s <= 2 * sms) best = s;
  }
  return best;
}

int attention_configure() {
  MSD_CUDA_CHECK(cudaFuncSetAttribute(attention_wgmma_kernel<128>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, ACfg<128>::SMEM));
  MSD_CUDA_CHECK(cudaFuncSetAttribute(attention_wgmma_kernel<64>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, ACfg<64>::SMEM));
  return 0;
}

// floats of the part_o workspace a launch with up to max_splits splits may need
size_t attention_workspace_floats(int nbatch, int heads, int Lq, int max_splits) {
  return static_cast<size_t>(nbatch) * Lq * heads * max_splits * HD;
}

int launch_attention(const AttnArgs& a, cudaStream_t stream) {
  static int configured = attention_configure();
  if (configured != 0) return configured;
  const int bkv = attention_bkv(a.Lk);
  MSD_REQUIRE(a.Lq % BQ == 0 && a.Lk % 128 == 0,
              "attention: Lq=%d and Lk=%d must be multiples of 128", a.Lq, a.Lk);
  MSD_REQUIRE(a.Lk / bkv <= 64, "attention: Lk=%d exceeds 64 key blocks", a.Lk);
  MSD_REQUIRE(a.nbatch > 0 && a.heads > 0, "attention: empty problem");
  MSD_REQUIRE(a.ldo % 8 == 0, "attention: ldo must be a multiple of 8");
  if (a.mask_bits)
    MSD_REQUIRE(a.mask_stride_words % 4 == 0 &&
                    (reinterpret_cast<uintptr_t>(a.mask_bits) & 15) == 0,
                "attention: mask words must be 16-byte aligned per row");
  CUtensorMap tq, tk, tv;
  const int width = a.heads * HD;
  if (int rc = make_tmap_bf16_2d(&tq, a.Q, (uint64_t)a.nbatch * a.Lq, width, a.ldq, BQ)) return rc;
  const int kv_batch_rows = a.kv_batch_rows > 0 ? a.kv_batch_rows : a.Lk;
  MSD_REQUIRE(a.kv_row0 >= 0 && a.kv_row0 + a.Lk <= kv_batch_rows,
              "attention: key rows [%d, %d) exceed the %d rows per batch", a.kv_row0, a.kv_row0 + a.Lk,
              kv_batch_rows);
  const uint64_t kv_rows = (uint64_t)a.nbatch * kv_batch_rows;
  if (int rc = make_tmap_bf16_2d(&tk, a.K, kv_rows, width, a.ldk, bkv)) return rc;
  if (int rc = make_tmap_bf16_2d(&tv, a.V, kv_rows, width, a.ldv, bkv)) return rc;
  AttnDev d;
  d.O = a.O; d.ldo = a.ldo; d.heads = a.heads; d.Lq = a.Lq; d.Lk = a.Lk;
  d.mask_bits = a.mask_bits; d.mask_stride_words = a.mask_stride_words;
  const int nkb = a.Lk / bkv;
  int splits = (a.part_o != nullptr && a.part_ml != nullptr)
                   ? (a.splits > 0 ? a.splits : attention_pick_splits(a.nbatch, a.heads, a.Lq, a.Lk))
                   : 1;
  if (splits > a.max_splits) splits = a.max_splits > 0 ? a.max_splits : 1;
  MSD_REQUIRE(nkb % splits == 0, "attention: %d key blocks not divisible by %d splits", nkb, splits);
  MSD_REQUIRE(a.tail < nkb, "attention: tail %d must be below %d key blocks", a.tail, nkb);
  // a forced tail (128-key instance, otherwise unsplit launch) runs as an uneven two-way split
  d.tail = 0;
  if (bkv == 128 && splits == 1 && a.tail > 0 && a.part_o != nullptr && a.part_ml != nullptr &&
      a.max_splits >= 2) {
    d.tail = a.tail;
    splits = 2;
  }
  d.splits = splits; d.part_o = a.part_o; d.part_ml = a.part_ml;
  d.kv_static = a.kv_static;
  d.kv_batch_rows = kv_batch_rows; d.kv_row0 = a.kv_row0;
  dim3 grid(a.Lq / BQ, a.heads, a.nbatch * splits);
  if (getenv("MSD_ATTN_DEBUG"))
    fprintf(stderr, "[attn] nb=%d Lq=%d Lk=%d bkv=%d ctas=%d splits=%d tail=%d\n", a.nbatch, a.Lq, a.Lk,
            bkv, grid.x * grid.y * a.nbatch, splits, d.tail);
  ProfScope prof(KC_ATTENTION, 4.0 * a.nbatch * a.heads * static_cast<double>(a.Lq) * a.Lk * HD,
                 2.0 * a.nbatch * a.heads * HD * (2.0 * a.Lq + 2.0 * a.Lk), stream);
  if (bkv == 64)
    MSD_CUDA_CHECK(launch_kernel(attention_wgmma_kernel<64>, grid, dim3(ATTN_THREADS), ACfg<64>::SMEM,
                                 stream, tq, tk, tv, d));
  else
    MSD_CUDA_CHECK(launch_kernel(attention_wgmma_kernel<128>, grid, dim3(ATTN_THREADS),
                                 ACfg<128>::SMEM, stream, tq, tk, tv, d));
  ++g_launch_count;
  if (splits > 1) {
    const long long n_rh = static_cast<long long>(a.nbatch) * a.Lq * a.heads;
    const long long threads = n_rh * 16;
    MSD_CUDA_CHECK(launch_kernel(attention_combine_kernel, dim3(static_cast<unsigned>((threads + 255) / 256)),
                                 dim3(256), 0, stream, static_cast<const float*>(a.part_o),
                                 static_cast<const float*>(a.part_ml), a.O, a.ldo, a.heads, splits,
                                 n_rh));
    ++g_launch_count;
  }
  return 0;
}

}  // namespace msd
