// bf16 GEMM on the Hopper tensor cores: D[M,N] = A[M,K] * B[N,K]^T.
//
// Persistent CTAs (at most one per SM), each walking 128 x BN output tiles, three warpgroups:
//   warpgroup 0 (one lane)  TMA producer: cp.async.bulk.tensor 2D tiles (SWIZZLE_128B) into a
//                           STAGES-deep smem ring, completion on `full` mbarriers, running ahead
//                           into the CTA's next tile; its register allowance goes to the consumers
//                           (setmaxnreg)
//   warpgroups 1, 2         consumers: 64 rows each, wgmma.mma_async m64 x nBN x k16 straight from
//                           the ring (fp32 accumulator fragment in registers), one MMA group kept
//                           in flight while the previous ring slot is handed back (`empty`), then
//                           the fused epilogue (residual / gated-GELU / position-add / deferred
//                           normalisation) from the accumulator fragment: bf16 outputs through
//                           shared-memory staging and TMA stores the drain does not wait for; fp32
//                           outputs straight from the fragment, a quad of lanes owning 8
//                           consecutive columns of a row (whole 32-byte sectors).  The tile's bias row /
//                           column gains are staged in shared memory (cp.async) during the main
//                           loop, so the drain's only global loads are the residual / position rows
//
// Replaces the XLA dot_general lowering of DenseGeneral (msd/layers.py:397-442) for every
// projection on the hot path (SURVEY §2.2 K2, K4, K5, K6, K8, K9).
#include "common.cuh"
#include "kernels.h"
#include "wgmma.cuh"

namespace msd {

namespace {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 64;  // 64 bf16 = 128 bytes = one swizzle atom row
constexpr int MMA_K = 16;
constexpr int A_STAGE_BYTES = BLOCK_M * BLOCK_K * 2;
constexpr int GEMM_THREADS = 384;
// Epilogues that read a row (residual, position table, column gains) issue the loads of
// EPI_CHUNK column groups together, ahead of the chunk's stores.  Interleaved one by one, every
// load's latency was paid in full: the compiler cannot move a load above a store to the output,
// which may alias the row being read (it is the same row for the in-place residual).
constexpr int EPI_CHUNK = 8;
// The bf16 outputs leave through shared memory: each consumer warpgroup owns two staging buffers
// of one 64-row x 32-column sub-tile (64-byte rows, the box of the SWIZZLE_64B output map).
constexpr int STG_BUF_BYTES = 64 * 64;

__host__ __device__ inline bool epi_is_bf16_out(int e) {
  return e == EPI_BF16 || e == EPI_GATED_GELU || e == EPI_GATED_GELU_SPLIT3;
}

// exact-tanh GELU of the fp32-accurate mode (flax.linen.gelu(approximate=True))
__device__ __forceinline__ float gelu_tanh_exact(float x) {
  const float k0 = 0.7978845608028654f;
  return 0.5f * x * (1.0f + tanhf(k0 * (x + 0.044715f * x * x * x)));
}

struct GemmDev {
  int M, N, K;
  int epilogue;
  void* out;
  int ldo;
  const float* resid;
  const float* pos;
  int pos_rows;
  const int* pos_shift;
  int dup_rows;
  // debugging (MSD_GEMM_TRACE with msd_bench_gemm): per-tile stamps, see the kernel
  long long* trace;
  GemmPrep prep;       // EPI_RESID_PREP
  GemmRowScale rs;     // row scale + bias on EPI_BF16 / EPI_GATED_GELU
  const int* step;
};

template <int BN>
struct GemmCfg {
  static constexpr int B_STAGE_BYTES = BN * BLOCK_K * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int STAGE_BUDGET = 200 * 1024;
  static constexpr int STAGES = STAGE_BUDGET / STAGE_BYTES > 6 ? 6 : STAGE_BUDGET / STAGE_BYTES;
  static constexpr int CONST_BYTES = 2 /*warpgroups*/ * 2 /*rows*/ * BN * 4;
  // the staging buffers fit between the ring budget and the 227 KB limit at every width, so they
  // cost no ring stage (6 / 6 / 6 / 5 / 4 stages at BN 64 / 96 / 128 / 192 / 256)
  static constexpr int STG_BYTES = 2 /*warpgroups*/ * 2 * STG_BUF_BYTES;
  static constexpr int SMEM_BYTES =
      CONST_BYTES + 1024 /*align*/ + STAGES * STAGE_BYTES + STG_BYTES + 256 /*barriers*/;
};

// 8-byte asynchronous copy global -> shared (no register round trip); completed by cp_async_wait_all
__device__ __forceinline__ void cp_async_8(void* smem_dst, const void* gmem_src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src)
               : "memory");
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// barrier over the 128 threads of one consumer warpgroup (ids 1, 2; 0 is __syncthreads)
__device__ __forceinline__ void warpgroup_sync(int wg) {
  asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");
}

// One consumer warpgroup's two staging buffers of the bf16 outputs, and the thread's place in them:
// the 16-byte chunk c of local row r sits at chunk c ^ ((r >> 1) & 3) (SWIZZLE_64B), so the 4-byte
// writes of a warp (8 rows x 4 lanes, one chunk per row) fall on 32 distinct banks.  Bits 4-5 of
// `thr` hold its row's (r >> 1) & 3, so XOR-ing the chunk into them places it.
struct Staging {
  uint8_t* buf;  // buffer b at buf + b * STG_BUF_BYTES
  uint32_t thr;  // shared address of the thread's first element pair in buffer 0
  int wg, tid;
  int count;     // sub-tiles the warpgroup has staged so far, across all of the CTA's tiles
};

// Drains a tile's bf16 output through the staging buffers, one 64-row x 32-column sub-tile at a
// time, and moves on without waiting for the global writes.  Sub-tile s: the thread's element pairs
// pair(s, h, jj) (row h * 8 of its quad's rows, column group jj) go into buffer count & 1, then
// fence.proxy.async, lane 0 waits until every store issued so far has read its buffer, a warpgroup
// barrier, and lane 0 stores the buffer at output column cols(s).x (and .y when >= 0) of rows
// [row, row + 64) and commits the group.  So a buffer is written only after the store that last
// read it, two sub-tiles earlier in the running count, has been waited for, in whichever tile that
// was.
template <int SUBTILES, class Pair, class Cols>
__device__ __forceinline__ void drain_staged(Staging& st, const CUtensorMap* tmap_o, int row, Pair pair,
                                             Cols cols) {
#pragma unroll
  for (int s = 0; s < SUBTILES; ++s, ++st.count) {
    const uint32_t b = (st.count & 1) * STG_BUF_BYTES;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) st_shared_u32((st.thr ^ (jj << 4)) + b + h * 8 * 64, pair(s, h, jj));
    }
    fence_proxy_async_smem();
    if (st.tid == 0) bulk_wait_group_read<0>();
    warpgroup_sync(st.wg);
    if (st.tid == 0) {
      const int2 c = cols(s);
      for (int k = 0; k < (c.y >= 0 ? 2 : 1); ++k) tma_store_2d(tmap_o, st.buf + b, k ? c.y : c.x, row);
      bulk_commit_group();
    }
  }
}

// Drains a tile's fp32 output (EPI_F32 / EPI_RESID_F32 / EPI_POS_F32, or EPI_RESID_PREP when PREP)
// straight from the fragment, for the thread's two rows: out = acc + the residual or (rolled)
// position row, if any, and with EPI_POS_F32 the same again dup_rows rows further down.  PREP, the
// deferred normalisation's producer side (the residual is the output row, updated in place): also
// the next GEMM's operand bf16(x * g), with the tile's gains staged at cst, and the tile's share of
// the row's sum of squares.  Each chunk's EPI_CHUNK row loads are issued ahead of its stores.
template <int BN, bool PREP>
__device__ __forceinline__ void drain_f32(const GemmDev& p, const float (&acc)[BN / 2], int row_first,
                                          int n0, int q, const float* cst) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row_first + 8 * h;
    float* out = reinterpret_cast<float*>(p.out) + static_cast<size_t>(row) * p.ldo;
    const float* add = nullptr;  // row added to the accumulator
    if (PREP || p.epilogue == EPI_RESID_F32) {
      add = p.resid + static_cast<size_t>(row) * p.ldo;
    } else if (p.epilogue == EPI_POS_F32) {
      const int seq = row / p.pos_rows;
      int pr = row - seq * p.pos_rows;
      if (p.pos_shift != nullptr) {
        pr -= p.pos_shift[seq];
        if (pr < 0) pr += p.pos_rows;
      }
      add = p.pos + static_cast<size_t>(pr) * p.N;
    }
    const bool dup = !PREP && p.epilogue == EPI_POS_F32 && p.dup_rows > 0;
    bf16* arow = PREP ? p.prep.a + static_cast<size_t>(row) * p.prep.lda : nullptr;
    const float* gvec = row < p.prep.split_row ? cst : cst + BN;
    float ssum = 0.f;
#pragma unroll
    for (int j0 = 0; j0 < BN / 8; j0 += EPI_CHUNK) {
      float2 x[EPI_CHUNK];
      if (PREP || add != nullptr) {
#pragma unroll
        for (int jj = 0; jj < EPI_CHUNK; ++jj)
          if (j0 + jj < BN / 8) x[jj] = *reinterpret_cast<const float2*>(add + n0 + 8 * (j0 + jj) + 2 * q);
      }
#pragma unroll
      for (int jj = 0; jj < EPI_CHUNK; ++jj) {
        const int j = j0 + jj, col = n0 + 8 * j + 2 * q;
        if (j >= BN / 8) continue;
        float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        if (PREP || add != nullptr) {
          v0 += x[jj].x; v1 += x[jj].y;
        }
        *reinterpret_cast<float2*>(out + col) = make_float2(v0, v1);
        if constexpr (PREP) {
          const float2 g = *reinterpret_cast<const float2*>(gvec + 8 * j + 2 * q);
          ssum = fmaf(v0, v0, ssum);
          ssum = fmaf(v1, v1, ssum);
          *reinterpret_cast<uint32_t*>(arow + col) = pack_bf16(v0 * g.x, v1 * g.y);
        }
        if (dup)
          *reinterpret_cast<float2*>(out + static_cast<size_t>(p.dup_rows) * p.ldo + col) =
              make_float2(v0, v1);
      }
    }
    if constexpr (PREP) {
      ssum += __shfl_xor_sync(0xffffffffu, ssum, 1);
      ssum += __shfl_xor_sync(0xffffffffu, ssum, 2);
      if (q == 0) p.prep.ss[static_cast<size_t>(n0 / BN) * p.prep.ss_stride + row] = ssum;
    }
  }
}

// Persistent: gridDim.x CTAs (at most one per SM) walk the 128 x BN output tiles in the static
// order tile = blockIdx.x + i * gridDim.x, column tiles fastest.  The ring's slot / phase counter
// runs on across tiles, so the producer streams the next tile's k-blocks while the consumers drain
// the current one.
template <int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_a,
                       const __grid_constant__ CUtensorMap tmap_b,
                       const __grid_constant__ CUtensorMap tmap_o, const GemmDev p) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  // per consumer warpgroup: the tile's column constants, [0] bias row or g_lo, [1] g_hi (BN each);
  // addressed from the shared array itself, so that the drain reads them with LDS (generic loads
  // would be ordered behind its global stores)
  float* s_const = reinterpret_cast<float*>(smem_raw);
  uint8_t* smem = reinterpret_cast<uint8_t*>(
      (reinterpret_cast<uintptr_t>(smem_raw + Cfg::CONST_BYTES) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_STAGE_BYTES;
  uint8_t* s_stg = sB + STAGES * Cfg::B_STAGE_BYTES;  // 1024-aligned, as the swizzle pattern needs
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_stg + Cfg::STG_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;

  const int warp = __shfl_sync(0xffffffffu, static_cast<int>(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int n_tiles = p.N / BN;
  const int tiles = n_tiles * (p.M / BLOCK_M);
  const int num_kb = p.K / BLOCK_K;
  // per-tile stamps, 8 int64 per tile (first 512 tiles): smid, globaltimer at tile start / end,
  // cycles in the tile, then clock64 offsets from its start of: set-up done (first tile of a CTA
  // only), main loop entered, accumulator complete and dependency wait returned, last sub-tile
  // handed to TMA (bf16 outputs) / last store issued (fp32 outputs)
  const bool tracing = p.trace != nullptr && threadIdx.x == 128;
  long long t_tile = tracing ? clock64() : 0;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_b);
    if (epi_is_bf16_out(p.epilogue)) tma_prefetch_desc(&tmap_o);
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);  // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (tracing && blockIdx.x < 512) p.trace[blockIdx.x * 8 + 4] = clock64() - t_tile;

  griddep_launch_dependents();
  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      int it = 0;  // k-blocks loaded so far: ring slot it % STAGES, phase (it / STAGES) & 1
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int n0 = (tile % n_tiles) * BN, m0 = (tile / n_tiles) * BLOCK_M;
        int kb = 0;
        if (tile == static_cast<int>(blockIdx.x)) {
          // The weight (B) tiles do not depend on the previous kernel: the first ring-full of them
          // is requested BEFORE griddepcontrol.wait so the fetch overlaps the predecessor's tail.
          const int prefetched = num_kb < STAGES ? num_kb : STAGES;
          for (int k = 0; k < prefetched; ++k) {
            mbar_arrive_expect_tx(&full_bar[k], Cfg::STAGE_BYTES);
            tma_load_2d(sB + k * Cfg::B_STAGE_BYTES, &tmap_b, &full_bar[k], k * BLOCK_K, n0);
          }
          griddep_wait();
          for (; kb < prefetched; ++kb, ++it)
            tma_load_2d(sA + kb * A_STAGE_BYTES, &tmap_a, &full_bar[kb], kb * BLOCK_K, m0);
        }
        for (; kb < num_kb; ++kb, ++it) {
          const int s = it % STAGES;
          if (it >= STAGES) mbar_wait(&empty_bar[s], ((it / STAGES) & 1) ^ 1u);
          mbar_arrive_expect_tx(&full_bar[s], Cfg::STAGE_BYTES);
          tma_load_2d(sA + s * A_STAGE_BYTES, &tmap_a, &full_bar[s], kb * BLOCK_K, m0);
          tma_load_2d(sB + s * Cfg::B_STAGE_BYTES, &tmap_b, &full_bar[s], kb * BLOCK_K, n0);
        }
      }
    }
    return;
  }

  // ------------------------------ consumers ------------------------------
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wg = (warp >> 2) - 1;  // 0 / 1: rows [64 wg, 64 wg + 64) of the tile
  const int tid = threadIdx.x & 127;
  const int q = lane & 3;
  float acc[BN / 2];
  float* cst = s_const + wg * 2 * BN;
  // The column constants (bias row of the row-scale epilogues, column gains of EPI_RESID_PREP) are
  // fixed for the whole step -- only the sampler, the step's last kernel, advances the step index,
  // and the step's first kernel is a plain launch -- so, like the weights, they are requested
  // before the dependency wait.
  const long long step = p.step != nullptr ? *p.step : 0;
  const float* const0 = nullptr;
  const float* const1 = nullptr;
  if (p.epilogue == EPI_RESID_PREP) {
    const0 = p.prep.g_lo + step * p.prep.g_lo_step_stride;
    const1 = p.prep.g_hi + step * p.prep.g_hi_step_stride;
  } else if (p.rs.ss_lo != nullptr && p.rs.col_bias != nullptr) {
    const0 = p.rs.col_bias + step * p.rs.bias_step_stride;
  }
  const int stg_row = (warp & 3) * 16 + (lane >> 2);
  uint8_t* const stg_buf = s_stg + wg * 2 * STG_BUF_BYTES;
  Staging stg{stg_buf, smem_u32(stg_buf) + stg_row * 64 + (((stg_row >> 1) & 3) << 4) + 4 * q, wg, tid, 0};
  int it = 0;  // k-blocks consumed so far (same count as the producer's)
  for (int tile = blockIdx.x, i = 0; tile < tiles; tile += gridDim.x, ++i) {
    const int n0 = (tile % n_tiles) * BN, m0 = (tile / n_tiles) * BLOCK_M;
    long long* trc = tracing && tile < 512 ? p.trace + tile * 8 : nullptr;
    if (trc) {
      long long t;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      trc[1] = t;
      trc[5] = clock64() - t_tile;
    }
    if (const0 != nullptr) {
      if (i > 0) warpgroup_sync(wg);  // the previous tile's drain has read its constants
      for (int c = 2 * tid; c < BN; c += 256) {
        cp_async_8(cst + c, const0 + n0 + c);
        if (const1 != nullptr) cp_async_8(cst + BN + c, const1 + n0 + c);
      }
    }
    {
      const uint64_t da0 = make_smem_desc_sw128(smem_u32(sA) + wg * 64 * 128);
      const uint64_t db0 = make_smem_desc_sw128(smem_u32(sB));
      for (int kb = 0; kb < num_kb; ++kb, ++it) {
        const int s = it % STAGES;
        mbar_wait(&full_bar[s], (it / STAGES) & 1);
        const uint64_t da = da0 + static_cast<uint64_t>(s * (A_STAGE_BYTES >> 4));
        const uint64_t db = db0 + static_cast<uint64_t>(s * (Cfg::B_STAGE_BYTES >> 4));
        wgmma_fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / MMA_K; ++k)
          WgmmaSS<BN>::mma(acc, da + k * 2, db + k * 2, (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();  // the MMAs of the previous k-block have retired: its slot is free
        if (kb > 0 && tid == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (tid == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
    }
    if (i == 0) griddep_wait();  // residual reads / output writes come after the predecessor is complete
    if (trc) trc[6] = clock64() - t_tile;
    if (const0 != nullptr) {
      cp_async_wait_all();
      warpgroup_sync(wg);  // every thread's share of the constants has landed
    }

    // ---------------- epilogue from the accumulator fragment ----------------
    const int row_first = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2);
    if (p.epilogue == EPI_RESID_PREP) {
      drain_f32<BN, true>(p, acc, row_first, n0, q, cst);
    } else if (!epi_is_bf16_out(p.epilogue)) {
      drain_f32<BN, false>(p, acc, row_first, n0, q, cst);
    } else if constexpr (BN % 64 == 0) {  // the launcher refuses width 96 for bf16 outputs
      // deferred normalisation, consumer side: both rows' scales before the first store, so the
      // partial-sum loads are in flight together
      float inv_r[2] = {1.0f, 1.0f};
      if (p.rs.ss_lo != nullptr) {
        const float* ssp[2];
        int parts[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = row_first + 8 * h;
          const bool lo = row < p.rs.split_row;
          ssp[h] = (lo ? p.rs.ss_lo : p.rs.ss_hi) + row;
          parts[h] = lo ? p.rs.parts_lo : p.rs.parts_hi;
        }
        float ss[2] = {0.f, 0.f};
        const int pmax = parts[0] > parts[1] ? parts[0] : parts[1];
#pragma unroll 4
        for (int t = 0; t < pmax; ++t) {
#pragma unroll
          for (int h = 0; h < 2; ++h)
            if (t < parts[h]) ss[h] += ssp[h][static_cast<size_t>(t) * p.rs.ss_stride];
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) inv_r[h] = rsqrtf(ss[h] * p.rs.inv_d + 1e-6f);
      }
      // columns 8 j + 2 q, 8 j + 2 q + 1 of the thread's row h, row-scaled and biased.  Without a
      // row scale inv_r is 1, which multiplies exactly, so no branch separates the bias loads of
      // the gated epilogue's two calls
      auto scaled = [&](int h, int j) {
        float v0 = acc[4 * j + 2 * h] * inv_r[h], v1 = acc[4 * j + 2 * h + 1] * inv_r[h];
        if (const0 != nullptr) {
          const float2 b = *reinterpret_cast<const float2*>(cst + 8 * j + 2 * q);
          v0 += b.x; v1 += b.y;
        }
        return make_float2(v0, v1);
      };
      const int row0 = m0 + wg * 64;
      if (p.epilogue == EPI_BF16) {
        drain_staged<BN / 32>(
            stg, &tmap_o, row0,
            [&](int s, int h, int jj) {
              const float2 v = scaled(h, 4 * s + jj);
              return pack_bf16(v.x, v.y);
            },
            [&](int s) { return make_int2(n0 + 32 * s, -1); });
      } else if (p.epilogue == EPI_GATED_GELU) {
        // 64 accumulator columns, 32 GELU inputs then their 32 gates, make one sub-tile
        drain_staged<BN / 64>(
            stg, &tmap_o, row0,
            [&](int s, int h, int jj) {
              const float2 r = scaled(h, 8 * s + jj), g = scaled(h, 8 * s + jj + 4);
              return pack_bf16(gelu_tanh(r.x) * g.x, gelu_tanh(r.y) * g.y);
            },
            [&](int s) { return make_int2(n0 / 2 + 32 * s, -1); });
      } else {
        // EPI_GATED_GELU_SPLIT3, the fp32-accurate mode: exact tanh, the result kept to ~16
        // mantissa bits as [hi | lo | hi], F columns each.  Per 64 accumulator columns, the hi
        // sub-tile (stored twice), then the lo sub-tile, whose pairs the hi sub-tile computed
        const int F = p.N / 2;
        uint32_t lo[2][4] = {};
        drain_staged<BN / 32>(
            stg, &tmap_o, row0,
            [&](int s, int h, int jj) {
              if (s & 1) return lo[h][jj];
              const int jr = 8 * (s / 2) + jj, jg = jr + 4;
              const float v0 = gelu_tanh_exact(acc[4 * jr + 2 * h]) * acc[4 * jg + 2 * h];
              const float v1 = gelu_tanh_exact(acc[4 * jr + 2 * h + 1]) * acc[4 * jg + 2 * h + 1];
              lo[h][jj] = pack_bf16(v0 - __bfloat162float(__float2bfloat16_rn(v0)),
                                    v1 - __bfloat162float(__float2bfloat16_rn(v1)));
              return pack_bf16(v0, v1);
            },
            [&](int s) {
              const int oc = n0 / 2 + 32 * (s / 2);
              return s & 1 ? make_int2(F + oc, -1) : make_int2(oc, 2 * F + oc);
            });
      }
      // after the CTA's last tile the staged stores must have landed before the grid counts as
      // complete: dependent kernels read them (only lane 0 of each warpgroup has issued any; for
      // the others the wait returns at once)
      if (tile + static_cast<int>(gridDim.x) >= tiles) bulk_wait_group_all();
    }
    if (tracing) {
      const long long t_end = clock64();
      if (trc) {
        uint32_t smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        trc[0] = smid;
        trc[2] = t;
        trc[3] = trc[7] = t_end - t_tile;
      }
      t_tile = t_end;
    }
  }
}

template <int BN>
int launch_bn(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const GemmDev& d,
              cudaStream_t st) {
  using Cfg = GemmCfg<BN>;
  static_assert(Cfg::SMEM_BYTES <= 227 * 1024 && Cfg::STAGES >= 3, "smem budget");
  const int tiles = (d.N / BN) * (d.M / BLOCK_M);
  const int sms = device_sm_count();  // one CTA is resident per SM
  dim3 grid(tiles < sms ? tiles : sms);
  ProfScope prof(KC_GEMM, 2.0 * d.M * d.N * d.K,
                 2.0 * (static_cast<double>(d.M) * d.K + static_cast<double>(d.N) * d.K) +
                     4.0 * d.M * d.N, st);
  MSD_CUDA_CHECK(launch_kernel(gemm_bf16_wgmma_kernel<BN>, grid, dim3(GEMM_THREADS), Cfg::SMEM_BYTES,
                               st, ta, tb, to, d));
  ++g_launch_count;
  return 0;
}

template <int BN>
int configure_bn() {
  MSD_CUDA_CHECK(cudaFuncSetAttribute(gemm_bf16_wgmma_kernel<BN>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      GemmCfg<BN>::SMEM_BYTES));
  return 0;
}

}  // namespace

int gemm_configure() {
  if (int rc = configure_bn<64>()) return rc;
  if (int rc = configure_bn<96>()) return rc;
  if (int rc = configure_bn<128>()) return rc;
  if (int rc = configure_bn<192>()) return rc;
  return configure_bn<256>();
}

// The tile width launch_gemm runs with when block_n is 0.  The CTAs are persistent, one per SM, so
// a launch takes ceil(tiles / SMs) tile times, and a tile's k-block costs about 4 (BN + 64) cycles
// (measured 515 / 690 / 983 / 1168 at BN 64 / 128 / 192 / 256): take the width with the least
// ceil(tiles / SMs) * (BN + 64), the wider one on a tie (it re-reads the least of A and B per FLOP).
// 96 only for the fp32-output epilogues.
static int gemm_pick_wide_bn(int M, int N, int epilogue) {
  const int m_tiles = (M + BLOCK_M - 1) / BLOCK_M;
  const int widths[5] = {256, 192, 128, 96, 64};
  const int sms = device_sm_count();
  int best = 0;
  long long best_cost = 0;
  for (int i = 0; i < 5; ++i) {
    const int bn = widths[i];
    if (N % bn != 0 || (bn == 96 && epi_is_bf16_out(epilogue))) continue;
    const long long tiles = static_cast<long long>(m_tiles) * (N / bn);
    const long long cost = (tiles + sms - 1) / sms * (bn + 64);
    if (best == 0 || cost < best_cost) { best = bn; best_cost = cost; }
  }
  return best;
}

int gemm_resolve_block_n(const GemmArgs& a) {
  const int bn = a.block_n ? a.block_n : gemm_pick_wide_bn(a.M, a.N, a.epilogue);
  const bool allowed = bn == 64 || bn == 128 || bn == 192 || bn == 256 ||
                       (bn == 96 && !epi_is_bf16_out(a.epilogue));
  return allowed && a.N % bn == 0 ? bn : 0;
}

int launch_gemm(const GemmArgs& a, cudaStream_t stream) {
  static int configured = gemm_configure();
  if (configured != 0) return configured;
  MSD_REQUIRE(a.M > 0 && a.N > 0 && a.K > 0, "gemm: empty problem M=%d N=%d K=%d", a.M, a.N, a.K);
  MSD_REQUIRE(a.K % BLOCK_K == 0, "gemm: K=%d must be a multiple of %d", a.K, BLOCK_K);
  MSD_REQUIRE(a.M % BLOCK_M == 0, "gemm: M=%d must be a multiple of %d", a.M, BLOCK_M);
  const int bn = gemm_resolve_block_n(a);
  MSD_REQUIRE(bn != 0, "gemm: N=%d has no valid tile width (block_n %d)", a.N, a.block_n);
  MSD_REQUIRE(a.ldo % 8 == 0, "gemm: ldo=%d must be a multiple of 8", a.ldo);

  CUtensorMap ta, tb;
  if (int rc = make_tmap_bf16_2d(&ta, a.A, a.M, a.K, a.lda, BLOCK_M)) return rc;
  if (int rc = make_tmap_bf16_2d(&tb, a.B, a.N, a.K, a.ldb, bn)) return rc;
  // bf16 outputs are stored by TMA in 64-row x 32-column boxes; the map refuses an output view
  // whose base is not 16-byte aligned
  CUtensorMap to;
  memset(&to, 0, sizeof(to));
  if (epi_is_bf16_out(a.epilogue)) {
    const int cols = a.epilogue == EPI_BF16 ? a.N : a.epilogue == EPI_GATED_GELU ? a.N / 2 : 3 * (a.N / 2);
    if (int rc = make_tmap_bf16_2d(&to, a.out, a.M, cols, a.ldo, 64, 64)) return rc;
  }
  GemmDev d;
  d.M = a.M; d.N = a.N; d.K = a.K;
  d.epilogue = a.epilogue;
  d.out = a.out; d.ldo = a.ldo;
  d.resid = a.resid; d.pos = a.pos; d.pos_rows = a.pos_rows > 0 ? a.pos_rows : 1;
  d.pos_shift = a.pos_shift; d.dup_rows = a.dup_rows;
  d.trace = a.trace;
  d.prep = a.prep; d.rs = a.rs; d.step = a.step;
  if (a.epilogue == EPI_RESID_F32)
    MSD_REQUIRE(a.resid != nullptr, "gemm: EPI_RESID_F32 needs the residual");
  if (a.epilogue == EPI_RESID_PREP) {
    MSD_REQUIRE(a.resid != nullptr && a.resid == a.out, "gemm: EPI_RESID_PREP works in place (out == resid)");
    MSD_REQUIRE(a.prep.a && a.prep.ss && a.prep.g_lo && a.prep.g_hi && a.prep.lda % 8 == 0 &&
                    a.prep.ss_stride >= a.M,
                "gemm: EPI_RESID_PREP needs prep.a / ss / g_lo / g_hi (lda %% 8 == 0, ss_stride >= M)");
    MSD_REQUIRE(a.step != nullptr || (a.prep.g_lo_step_stride == 0 && a.prep.g_hi_step_stride == 0),
                "gemm: step-dependent column scales need the device step index");
  }
  if (a.rs.ss_lo != nullptr) {
    MSD_REQUIRE(a.epilogue == EPI_BF16 || a.epilogue == EPI_GATED_GELU,
                "gemm: the row scale applies to the bf16 and gated epilogues only");
    MSD_REQUIRE(a.rs.ss_hi != nullptr && a.rs.parts_lo > 0 && a.rs.parts_hi > 0 && a.rs.inv_d > 0.f,
                "gemm: incomplete row-scale description");
    MSD_REQUIRE(a.step != nullptr || a.rs.col_bias == nullptr || a.rs.bias_step_stride == 0,
                "gemm: a step-dependent bias row needs the device step index");
  }
  switch (bn) {
    case 64: return launch_bn<64>(ta, tb, to, d, stream);
    case 96: return launch_bn<96>(ta, tb, to, d, stream);
    case 128: return launch_bn<128>(ta, tb, to, d, stream);
    case 192: return launch_bn<192>(ta, tb, to, d, stream);
    default: return launch_bn<256>(ta, tb, to, d, stream);
  }
}

}  // namespace msd
