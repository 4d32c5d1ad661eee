// fp32 attention for the fp32-accurate mode (BASELINE config 2: "fp32 vs reference tolerance
// check"): O = softmax(Q K^T + keymask) V with every product, the softmax and the accumulation in
// fp32 (exact expf), NO 1/sqrt(d) (msd/layers.py:158-181, 254-258), key-padding mask as
// msd/layers.py:341-348, rows without an attendable key -> 0 (msd/layers.py:882-902).
//
// The reference computes this path in fp32 (gin/models/diffusion/context/t5_base.gin:72); the
// tensor-core kernel (attention_wgmma.cu) rounds Q, K, V and P to bf16.  This one is a plain
// CUDA-core flash-attention: one CTA per (32 queries, head, batch row), 128 threads, 64-key
// blocks staged in shared memory, online softmax per query row, thread = 4 rows x 4 columns of
// the 32 x 64 score / output tiles.  It is the accuracy mode, not the fast path: ~25 TFLOP/s.
// The result leaves as bf16 [hi | lo | hi] (16 mantissa bits), the A operand of the 3 x bf16
// split-precision output projection that follows.
#include "common.cuh"
#include "kernels.h"

namespace msd {

namespace {

constexpr int FQ = 32;    // queries per CTA
constexpr int FK = 64;    // keys per block
constexpr int FD = 64;    // head dim
constexpr int FLD = 68;   // padded row length (floats): 16-byte aligned rows, conflict-free LDS.128
constexpr int F32_THREADS = 128;
constexpr int F32_SMEM = (FQ * FLD + 2 * FK * FLD + FQ * FLD) * 4;  // Q, K, V, P

struct AttnF32Dev {
  const float* Q; int ldq;
  const float* K; int ldk;
  const float* V; int ldv;
  bf16* O; int o_third;
  int heads, Lq, Lk;
  const uint32_t* mask_bits; int mask_stride_words;
  int kv_batch_rows, kv_row0;
  // split-KV (small grids, e.g. one segment's cross-attention: 96 CTAs): blockIdx.z = batch *
  // splits + split; each split covers nkb / splits key blocks and leaves an unnormalised partial
  // (o, m, l) that attention_f32_combine_kernel merges.  More CTAs per SM also hides the
  // synchronous K/V tile loads.
  int splits;
  float* part_o;   // [rows * heads * splits][64]
  float* part_ml;  // [rows * heads * splits][2]
};

__global__ void __launch_bounds__(F32_THREADS)
attention_f32_kernel(const AttnF32Dev p) {
  extern __shared__ __align__(16) float smem_f[];
  float* sQ = smem_f;                 // [FQ][FLD]
  float* sK = sQ + FQ * FLD;          // [FK][FLD]
  float* sV = sK + FK * FLD;          // [FK][FLD]
  float* sP = sV + FK * FLD;          // [FQ][FLD]
  griddep_launch_dependents();
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;   // tx: key / dim group, ty: row group (4 rows)
  const int q0 = blockIdx.x * FQ, head = blockIdx.y;
  const int b = static_cast<int>(blockIdx.z) / p.splits;
  const int split = static_cast<int>(blockIdx.z) - b * p.splits;
  const uint32_t* mrow =
      p.mask_bits ? p.mask_bits + static_cast<size_t>(b) * p.mask_stride_words : nullptr;
  griddep_wait();

  // Q tile: 32 rows x 64 floats = 512 float4, 4 per thread
  {
    const float* qb = p.Q + static_cast<size_t>(b * p.Lq + q0) * p.ldq + head * FD;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = tid + i * F32_THREADS;
      const int r = e >> 4, c4 = e & 15;
      *reinterpret_cast<float4*>(sQ + r * FLD + c4 * 4) =
          *reinterpret_cast<const float4*>(qb + static_cast<size_t>(r) * p.ldq + c4 * 4);
    }
  }
  float m[4], l[4], o[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    m[r] = -INFINITY;
    l[r] = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) o[r][c] = 0.f;
  }
  const int nkb_all = p.Lk / FK;
  const int kb0 = split * nkb_all / p.splits, nkb = (split + 1) * nkb_all / p.splits;
  for (int j = kb0; j < nkb; ++j) {
    uint32_t w0 = 0xffffffffu, w1 = 0xffffffffu;
    if (mrow != nullptr) {
      w0 = mrow[2 * j];
      w1 = mrow[2 * j + 1];
      if ((w0 | w1) == 0u) continue;   // block-uniform: nothing attendable in this key block
    }
    __syncthreads();   // previous block's K / V / P reads are done (also covers the Q stores)
    {
      const size_t krow0 = static_cast<size_t>(b) * p.kv_batch_rows + p.kv_row0 + j * FK;
      const float* kb = p.K + krow0 * p.ldk + head * FD;
      const float* vb = p.V + krow0 * p.ldv + head * FD;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int e = tid + i * F32_THREADS;
        const int r = e >> 4, c4 = e & 15;
        *reinterpret_cast<float4*>(sK + r * FLD + c4 * 4) =
            *reinterpret_cast<const float4*>(kb + static_cast<size_t>(r) * p.ldk + c4 * 4);
        *reinterpret_cast<float4*>(sV + r * FLD + c4 * 4) =
            *reinterpret_cast<const float4*>(vb + static_cast<size_t>(r) * p.ldv + c4 * 4);
      }
    }
    __syncthreads();
    // S[r][i] = q(ty*4 + r) . k(tx + 16 i)
    float s[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int i = 0; i < 4; ++i) s[r][i] = 0.f;
#pragma unroll 4
    for (int d = 0; d < FD; d += 4) {
      float4 q4[4], k4[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) q4[r] = *reinterpret_cast<const float4*>(sQ + (ty * 4 + r) * FLD + d);
#pragma unroll
      for (int i = 0; i < 4; ++i) k4[i] = *reinterpret_cast<const float4*>(sK + (tx + 16 * i) * FLD + d);
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          s[r][i] = fmaf(q4[r].x, k4[i].x, s[r][i]);
          s[r][i] = fmaf(q4[r].y, k4[i].y, s[r][i]);
          s[r][i] = fmaf(q4[r].z, k4[i].z, s[r][i]);
          s[r][i] = fmaf(q4[r].w, k4[i].w, s[r][i]);
        }
    }
    // key (tx + 16 i) of this block attendable?
    bool ok[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int key = tx + 16 * i;
      ok[i] = ((key < 32 ? (w0 >> key) : (w1 >> (key - 32))) & 1u) != 0u;
    }
    // online softmax per row (the 16 lanes sharing ty hold the row's 64 logits)
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      float bm = -INFINITY;
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (ok[i]) bm = fmaxf(bm, s[r][i]);
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) bm = fmaxf(bm, __shfl_xor_sync(0xffffffffu, bm, off));
      const float mn = fmaxf(m[r], bm);   // finite: the block has at least one attendable key
      const float alpha = (m[r] == -INFINITY) ? 0.f : expf(m[r] - mn);
      float ps = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float pv = ok[i] ? expf(s[r][i] - mn) : 0.f;
        ps += pv;
        sP[(ty * 4 + r) * FLD + tx + 16 * i] = pv;
      }
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) ps += __shfl_xor_sync(0xffffffffu, ps, off);
      l[r] = l[r] * alpha + ps;
      m[r] = mn;
#pragma unroll
      for (int c = 0; c < 4; ++c) o[r][c] *= alpha;
    }
    __syncwarp();   // a row's P values are written and read by the 16 lanes of one half-warp
    // O[r][c] += sum_k P[ty*4 + r][k] * V[k][tx*4 + c]
#pragma unroll 4
    for (int k = 0; k < FK; k += 4) {
      float4 p4[4], v4[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) p4[r] = *reinterpret_cast<const float4*>(sP + (ty * 4 + r) * FLD + k);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) v4[kk] = *reinterpret_cast<const float4*>(sV + (k + kk) * FLD + tx * 4);
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        o[r][0] = fmaf(p4[r].x, v4[0].x, o[r][0]); o[r][1] = fmaf(p4[r].x, v4[0].y, o[r][1]);
        o[r][2] = fmaf(p4[r].x, v4[0].z, o[r][2]); o[r][3] = fmaf(p4[r].x, v4[0].w, o[r][3]);
        o[r][0] = fmaf(p4[r].y, v4[1].x, o[r][0]); o[r][1] = fmaf(p4[r].y, v4[1].y, o[r][1]);
        o[r][2] = fmaf(p4[r].y, v4[1].z, o[r][2]); o[r][3] = fmaf(p4[r].y, v4[1].w, o[r][3]);
        o[r][0] = fmaf(p4[r].z, v4[2].x, o[r][0]); o[r][1] = fmaf(p4[r].z, v4[2].y, o[r][1]);
        o[r][2] = fmaf(p4[r].z, v4[2].z, o[r][2]); o[r][3] = fmaf(p4[r].z, v4[2].w, o[r][3]);
        o[r][0] = fmaf(p4[r].w, v4[3].x, o[r][0]); o[r][1] = fmaf(p4[r].w, v4[3].y, o[r][1]);
        o[r][2] = fmaf(p4[r].w, v4[3].z, o[r][2]); o[r][3] = fmaf(p4[r].w, v4[3].w, o[r][3]);
      }
    }
  }
  if (p.splits > 1) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const size_t prow =
          (static_cast<size_t>(b * p.Lq + q0 + ty * 4 + r) * p.heads + head) * p.splits + split;
      *reinterpret_cast<float4*>(p.part_o + prow * FD + tx * 4) =
          make_float4(o[r][0], o[r][1], o[r][2], o[r][3]);
      if (tx == 0) *reinterpret_cast<float2*>(p.part_ml + prow * 2) = make_float2(m[r], l[r]);
    }
    return;
  }
  // normalise and write [hi | lo | hi]; thread: rows ty*4 + r, dims tx*4 .. +3 (8 bytes each)
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const float inv = l[r] > 0.f ? 1.0f / l[r] : 0.f;
    float v[4], lo[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      v[c] = o[r][c] * inv;
      lo[c] = v[c] - __bfloat162float(__float2bfloat16_rn(v[c]));
    }
    const uint2 uh = make_uint2(pack_bf16(v[0], v[1]), pack_bf16(v[2], v[3]));
    const uint2 ul = make_uint2(pack_bf16(lo[0], lo[1]), pack_bf16(lo[2], lo[3]));
    bf16* orow = p.O + static_cast<size_t>(b * p.Lq + q0 + ty * 4 + r) * (3 * p.o_third) +
                 head * FD + tx * 4;
    *reinterpret_cast<uint2*>(orow) = uh;
    *reinterpret_cast<uint2*>(orow + p.o_third) = ul;
    *reinterpret_cast<uint2*>(orow + 2 * p.o_third) = uh;
  }
}

// out = sum_s w_s O_s / sum_s w_s l_s, w_s = exp(m_s - max_s m_s), written as [hi | lo | hi]
__global__ void __launch_bounds__(256)
attention_f32_combine_kernel(const float* __restrict__ part_o, const float* __restrict__ part_ml,
                             bf16* __restrict__ O, int o_third, int heads, int splits,
                             long long n_rh) {
  griddep_launch_dependents();
  const long long gid = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long rh = gid >> 4;  // (row, head) pair; 16 threads x 4 columns each
  const int c4 = static_cast<int>(gid & 15);
  if (rh >= n_rh) return;
  griddep_wait();
  float mmax = -INFINITY;
  for (int s = 0; s < splits; ++s) mmax = fmaxf(mmax, part_ml[(rh * splits + s) * 2]);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  float lt = 0.f;
  for (int s = 0; s < splits; ++s) {
    const float2 ml = *reinterpret_cast<const float2*>(part_ml + (rh * splits + s) * 2);
    const float w = (ml.x == -INFINITY) ? 0.f : expf(ml.x - mmax);
    const float4 v = *reinterpret_cast<const float4*>(part_o + (rh * splits + s) * FD + c4 * 4);
    acc[0] += w * v.x; acc[1] += w * v.y; acc[2] += w * v.z; acc[3] += w * v.w;
    lt += w * ml.y;
  }
  const float inv = lt > 0.f ? 1.0f / lt : 0.f;
  float lo[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    acc[c] *= inv;
    lo[c] = acc[c] - __bfloat162float(__float2bfloat16_rn(acc[c]));
  }
  const long long row = rh / heads;
  const int head = static_cast<int>(rh - row * heads);
  const uint2 uh = make_uint2(pack_bf16(acc[0], acc[1]), pack_bf16(acc[2], acc[3]));
  const uint2 ul = make_uint2(pack_bf16(lo[0], lo[1]), pack_bf16(lo[2], lo[3]));
  bf16* orow = O + row * (3LL * o_third) + head * FD + c4 * 4;
  *reinterpret_cast<uint2*>(orow) = uh;
  *reinterpret_cast<uint2*>(orow + o_third) = ul;
  *reinterpret_cast<uint2*>(orow + 2 * o_third) = uh;
}

}  // namespace

int launch_attention_f32(const AttnF32Args& a, cudaStream_t stream) {
  MSD_REQUIRE(a.Lq % FQ == 0 && a.Lk % FK == 0, "attention_f32: Lq=%d / Lk=%d must be multiples of %d / %d",
              a.Lq, a.Lk, FQ, FK);
  MSD_REQUIRE(a.nbatch > 0 && a.heads > 0, "attention_f32: empty problem");
  MSD_REQUIRE(a.ldq % 4 == 0 && a.ldk % 4 == 0 && a.ldv % 4 == 0 && a.o_third % 4 == 0,
              "attention_f32: leading dimensions must be multiples of 4");
  static const int configured = [] {
    return cudaFuncSetAttribute(attention_f32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                F32_SMEM) == cudaSuccess ? 0 : -2;
  }();
  MSD_REQUIRE(configured == 0, "attention_f32: cannot opt in to %d bytes of shared memory", F32_SMEM);
  const int kv_batch_rows = a.kv_batch_rows > 0 ? a.kv_batch_rows : a.Lk;
  MSD_REQUIRE(a.kv_row0 >= 0 && a.kv_row0 + a.Lk <= kv_batch_rows && a.kv_row0 % 64 == 0,
              "attention_f32: key rows [%d, %d) exceed the %d rows per batch", a.kv_row0,
              a.kv_row0 + a.Lk, kv_batch_rows);
  AttnF32Dev d;
  d.Q = a.Q; d.ldq = a.ldq; d.K = a.K; d.ldk = a.ldk; d.V = a.V; d.ldv = a.ldv;
  d.O = a.O; d.o_third = a.o_third; d.heads = a.heads; d.Lq = a.Lq; d.Lk = a.Lk;
  d.mask_bits = a.mask_bits; d.mask_stride_words = a.mask_stride_words;
  d.kv_batch_rows = kv_batch_rows; d.kv_row0 = a.kv_row0;
  // split the keys when the grid would leave SMs idle (one segment's cross-attention)
  int splits = 1;
  const int ctas = (a.Lq / FQ) * a.heads * a.nbatch, nkb = a.Lk / FK;
  if (a.part_o != nullptr && a.part_ml != nullptr) {
    if (a.splits > 0) {
      splits = a.splits;
    } else {
      const int sms = device_sm_count();
      for (int s = 2; s <= a.max_splits && ctas * (s - 1) < 3 * sms; ++s)
        if (nkb % s == 0 && nkb / s >= 4) splits = s;
    }
    if (splits > a.max_splits) splits = a.max_splits > 0 ? a.max_splits : 1;
  }
  MSD_REQUIRE(nkb % splits == 0, "attention_f32: %d key blocks not divisible by %d splits", nkb, splits);
  d.splits = splits; d.part_o = a.part_o; d.part_ml = a.part_ml;
  ProfScope prof(KC_ATTENTION, 4.0 * a.nbatch * a.heads * static_cast<double>(a.Lq) * a.Lk * FD,
                 4.0 * a.nbatch * a.heads * FD * (2.0 * a.Lq + 2.0 * a.Lk), stream);
  MSD_CUDA_CHECK(launch_kernel(attention_f32_kernel, dim3(a.Lq / FQ, a.heads, a.nbatch * splits),
                               dim3(F32_THREADS), F32_SMEM, stream, d));
  ++g_launch_count;
  if (splits > 1) {
    const long long n_rh = static_cast<long long>(a.nbatch) * a.Lq * a.heads;
    MSD_CUDA_CHECK(launch_kernel(attention_f32_combine_kernel,
                                 dim3(static_cast<unsigned>((n_rh * 16 + 255) / 256)), dim3(256), 0,
                                 stream, static_cast<const float*>(a.part_o),
                                 static_cast<const float*>(a.part_ml), a.O, a.o_third, a.heads,
                                 splits, n_rh));
    ++g_launch_count;
  }
  return 0;
}

}  // namespace msd
