// wgrad_tc.cu -- the DCRNN weight / bias gradient contraction on the tensor cores (wgmma, TF32, K-major operands).
//
//   dW_zr [3C x 64] = S1^T dpre_zr,   dW_h [3C x 32] = S2^T dpre_h,   db = 1^T dpre        over all rows = T*B*N (159 k at B = 64)
//
// (what autograd accumulates for the matmul(basis, W) + bias of torch_geometric_temporal/nn/recurrent/dcrnn.py:86-111 across steps, gates
// and hops).  The contraction axis is the ROW axis of the row-major operands; TF32 wgmma takes K-major operands only, so a 16-row tile
// is transposed while it is converted: operand row m (a column of S, or of dpre) holds the tile's 16 k values, 64 bytes, in the
// canonical K-major SWIZZLE_64B layout (8-row atoms of 512 B, the four 16-byte chunks of a row XOR-ed with (row / 2) % 4).  fp16 hi/lo
// splits (the forward kernel's trick) would need a gradient scale -- d pre-activations of a mean loss are ~1e-5 and fall into fp16
// subnormals -- so the split is TF32 hi + TF32 lo (fp32 exponent range, 21+ mantissa bits together): three passes hi*hi + lo*hi + hi*lo
// per product, accumulators in registers (two sets used alternately).
//
// Per CTA (one per SM; 8 converting warps = 2 warpgroups + 1 TMA producer warp): a 6-stage ring of 16-row fp32 tiles S1 | S2 | dpre_zr |
// dpre_h filled by TMA bulk copies; the two warpgroups convert a tile into one of two operand buffers (hi and lo copies) and then each
// issues the MMAs of its 64 rows of the weight gradient.  (ptxas serializes these wgmmas -- the accumulator set is chosen per tile -- so
// a tile's MMAs complete before the next tile is converted; the two operand buffers still let the TMA ring run ahead.)
// The bias row-sums ride along as a row of ones at m = 127 of the A operands.  Epilogue: one partial per CTA, summed in a fixed order by
// k_dcrnn_wgrad_reduce (train.cu) straight into the module's weight layout.
#include "tc_common.cuh"

namespace stmp {
namespace {

constexpr int kCo = 32;
constexpr int kTK = 16;                  // rows per tile = two k-steps of 8 (one TF32 wgmma consumes K = 8)
constexpr int kStages = 6;
constexpr int kConvThreads = 256;        // warps 0..7 convert and issue the MMAs (two warpgroups); warp 8 = TMA producer
constexpr int kThreads = kConvThreads + 32;
constexpr int kObBytes = 45056;          // one operand buffer: A1 hi|lo 2 x 8 KB, A2 hi|lo 2 x 8 KB, B1 hi|lo 2 x 4 KB, B2 hi|lo 2 x 2 KB
constexpr int kOffA1 = 0, kOffA2 = 16384, kOffB1 = 32768, kOffB2 = 40960;
constexpr int kLoA = 8192, kLoB1 = 4096, kLoB2 = 2048;   // offset of the lo copy behind the hi copy

struct WgTcParams {
  const float* S1; const float* S2; const float* dpzr; const float* dph;
  long long rows;
  int ld, n_tiles, MG, C3;               // C3 = (n_ops + 1)(cin + cout) (DCRNN: 3 blocks): columns >= C3 of S are padding
  float* partial;                        // [grid][MG*8*96 + 96]
};

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// barrier of the converting warps only (the producer warp has left)
__device__ __forceinline__ void conv_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kConvThreads) : "memory"); }
__device__ __forceinline__ float tf32_rna(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return __uint_as_float(r);
}
// byte offset of k values 4q..4q+3 (q = 0..3) of operand row m: K-major SWIZZLE_64B
__device__ __forceinline__ int kmaj64(int m, int q) { return (m >> 3) * 512 + (m & 7) * 64 + ((q ^ ((m >> 1) & 3)) << 4); }
__device__ __forceinline__ uint64_t desc64(uint32_t saddr) { return gmma_desc(saddr, 512, 2); }

__device__ __forceinline__ void store_split_tf32(unsigned char* hi, int lo_off, int off, float4 v) {
  const float4 h = make_float4(tf32_rna(v.x), tf32_rna(v.y), tf32_rna(v.z), tf32_rna(v.w));
  *reinterpret_cast<float4*>(hi + off) = h;
  *reinterpret_cast<float4*>(hi + lo_off + off) = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
}

struct WgAcc { float z0[16], z1[16], h[16]; };   // m64 rows of D_zr columns [0,32) [32,64) and of D_h

__global__ void __launch_bounds__(kThreads, 1) k_dcrnn_wgrad_tc(WgTcParams p) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ld = p.ld;
  const int stage_bytes = kTK * (2 * ld + 3 * kCo) * 4;
  unsigned char* ob0 = smem;                                   // two operand buffers (1024-byte aligned)
  unsigned char* raw = smem + 2 * kObBytes;                    // kStages raw fp32 tiles
  // mbarriers: raw_full[s] (TMA bytes landed) | raw_free[s] (both warpgroups have read the stage)
  uint64_t* raw_full = reinterpret_cast<uint64_t*>(raw + (size_t)kStages * stage_bytes);
  uint64_t* raw_free = raw_full + kStages;

  if (tid == 0) {
    for (int i = 0; i < kStages; ++i) { mbar_init(&raw_full[i], 1); mbar_init(&raw_free[i], kConvThreads / 32); }
    fence_mbar_init();
  }
  // operand buffers: zero (rows >= ld of A are never written again), then the row of ones at m = 127 of A1 hi / A2 hi
  for (int i = tid; i < 2 * kObBytes / 16; i += kThreads) reinterpret_cast<uint4*>(ob0)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  if (tid < 2 * 2 * 4) {                                       // (buffer, operand, k chunk)
    const int q = tid & 3, which = (tid >> 2) & 1, b = tid >> 3;
    *reinterpret_cast<float4*>(ob0 + b * kObBytes + (which ? kOffA2 : kOffA1) + kmaj64(127, q)) = make_float4(1.f, 1.f, 1.f, 1.f);
  }
  fence_proxy_async();
  __syncthreads();

  auto issue_tma = [&](int tile, int s) {
    const long long r0 = (long long)tile * kTK;
    const int nr = (int)((p.rows - r0) < kTK ? (p.rows - r0) : kTK);
    float* st = reinterpret_cast<float*>(raw + (size_t)s * stage_bytes);
    const uint32_t bs = (uint32_t)nr * ld * 4u, bzr = (uint32_t)nr * 2 * kCo * 4u, bh = (uint32_t)nr * kCo * 4u;
    mbar_arrive_expect_tx(&raw_full[s], 2 * bs + bzr + bh);
    tma_bulk_g2s(st, p.S1 + r0 * ld, bs, &raw_full[s]);
    tma_bulk_g2s(st + kTK * ld, p.S2 + r0 * ld, bs, &raw_full[s]);
    tma_bulk_g2s(st + 2 * kTK * ld, p.dpzr + r0 * 2 * kCo, bzr, &raw_full[s]);
    tma_bulk_g2s(st + 2 * kTK * ld + kTK * 2 * kCo, p.dph + r0 * kCo, bh, &raw_full[s]);
  };

  int n_local = 0;                                               // tiles of this CTA
  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) ++n_local;

  if (warp == kConvThreads / 32) {
    // ---- producer warp: one lane keeps the TMA ring full -------------------------------------------------------------------------
    if (lane == 0) {
      for (int q = 0; q < kStages && q < n_local; ++q) issue_tma(blockIdx.x + q * gridDim.x, q);
      for (int it = kStages; it < n_local; ++it) {
        const int sp = it % kStages;                             // last used by tile it - kStages
        mbar_wait(&raw_free[sp], ((it - kStages) / kStages) & 1);
        issue_tma(blockIdx.x + it * gridDim.x, sp);
      }
    }
    return;
  }

  // ---- converting / MMA warps ------------------------------------------------------------------------------------------------------
  // Conversion work of a thread is the same for every tile (k = row of the raw tile):
  //   A1, A2     operand row m = tid & 127, k chunk pair (tid >> 7) * 2 + {0, 1}   (idle when m >= ld)
  //   B1         row n = tid & 63, k chunk tid >> 6                                 B2   row n = tid & 31, k chunk tid >> 5 (tid < 128)
  const int wg = warp >> 2, wt = tid & 127;
  const int am = tid & 127, aq0 = (tid >> 7) * 2;
  const bool a_on = am < ld;
  const bool a_zero = am >= p.C3;                                // padding columns of S hold garbage: they must never reach a result
  const int b1n = tid & 63, b1q = tid >> 6, b2n = tid & 31, b2q = tid >> 5;
  WgAcc acc[2];
#pragma unroll
  for (int s = 0; s < 2; ++s)
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[s].z0[i] = acc[s].z1[i] = acc[s].h[i] = 0.f;

  auto issue = [&](WgAcc& a, uint32_t ob_s) {
    wgmma_fence();
#pragma unroll
    for (int kg = 0; kg < 2; ++kg) {
      // one TF32 wgmma consumes K = 8 = 32 bytes of each operand row
      const uint32_t a1 = ob_s + kOffA1 + wg * 64 * 64 + kg * 32, a2 = ob_s + kOffA2 + wg * 64 * 64 + kg * 32;
      const uint32_t b1 = ob_s + kOffB1 + kg * 32, b2 = ob_s + kOffB2 + kg * 32;
#pragma unroll
      for (int pass = 0; pass < 3; ++pass) {           // lo*hi, hi*lo, hi*hi (small terms first)
        const uint32_t ao = pass == 0 ? kLoA : 0, b1o = pass == 1 ? kLoB1 : 0, b2o = pass == 1 ? kLoB2 : 0;
        wgmma_tf32_n32(a.z0, desc64(a1 + ao), desc64(b1 + b1o));
        wgmma_tf32_n32(a.z1, desc64(a1 + ao), desc64(b1 + b1o + 32 * 64));
        wgmma_tf32_n32(a.h, desc64(a2 + ao), desc64(b2 + b2o));
      }
    }
    wgmma_commit();
  };

  for (int it = 0; it < n_local; ++it) {
    const int s = it % kStages, ob = it & 1;
    const long long r0 = ((long long)blockIdx.x + (long long)it * gridDim.x) * kTK;
    const int nr = (int)((p.rows - r0) < kTK ? (p.rows - r0) : kTK);                  // < 16 only for the last tile: missing rows become zeros
    mbar_wait(&raw_full[s], (it / kStages) & 1);
    const float* st = reinterpret_cast<const float*>(raw + (size_t)s * stage_bytes);
    auto col4 = [&](const float* base, int pitch, int q, int n) {                      // rows 4q..4q+3 of column n
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = 4 * q + e < nr ? base[(4 * q + e) * pitch + n] : 0.f;
      return make_float4(v[0], v[1], v[2], v[3]);
    };
    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 s1[2], s2[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      s1[i] = (a_on && !a_zero) ? col4(st, ld, aq0 + i, am) : zero4;
      s2[i] = (a_on && !a_zero) ? col4(st + kTK * ld, ld, aq0 + i, am) : zero4;
    }
    const float4 v1 = col4(st + 2 * kTK * ld, 2 * kCo, b1q, b1n);
    const float4 v2 = tid < 128 ? col4(st + 2 * kTK * ld + kTK * 2 * kCo, kCo, b2q, b2n) : zero4;
    __syncwarp();
    if (lane == 0) mbar_arrive(&raw_free[s]);
    wgmma_wait<1>();            // my MMAs of tile it - 2 (operand buffer ob) are done; those of tile it - 1 keep running
    conv_sync();                // ... and the other warpgroup's
    unsigned char* o = ob0 + ob * kObBytes;
    if (a_on) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        store_split_tf32(o + kOffA1, kLoA, kmaj64(am, aq0 + i), s1[i]);
        store_split_tf32(o + kOffA2, kLoA, kmaj64(am, aq0 + i), s2[i]);
      }
    }
    store_split_tf32(o + kOffB1, kLoB1, kmaj64(b1n, b1q), v1);
    if (tid < 128) store_split_tf32(o + kOffB2, kLoB2, kmaj64(b2n, b2q), v2);
    fence_proxy_async();          // generic-proxy operand stores -> visible to the tensor core
    conv_sync();
    // two accumulator sets used alternately: the tensor core's fp32 accumulation is not round-to-nearest, a shorter chain per set (and an
    // fp32 sum of the sets in the epilogue) keeps the result close to the fp32 FFMA kernel
    if (it & 1) issue(acc[1], smem_u32(o)); else issue(acc[0], smem_u32(o));
  }
  wgmma_wait<0>();
#pragma unroll
  for (int s = 0; s < 2; ++s) { acc_fence(acc[s].z0); acc_fence(acc[s].z1); acc_fence(acc[s].h); }

  // ---- epilogue: fragment rows m = 64 wg + 16 (wt / 32) + (lane / 4) (+8), columns 8 j + 2 (lane % 4) (+1) ------------------------
  const int MG8 = p.MG * 8;
  float* out = p.partial + (size_t)blockIdx.x * ((size_t)MG8 * 3 * kCo + 3 * kCo);
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int m = 64 * wg + 16 * (wt >> 5) + ((wt & 31) >> 2) + 8 * hr;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = 8 * j + 2 * (wt & 3), a = 4 * j + 2 * hr;
      const float2 z0 = make_float2(acc[0].z0[a] + acc[1].z0[a], acc[0].z0[a + 1] + acc[1].z0[a + 1]);
      const float2 z1 = make_float2(acc[0].z1[a] + acc[1].z1[a], acc[0].z1[a + 1] + acc[1].z1[a + 1]);
      const float2 h = make_float2(acc[0].h[a] + acc[1].h[a], acc[0].h[a + 1] + acc[1].h[a + 1]);
      if (m < MG8) {
        *reinterpret_cast<float2*>(out + (size_t)m * 2 * kCo + n) = z0;
        *reinterpret_cast<float2*>(out + (size_t)m * 2 * kCo + 32 + n) = z1;
        *reinterpret_cast<float2*>(out + (size_t)MG8 * 2 * kCo + (size_t)m * kCo + n) = h;
      } else if (m == 127) {                                    // the ones row: bias sums z | r | h
        float* bsum = out + (size_t)MG8 * 3 * kCo;
        *reinterpret_cast<float2*>(bsum + n) = z0;
        *reinterpret_cast<float2*>(bsum + 32 + n) = z1;
        *reinterpret_cast<float2*>(bsum + 64 + n) = h;
      }
    }
  }
}

}  // namespace

// launched by stmp_dcrnn_bwd_wgrad / stmp_gru_bwd_wgrad (train.cu), c3 = used basis columns; returns the number of partials written (= grid)
int wgrad_tc_launch(int c3, long long rows, int ld, const float* S1, const float* S2, const float* dpzr, const float* dph, float* partial,
                    int max_parts, cudaStream_t st, int* parts) {
  WgTcParams p;
  p.S1 = S1; p.S2 = S2; p.dpzr = dpzr; p.dph = dph; p.rows = rows; p.ld = ld;
  p.C3 = c3; p.MG = (p.C3 + 7) / 8;
  p.n_tiles = (int)((rows + kTK - 1) / kTK);
  p.partial = partial;
  int dev = 0, sms = 132;
  STMP_CUDA_OK(cudaGetDevice(&dev));
  STMP_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  int grid = sms < max_parts ? sms : max_parts;
  if (p.n_tiles < grid) grid = p.n_tiles > 0 ? p.n_tiles : 1;
  const int smem = 2 * kObBytes + kStages * kTK * (2 * ld + 3 * kCo) * 4 + 2 * kStages * 8;
  STMP_CUDA_OK(cudaFuncSetAttribute(k_dcrnn_wgrad_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_dcrnn_wgrad_tc<<<grid, kThreads, smem, st>>>(p);
  STMP_LAUNCH_OK("k_dcrnn_wgrad_tc");
  *parts = grid;
  return STMP_OK;
}

}  // namespace stmp
