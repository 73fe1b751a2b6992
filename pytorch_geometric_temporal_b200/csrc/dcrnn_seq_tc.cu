// dcrnn_seq_tc.cu -- fused DCRNN recurrence with the dense contraction on the Hopper tensor cores (wgmma).
//
// Same contract as k_dcrnn_seq (dcrnn_seq.cu) for K=2, Cout=32, Cin<=4, N<=255; what changes is WHERE the
// S @ [Wz|Wr] and S @ Wh contractions run: warpgroup MMAs (wgmma, fp32 accumulators in registers) instead of FFMA.
// Two kernels: k_dcrnn_seq_rf (one CTA per window, A operands gathered straight into registers; below, "the one-CTA kernel") and
// k_dcrnn_seq_tc<CIN, 2> (a 2-CTA cluster per window for small batches, A operands in shared-memory panels; described first).
//
// fp32 accuracy on fp16 tensor cores: every fp32 operand v is split on the fly into hi = fp16(v) and
// lo = fp16(v - hi) (22 mantissa bits together; products of fp16 pairs are exact in the fp32 accumulator) and
// the product is formed as lo*hi + hi*lo + hi*hi -- three MMAs.  The tests hold the result to the fp32 oracle at
// rtol 1e-4 / atol 1e-5 (tests/test_gpu_dcrnn.py).
//
// Shared memory (~204 KB of 227), all operands written by hand in the canonical K-major SWIZZLE_128B layout
// (row pitch 128 B = 64 fp16, 16-byte chunk index XOR (row % 8), 8-row atoms of 1024 B):
//   A_hi / A_lo : 2 K-panels x 208 rows   k = [H|H*R (32) , P_o H (32)] , [P_i H (32), X(4) P_oX(4) P_iX(4) 0(4)]
//   B_hi / B_lo : 2 K-panels x 96 rows    rows = output channels of z | r | h, same k order (7 k-steps of 16)
//   U  fp32 [208][36] = H (or H*R) + 16 B of row padding: the gather source of the diffusion (tensor cores only see the fp16 split); row 207 = 0
//   graph image (graph_image.cuh: balanced warp-task lists, 8-bit source rows four per word, values four per 128 bits),
//   biases, one mbarrier (prologue TMA).
// 16 warps = 4 warpgroups; warpgroup wg = one 64-row MMA subtile, rows [64 wg, 64 wg + 64) (warpgroups 0-1 form row tile 0, 2-3 tile 1).
// Per k-step and pass it issues one m64n64k16 for GEMM 1 (B rows 0..63 = z | r) and one m64n32k16 for GEMM 2 (the candidate), so the
// A rows of a subtile are read once per MMA k-step, and keeps the accumulators in registers: every thread applies the gates to the
// (row, channel) pairs its fragment holds -- rows 64 wg + 16 w + l/4 (+8), channels 8 jj + 2 (l % 4) (+1), jj = 0..3 -- with z, r
// and the candidate of a pair in the same thread.  It keeps H of those pairs in registers and writes H*R / H_t back as fp32 (U), as
// fp16 hi/lo (A panel) and to HBM.
// The wgmmas are issued on paths ptxas can prove warpgroup-uniform (no run-time row guards; the role comes from a warp broadcast), so
// they run asynchronously: the H | X group under the gather of tile 0, tile 0's P groups under the gather of tile 1.
#include <cuda_fp16.h>

#include <cstdlib>

#include "common.cuh"
#include "dcrnn_common.cuh"
#include "graph_image.cuh"
#include "row_image.cuh"
#include "tc_common.cuh"

namespace stmp {
namespace {

constexpr int kMaxSmemTc = 232448;
constexpr int TC_UP = 36;                  // U row pitch (floats): a 128-byte row of H (or of T*Cin X values in the window prologue) + 16 B, so that the
                                           // epilogue's row-strided 16-byte stores rotate through the banks (pitch 32: 8-way conflicts, measured -14 %)
constexpr int TC_UROWS = 208;              // rows of U; row 207 is the all-zero row that pad entries of the graph image point at
constexpr int TC_AROWS = 208;              // rows stored per A panel (subtile 3 over-reads into the next buffer: harmless)
constexpr int TC_PANEL_A = TC_AROWS * 128;
constexpr int TC_PANEL_B = 96 * 128;

struct TcParams {
  int N, CIN, T;
  long long B;
  const float* x;
  const long long* win_start;
  long long x_bstride, x_tstride;
  const float* w[3];
  const float* bias[3];
  const float* h0;
  long long h0_bstride;   // elements between windows' H0 (0: every window starts from the same H0)
  const float* wcat;      // optional prepacked fp32 weights [96][112] in the kernel's k order (else: DConv weights p.w[])
  const float* bcat;      // with wcat: biases [96]
  int n_ops;              // 2: DConv (P_o, P_i); 1: single operator (ChebConv K=2 / GCN); 0: no propagation
  const void* gimg;       // plan's prebuilt shared-memory graph image for n_ops operators (TMA bulk source; cluster pair)
  GraphImageLayout gl;    // its internal offsets
  const void* rimg;       // plan's row image for n_ops operators (one-CTA kernel; null for n_ops = 0)
  RowImageLayout rl;      // its offsets
  const void* wimage;     // prebuilt B-operand image (fp16 hi/lo, swizzled, + biases) or null
  float* out;
  float* stash;
  float* ws;              // workspace [grid][N][2 operators][ws_pitch] for P_o X / P_i X of a window's steps, or null (park them in `out`)
  int ws_pitch;
  int off_A, off_B, off_U, off_img, off_bias, off_bar;
};

// CW = 32 (whole row) or 16 (channel half `half`): chunks [half*CW/8, +CW/8) of panel 0
template <int CW>
__device__ __forceinline__ void store_split_row(unsigned char* a_hi, unsigned char* a_lo, int row, int half, const float (&v)[CW]) {
#pragma unroll
  for (int c = 0; c < CW / 8; ++c) {
    uint32_t hw[4], lw[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float a = v[8 * c + 2 * j], b = v[8 * c + 2 * j + 1];
      const __half2 h = __floats2half2_rn(a, b);
      const float2 f = __half22float2(h);
      hw[j] = pack_h2(h);
      lw[j] = pack_h2(__floats2half2_rn(a - f.x, b - f.y));
    }
    const int off = row * 128 + (((half * (CW / 8) + c) ^ (row & 7)) << 4);
    *reinterpret_cast<uint4*>(a_hi + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
    *reinterpret_cast<uint4*>(a_lo + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
  }
}

constexpr int TC_WIMAGE_BYTES = 4 * TC_PANEL_B + 96 * 4;   // B hi (2 panels) | B lo (2 panels) | 96 biases

// fp32 weight of output row n (gate*32 + channel) at k position kk (kernel k order, 0..111)
__device__ __forceinline__ float tc_weight_value(const float* wcat, const float* w0, const float* w1, const float* w2, int CIN, int n,
                                                 int kk) {
  if (wcat) return wcat[n * 112 + kk];
  const int C = 32 + CIN;
  const int gte = n >> 5, o = n & 31;
  const int panel = kk >= 64 ? 1 : 0, kin = kk - 64 * panel;
  int blk, ch;  // blk 0: U, 1: P_o, 2: P_i ; ch = reference channel index or -1
  if (panel == 0) { blk = kin < 32 ? 0 : 1; ch = CIN + (kin & 31); }
  else if (kin < 32) { blk = 2; ch = CIN + kin; }
  else { const int qq = kin - 32; blk = qq >> 2; const int c = qq & 3; ch = (blk < 3 && c < CIN) ? c : -1; }
  if (ch < 0) return 0.f;
  const float* wg = gte == 0 ? w0 : (gte == 1 ? w1 : w2);
  if (blk == 0) return wg[((0 * 2 + 0) * C + ch) * 32 + o] + wg[((1 * 2 + 0) * C + ch) * 32 + o];
  return wg[(((blk - 1) * 2 + 1) * C + ch) * 32 + o];
}

// Builds the B-operand image once per weight update (stmp_*_pack_weights); the fused kernel then TMA-copies it.
__global__ void k_pack_weight_image(const float* wcat, const float* bcat, const float* w0, const float* w1, const float* w2,
                                    const float* b0, const float* b1, const float* b2, int CIN, unsigned char* image) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < 96 * 128) {
    const int n = idx >> 7, kk = idx & 127;
    const float v = kk < 112 ? tc_weight_value(wcat, w0, w1, w2, CIN, n, kk) : 0.f;
    const __half h = __float2half_rn(v);
    const __half l = __float2half_rn(v - __half2float(h));
    const int off = (kk >> 6) * TC_PANEL_B + sw128(n, kk & 63);
    *reinterpret_cast<__half*>(image + off) = h;
    *reinterpret_cast<__half*>(image + 2 * TC_PANEL_B + off) = l;
  } else if (idx < 96 * 128 + 96) {
    const int j = idx - 96 * 128, gte = j >> 5;
    const float* bg = gte == 0 ? b0 : (gte == 1 ? b1 : b2);
    reinterpret_cast<float*>(image + 4 * TC_PANEL_B)[j] = bcat ? bcat[j] : (bg ? bg[j & 31] : 0.f);
  }
}

// fast, accurate-enough gates (abs err ~2e-7): ex2.approx + rcp.approx
__device__ __forceinline__ float sigmoid_fast(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float tanh_fast(float x) { return 2.0f * __fdividef(1.0f, 1.0f + __expf(-2.0f * x)) - 1.0f; }

// ---- gather ------------------------------------------------------------------------------------------------------------
// Weighted sum of the source rows of one task (graph_image.cuh): quarter-warp lane j accumulates floats 4j..4j+3 of the row.
// Four edges per group: one broadcast 32-bit load carries their four 8-bit source rows, one 128-bit load their values; the
// next group's entries are fetched while the current group's four feature rows are in flight.  Summation order = CSR order
// (the reference's scatter order), products by FMA as in the round-1 kernel.
__device__ __forceinline__ float4 gather_groups(const float* __restrict__ Uj, const uint32_t* __restrict__ idx4,
                                                const float4* __restrict__ val4, int g0, int ng) {
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  uint32_t u = idx4[g0];
  float4 v = val4[g0];
#pragma unroll 2    // a task has 2-3 groups on average: the rolled loop's branch and convergence barrier were 10 % of the issued instructions
  for (int g = 1; g <= ng; ++g) {
    const uint32_t un = idx4[g0 + g];      // (one spare group at the end of the arrays)
    const float4 vn = val4[g0 + g];
    // (predicating the loads of pad entries off saves their wavefronts but costs more in compares / selects: measured -2 %, A/B on one box)
    const float4 x0 = ld4(Uj + (u & 0xffu) * TC_UP);
    const float4 x1 = ld4(Uj + ((u >> 8) & 0xffu) * TC_UP);
    const float4 x2 = ld4(Uj + ((u >> 16) & 0xffu) * TC_UP);
    const float4 x3 = ld4(Uj + (u >> 24) * TC_UP);
    fma4(acc, v.x, x0);
    fma4(acc, v.y, x1);
    fma4(acc, v.z, x2);
    fma4(acc, v.w, x3);
    u = un;
    v = vn;
  }
  return acc;
}

// Step anatomy (all 16 warps = 4 warpgroups; T_k = MMA row tile k = rows [128k, 128k+128)):
//   round 1  every warpgroup issues the H | X k-steps of GEMM1 for its subtile; all warps gather [P_o H | P_i H] of T_0's rows -> A panels
//            barrier; T_0's warpgroups issue their P_o / P_i k-steps, then (with their MMAs in flight) gather T_1's rows
//            barrier; T_1's warpgroups issue their k-steps
//   epi 1    wait GEMM1 (own MMAs): R, H*R; barrier (every MMA has read the A panels); H*R -> U, A panel                      barrier
//   round 2  same gathers over H*R, GEMM2 (candidate)
//   epi 2    wait GEMM2: Z (from the GEMM1 accumulators, still in registers), H~, H_t; barrier; H_t -> U, A panel, HBM;
//            X_{t+1} k-step                                                                                                  barrier
// A warpgroup issues the wgmmas of its own subtile: the accumulator fragments then sit in the threads that apply the gates, so the
// epilogue is register-local.  Thread (warp w of the group, lane l) owns rows row0 + 16 w + l/4 (+8) and channels ch0 + 8 jj + 2 (l % 4)
// (+1), jj < NJ.
// The task lists of the gather are balanced over the warps when the plan is built (graph_image.cuh), which is what makes the extra
// barriers cheap (round 1 profile: 25 % of all warp time was barrier wait behind the warp that always drew the longest rows).
// X is never gathered per step: P_o X_t, P_i X_t of ALL steps of a window are produced by one gather pass over rows of
// T*Cin floats in the window prologue and parked in the window's own (not yet written) output rows out[b, t, :, 0:8].
// SPLIT = 2 (small batches: 2 B CTAs still fit the machine, N > 128): a window is served by a 2-CTA thread-block cluster.  CTA c owns MMA
// row tile c -- its gather tasks, its MMAs, its epilogue (warpgroup = subtile x channel half: m64n16 per gate) -- and pushes the rows of H*R / H_t it
// produces into the partner's gather buffer U through distributed shared memory, so both gathers stay local.  Per round: "done reading U"
// is a relaxed cluster arrival right after the gather, waited for just before the epilogue overwrites U; the barrier that closes an epilogue is
// a release / acquire cluster barrier (the pushed rows are visible).
template <int CIN, int SPLIT>
__global__ void __launch_bounds__(512, 1) k_dcrnn_seq_tc(const TcParams p) {
  constexpr int NJ = SPLIT == 2 ? 2 : 4;    // 8-channel groups of a warpgroup (all 32 channels / a half)
  constexpr int NE = 2;                     // rows of a thread's accumulator fragment
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int N = p.N, T = p.T;
  unsigned char* a_hi = smem + p.off_A;
  unsigned char* a_lo = a_hi + 2 * TC_PANEL_A;
  unsigned char* b_hi = smem + p.off_B;
  unsigned char* b_lo = b_hi + 2 * TC_PANEL_B;
  float* U = reinterpret_cast<float*>(smem + p.off_U);
  const unsigned char* img = smem + p.off_img;
  const uint16_t* s_wstart = reinterpret_cast<const uint16_t*>(img + p.gl.off_wstart);
  const uint16_t* s_wcount = reinterpret_cast<const uint16_t*>(img + p.gl.off_wcount);
  const uint32_t* s_wt = reinterpret_cast<const uint32_t*>(img + p.gl.off_wt);
  const uint32_t* s_idx = reinterpret_cast<const uint32_t*>(img + p.gl.off_idx);
  const float4* s_val = reinterpret_cast<const float4*>(img + p.gl.off_val);
  float* Bs = reinterpret_cast<float*>(smem + p.off_bias);
  uint64_t* tma_bar = reinterpret_cast<uint64_t*>(smem + p.off_bar);   // prologue TMA (graph and weight images)

  const int crank = SPLIT == 2 ? (int)cluster_rank() : 0;
  const long long cta = blockIdx.x / SPLIT, n_cta = gridDim.x / SPLIT;
  if (cta >= p.B) return;

  // ---- one-time per CTA ------------------------------------------------------------------------------------
  if (tid == 0) {
    mbar_init(tma_bar, 1);
    fence_mbar_init();
    const uint32_t tx = (p.n_ops ? (uint32_t)p.gl.bytes : 0u) + (p.wimage ? (uint32_t)TC_WIMAGE_BYTES : 0u);
    if (tx) {   // graph image and weight image arrive by TMA bulk copies while the CTA zeroes its panels
      mbar_arrive_expect_tx(tma_bar, tx);
      if (p.n_ops) tma_bulk_g2s(smem + p.off_img, p.gimg, (uint32_t)p.gl.bytes, tma_bar);
      if (p.wimage) {
        tma_bulk_g2s(b_hi, p.wimage, 4u * TC_PANEL_B, tma_bar);
        tma_bulk_g2s(Bs, reinterpret_cast<const unsigned char*>(p.wimage) + 4 * TC_PANEL_B, 96u * 4u, tma_bar);
      }
    }
  }
  {  // zero A (pad columns / rows must be finite) and U (row 207 stays the zero row); B too unless the TMA image overwrites all of it
    uint4* z = reinterpret_cast<uint4*>(a_hi);
    const int nz = (4 * TC_PANEL_A + (p.wimage ? 0 : 4 * TC_PANEL_B)) / 16;
    for (int i = tid; i < nz; i += 512) z[i] = make_uint4(0, 0, 0, 0);
    for (int i = tid; i < TC_UROWS * TC_UP; i += 512) U[i] = 0.f;
  }
  __syncthreads();
  if (!p.wimage) {
    // weights -> B operand (fp16 hi/lo, swizzled).  Row n = gate*32 + out channel; k order as the A panels.
    for (int idx = tid; idx < 96 * 112; idx += 512) {
      const int n = idx / 112, kk = idx - n * 112;
      const float v = tc_weight_value(p.wcat, p.w[0], p.w[1], p.w[2], CIN, n, kk);
      const __half h = __float2half_rn(v);
      const __half l = __float2half_rn(v - __half2float(h));
      const int off = (kk >> 6) * TC_PANEL_B + sw128(n, kk & 63);
      *reinterpret_cast<__half*>(b_hi + off) = h;
      *reinterpret_cast<__half*>(b_lo + off) = l;
    }
    for (int idx = tid; idx < 96; idx += 512) {
      const int gte = idx >> 5;
      const float* bg = gte == 0 ? p.bias[0] : (gte == 1 ? p.bias[1] : p.bias[2]);
      Bs[idx] = p.bcat ? p.bcat[idx] : (bg ? bg[idx & 31] : 0.f);
    }
  }
  if (p.n_ops || p.wimage) mbar_wait(tma_bar, 0);
  fence_proxy_async();
  __syncthreads();

  // Warpgroup wg owns one 64-row subtile (rows [64 sub, 64 sub + 64)) and 8 NJ channels of it.  SPLIT 1: sub = wg, all channels (tile
  // wg / 2); cluster pair: sub = 2 rank + wg % 2, channel half wg / 2.  wg is broadcast from lane 0 so that the compiler knows it is
  // warp-uniform: the wgmma issue branches on it, and a branch it cannot prove uniform makes ptxas serialize every wgmma of the kernel.
  const int wg = __shfl_sync(~0u, tid >> 7, 0), wt = tid & 127;
  const int tile = SPLIT == 2 ? crank : (wg >> 1);
  const int ch0 = SPLIT == 2 ? 16 * (wg >> 1) : 0;                  // my first channel
  const int row0 = 64 * (SPLIT == 2 ? 2 * crank + (wg & 1) : wg);   // first row of my subtile
  const int fr = row0 + 16 * (wt >> 5) + ((wt & 31) >> 2);          // my first row; the other is +8
  const int fc = 2 * (wt & 3);                                      // my first channel offset; the others are +1 and +8 jj, +8 jj + 1
  auto frow = [&](int e) { return fr + 8 * e; };                    // e = row of the fragment
  const uint32_t a_hi_s = smem_u32(a_hi), a_lo_s = smem_u32(a_lo), b_hi_s = smem_u32(b_hi), b_lo_s = smem_u32(b_lo);
  const bool two_tiles = N > 128;
  const int j = lane & 7, quarter = lane >> 3;
  const float* Uj = U + 4 * j;
  // the thread that feeds row `xrow`'s X k-step (one row per thread; the cluster pair feeds the rows of its own tile)
  const int xrow = SPLIT == 2 ? crank * 128 + tid : tid;
  const bool x_owner = (SPLIT == 2 ? tid < 128 : true) && xrow < N;
  uint32_t peer_U = 0;
  if constexpr (SPLIT == 2) peer_U = map_to_peer(U, (uint32_t)(crank ^ 1));
  // store two floats of a row into U -- and into the partner's U in the cluster-pair variant
  auto put_u = [&](int off, float2 v) {
    *reinterpret_cast<float2*>(U + off) = v;
    if constexpr (SPLIT == 2) st2_cluster(peer_U + (uint32_t)off * 4u, v);
  };
  // two channels (c, c+1) of a row -> panel 0 as fp16 hi / lo
  auto store_split2 = [&](int row, int c, float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    const float2 f = __half22float2(h);
    const int off = sw128(row, c);
    *reinterpret_cast<uint32_t*>(a_hi + off) = pack_h2(h);
    *reinterpret_cast<uint32_t*>(a_lo + off) = pack_h2(__floats2half2_rn(a - f.x, b - f.y));
  };
  // barrier that closes an epilogue / the window prologue: operand + U stores of everybody visible to the MMAs and the next gather
  auto close_phase = [&]() {
    fence_proxy_async();
    if constexpr (SPLIT == 2) cluster_sync_all(); else __syncthreads();
  };

  // Accumulators of my subtile.  GEMM 1: z in fragment columns [0, 8 NJ), r in [8 NJ, 16 NJ); GEMM 2: the candidate.  SPLIT 1 issues a
  // k-step as one m64n64 (B rows 0..63 = z | r) and one m64n32 (rows 64..95), the cluster pair as one m64n16 per gate.
  // Thread (warp w of the group, lane l) holds for fragment row e (row frow(e)) and channel ch0 + 8 jj + fc + x:
  //   z = acc1[4 jj + 2 e + x],  r = acc1[4 NJ + 4 jj + 2 e + x],  candidate = acc2[4 jj + 2 e + x]
  float acc1[8 * NJ], acc2[4 * NJ];
  // The 3 x 7 k-steps of one gemm are issued in three commit groups, each as soon as its k-steps are in shared memory:
  //   group 0: k-steps of H | H*R and X  -- complete when the round starts; its first MMA overwrites the accumulator
  //   group 1: k-steps of P_o H          -- after the last warp finished the tile's P_o tasks
  //   group 2: k-steps of P_i H          -- after the last warp finished the tile's P_i tasks
  // No MMA is skipped at run time (a wgmma under a branch ptxas cannot prove uniform is serialized): rows past N are issued too.  Their
  // operands are finite -- zeroed, or over-read from the buffer behind the panel -- and their results are never stored.
  auto issue_group = [&](int gm, int grp) {
    const int ks0 = grp == 0 ? 0 : (grp == 1 ? 2 : 4);
    wgmma_fence();
#pragma unroll
    for (int pass = 0; pass < 3; ++pass) {           // lo*hi, hi*lo, hi*hi (small terms first)
      const uint32_t ab = (pass == 0 ? a_lo_s : a_hi_s) + row0 * 128;
      const uint32_t bb = pass == 1 ? b_lo_s : b_hi_s;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        if (i == 2 && grp != 0) continue;
        const int ks = i == 2 ? 6 : ks0 + i;
        const int panel = ks >> 2, kin = (ks & 3) * 16;
        const uint32_t sc = (grp == 0 && pass == 0 && i == 0) ? 0u : 1u;
        const uint32_t bk = bb + panel * TC_PANEL_B + kin * 2;
        const uint64_t da = gmma_desc_sw128(ab + panel * TC_PANEL_A + kin * 2);
        if (gm == 1) {
          wgmma_f16<8 * NJ>(acc2, da, gmma_desc_sw128(bk + (64 + ch0) * 128), sc);
        } else if constexpr (NJ == 4) {
          wgmma_f16<64>(acc1, da, gmma_desc_sw128(bk), sc);
        } else {
          wgmma_f16<16>(*reinterpret_cast<float(*)[8]>(&acc1[0]), da, gmma_desc_sw128(bk + ch0 * 128), sc);
          wgmma_f16<16>(*reinterpret_cast<float(*)[8]>(&acc1[8]), da, gmma_desc_sw128(bk + (32 + ch0) * 128), sc);
        }
      }
    }
    wgmma_commit();
  };
  auto wait_gemm = [&](int gm) {
    wgmma_wait<0>();
    if (gm == 0) acc_fence(acc1); else acc_fence(acc2);
  };

  // this warp's warp-tasks of segment `seg` = (MMA tile of the destination rows) * 2 + operator: results -> A panels as fp16 hi/lo
  //   op 0 (P_o): panel 0 k 32..63        op 1 (P_i): panel 1 k 0..31
  auto gather_segment = [&](int seg) {
    const int ws = s_wstart[warp * 4 + seg], wc = s_wcount[warp * 4 + seg];
    const int op = seg & 1;
    unsigned char* dh = a_hi + (op ? TC_PANEL_A : 0);
    unsigned char* dl = a_lo + (op ? TC_PANEL_A : 0);
    const int kcol = (op ? 0 : 32) + 4 * j;
    for (int i = 0; i < wc; ++i) {
      const uint32_t d = s_wt[(ws + i) * 4 + quarter];
      if (d != kImgNoTask) {
        const float4 acc = gather_groups(Uj, s_idx, s_val, (int)(d >> 16), (int)((d >> 9) & 0x7f));
        store_split4(dh, dl, (int)(d & 0xff), kcol, acc);
      }
    }
  };
  // One gather round.  Every warpgroup issues the static group (H | X k-steps) of its tile right away (the block barrier in front of
  // the round ordered those operand stores), tile 0's warpgroups their P_o / P_i groups behind the barrier that closes tile 0's tasks,
  // and tile 1's warpgroups theirs behind the closing barrier.  The task
  // lists are balanced (graph_image.cuh), so the two barriers are cheap; the closing one also tells the epilogue that nobody reads U any more.
  auto gather_round = [&](int gm) {
    if constexpr (SPLIT == 2) {
      issue_group(gm, 0);
      if (p.n_ops > 0) gather_segment(2 * crank);
      if (p.n_ops > 1) gather_segment(2 * crank + 1);
      cluster_arrive_relaxed();   // this CTA has finished reading U (waited for by the partner before its epilogue overwrites my U)
      fence_proxy_async();
      __syncthreads();
      issue_group(gm, 1);
      issue_group(gm, 2);
      return;
    }
    issue_group(gm, 0);
    if (p.n_ops > 0) gather_segment(0);
    if (p.n_ops > 1) gather_segment(1);
    fence_proxy_async();        // my generic-proxy stores to the A panels -> visible to the tensor core (async proxy)
    __syncthreads();
    if (tile == 0) {
      issue_group(gm, 1);
      issue_group(gm, 2);
    }
    if (two_tiles) {
      if (p.n_ops > 0) gather_segment(2);
      if (p.n_ops > 1) gather_segment(3);
    }
    fence_proxy_async();
    __syncthreads();
    if (tile == 1) {
      issue_group(gm, 1);
      issue_group(gm, 2);
    }
  };
  // every MMA of the CTA has read the A panels (each is issued by the warpgroup of its subtile / channel quarter): only then are they
  // overwritten
  auto operands_free = [&]() {
    __syncthreads();
    if constexpr (SPLIT == 2) cluster_wait();       // the partner is done gathering from its U
  };

  auto x_base = [&](long long b) -> const float* { return p.x + (p.win_start ? p.win_start[b] * p.x_tstride : b * p.x_bstride); };
  // [X_t | P_o X_t | P_i X_t] of row xrow -> k 32..43 of panel 1 (weights of absent channels / operators are zero, but the
  // operand itself must be finite: everything not produced is written as 0 -- at store time, so the loads stay in flight)
  auto load_x = [&](const float* xb, long long b, int t, float4& xv, float4& po, float4& pi) {
    float xn[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int c = 0; c < CIN; ++c) xn[c] = __ldg(xb + t * p.x_tstride + xrow * CIN + c);
    xv = make_float4(xn[0], xn[1], xn[2], xn[3]);
    po = pi = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.ws) {             // per-CTA workspace rows [row][op][t*CIN + c]: rewritten every window, so they stay in L2
      const float* w0 = p.ws + (((long long)blockIdx.x * N + xrow) * 2) * p.ws_pitch + t * CIN;
      float a0[4] = {0.f, 0.f, 0.f, 0.f}, a1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int c = 0; c < CIN; ++c) {
        if (p.n_ops >= 1) a0[c] = w0[c];
        if (p.n_ops >= 2) a1[c] = w0[p.ws_pitch + c];
      }
      po = make_float4(a0[0], a0[1], a0[2], a0[3]);
      pi = make_float4(a1[0], a1[1], a1[2], a1[3]);
      return;
    }
    const float* sc = p.out + ((b * T + t) * (long long)N + xrow) * 32;  // parked there by the window prologue (plain loads:
    if (p.n_ops >= 1) po = *reinterpret_cast<const float4*>(sc);         //  written by this CTA earlier in this launch)
    if (p.n_ops >= 2) pi = *reinterpret_cast<const float4*>(sc + 4);
  };
  auto mask_c = [&](float4 v) {
    if (CIN < 4) v.w = 0.f;
    if (CIN < 3) v.z = 0.f;
    if (CIN < 2) v.y = 0.f;
    return v;
  };
  auto store_x = [&](const float4& xv, const float4& po, const float4& pi) {
    store_split4(a_hi + TC_PANEL_A, a_lo + TC_PANEL_A, xrow, 32, xv);
    store_split4(a_hi + TC_PANEL_A, a_lo + TC_PANEL_A, xrow, 36, mask_c(po));
    store_split4(a_hi + TC_PANEL_A, a_lo + TC_PANEL_A, xrow, 40, mask_c(pi));
  };

  for (long long b = cta; b < p.B; b += n_cta) {
    const float* xb = x_base(b);
    // ---- window prologue A: P_o X_t, P_i X_t for every step of the window, TCH steps per gather pass ------------------------
    if (p.n_ops) {
      constexpr int TCH = 32 / CIN;
      for (int t0 = 0; t0 < T; t0 += TCH) {
        const int tn = (T - t0) < TCH ? (T - t0) : TCH;
        const int F = tn * CIN, NC = N * CIN;
        // U[n][tt*CIN + c] = X[b, t0+tt, n, c]: all loads of a thread are issued before the first store (one HBM/L2 latency)
        for (int base = 0; base < tn * NC; base += 512 * 8) {
          float xv8[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const int idx = base + u * 512 + tid;
            xv8[u] = 0.f;
            if (idx < tn * NC) {
              const int tt = idx / NC, r = idx - tt * NC;
              xv8[u] = __ldg(xb + (long long)(t0 + tt) * p.x_tstride + r);
            }
          }
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const int idx = base + u * 512 + tid;
            if (idx < tn * NC) {
              const int tt = idx / NC, r = idx - tt * NC;
              const int n = r / CIN, c = r - n * CIN;
              U[n * TC_UP + tt * CIN + c] = xv8[u];
            }
          }
        }
        __syncthreads();
        for (int seg = SPLIT == 2 ? 2 * crank : 0; seg < (SPLIT == 2 ? 2 * crank + 2 : 4); ++seg) {
          const int ws = s_wstart[warp * 4 + seg], wc = s_wcount[warp * 4 + seg];
          for (int i = 0; i < wc; ++i) {
            const uint32_t d = s_wt[(ws + i) * 4 + quarter];
            if (d != kImgNoTask && 4 * j < F) {
              const float4 acc = gather_groups(Uj, s_idx, s_val, (int)(d >> 16), (int)((d >> 9) & 0x7f));
              const float av[4] = {acc.x, acc.y, acc.z, acc.w};
              const int drow = d & 0xff, op = (d >> 8) & 1;
              float* orow = p.out + ((b * T + t0) * (long long)N + drow) * 32 + op * 4;
              const long long tstep = (long long)N * 32;
              if (p.ws) {               // floats 4j..4j+3 of the row are consecutive (t, c) pairs: one 16-byte store, full sectors
                float* wrow = p.ws + (((long long)blockIdx.x * N + drow) * 2 + op) * p.ws_pitch + t0 * CIN + 4 * j;
                if (4 * j + 4 <= F) {
                  *reinterpret_cast<float4*>(wrow) = acc;
                } else {
#pragma unroll
                  for (int k = 0; k < 4; ++k)
                    if (4 * j + k < F) wrow[k] = av[k];
                }
              } else if (CIN == 2) {           // floats 4j..4j+3 = (t, c) = (2j,0) (2j,1) (2j+1,0) (2j+1,1): two 8-byte stores
                *reinterpret_cast<float2*>(orow + (2 * j) * tstep) = make_float2(av[0], av[1]);
                if (4 * j + 2 < F) *reinterpret_cast<float2*>(orow + (2 * j + 1) * tstep) = make_float2(av[2], av[3]);
              } else if (CIN == 4) {    // one timestep per lane: a 16-byte store
                *reinterpret_cast<float4*>(orow + j * tstep) = acc;
              } else {
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                  const int f = 4 * j + k;
                  if (f < F) {
                    const int tt = f / CIN, c = f - tt * CIN;
                    orow[tt * tstep + c] = av[k];
                  }
                }
              }
            }
          }
        }
        __syncthreads();
      }
    }
    // ---- window prologue B: H_0 into U (fp32) and the A panels (fp16 hi/lo); the X k-step of step 0 ---------------------------
    float hreg[NE][2 * NJ];     // [fragment row e][channel ch0 + 8 jj + fc + x at 2 jj + x]
    if constexpr (SPLIT == 2) {   // the partner has finished the X gather of its prologue: its U may be overwritten
      cluster_arrive_relaxed();
      cluster_wait();
    }
#pragma unroll
    for (int e = 0; e < NE; ++e) {
      const int row = frow(e);
#pragma unroll
      for (int jj = 0; jj < NJ; ++jj) {
        const int c = ch0 + 8 * jj + fc;
        float2 h = make_float2(0.f, 0.f);
        if (row < N && p.h0) h = __ldg(reinterpret_cast<const float2*>(p.h0 + b * p.h0_bstride + row * 32 + c));
        hreg[e][2 * jj] = h.x; hreg[e][2 * jj + 1] = h.y;
        if (row < N) {
          put_u(row * TC_UP + c, h);
          store_split2(row, c, h.x, h.y);
        }
      }
    }
    if (x_owner) {
      float4 xv, po, pi;
      load_x(xb, b, 0, xv, po, pi);
      store_x(xv, po, pi);
    }
    close_phase();             // the first MMA group of step 0 is issued right behind this barrier

    for (int t = 0; t < T; ++t) {
      // ---- round 1: diffuse H ------------------------------------------------------------------------------------------
      gather_round(0);
      // ---- epilogue 1: r gate; H*R ---------------------------------------------------------------------------------------
      wait_gemm(0);
      const long long obase = (b * T + t) * (long long)N;
      {
        float hr[NE][2 * NJ], rv[NE][2 * NJ];
#pragma unroll
        for (int e = 0; e < NE; ++e)
#pragma unroll
          for (int jj = 0; jj < NJ; ++jj)
#pragma unroll
            for (int x = 0; x < 2; ++x) {
              const float r = sigmoid_fast(acc1[4 * NJ + 4 * jj + 2 * e + x] + Bs[32 + ch0 + 8 * jj + fc + x]);
              hr[e][2 * jj + x] = hreg[e][2 * jj + x] * r;
              rv[e][2 * jj + x] = r;
            }
        operands_free();
#pragma unroll
        for (int e = 0; e < NE; ++e) {
          const int row = frow(e);
          if (row < N) {
#pragma unroll
            for (int jj = 0; jj < NJ; ++jj) {
              const int c = ch0 + 8 * jj + fc;
              put_u(row * TC_UP + c, make_float2(hr[e][2 * jj], hr[e][2 * jj + 1]));
              store_split2(row, c, hr[e][2 * jj], hr[e][2 * jj + 1]);
              if (p.stash)
                *reinterpret_cast<float2*>(p.stash + ((obase * 3) + row) * 32 + (long long)N * 32 + c) = make_float2(rv[e][2 * jj], rv[e][2 * jj + 1]);
            }
          }
        }
      }
      close_phase();
      // ---- round 2: re-diffuse H*R ---------------------------------------------------------------------------------------
      gather_round(1);
      // ---- epilogue 2: candidate, H_t --------------------------------------------------------------------------------------
      float4 xv, po, pi;
      const bool feed_x = x_owner && t + 1 < T;
      if (feed_x) load_x(xb, b, t + 1, xv, po, pi);      // in flight under the MMA wait
      wait_gemm(1);
      {
        // Z comes from its GEMM-1 accumulators, which stay in registers until the next step's GEMM 1
        float ht[NE][2 * NJ], zreg[NE][2 * NJ];
#pragma unroll
        for (int e = 0; e < NE; ++e)
#pragma unroll
          for (int jj = 0; jj < NJ; ++jj)
#pragma unroll
            for (int x = 0; x < 2; ++x) {
              const int c = ch0 + 8 * jj + fc + x, a = 4 * jj + 2 * e + x;
              const float z = sigmoid_fast(acc1[a] + Bs[c]);
              const float h = tanh_fast(acc2[a] + Bs[64 + c]);
              zreg[e][2 * jj + x] = z;
              ht[e][2 * jj + x] = h;
              hreg[e][2 * jj + x] = z * hreg[e][2 * jj + x] + (1.0f - z) * h;   // dcrnn.py:190-192
            }
        operands_free();
#pragma unroll
        for (int e = 0; e < NE; ++e) {
          const int row = frow(e);
          if (row < N) {
            float* op = p.out + (obase + row) * 32;
#pragma unroll
            for (int jj = 0; jj < NJ; ++jj) {
              const int c = ch0 + 8 * jj + fc;
              const float2 hv = make_float2(hreg[e][2 * jj], hreg[e][2 * jj + 1]);
              put_u(row * TC_UP + c, hv);
              *reinterpret_cast<float2*>(op + c) = hv;
              store_split2(row, c, hv.x, hv.y);
              if (p.stash) {
                float* sp = p.stash + ((obase * 3) + row) * 32;
                *reinterpret_cast<float2*>(sp + c) = make_float2(zreg[e][2 * jj], zreg[e][2 * jj + 1]);
                *reinterpret_cast<float2*>(sp + 2 * (long long)N * 32 + c) = make_float2(ht[e][2 * jj], ht[e][2 * jj + 1]);
              }
            }
          }
        }
        if (feed_x) store_x(xv, po, pi);
      }
      close_phase();
    }
  }
}

// ---- the one-CTA kernel: A operands from registers ----------------------------------------------------------------------
// Warpgroup wg owns MMA rows [64 wg, 64 wg + 64); the plan's row image (row_image.cuh) maps graph nodes onto these 256 positions so
// that the gather work is balanced.  Thread (warp w, lane l; quad = l / 4, q = l % 4) owns positions 16 w + quad (slot 0) and +8
// (slot 1) and, of every 32-channel block, the channels 8 jj + 2q (+1), jj = 0..3: exactly the (row, k) pairs of its m64nNk16 A
// fragment and of its accumulator fragment.  So it gathers the diffusion of its own two rows straight into A fragments (split into fp16
// hi / lo in registers) and applies the gates to the accumulators of the same rows; no operand goes through shared memory but B.
//
// Gather buffers U_H (H) and U_R (H*R): fp32 [256 positions][32], 128-byte rows without padding, channels permuted so that the 8
// channels of quad lane q sit in 32 contiguous bytes (float 8q + 2jj + x = channel 8jj + 2q + x): a lane reads a source row with
// two 16-byte loads, odd quads in the opposite order, so the two quads of a load phase touch disjoint banks whatever rows they read.
//
// Step:  round 1  gather P_o H of my rows -> issue the H | X and P_o k-steps -> gather P_i H while they run -> issue the P_i k-steps
//                 -> wait -> r, H*R -> U_R                                                                            barrier
//        round 2  the same over U_R (GEMM 2) -> z, candidate, H_t -> U_H, HBM                                         barrier
// Between the two barriers a warpgroup depends only on itself.  The k-steps of a gemm are issued in the order of the cluster kernel
// (k-steps 0, 1, 6, then 2, 3, then 4, 5, each pass-major lo*hi, hi*lo, hi*hi) and the gather sums the same entries in CSR order, so
// the outputs are bit-identical to it.
constexpr int RF_UBUF = kRiPos * 32;   // floats per gather buffer

// Measurement only, never set in a shipped build: -DSTMP_RF_OMIT=1 compiles the per-step gathers of k_dcrnn_seq_rf out (the
// diffusion fragments are zero), -DSTMP_RF_OMIT=2 its wgmmas (the gates read zero accumulators).  The results are wrong; the launch
// times of the two builds against the full one give the step's phase breakdown (DESIGN §4).
#ifndef STMP_RF_OMIT
#define STMP_RF_OMIT 0
#endif

// 8 floats of a row in fragment order (v[2jj + x] = channel 8jj + 2q + x) <-> the two 16-byte chunks 2q, 2q+1 of the row; `par`
// (quad parity) selects which chunk is touched first
__device__ __forceinline__ void rf_ld_row(const float* row, int q, int par, float (&v)[8]) {
  const float4 a = ld4(row + 4 * (2 * q + par)), b = ld4(row + 4 * (2 * q + 1 - par));
  const float4 lo = par ? b : a, hi = par ? a : b;
  v[0] = lo.x; v[1] = lo.y; v[2] = lo.z; v[3] = lo.w; v[4] = hi.x; v[5] = hi.y; v[6] = hi.z; v[7] = hi.w;
}
__device__ __forceinline__ void rf_st_row(float* row, int q, int par, const float (&v)[8]) {
  const float4 lo = make_float4(v[0], v[1], v[2], v[3]), hi = make_float4(v[4], v[5], v[6], v[7]);
  st4(row + 4 * (2 * q + par), par ? hi : lo);
  st4(row + 4 * (2 * q + 1 - par), par ? lo : hi);
}
// fp16 hi / lo of a pair (as store_split2)
__device__ __forceinline__ void rf_split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(a, b);
  const float2 f = __half22float2(h);
  hi = pack_h2(h);
  lo = pack_h2(__floats2half2_rn(a - f.x, b - f.y));
}
// A-fragment registers of the two k-steps of a 32-channel block that hold my fragment row e, from its values v in fragment order
__device__ __forceinline__ void rf_split_row(const float (&v)[8], int e, uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
#pragma unroll
  for (int s = 0; s < 2; ++s) {
    rf_split2(v[4 * s], v[4 * s + 1], hi[s][e], lo[s][e]);
    rf_split2(v[4 * s + 2], v[4 * s + 3], hi[s][2 + e], lo[s][2 + e]);
  }
}
// Weighted sum over one gather list (a (warp, operator, slot) of the row image) of the 8 floats of my quad lane: v in the order of
// the row's chunks 2q, 2q+1.  Four entries per group as gather_groups, the next group's entries fetched while the current one's rows
// are in flight; summation order = CSR order, products by FMA.
__device__ __forceinline__ void rf_gather(const float* __restrict__ Ub, const uint32_t* __restrict__ idx, const float4* __restrict__ val,
                                          int g0, int ng, int quad, int q, int par, float (&v)[8]) {
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
  const int cf = 4 * (2 * q + par), cs = 4 * (2 * q + 1 - par);
  const uint32_t* ix = idx + g0 * 8 + quad;
  const float4* vx = val + g0 * 8 + quad;
  uint32_t u = ix[0];
  float4 w = vx[0];
#pragma unroll 2
  for (int g = 1; g <= ng; ++g) {
    const uint32_t un = ix[8 * g];          // (one spare group row at the end of the arrays)
    const float4 wn = vx[8 * g];
    const float* r0 = Ub + (u & 0xffu) * 32;
    const float* r1 = Ub + ((u >> 8) & 0xffu) * 32;
    const float* r2 = Ub + ((u >> 16) & 0xffu) * 32;
    const float* r3 = Ub + (u >> 24) * 32;
    const float4 x0 = ld4(r0 + cf), y0 = ld4(r0 + cs);
    const float4 x1 = ld4(r1 + cf), y1 = ld4(r1 + cs);
    const float4 x2 = ld4(r2 + cf), y2 = ld4(r2 + cs);
    const float4 x3 = ld4(r3 + cf), y3 = ld4(r3 + cs);
    fma4(a, w.x, x0); fma4(b, w.x, y0);
    fma4(a, w.y, x1); fma4(b, w.y, y1);
    fma4(a, w.z, x2); fma4(b, w.z, y2);
    fma4(a, w.w, x3); fma4(b, w.w, y3);
    u = un;
    w = wn;
  }
  const float4 lo = par ? b : a, hi = par ? a : b;
  v[0] = lo.x; v[1] = lo.y; v[2] = lo.z; v[3] = lo.w; v[4] = hi.x; v[5] = hi.y; v[6] = hi.z; v[7] = hi.w;
}

template <int CIN>
__global__ void __launch_bounds__(512, 1) k_dcrnn_seq_rf(const TcParams p) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int N = p.N, T = p.T;
  unsigned char* b_hi = smem + p.off_B;
  unsigned char* b_lo = b_hi + 2 * TC_PANEL_B;
  float* UH = reinterpret_cast<float*>(smem + p.off_U);
  float* UR = UH + RF_UBUF;
  unsigned char* img = smem + p.off_img;
  int16_t* s_perm = reinterpret_cast<int16_t*>(img + kRiOffPerm);
  const uint8_t* s_ipos = img + kRiOffIpos;
  const uint16_t* s_gstart = reinterpret_cast<const uint16_t*>(img + kRiOffGstart);
  const uint16_t* s_gcount = reinterpret_cast<const uint16_t*>(img + kRiOffGcount);
  const uint32_t* s_idx = reinterpret_cast<const uint32_t*>(img + kRiOffIdx);
  const float4* s_val = reinterpret_cast<const float4*>(img + p.rl.off_val);
  float* Bs = reinterpret_cast<float*>(smem + p.off_bias);
  uint64_t* tma_bar = reinterpret_cast<uint64_t*>(smem + p.off_bar);
  if (blockIdx.x >= p.B) return;

  // ---- one-time per CTA ------------------------------------------------------------------------------------
  if (tid == 0) {
    mbar_init(tma_bar, 1);
    fence_mbar_init();
    const uint32_t tx = (p.rimg ? (uint32_t)p.rl.bytes : 0u) + (p.wimage ? (uint32_t)TC_WIMAGE_BYTES : 0u);
    if (tx) {
      mbar_arrive_expect_tx(tma_bar, tx);
      if (p.rimg) tma_bulk_g2s(img, p.rimg, (uint32_t)p.rl.bytes, tma_bar);
      if (p.wimage) {
        tma_bulk_g2s(b_hi, p.wimage, 4u * TC_PANEL_B, tma_bar);
        tma_bulk_g2s(Bs, reinterpret_cast<const unsigned char*>(p.wimage) + 4 * TC_PANEL_B, 96u * 4u, tma_bar);
      }
    }
  }
  {  // zero both gather buffers (the rows of empty positions stay zero for good); B too unless the TMA image overwrites it
    for (int i = tid; i < 2 * RF_UBUF; i += 512) UH[i] = 0.f;
    if (!p.wimage) {
      uint4* z = reinterpret_cast<uint4*>(b_hi);
      for (int i = tid; i < 4 * TC_PANEL_B / 16; i += 512) z[i] = make_uint4(0, 0, 0, 0);
    }
    if (!p.rimg)   // no operator: the identity map
      for (int i = tid; i < kRiPos; i += 512) s_perm[i] = (int16_t)(i < N ? i : -1);
  }
  __syncthreads();
  if (!p.wimage) {
    for (int idx = tid; idx < 96 * 112; idx += 512) {
      const int n = idx / 112, kk = idx - n * 112;
      const float v = tc_weight_value(p.wcat, p.w[0], p.w[1], p.w[2], CIN, n, kk);
      const __half h = __float2half_rn(v);
      const __half l = __float2half_rn(v - __half2float(h));
      const int off = (kk >> 6) * TC_PANEL_B + sw128(n, kk & 63);
      *reinterpret_cast<__half*>(b_hi + off) = h;
      *reinterpret_cast<__half*>(b_lo + off) = l;
    }
    for (int idx = tid; idx < 96; idx += 512) {
      const int gte = idx >> 5;
      const float* bg = gte == 0 ? p.bias[0] : (gte == 1 ? p.bias[1] : p.bias[2]);
      Bs[idx] = p.bcat ? p.bcat[idx] : (bg ? bg[idx & 31] : 0.f);
    }
  }
  if (p.rimg || p.wimage) mbar_wait(tma_bar, 0);
  fence_proxy_async();
  __syncthreads();

  const int quad = lane >> 2, q = lane & 3, par = quad & 1;
  const int pos[2] = {16 * warp + quad, 16 * warp + quad + 8};   // my MMA rows (fragment slots 0, 1)
  // graph node of my fragment row e (-1: empty), re-read where it is used: a register held across the step costs more
  auto node_of = [&](int e) -> int { return s_perm[pos[e]]; };
  const uint32_t b_hi_s = smem_u32(b_hi), b_lo_s = smem_u32(b_lo);

  // Accumulators: GEMM 1 z in [0, 16), r in [16, 32); GEMM 2 the candidate.  Value of fragment row e, channel 8jj + 2q + x at
  // 4jj + 2e + x (+16 for r).
  float acc1[32], acc2[16];
  if (STMP_RF_OMIT == 2) {
#pragma unroll
    for (int i = 0; i < 32; ++i) acc1[i] = 0.f;
#pragma unroll
    for (int i = 0; i < 16; ++i) acc2[i] = 0.f;
  }
  // A fragments, [k-step of the block][register]: H | H*R (k-steps 0, 1), P_o (2, 3), P_i (4, 5); X (k-step 6)
  uint32_t aH_hi[2][4], aH_lo[2][4], aO_hi[2][4], aO_lo[2][4], aI_hi[2][4], aI_lo[2][4], aX_hi[4], aX_lo[4];

  auto mma = [&](int gm, int ks, int pass, const uint32_t (&a)[4]) {
    if (STMP_RF_OMIT == 2) return;
    const uint32_t bb = pass == 1 ? b_lo_s : b_hi_s;
    const uint32_t bk = bb + (ks >> 2) * TC_PANEL_B + (ks & 3) * 32;
    const bool first = ks == 0 && pass == 0;   // overwrites the accumulator
    if (gm == 1) {
      if (first) wgmma_f16_rs_n32_first(acc2, a, gmma_desc_sw128(bk + 64 * 128));
      else wgmma_f16_rs_n32(acc2, a, gmma_desc_sw128(bk + 64 * 128), 1u);
    } else {
      if (first) wgmma_f16_rs_n64_first(acc1, a, gmma_desc_sw128(bk));
      else wgmma_f16_rs_n64(acc1, a, gmma_desc_sw128(bk), 1u);
    }
  };
  // k-steps 0, 1, 6 (H | H*R, X) and 2, 3 (P_o), each group pass-major: lo*hi, hi*lo, hi*hi
  auto issue_hxo = [&](int gm) {
    wgmma_fence();
#pragma unroll
    for (int pass = 0; pass < 3; ++pass) {
      mma(gm, 0, pass, pass == 0 ? aH_lo[0] : aH_hi[0]);
      mma(gm, 1, pass, pass == 0 ? aH_lo[1] : aH_hi[1]);
      mma(gm, 6, pass, pass == 0 ? aX_lo : aX_hi);
    }
#pragma unroll
    for (int pass = 0; pass < 3; ++pass) {
      mma(gm, 2, pass, pass == 0 ? aO_lo[0] : aO_hi[0]);
      mma(gm, 3, pass, pass == 0 ? aO_lo[1] : aO_hi[1]);
    }
    wgmma_commit();
  };
  auto issue_i = [&](int gm) {
    wgmma_fence();
#pragma unroll
    for (int pass = 0; pass < 3; ++pass) {
      mma(gm, 4, pass, pass == 0 ? aI_lo[0] : aI_hi[0]);
      mma(gm, 5, pass, pass == 0 ? aI_lo[1] : aI_hi[1]);
    }
    wgmma_commit();
  };
  // diffusion by operator `op` of my two rows from gather buffer Ub -> A fragments (zero when the operator is absent)
  auto gather_op = [&](const float* Ub, int op, uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float v[8];
      if (STMP_RF_OMIT != 1 && p.n_ops > op) {
        rf_gather(Ub, s_idx, s_val, s_gstart[ri_list(warp, op, e)], s_gcount[ri_list(warp, op, e)], quad, q, par, v);
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = 0.f;
      }
      rf_split_row(v, e, hi, lo);
    }
  };

  auto x_base = [&](long long b) -> const float* { return p.x + (p.win_start ? p.win_start[b] * p.x_tstride : b * p.x_bstride); };
  // My values of the X k-step (k = X c0..3 | P_o X c0..3 | P_i X c0..3 | 0): k 2q, 2q+1 -> xr[4e], xr[4e+1]; k 8+2q, 9+2q ->
  // xr[4e+2], xr[4e+3] (fragment row e).  Absent channels / operators and empty rows are 0 (the weights there are zero, the operand
  // must be finite).
  auto load_x = [&](const float* xb, long long b, int t, float (&xr)[8]) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int n = node_of(e);
#pragma unroll
      for (int x = 0; x < 2; ++x) {
        const int c = 2 * (q & 1) + x;
        float va = 0.f, vb = 0.f;
        if (n >= 0 && c < CIN) {
          auto ld_p = [&](int op) -> float {     // P_op X_t of row n, channel c: workspace or the parked output row
            if (p.ws) return p.ws[(((long long)blockIdx.x * N + n) * 2 + op) * p.ws_pitch + t * CIN + c];
            return p.out[((b * T + t) * (long long)N + n) * 32 + op * 4 + c];
          };
          if (q < 2) {
            va = __ldg(xb + t * p.x_tstride + n * CIN + c);
            if (p.n_ops >= 2) vb = ld_p(1);
          } else if (p.n_ops >= 1) {
            va = ld_p(0);
          }
        }
        xr[4 * e + x] = va;
        xr[4 * e + 2 + x] = vb;
      }
    }
  };
  auto split_x = [&](const float (&xr)[8]) {
    rf_split2(xr[0], xr[1], aX_hi[0], aX_lo[0]);
    rf_split2(xr[4], xr[5], aX_hi[1], aX_lo[1]);
    rf_split2(xr[2], xr[3], aX_hi[2], aX_lo[2]);
    rf_split2(xr[6], xr[7], aX_hi[3], aX_lo[3]);
  };

  for (long long b = blockIdx.x; b < p.B; b += gridDim.x) {
    const float* xb = x_base(b);
    // ---- window prologue A: P_o X_t, P_i X_t for every step of the window, TCH steps per gather pass (rows of T*Cin floats in U_R)
    if (p.n_ops) {
      constexpr int TCH = 32 / CIN;
      for (int t0 = 0; t0 < T; t0 += TCH) {
        const int tn = (T - t0) < TCH ? (T - t0) : TCH;
        const int F = tn * CIN, NC = N * CIN;
        for (int base = 0; base < tn * NC; base += 512 * 8) {
          float xv8[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const int idx = base + u * 512 + tid;
            xv8[u] = 0.f;
            if (idx < tn * NC) {
              const int tt = idx / NC, r = idx - tt * NC;
              xv8[u] = __ldg(xb + (long long)(t0 + tt) * p.x_tstride + r);
            }
          }
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            const int idx = base + u * 512 + tid;
            if (idx < tn * NC) {
              const int tt = idx / NC, r = idx - tt * NC;
              const int n = r / CIN, c = r - n * CIN;
              UR[s_ipos[n] * 32 + tt * CIN + c] = xv8[u];
            }
          }
        }
        __syncthreads();
        for (int op = 0; op < p.n_ops; ++op)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float v[8];   // floats 8q .. 8q+7 of the row = (t, c) pairs in order
            rf_gather(UR, s_idx, s_val, s_gstart[ri_list(warp, op, e)], s_gcount[ri_list(warp, op, e)], quad, q, par, v);
            const int n = node_of(e);
            if (n < 0 || 8 * q >= F) continue;
            if (p.ws) {
              float* wrow = p.ws + (((long long)blockIdx.x * N + n) * 2 + op) * p.ws_pitch + t0 * CIN + 8 * q;
              if (CIN != 3 && 8 * q + 8 <= F) {      // 16-byte aligned: t0 * CIN is a multiple of 32 for CIN = 1, 2, 4
                st4(wrow, make_float4(v[0], v[1], v[2], v[3]));
                st4(wrow + 4, make_float4(v[4], v[5], v[6], v[7]));
              } else {
#pragma unroll
                for (int k = 0; k < 8; ++k)
                  if (8 * q + k < F) wrow[k] = v[k];
              }
            } else {
#pragma unroll
              for (int k = 0; k < 8; ++k) {
                const int f = 8 * q + k;
                if (f < F) {
                  const int tt = f / CIN, c = f - tt * CIN;
                  p.out[((b * T + t0 + tt) * (long long)N + n) * 32 + op * 4 + c] = v[k];
                }
              }
            }
          }
        __syncthreads();
      }
    }
    // ---- window prologue B: H_0 into U_H and the A fragments; the X k-step of step 0 -----------------------------------------
    {
      float hv[2][8];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = node_of(e);
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          float2 h = make_float2(0.f, 0.f);
          if (n >= 0 && p.h0) h = __ldg(reinterpret_cast<const float2*>(p.h0 + b * p.h0_bstride + n * 32 + 8 * jj + 2 * q));
          hv[e][2 * jj] = h.x; hv[e][2 * jj + 1] = h.y;
        }
        if (n >= 0) rf_st_row(UH + pos[e] * 32, q, par, hv[e]);
        rf_split_row(hv[e], e, aH_hi, aH_lo);
      }
      float xr[8];
      load_x(xb, b, 0, xr);
      split_x(xr);
    }
    __syncthreads();

    for (int t = 0; t < T; ++t) {
      const long long obase = (b * T + t) * (long long)N;
      // ---- round 1: diffuse H (GEMM 1: z | r) -----------------------------------------------------------------------------
      gather_op(UH, 0, aO_hi, aO_lo);
      issue_hxo(0);
      gather_op(UH, 1, aI_hi, aI_lo);
      issue_i(0);
      wgmma_wait<0>();
      acc_fence(acc1);
      // ---- epilogue 1: r gate; H*R -> U_R and the A fragments of round 2 --------------------------------------------------
      {
        float hr[2][8];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float h[8];
          rf_ld_row(UH + pos[e] * 32, q, par, h);
          float rv[8];
#pragma unroll
          for (int jj = 0; jj < 4; ++jj)
#pragma unroll
            for (int x = 0; x < 2; ++x) {
              const float r = sigmoid_fast(acc1[16 + 4 * jj + 2 * e + x] + Bs[32 + 8 * jj + 2 * q + x]);
              hr[e][2 * jj + x] = h[2 * jj + x] * r;
              rv[2 * jj + x] = r;
            }
          const int n = node_of(e);
          if (n >= 0) {
            rf_st_row(UR + pos[e] * 32, q, par, hr[e]);
            if (p.stash)
#pragma unroll
              for (int jj = 0; jj < 4; ++jj)
                *reinterpret_cast<float2*>(p.stash + ((obase * 3) + n) * 32 + (long long)N * 32 + 8 * jj + 2 * q) =
                    make_float2(rv[2 * jj], rv[2 * jj + 1]);
          }
          rf_split_row(hr[e], e, aH_hi, aH_lo);
        }
      }
      __syncthreads();   // U_R complete
      // ---- round 2: re-diffuse H*R (GEMM 2: candidate) ----------------------------------------------------------------------
      gather_op(UR, 0, aO_hi, aO_lo);
      issue_hxo(1);
      gather_op(UR, 1, aI_hi, aI_lo);
      issue_i(1);
      wgmma_wait<0>();
      acc_fence(acc2);
      // ---- epilogue 2: candidate, H_t -> U_H, HBM and the A fragments of the next step ----------------------------------------
      {
        float hn[2][8];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float h[8], zv[8], ht[8];
          rf_ld_row(UH + pos[e] * 32, q, par, h);
#pragma unroll
          for (int jj = 0; jj < 4; ++jj)
#pragma unroll
            for (int x = 0; x < 2; ++x) {
              const int c = 8 * jj + 2 * q + x, a = 4 * jj + 2 * e + x;
              const float z = sigmoid_fast(acc1[a] + Bs[c]);
              const float hc = tanh_fast(acc2[a] + Bs[64 + c]);
              zv[2 * jj + x] = z;
              ht[2 * jj + x] = hc;
              hn[e][2 * jj + x] = z * h[2 * jj + x] + (1.0f - z) * hc;   // dcrnn.py:190-192
            }
          const int n = node_of(e);
          if (n >= 0) {
            rf_st_row(UH + pos[e] * 32, q, par, hn[e]);
            float* op = p.out + (obase + n) * 32;
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int c = 8 * jj + 2 * q;
              *reinterpret_cast<float2*>(op + c) = make_float2(hn[e][2 * jj], hn[e][2 * jj + 1]);
              if (p.stash) {
                float* sp = p.stash + ((obase * 3) + n) * 32;
                *reinterpret_cast<float2*>(sp + c) = make_float2(zv[2 * jj], zv[2 * jj + 1]);
                *reinterpret_cast<float2*>(sp + 2 * (long long)N * 32 + c) = make_float2(ht[2 * jj], ht[2 * jj + 1]);
              }
            }
          }
          rf_split_row(hn[e], e, aH_hi, aH_lo);
        }
        if (t + 1 < T) {   // the X k-step of the next step (loaded here: held across the gate math, the values spill)
          float xr[8];
          load_x(xb, b, t + 1, xr);
          split_x(xr);
        }
      }
      __syncthreads();   // U_H complete
    }
  }
}

// shared-memory layout of the one-CTA kernel for `n_ops` operators of `plan`
bool rf_layout(const stmp_plan* plan, int n_ops, TcParams* p, int* smem_bytes) {
  int off = 0;
  p->off_B = off; off += 4 * TC_PANEL_B;
  p->off_U = off; off += 2 * RF_UBUF * 4;
  p->rl = row_image_layout(n_ops && plan ? plan->rimg_groups[n_ops] : 0);
  p->off_img = off; off += p->rl.bytes;
  p->off_bias = off; off += 96 * 4;
  p->off_bar = off; off += 8;
  *smem_bytes = off;
  return off <= kMaxSmemTc;
}

// shared-memory layout of the cluster-pair kernel for `n_ops` operators of `plan`
bool tc_layout(const stmp_plan* plan, int n_ops, TcParams* p, int* smem_bytes) {
  int off = 0;
  p->off_A = off; off += 4 * TC_PANEL_A;
  p->off_B = off; off += 4 * TC_PANEL_B;
  p->off_U = off; off += TC_UROWS * TC_UP * 4;
  int nnz = 0;
  for (int op = 0; op < n_ops; ++op) nnz += plan->fwd[op].nnz;
  p->gl = graph_image_layout(n_ops * plan->n, nnz);
  p->off_img = off; off += n_ops ? p->gl.bytes : 0;
  p->off_bias = off; off += 96 * 4;
  p->off_bar = off; off += 8;
  *smem_bytes = off;
  return off <= kMaxSmemTc;
}

}  // namespace

// bytes of shared memory the kernel has left for a graph image: the plan builds no image larger than this (it could never be used)
int tc_graph_image_budget() {
  stmp_plan none;                           // no operators: tc_layout lays out everything but the image
  TcParams p;
  int smem = 0;
  tc_layout(&none, 0, &p, &smem);
  return kMaxSmemTc - smem;
}
// the same for the row image of the one-CTA kernel
int tc_row_image_budget() {
  TcParams p;
  int smem = 0;
  rf_layout(nullptr, 0, &p, &smem);       // lays out the image of no group rows
  return kMaxSmemTc - smem + p.rl.bytes;
}

int tc_ws_pitch(long long T, long long cin) { return (int)((T * cin + 7) / 8 * 8); }   // floats per (row, operator): whole 32-byte sectors

long long tc_workspace_bytes(const stmp_plan* plan, long long T, long long cin) {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return (long long)sms * plan->n * 2 * tc_ws_pitch(T, cin) * 4;
}

static bool tc_fits(const stmp_plan* plan, int n_ops) {
  if (!plan || plan->n > kImgMaxN || plan->n < 1) return false;
  if (n_ops > 0 && (!plan->gimg[n_ops] || !plan->rimg[n_ops])) return false;   // no image: graph too large / too dense
  TcParams p;
  int smem = 0;
  return tc_layout(plan, n_ops, &p, &smem) && rf_layout(plan, n_ops, &p, &smem);
}

bool gru_tc_supported(const stmp_plan* plan, long long cin, int n_ops) {
  if (!plan || cin < 1 || cin > 4 || n_ops < 0 || n_ops > 2 || n_ops > plan->n_ops) return false;
  return tc_fits(plan, n_ops);
}

bool dcrnn_tc_supported(const stmp_plan* plan, long long cin, long long cout, long long K) {
  if (!plan || plan->flavor != STMP_FLAVOR_DCONV || plan->n_ops != 2) return false;
  if (K != 2 || cout != 32 || cin < 1 || cin > 4) return false;
  return tc_fits(plan, 2);
}

static int tc_launch_params(const stmp_plan* plan, TcParams& p, cudaStream_t st);

int dcrnn_tc_launch(const stmp_plan* plan, long long B, long long T, long long cin, const float* x, const long long* win_start,
                    long long x_bstride, long long x_tstride, const float* w_z, const float* w_r, const float* w_h, const float* b_z,
                    const float* b_r, const float* b_h, const float* h0, float* out, float* stash, const void* wimage,
                    void* workspace, cudaStream_t st) {
  TcParams p;
  p.N = plan->n; p.CIN = (int)cin; p.T = (int)T; p.B = B;
  p.x = x; p.win_start = win_start; p.x_bstride = x_bstride; p.x_tstride = x_tstride;
  p.w[0] = w_z; p.w[1] = w_r; p.w[2] = w_h; p.bias[0] = b_z; p.bias[1] = b_r; p.bias[2] = b_h;
  p.h0 = h0; p.h0_bstride = (long long)plan->n * 32; p.wcat = nullptr; p.bcat = nullptr; p.n_ops = 2;
  p.out = out; p.stash = stash; p.wimage = wimage; p.ws = reinterpret_cast<float*>(workspace);
  return tc_launch_params(plan, p, st);
}

// generic graph-GRU: prepacked weights, any plan flavor with >= n_ops operators
int gru_tc_launch(const stmp_plan* plan, int n_ops, long long B, long long T, long long cin, const float* x, const long long* win_start,
                  long long x_bstride, long long x_tstride, const float* wcat, const float* bcat, const float* h0, long long h0_bstride,
                  float* out, float* stash, const void* wimage, void* workspace, cudaStream_t st) {
  TcParams p;
  p.N = plan->n; p.CIN = (int)cin; p.T = (int)T; p.B = B;
  p.x = x; p.win_start = win_start; p.x_bstride = x_bstride; p.x_tstride = x_tstride;
  for (int i = 0; i < 3; ++i) { p.w[i] = nullptr; p.bias[i] = nullptr; }
  p.h0 = h0; p.h0_bstride = h0_bstride; p.wcat = wcat; p.bcat = bcat; p.n_ops = n_ops;
  p.out = out; p.stash = stash; p.wimage = wimage; p.ws = reinterpret_cast<float*>(workspace);
  return tc_launch_params(plan, p, st);
}

static int tc_launch_params(const stmp_plan* plan, TcParams& p, cudaStream_t st) {
  int smem = 0;
  const long long B = p.B;
  int dev = 0, sms = 0;
  STMP_CUDA_OK(cudaGetDevice(&dev));
  STMP_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  // small batches: a CTA pair (thread-block cluster) per window when both tiles exist and 2 B CTAs fit the machine
  const bool split = g_fwd_split != 0 && plan->n > 128 && 2 * B <= sms;
  const int grid = split ? (int)(2 * B) : (int)(B < sms ? B : sms);
  if (!(split ? tc_layout(plan, p.n_ops, &p, &smem) : rf_layout(plan, p.n_ops, &p, &smem)))
    return set_error(STMP_EUNSUPPORTED, "tensor-core graph-GRU kernel needs %d B of shared memory", smem);
  p.gimg = p.n_ops && split ? plan->gimg[p.n_ops] : nullptr;
  p.rimg = p.n_ops && !split ? plan->rimg[p.n_ops] : nullptr;
  if (p.n_ops && !(split ? p.gimg : p.rimg))
    return set_error(STMP_EUNSUPPORTED, "tensor-core graph-GRU kernel: the plan has no shared-memory graph image");
  p.ws_pitch = tc_ws_pitch(p.T, p.CIN);
  switch (p.CIN) {
#define STMP_TC_CASE(C)                                                                                              \
  case C:                                                                                                            \
    if (split) {                                                                                                     \
      STMP_CUDA_OK(cudaFuncSetAttribute(k_dcrnn_seq_tc<C, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));   \
      cudaLaunchConfig_t cfg = {};                                                                                   \
      cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(512); cfg.dynamicSmemBytes = (size_t)smem; cfg.stream = st; \
      cudaLaunchAttribute at[1];                                                                                     \
      at[0].id = cudaLaunchAttributeClusterDimension;                                                                \
      at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;                            \
      cfg.attrs = at; cfg.numAttrs = 1;                                                                              \
      STMP_CUDA_OK(cudaLaunchKernelEx(&cfg, k_dcrnn_seq_tc<C, 2>, p));                                               \
    } else {                                                                                                         \
      STMP_CUDA_OK(cudaFuncSetAttribute(k_dcrnn_seq_rf<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));      \
      k_dcrnn_seq_rf<C><<<grid, 512, smem, st>>>(p);                                                                 \
    }                                                                                                                \
    break;
    STMP_TC_CASE(1) STMP_TC_CASE(2) STMP_TC_CASE(3) STMP_TC_CASE(4)
#undef STMP_TC_CASE
    default: return set_error(STMP_EUNSUPPORTED, "tensor-core graph-GRU kernel: cin %d not in 1..4", p.CIN);
  }
  STMP_LAUNCH_OK("k_dcrnn_seq_tc");
  if (split) { static const int slot2 = path_slot("k_dcrnn_seq_tc[cluster2]"); count_path(slot2); }
  return STMP_OK;
}

int tc_pack_weight_image(const float* wcat, const float* bcat, const float* w0, const float* w1, const float* w2, const float* b0,
                         const float* b1, const float* b2, int cin, void* image, cudaStream_t st) {
  const int total = 96 * 128 + 96;
  k_pack_weight_image<<<(total + 255) / 256, 256, 0, st>>>(wcat, bcat, w0, w1, w2, b0, b1, b2, cin, reinterpret_cast<unsigned char*>(image));
  STMP_LAUNCH_OK("k_pack_weight_image");
  return STMP_OK;
}
int tc_weight_image_bytes() { return TC_WIMAGE_BYTES; }

}  // namespace stmp
