// tgcn_attn.cu -- fused temporal-attention + GCN-GRU kernel: A3TGCN / A3TGCN2 (and a TGCN / TGCN2 cell as the one-period case)
// for graphs of ANY size (the wgmma graph-GRU kernel stops at 207 nodes; PEMS-BAY has 325).
//
// Reference (nn/recurrent/attentiontemporalgcn.py:130-157, temporalgcn.py:187-233): for every period t
//     G_g = GCNConv_g(X[..., t])            three GCNConvs = gcn_norm + Linear(in,out) + propagate over `out` channels
//     Z = sigma(L_z [G_z | H]),  R = sigma(L_r [G_r | H]),  H~ = tanh(L_h [G_h | H*R]),  H_t = Z*H + (1-Z)*H~
//     out += softmax(attention)[t] * H_t                                     (the SAME H enters every period)
// Because A^(X W) = (A^ X) W the graph part only ever touches the `in` channels: one gather per node yields A^X for ALL
// periods at once (a row of in*periods floats: lane = (feature, period)), and GCNConv's Linear and the gate Linear fold into
//     pre_g = (A^X_t) A_g + H' B_g + c_g          A_g (in x out), B_g (out x out), c_g (out)   [host: TGCN._packed3]
// One warp per (batch row, node), lane = output channel.  H' B is an out x out mat-vec per node with the weight column in
// registers and H' handed round by shuffles; H B_z, H B_r are shared by all periods, only (H*R_t) B_h is per period.
// X[b] (N x in*periods floats, 31 KB at the PEMS-BAY shape) is staged into shared memory with ONE TMA bulk copy per CTA; the
// gather then runs out of shared memory.  Output and nothing else goes back to HBM: algorithmic bytes per (row, node) =
// 4*in*periods (X) + 4*out (H) + 4*out (out).
//
// 64 hidden channels (the *_wide_* entries): lane l owns channels l and l + 32 (NC = 2, as in gru_rows.cu / lstm_rows.cu).  A 64 x 192
// column of Bm would be 384 floats per lane, so the forward stages Bm in shared memory at pitch kWideBmLd next to the staged X, and the
// cell backward writes the per-row gate gradients and the two bases [A^X | H], [A^X | H*R] for the 64-wide weight-gradient contraction of
// rows.cuh instead of holding 384 dBm accumulators per lane.  The H = None backward is the 32-wide kernel templated on NC.
#include <cuda_runtime.h>

#include "common.cuh"
#include "rows.cuh"

namespace stmp {
namespace {

struct TgcnArgs {
  const int* rowptr;
  const int2* cv;
  int N, FIN, P, FP;      // FP = FIN * P floats per node of X[b]
  long long B;
  const float* x;         // [B][N][FIN][P] contiguous
  const float* h;         // [B][N][CO] (h_bstride) or null;  CO = 32 (k_tgcn_attn) or 64 (k_tgcn_wide_attn)
  long long h_bstride;
  const float* A;         // [FIN][3 CO]   columns z | r | h
  const float* Bm;        // [CO][3 CO]
  const float* c;         // [3 CO]
  const float* probs;     // [P] or null (one period, weight 1)
  float* out;             // [B][N][CO]
  int stage;              // 1: X[b] staged in shared memory by TMA; 0: gathered from global memory (huge graphs)
};

__device__ __forceinline__ float sigmoid_f(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }
__device__ __forceinline__ float tanh_f(float x) { return 2.0f * __fdividef(1.0f, 1.0f + __expf(-2.0f * x)) - 1.0f; }

constexpr int kNodesPerBlock = 64;

// Thread 0 starts ONE TMA bulk copy of X[b] into shared memory; the CTA waits for it with __syncthreads() + mbar_wait(bar, 0).
__device__ __forceinline__ void stage_x_begin(uint64_t* bar, float* Xs, const float* xb, uint32_t bytes) {
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(bar, bytes);
    tma_bulk_g2s(Xs, xb, bytes, bar);
  }
}

// A^X of node n for all periods, in the reference's edge order: lane holds entries (q*32 + lane) of the node's FP-float row of X[b]
// (Xg: shared memory when staged, global memory otherwise).
template <int NQ>
__device__ __forceinline__ void gather_ax(const int* rowptr, const int2* cv, const float* Xg, int FP, int stage, int n, int lane,
                                          float (&ax)[NQ]) {
#pragma unroll
  for (int q = 0; q < NQ; ++q) ax[q] = 0.f;
  const int beg = __ldg(rowptr + n), end = __ldg(rowptr + n + 1);
  for (int k = beg; k < end; ++k) {
    const int2 e = __ldg(cv + k);
    const float w = __int_as_float(e.y);
    const float* xr = Xg + (long long)e.x * FP;
#pragma unroll
    for (int q = 0; q < NQ; ++q)
      if (q * 32 + lane < FP) ax[q] = __fadd_rn(ax[q], __fmul_rn(w, stage ? xr[q * 32 + lane] : __ldg(xr + q * 32 + lane)));
  }
}

// Sum of column i of `parts` per-CTA partials (row length `width`) in a fixed association: warp w sums its contiguous share of the
// partials, then the 8 sub-sums are added in warp order.  Valid in warp 0 only; i may depend on the lane only.  A warp's share is
// summed with Kahan compensation: at 65 535 batch rows a share is 8 192 partials, and a plain running sum lost ~3e-6 of the total.
__device__ __forceinline__ float sum_partials(int parts, int width, const float* __restrict__ partial, int i, float (&sub)[8][32]) {
  const int x = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int per = (parts + 7) / 8, q0 = w * per, q1 = (q0 + per < parts) ? q0 + per : parts;
  float s = 0.f, comp = 0.f;
  if (i < width)
    for (int q = q0; q < q1; ++q) {
      const float y = __fsub_rn(partial[(size_t)q * width + i], comp);
      const float t = __fadd_rn(s, y);
      comp = __fsub_rn(__fsub_rn(t, s), y);
      s = t;
    }
  sub[w][x] = s;
  __syncthreads();
  float t = sub[0][x];
#pragma unroll
  for (int k = 1; k < 8; ++k) t += sub[k][x];
  return t;
}

template <int NQ, bool HAS_H>
__global__ void __launch_bounds__(256) k_tgcn_attn(const TgcnArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* Xs = reinterpret_cast<float*>(smem_raw);
  __shared__ __align__(8) uint64_t bar;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long b = blockIdx.y;
  const int n0 = blockIdx.x * kNodesPerBlock;
  const float* xb = a.x + b * (long long)a.N * a.FP;
  if (a.stage) stage_x_begin(&bar, Xs, xb, (uint32_t)a.N * a.FP * 4u);
  // weights of my output channel (lane) while the copy is in flight
  float Az[4], Ar[4], Ah[4];
#pragma unroll
  for (int f = 0; f < 4; ++f) {
    Az[f] = f < a.FIN ? __ldg(a.A + f * 96 + lane) : 0.f;
    Ar[f] = f < a.FIN ? __ldg(a.A + f * 96 + 32 + lane) : 0.f;
    Ah[f] = f < a.FIN ? __ldg(a.A + f * 96 + 64 + lane) : 0.f;
  }
  const float cz = __ldg(a.c + lane), cr = __ldg(a.c + 32 + lane), ch = __ldg(a.c + 64 + lane);
  float Bz[HAS_H ? 32 : 1], Br[HAS_H ? 32 : 1], Bh[HAS_H ? 32 : 1];
  if (HAS_H) {
#pragma unroll
    for (int k = 0; k < 32; ++k) {
      Bz[k] = __ldg(a.Bm + k * 96 + lane);
      Br[k] = __ldg(a.Bm + k * 96 + 32 + lane);
      Bh[k] = __ldg(a.Bm + k * 96 + 64 + lane);
    }
  }
  if (a.stage) {
    __syncthreads();          // barrier initialised before anyone waits on it
    mbar_wait(&bar, 0);
  }
  const float* Xg = a.stage ? Xs : xb;
  const int FP = a.FP, P = a.P;
  const int nend = min(n0 + kNodesPerBlock, a.N);
  for (int n = n0 + warp; n < nend; n += 8) {
    // ---- A^X for all periods: lane holds entries (q*32 + lane) of the node's in*periods row, reference's edge order --------
    float ax[NQ];
    gather_ax<NQ>(a.rowptr, a.cv, Xg, FP, a.stage, n, lane, ax);
    float h = 0.f, hz = cz, hr = cr;
    if (HAS_H) {
      h = __ldg(a.h + b * a.h_bstride + (long long)n * 32 + lane);
#pragma unroll
      for (int k = 0; k < 32; ++k) {
        const float hk = __shfl_sync(0xffffffffu, h, k);
        hz = fmaf(hk, Bz[k], hz);
        hr = fmaf(hk, Br[k], hr);
      }
    }
    float acc = 0.f;
    for (int t = 0; t < P; ++t) {
      float pz = hz, pr = hr, ph = ch;
#pragma unroll
      for (int f = 0; f < 4; ++f) {
        if (f < a.FIN) {
          const int idx = f * P + t;
          float src = ax[0];
#pragma unroll
          for (int q = 1; q < NQ; ++q) src = (idx >> 5) == q ? ax[q] : src;
          const float v = __shfl_sync(0xffffffffu, src, idx & 31);
          pz = fmaf(v, Az[f], pz);
          pr = fmaf(v, Ar[f], pr);
          ph = fmaf(v, Ah[f], ph);
        }
      }
      const float Z = sigmoid_f(pz);
      float hn;
      if (HAS_H) {
        const float hrr = h * sigmoid_f(pr);
#pragma unroll
        for (int k = 0; k < 32; ++k) ph = fmaf(__shfl_sync(0xffffffffu, hrr, k), Bh[k], ph);
        hn = Z * h + (1.0f - Z) * tanh_f(ph);
      } else {
        hn = (1.0f - Z) * tanh_f(ph);       // H = 0: Z*H vanishes, R is irrelevant
      }
      acc = a.probs ? fmaf(__ldg(a.probs + t), hn, acc) : hn;
    }
    a.out[(b * a.N + n) * 32 + lane] = acc;
  }
}

// ---- 64 hidden channels: Bm (64 x 192) in shared memory ------------------------------------------------------------------------
// The pitch 193 makes both access patterns conflict-free: column reads (lane = column, the forward's products) and row reads
// (lane = row, the backward's transposed products).
constexpr int kWideBmLd = 193;
constexpr int kWideBmBytes = 64 * kWideBmLd * 4;

__device__ __forceinline__ void stage_bm_wide(float* Bs, const float* __restrict__ Bm) {
  for (int i = threadIdx.x; i < 64 * 192; i += 256) Bs[(i / 192) * kWideBmLd + i % 192] = __ldg(Bm + i);
}

// p[g][j] += sum_k v_k Bm[k][col0 + 64 g + lane + 32 j] over k = 0..63 in order, where v_k is channel k of the warp's 64-vector v
// (lane l holds v_l in v[0] and v_{l+32} in v[1]).  One shuffle per k serves all G column blocks.
template <int G>
__device__ __forceinline__ void matvec_wide(const float* Bs, int col0, const float (&v)[2], int lane, float (&p)[G][2]) {
#pragma unroll
  for (int k = 0; k < 64; ++k) {
    const float vk = __shfl_sync(0xffffffffu, v[k >> 5], k & 31);
    const float* row = Bs + k * kWideBmLd + col0 + lane;
#pragma unroll
    for (int g = 0; g < G; ++g) {
      p[g][0] = fmaf(vk, row[64 * g], p[g][0]);
      p[g][1] = fmaf(vk, row[64 * g + 32], p[g][1]);
    }
  }
}

// p[j] += sum_k sum_g v[g]_k Bm[lane + 32 j][col0 + 64 g + k] over k = 0..63 in order (g inner): the transposed products of the backward
template <int G>
__device__ __forceinline__ void matvec_wide_t(const float* Bs, int col0, const float (&v)[G][2], int lane, float (&p)[2]) {
  const float* r0 = Bs + lane * kWideBmLd + col0;
  const float* r1 = r0 + 32 * kWideBmLd;
#pragma unroll
  for (int k = 0; k < 64; ++k) {
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const float vk = __shfl_sync(0xffffffffu, v[g][k >> 5], k & 31);
      p[0] = fmaf(vk, r0[64 * g + k], p[0]);
      p[1] = fmaf(vk, r1[64 * g + k], p[1]);
    }
  }
}

// the A and c columns of lane's channels: Aw[gate][f][j] = A[f][64 gate + lane + 32 j] (zero for f >= FIN), cw[gate][j] = c[64 gate + ...]
__device__ __forceinline__ void load_ac_wide(const float* __restrict__ A, const float* __restrict__ c, int FIN, int lane,
                                             float (&Aw)[3][4][2], float (&cw)[3][2]) {
#pragma unroll
  for (int g = 0; g < 3; ++g)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
#pragma unroll
      for (int f = 0; f < 4; ++f) Aw[g][f][j] = f < FIN ? __ldg(A + f * 192 + 64 * g + 32 * j + lane) : 0.f;
      cw[g][j] = __ldg(c + 64 * g + 32 * j + lane);
    }
}

// k_tgcn_attn at 64 channels, one warp per (batch row, node).  With H, Bm is staged after X in dynamic shared memory; H Bm_{z,r} is
// shared by all periods and (H*R_t) Bm_h is per period, as at 32 channels.  The order of every per-channel sum is the 32-wide kernel's.
// Two CTAs per SM: without the bound ptxas stops at 64 registers and spills.
template <int NQ, bool HAS_H>
__global__ void __launch_bounds__(256, 2) k_tgcn_wide_attn(const TgcnArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* Xs = reinterpret_cast<float*>(smem_raw);
  float* Bs = reinterpret_cast<float*>(smem_raw + (a.stage ? (size_t)a.N * a.FP * 4 : 0));
  __shared__ __align__(8) uint64_t bar;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long b = blockIdx.y;
  const int n0 = blockIdx.x * kNodesPerBlock;
  const float* xb = a.x + b * (long long)a.N * a.FP;
  if (a.stage) stage_x_begin(&bar, Xs, xb, (uint32_t)a.N * a.FP * 4u);
  if (HAS_H) stage_bm_wide(Bs, a.Bm);
  float Aw[3][4][2], cw[3][2];
  load_ac_wide(a.A, a.c, a.FIN, lane, Aw, cw);
  if (a.stage || HAS_H) __syncthreads();      // Bs written; barrier initialised before anyone waits on it
  if (a.stage) mbar_wait(&bar, 0);
  const float* Xg = a.stage ? Xs : xb;
  const int FP = a.FP, P = a.P;
  const int nend = min(n0 + kNodesPerBlock, a.N);
  for (int n = n0 + warp; n < nend; n += 8) {
    float ax[NQ];
    gather_ax<NQ>(a.rowptr, a.cv, Xg, FP, a.stage, n, lane, ax);
    float h[2] = {0.f, 0.f}, hzr[2][2] = {{cw[0][0], cw[0][1]}, {cw[1][0], cw[1][1]}};
    if (HAS_H) {
      const float* hp = a.h + b * a.h_bstride + (long long)n * 64 + lane;
      h[0] = __ldg(hp);
      h[1] = __ldg(hp + 32);
      matvec_wide<2>(Bs, 0, h, lane, hzr);
    }
    float acc[2] = {0.f, 0.f};
    for (int t = 0; t < P; ++t) {
      float pz[2] = {hzr[0][0], hzr[0][1]}, pr[2] = {hzr[1][0], hzr[1][1]}, ph[1][2] = {{cw[2][0], cw[2][1]}};
#pragma unroll
      for (int f = 0; f < 4; ++f) {
        if (f < a.FIN) {
          const int idx = f * P + t;
          float src = ax[0];
#pragma unroll
          for (int q = 1; q < NQ; ++q) src = (idx >> 5) == q ? ax[q] : src;
          const float v = __shfl_sync(0xffffffffu, src, idx & 31);
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            pz[j] = fmaf(v, Aw[0][f][j], pz[j]);
            pr[j] = fmaf(v, Aw[1][f][j], pr[j]);
            ph[0][j] = fmaf(v, Aw[2][f][j], ph[0][j]);
          }
        }
      }
      float Z[2], hn[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) Z[j] = sigmoid_f(pz[j]);
      if (HAS_H) {
        float hrr[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) hrr[j] = h[j] * sigmoid_f(pr[j]);
        matvec_wide<1>(Bs, 128, hrr, lane, ph);
#pragma unroll
        for (int j = 0; j < 2; ++j) hn[j] = Z[j] * h[j] + (1.0f - Z[j]) * tanh_f(ph[0][j]);
      } else {
#pragma unroll
        for (int j = 0; j < 2; ++j) hn[j] = (1.0f - Z[j]) * tanh_f(ph[0][j]);      // H = 0: Z*H vanishes, R is irrelevant
      }
#pragma unroll
      for (int j = 0; j < 2; ++j) acc[j] = a.probs ? fmaf(__ldg(a.probs + t), hn[j], acc[j]) : hn[j];
    }
    float* o = a.out + (b * a.N + n) * 64 + lane;
    o[0] = acc[0];
    o[32] = acc[1];
  }
}

// ---- backward (H = None: the training configuration of the reference's A3TGCN2 example) ---------------------------------------
// What autograd records for attentiontemporalgcn.py:130-157 with H = 0: per period  Z = sigma(pz), H~ = tanh(ph), H_t = (1 - Z) H~,
// out = sum_t probs[t] H_t with pz = (A^X_t) A_z + c_z, ph = (A^X_t) A_h + c_h (the r gate multiplies H = 0 and has no gradient).
// Given g = dL/dout the kernel recomputes A^X (same gather as the forward) and the gates, and reduces
//     dA_z[f] = sum ax[f,t] dpz,  dA_h[f] = sum ax[f,t] dph,  dc_z = sum dpz,  dc_h = sum dph,  dprobs[t] = sum_j g_j H_t,j
// with dH_t = probs[t] g, dpz = -dH_t H~ Z (1 - Z), dph = dH_t (1 - Z)(1 - H~^2), over all (batch row, node, period).  One warp per
// (row, node), lane = output channel; per-CTA partials (fixed order inside the CTA) and a second launch that sums them in launch order:
// deterministic.  The gradient w.r.t. X is not produced (callers that need it take the op-for-op path).
struct TgcnBwdArgs {
  const int* rowptr;
  const int2* cv;
  int N, FIN, P, FP;
  const float* x; const float* A; const float* c; const float* probs; const float* gout;
  float* partial;         // [gridDim.y * gridDim.x][bwd_partial(NC)]: dA_z[4][CO] | dA_h[4][CO] | dc_z[CO] | dc_h[CO] | dprobs[128]
  int stage;
};
constexpr int bwd_partial(int nc) { return 10 * 32 * nc + 128; }

// NC = channels per lane (CO = 32 NC output channels, lane l owns channels l + 32 j); dprobs[t] sums the NC products of a lane, then the warp.
// NC = 1 keeps the 32-wide kernel's launch bounds; at NC = 2 the bound of two CTAs per SM lets ptxas take the registers it needs (no spills).
template <int NQ, int NC>
__global__ void __launch_bounds__(256, NC == 1 ? 0 : 2) k_tgcn_attn_bwd(const TgcnBwdArgs a) {
  constexpr int CO = 32 * NC, W = bwd_partial(NC);
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* Xs = reinterpret_cast<float*>(smem_raw);
  __shared__ __align__(8) uint64_t bar;
  __shared__ float red[8][W];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long b = blockIdx.y;
  const int n0 = blockIdx.x * kNodesPerBlock;
  const float* xb = a.x + b * (long long)a.N * a.FP;
  if (a.stage) stage_x_begin(&bar, Xs, xb, (uint32_t)a.N * a.FP * 4u);
  float Az[4][NC], Ah[4][NC], cz[NC], ch[NC];
#pragma unroll
  for (int j = 0; j < NC; ++j) {
#pragma unroll
    for (int f = 0; f < 4; ++f) {
      Az[f][j] = f < a.FIN ? __ldg(a.A + f * 3 * CO + 32 * j + lane) : 0.f;
      Ah[f][j] = f < a.FIN ? __ldg(a.A + f * 3 * CO + 2 * CO + 32 * j + lane) : 0.f;
    }
    cz[j] = __ldg(a.c + 32 * j + lane);
    ch[j] = __ldg(a.c + 2 * CO + 32 * j + lane);
  }
  if (a.stage) {
    __syncthreads();
    mbar_wait(&bar, 0);
  }
  const float* Xg = a.stage ? Xs : xb;
  const int FP = a.FP, P = a.P;
  const int nend = min(n0 + kNodesPerBlock, a.N);
  float dAz[4][NC], dAh[4][NC], dcz[NC], dch[NC], dpr[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int j = 0; j < NC; ++j) {
#pragma unroll
    for (int f = 0; f < 4; ++f) dAz[f][j] = dAh[f][j] = 0.f;
    dcz[j] = dch[j] = 0.f;
  }
  for (int n = n0 + warp; n < nend; n += 8) {
    float ax[NQ];
    gather_ax<NQ>(a.rowptr, a.cv, Xg, FP, a.stage, n, lane, ax);
    float g[NC];
#pragma unroll
    for (int j = 0; j < NC; ++j) g[j] = __ldg(a.gout + (b * a.N + n) * CO + 32 * j + lane);
    for (int t = 0; t < P; ++t) {
      float pz[NC], ph[NC], v[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int j = 0; j < NC; ++j) { pz[j] = cz[j]; ph[j] = ch[j]; }
#pragma unroll
      for (int f = 0; f < 4; ++f) {
        if (f < a.FIN) {
          const int idx = f * P + t;
          float src = ax[0];
#pragma unroll
          for (int q = 1; q < NQ; ++q) src = (idx >> 5) == q ? ax[q] : src;
          v[f] = __shfl_sync(0xffffffffu, src, idx & 31);
#pragma unroll
          for (int j = 0; j < NC; ++j) {
            pz[j] = fmaf(v[f], Az[f][j], pz[j]);
            ph[j] = fmaf(v[f], Ah[f][j], ph[j]);
          }
        }
      }
      float s = 0.f;                                      // dprobs[t] += sum over channels
#pragma unroll
      for (int j = 0; j < NC; ++j) {
        const float Z = sigmoid_f(pz[j]), Ht = tanh_f(ph[j]), hn = (1.0f - Z) * Ht;
        const float dh = (a.probs ? __ldg(a.probs + t) : 1.0f) * g[j];
        const float dpz = -dh * Ht * Z * (1.0f - Z), dph = dh * (1.0f - Z) * (1.0f - Ht * Ht);
#pragma unroll
        for (int f = 0; f < 4; ++f) {
          dAz[f][j] = fmaf(v[f], dpz, dAz[f][j]);
          dAh[f][j] = fmaf(v[f], dph, dAh[f][j]);
        }
        dcz[j] += dpz;
        dch[j] += dph;
        s = j == 0 ? g[j] * hn : fmaf(g[j], hn, s);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == (t & 31)) {
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if ((t >> 5) == q) dpr[q] += s;
      }
    }
  }
  // ---- CTA reduction in warp order, one partial per CTA ----------------------------------------------------------------------
  float* r = red[warp];
#pragma unroll
  for (int j = 0; j < NC; ++j) {
#pragma unroll
    for (int f = 0; f < 4; ++f) { r[f * CO + 32 * j + lane] = dAz[f][j]; r[4 * CO + f * CO + 32 * j + lane] = dAh[f][j]; }
    r[8 * CO + 32 * j + lane] = dcz[j];
    r[9 * CO + 32 * j + lane] = dch[j];
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) r[10 * CO + q * 32 + lane] = dpr[q];
  __syncthreads();
  float* out = a.partial + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * W;
  for (int i = threadIdx.x; i < W; i += 256) {
    float s = red[0][i];
#pragma unroll
    for (int w = 1; w < 8; ++w) s += red[w][i];
    out[i] = s;
  }
}

// dA (FIN x 3 CO, r columns zero), dc (3 CO), dprobs (P): sums of the per-CTA partials, 8 sub-sums per output in a fixed association
template <int NC>
__global__ void __launch_bounds__(256) k_tgcn_attn_bwd_reduce(int parts, int FIN, int P, const float* __restrict__ partial, float* __restrict__ dA,
                                                              float* __restrict__ dc, float* __restrict__ dprobs) {
  constexpr int CO = 32 * NC, W = bwd_partial(NC);
  __shared__ float sub[8][32];
  const int i = blockIdx.x * 32 + (threadIdx.x & 31);   // index into the partial layout
  const float t = sum_partials(parts, W, partial, i, sub);
  if (threadIdx.x >= 32 || i >= W) return;
  if (i < 4 * CO) { const int f = i / CO; if (f < FIN) dA[f * 3 * CO + i % CO] = t; }
  else if (i < 8 * CO) { const int f = (i - 4 * CO) / CO; if (f < FIN) dA[f * 3 * CO + 2 * CO + i % CO] = t; }
  else if (i < 9 * CO) dc[i - 8 * CO] = t;
  else if (i < 10 * CO) dc[2 * CO + i - 9 * CO] = t;
  else if (i - 10 * CO < P && dprobs) dprobs[i - 10 * CO] = t;
}

// ---- backward of one TGCN cell step WITH an incoming state (periods = 1): the steps t >= 1 of the reference's BatchedTGCN loop ----
// Forward (k_tgcn_attn<1, true>):  pre_g = (A^X) A_g + H' Bm_g + c_g,  Z = sigma(pre_z), R = sigma(pre_r) with H' = H,
// H~ = tanh(pre_h) with H' = H*R,  H_new = Z*H + (1-Z)*H~.  Given g = dL/dH_new the kernel recomputes A^X (the forward's gather) and
// the gates, then per (row, node), lane j = output channel:
//     dpz = g (H - H~) Z (1-Z),  dph = g (1-Z)(1 - H~^2),  d(H*R)_j = sum_k dph_k Bm_h[j][k],  dpr = d(H*R) H R (1-R)
//     dH_j = g_j Z_j + d(H*R)_j R_j + sum_k dpz_k Bm_z[j][k] + sum_k dpr_k Bm_r[j][k]            (only when dh != NULL)
// and accumulates  dA_g[f][j] += A^X_f dp_g,  dBm_{z,r}[k][j] += H_k dp_{z,r},  dBm_h[k][j] += (H*R)_k dph,  dc_g[j] += dp_g.
// The graph only touches X, so no transposed SpMM is needed.  Bm is staged in shared memory with a padded row (kBmLd = 97) so that
// both the column reads of the recompute (lane = column) and the row reads of the transposed products (lane = row) are free of bank
// conflicts; the 96 dBm accumulators of a lane stay in registers.  Per-CTA partials are summed over the 8 warps in warp order, and
// k_tgcn_cell_bwd_reduce adds the partials in a fixed association: the same inputs give the same bits.
struct TgcnCellBwdArgs {
  const int* rowptr;
  const int2* cv;
  int N, FIN;
  const float* x;         // [B][N][FIN] contiguous
  const float* h;         // [B][N][32] at h_bstride
  long long h_bstride;
  const float* A; const float* Bm; const float* c;
  const float* gout;      // [B][N][32]
  float* dh;              // [B][N][32] or null
  float* partial;         // [gridDim.y * gridDim.x][kCellPartial]: dA[4][96] | dBm[32][96] | dc[96] (the output layouts)
  int stage;
};
constexpr int kCellPartial = 4 * 96 + 32 * 96 + 96;
constexpr int kBmLd = 97;

__global__ void __launch_bounds__(256, 1) k_tgcn_cell_bwd(const TgcnCellBwdArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* Xs = reinterpret_cast<float*>(smem_raw);
  __shared__ __align__(8) uint64_t bar;
  __shared__ float Bs[32 * kBmLd];
  __shared__ float red[8][1024];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long b = blockIdx.y;
  const int n0 = blockIdx.x * kNodesPerBlock;
  const float* xb = a.x + b * (long long)a.N * a.FIN;
  if (a.stage) stage_x_begin(&bar, Xs, xb, (uint32_t)a.N * a.FIN * 4u);
  for (int i = threadIdx.x; i < 32 * 96; i += 256) Bs[(i / 96) * kBmLd + i % 96] = __ldg(a.Bm + i);
  float Az[4], Ar[4], Ah[4];
#pragma unroll
  for (int f = 0; f < 4; ++f) {
    Az[f] = f < a.FIN ? __ldg(a.A + f * 96 + lane) : 0.f;
    Ar[f] = f < a.FIN ? __ldg(a.A + f * 96 + 32 + lane) : 0.f;
    Ah[f] = f < a.FIN ? __ldg(a.A + f * 96 + 64 + lane) : 0.f;
  }
  const float cz = __ldg(a.c + lane), cr = __ldg(a.c + 32 + lane), ch = __ldg(a.c + 64 + lane);
  __syncthreads();            // Bs written; barrier initialised before anyone waits on it
  if (a.stage) mbar_wait(&bar, 0);
  const float* Xg = a.stage ? Xs : xb;
  const float* Bl = Bs + lane * kBmLd;          // row `lane` of Bm (transposed products)
  const int nend = min(n0 + kNodesPerBlock, a.N);
  float dAz[4] = {0.f, 0.f, 0.f, 0.f}, dAr[4] = {0.f, 0.f, 0.f, 0.f}, dAh[4] = {0.f, 0.f, 0.f, 0.f};
  float dcz = 0.f, dcr = 0.f, dch = 0.f;
  float dBz[32], dBr[32], dBh[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) dBz[k] = dBr[k] = dBh[k] = 0.f;
  for (int n = n0 + warp; n < nend; n += 8) {
    float ax[1];
    gather_ax<1>(a.rowptr, a.cv, Xg, a.FIN, a.stage, n, lane, ax);
    // ---- recompute the gates in the forward's order of operations -----------------------------------------------------------
    const float h = __ldg(a.h + b * a.h_bstride + (long long)n * 32 + lane);
    float pz = cz, pr = cr, ph = ch;
#pragma unroll
    for (int k = 0; k < 32; ++k) {
      const float hk = __shfl_sync(0xffffffffu, h, k);
      pz = fmaf(hk, Bs[k * kBmLd + lane], pz);
      pr = fmaf(hk, Bs[k * kBmLd + 32 + lane], pr);
    }
    float v[4];
#pragma unroll
    for (int f = 0; f < 4; ++f) {
      v[f] = __shfl_sync(0xffffffffu, ax[0], f);
      if (f < a.FIN) {
        pz = fmaf(v[f], Az[f], pz);
        pr = fmaf(v[f], Ar[f], pr);
        ph = fmaf(v[f], Ah[f], ph);
      } else {
        v[f] = 0.f;
      }
    }
    const float Z = sigmoid_f(pz), R = sigmoid_f(pr), hr = h * R;
#pragma unroll
    for (int k = 0; k < 32; ++k) ph = fmaf(__shfl_sync(0xffffffffu, hr, k), Bs[k * kBmLd + 64 + lane], ph);
    const float Ht = tanh_f(ph);
    // ---- gate backward ------------------------------------------------------------------------------------------------------
    const long long row = b * a.N + n;
    const float g = __ldg(a.gout + row * 32 + lane);
    const float dpz = g * (h - Ht) * Z * (1.0f - Z);
    const float dph = g * (1.0f - Z) * (1.0f - Ht * Ht);
    float dhr = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) dhr = fmaf(__shfl_sync(0xffffffffu, dph, k), Bl[64 + k], dhr);
    const float dpr = dhr * h * R * (1.0f - R);
    if (a.dh) {
      float d = fmaf(g, Z, dhr * R);
#pragma unroll
      for (int k = 0; k < 32; ++k) {
        d = fmaf(__shfl_sync(0xffffffffu, dpz, k), Bl[k], d);
        d = fmaf(__shfl_sync(0xffffffffu, dpr, k), Bl[32 + k], d);
      }
      a.dh[row * 32 + lane] = d;
    }
    // ---- weight-gradient accumulation ---------------------------------------------------------------------------------------
#pragma unroll
    for (int f = 0; f < 4; ++f) {
      dAz[f] = fmaf(v[f], dpz, dAz[f]);
      dAr[f] = fmaf(v[f], dpr, dAr[f]);
      dAh[f] = fmaf(v[f], dph, dAh[f]);
    }
    dcz += dpz;
    dcr += dpr;
    dch += dph;
#pragma unroll
    for (int k = 0; k < 32; ++k) {
      const float hk = __shfl_sync(0xffffffffu, h, k), hrk = __shfl_sync(0xffffffffu, hr, k);
      dBz[k] = fmaf(hk, dpz, dBz[k]);
      dBr[k] = fmaf(hk, dpr, dBr[k]);
      dBh[k] = fmaf(hrk, dph, dBh[k]);
    }
  }
  // ---- CTA reduction in warp order, one partial per CTA: dBm one gate (32 x 32) at a time, then dA | dc ----------------------
  float* out = a.partial + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * kCellPartial;
  float* r = red[warp];
#pragma unroll
  for (int gt = 0; gt < 3; ++gt) {
#pragma unroll
    for (int k = 0; k < 32; ++k) r[k * 32 + lane] = gt == 0 ? dBz[k] : (gt == 1 ? dBr[k] : dBh[k]);
    __syncthreads();
    for (int i = threadIdx.x; i < 1024; i += 256) {
      float s = red[0][i];
#pragma unroll
      for (int w = 1; w < 8; ++w) s += red[w][i];
      out[4 * 96 + (i >> 5) * 96 + gt * 32 + (i & 31)] = s;
    }
    __syncthreads();
  }
#pragma unroll
  for (int f = 0; f < 4; ++f) { r[f * 96 + lane] = dAz[f]; r[f * 96 + 32 + lane] = dAr[f]; r[f * 96 + 64 + lane] = dAh[f]; }
  r[384 + lane] = dcz;
  r[416 + lane] = dcr;
  r[448 + lane] = dch;
  __syncthreads();
  for (int i = threadIdx.x; i < 480; i += 256) {
    float s = red[0][i];
#pragma unroll
    for (int w = 1; w < 8; ++w) s += red[w][i];
    out[i < 384 ? i : 4 * 96 + 32 * 96 + (i - 384)] = s;
  }
}

// dA (FIN x 96), dBm (32 x 96), dc (96): sums of the per-CTA partials, 8 sub-sums per output in a fixed association
__global__ void __launch_bounds__(256) k_tgcn_cell_bwd_reduce(int parts, int FIN, const float* __restrict__ partial, float* __restrict__ dA,
                                                              float* __restrict__ dBm, float* __restrict__ dc) {
  __shared__ float sub[8][32];
  const int i = blockIdx.x * 32 + (threadIdx.x & 31);
  const float t = sum_partials(parts, kCellPartial, partial, i, sub);
  if (threadIdx.x >= 32 || i >= kCellPartial) return;
  if (i < 4 * 96) { if (i / 96 < FIN) dA[i] = t; }
  else if (i < 4 * 96 + 32 * 96) dBm[i - 4 * 96] = t;
  else dc[i - 4 * 96 - 32 * 96] = t;
}

// ---- the cell backward at 64 channels -----------------------------------------------------------------------------------------
// k_tgcn_cell_bwd's per-node algebra with lane l owning channels l and l + 32 and every product against Bm read from the staged Bs.  It
// writes dH and, per row (b, n), the gate gradients dp = [dpz | dpr | dph] (rows x 192) and the bases S1 = [A^X | H | 0] and
// S2 = [A^X | H*R | 0] (rows x kWideLd).  pre_g = (A^X) A_g + H' Bm_g + c_g is GConvGRU's gate shape with no operator hops, so
// k_wide_rows_wgrad<3> + k_wide_rows_wgrad_reduce<3> (rows.cuh) give dw [192][FIN + 64] = dp^T S and db = 1^T dp in a fixed order, and
// k_tgcn_wide_wgrad_unpack transposes dw into dA and dBm.
constexpr int kWideLd = 72;               // FIN + 64 <= 68 basis columns, padded to a multiple of 8 for the contraction
struct TgcnWideCellBwdArgs {
  const int* rowptr;
  const int2* cv;
  int N, FIN;
  const float* x;         // [B][N][FIN] contiguous
  const float* h;         // [B][N][64] at h_bstride
  long long h_bstride;
  const float* A; const float* Bm; const float* c;
  const float* gout;      // [B][N][64]
  float* dh;              // [B][N][64] or null
  float* dp;              // [B N][192]
  float* S1; float* S2;   // [B N][kWideLd]
  int stage;
};

__global__ void __launch_bounds__(256) k_tgcn_wide_cell_bwd(const TgcnWideCellBwdArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  float* Xs = reinterpret_cast<float*>(smem_raw);
  float* Bs = reinterpret_cast<float*>(smem_raw + (a.stage ? (size_t)a.N * a.FIN * 4 : 0));
  __shared__ __align__(8) uint64_t bar;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long b = blockIdx.y;
  const int n0 = blockIdx.x * kNodesPerBlock;
  const float* xb = a.x + b * (long long)a.N * a.FIN;
  if (a.stage) stage_x_begin(&bar, Xs, xb, (uint32_t)a.N * a.FIN * 4u);
  stage_bm_wide(Bs, a.Bm);
  float Aw[3][4][2], cw[3][2];
  load_ac_wide(a.A, a.c, a.FIN, lane, Aw, cw);
  __syncthreads();            // Bs written; barrier initialised before anyone waits on it
  if (a.stage) mbar_wait(&bar, 0);
  const float* Xg = a.stage ? Xs : xb;
  const int FIN = a.FIN;
  const int nend = min(n0 + kNodesPerBlock, a.N);
  for (int n = n0 + warp; n < nend; n += 8) {
    float ax[1];
    gather_ax<1>(a.rowptr, a.cv, Xg, FIN, a.stage, n, lane, ax);
    // ---- recompute the gates in the forward's order of operations -----------------------------------------------------------
    const float* hp = a.h + b * a.h_bstride + (long long)n * 64 + lane;
    const float h[2] = {__ldg(hp), __ldg(hp + 32)};
    float pzr[2][2] = {{cw[0][0], cw[0][1]}, {cw[1][0], cw[1][1]}}, ph[1][2] = {{cw[2][0], cw[2][1]}};
    matvec_wide<2>(Bs, 0, h, lane, pzr);
#pragma unroll
    for (int f = 0; f < 4; ++f) {
      if (f < FIN) {
        const float v = __shfl_sync(0xffffffffu, ax[0], f);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          pzr[0][j] = fmaf(v, Aw[0][f][j], pzr[0][j]);
          pzr[1][j] = fmaf(v, Aw[1][f][j], pzr[1][j]);
          ph[0][j] = fmaf(v, Aw[2][f][j], ph[0][j]);
        }
      }
    }
    float Z[2], R[2], hr[2];
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      Z[j] = sigmoid_f(pzr[0][j]);
      R[j] = sigmoid_f(pzr[1][j]);
      hr[j] = h[j] * R[j];
    }
    matvec_wide<1>(Bs, 128, hr, lane, ph);
    // ---- gate backward ------------------------------------------------------------------------------------------------------
    const long long row = b * a.N + n;
    float dph[1][2], dzr[2][2], dhr[2] = {0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const float Ht = tanh_f(ph[0][j]), g = __ldg(a.gout + row * 64 + 32 * j + lane);
      dzr[0][j] = g * (h[j] - Ht) * Z[j] * (1.0f - Z[j]);
      dph[0][j] = g * (1.0f - Z[j]) * (1.0f - Ht * Ht);
    }
    matvec_wide_t<1>(Bs, 128, dph, lane, dhr);
#pragma unroll
    for (int j = 0; j < 2; ++j) dzr[1][j] = dhr[j] * h[j] * R[j] * (1.0f - R[j]);
    if (a.dh) {
      float d[2];
#pragma unroll
      for (int j = 0; j < 2; ++j) d[j] = fmaf(__ldg(a.gout + row * 64 + 32 * j + lane), Z[j], dhr[j] * R[j]);
      matvec_wide_t<2>(Bs, 0, dzr, lane, d);
      a.dh[row * 64 + lane] = d[0];
      a.dh[row * 64 + 32 + lane] = d[1];
    }
    // ---- the weight-gradient operands ----------------------------------------------------------------------------------------
    float* dp = a.dp + row * 192 + lane;
    float* s1 = a.S1 + row * kWideLd;
    float* s2 = a.S2 + row * kWideLd;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      dp[32 * j] = dzr[0][j];
      dp[64 + 32 * j] = dzr[1][j];
      dp[128 + 32 * j] = dph[0][j];
      s1[FIN + 32 * j + lane] = h[j];
      s2[FIN + 32 * j + lane] = hr[j];
    }
    if (lane < FIN) { s1[lane] = ax[0]; s2[lane] = ax[0]; }
    if (lane < kWideLd - 64 - FIN) { s1[FIN + 64 + lane] = 0.f; s2[FIN + 64 + lane] = 0.f; }
  }
}

// dw [192][FIN + 64] (row = gate column of A / Bm, basis column m = [A^X | H]) -> dA [FIN][192], dBm [64][192]
__global__ void __launch_bounds__(256) k_tgcn_wide_wgrad_unpack(int FIN, const float* __restrict__ dw, float* __restrict__ dA,
                                                                float* __restrict__ dBm) {
  const int nb = FIN + 64;
  const int i = blockIdx.x * 256 + threadIdx.x;      // output index: m * 192 + col
  if (i >= nb * 192) return;
  const int m = i / 192, col = i - m * 192;
  const float v = dw[col * nb + m];
  if (m < FIN) dA[i] = v;
  else dBm[i - FIN * 192] = v;
}

template <int NQ>
int launch_nq(const TgcnArgs& a, dim3 grid, size_t smem, cudaStream_t st) {
  if (a.h) {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_tgcn_attn<NQ, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_tgcn_attn<NQ, true><<<grid, 256, smem, st>>>(a);
  } else {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_tgcn_attn<NQ, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_tgcn_attn<NQ, false><<<grid, 256, smem, st>>>(a);
  }
  STMP_LAUNCH_OK("k_tgcn_attn");
  if (!a.stage) { static const int slotg = path_slot("k_tgcn_attn[x-global]"); count_path(slotg); }
  return STMP_OK;
}

template <int NQ>
int launch_wide_nq(const TgcnArgs& a, dim3 grid, size_t smem, cudaStream_t st) {
  if (a.h) {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_tgcn_wide_attn<NQ, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_tgcn_wide_attn<NQ, true><<<grid, 256, smem, st>>>(a);
  } else {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_tgcn_wide_attn<NQ, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_tgcn_wide_attn<NQ, false><<<grid, 256, smem, st>>>(a);
  }
  STMP_LAUNCH_OK("k_tgcn_wide_attn");
  if (!a.stage) { static const int slotg = path_slot("k_tgcn_wide_attn[x-global]"); count_path(slotg); }
  return STMP_OK;
}

// entry and launch names per width (NC channels per lane)
template <int NC> struct TgcnNames;
template <> struct TgcnNames<1> {
  static constexpr const char* fwd = "stmp_tgcn_attn_fwd";
  static constexpr const char* bwd = "stmp_tgcn_attn_bwd";
  static constexpr const char* k_bwd = "k_tgcn_attn_bwd";
  static constexpr const char* k_bwd_global = "k_tgcn_attn_bwd[x-global]";
  static constexpr const char* k_bwd_reduce = "k_tgcn_attn_bwd_reduce";
};
template <> struct TgcnNames<2> {
  static constexpr const char* fwd = "stmp_tgcn_wide_attn_fwd";
  static constexpr const char* bwd = "stmp_tgcn_wide_attn_bwd";
  static constexpr const char* k_bwd = "k_tgcn_wide_attn_bwd";
  static constexpr const char* k_bwd_global = "k_tgcn_wide_attn_bwd[x-global]";
  static constexpr const char* k_bwd_reduce = "k_tgcn_wide_attn_bwd_reduce";
};

// X[b] is staged while it takes at most this many bytes.  At 64 channels with H the staged Bm (kWideBmBytes) sits next to it:
// 160 KB + 48.3 KB fits the 227 KB a CTA may take.
constexpr size_t kFwdStageBytes = 160 * 1024;
// The backwards stage at most 128 KB of X: next to it the H = None backward keeps its 8 warps' partials (24 KB at 64 channels) and the
// 64-wide cell backward the staged Bm (48.3 KB).
constexpr size_t kBwdStageBytes = 128 * 1024;

template <int NC>
int tgcn_attn_fwd(const stmp_plan* plan, int64_t B, int64_t fin, int64_t periods, const float* x, const float* h, int64_t h_bstride,
                  const float* A, const float* Bm, const float* c, const float* probs, float* out, void* stream) {
  using Nm = TgcnNames<NC>;
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: plan is NULL", Nm::fwd);
  STMP_REQUIRE(plan->n_ops >= 1, STMP_EINVAL, "%s: plan has no operator", Nm::fwd);
  STMP_REQUIRE(x && A && Bm && c && out, STMP_EINVAL, "%s: NULL tensor", Nm::fwd);
  STMP_REQUIRE(B >= 0 && periods >= 1, STMP_EINVAL, "%s: bad B/periods", Nm::fwd);
  if (fin < 1 || fin > 4 || fin * periods > 128)
    return set_error(STMP_EUNSUPPORTED, "fused TGCN-attention kernel takes in_channels <= 4 and in_channels*periods <= 128 (got %lld x %lld)",
                     (long long)fin, (long long)periods);
  if (B == 0) return STMP_OK;
  STMP_REQUIRE(B < 65536, STMP_ESHAPE, "%s: batch too large for one launch", Nm::fwd);
  TgcnArgs a;
  a.rowptr = plan->fwd[0].rowptr; a.cv = plan->fwd[0].cv;
  a.N = plan->n; a.FIN = (int)fin; a.P = (int)periods; a.FP = (int)(fin * periods); a.B = B;
  a.x = x; a.h = h; a.h_bstride = h_bstride; a.A = A; a.Bm = Bm; a.c = c; a.probs = probs; a.out = out;
  const size_t bytes = (size_t)a.N * a.FP * 4;
  a.stage = (bytes <= kFwdStageBytes && bytes % 16 == 0 && (reinterpret_cast<uintptr_t>(x) % 16) == 0 && ((size_t)a.N * a.FP * 4) % 16 == 0) ? 1 : 0;
  dim3 grid((unsigned)((a.N + kNodesPerBlock - 1) / kNodesPerBlock), (unsigned)B);
  cudaStream_t st = (cudaStream_t)stream;
  const int nq = (a.FP + 31) / 32;
  if constexpr (NC == 1) {
    const size_t smem = a.stage ? bytes : 0;
    switch (nq) {
      case 1: return launch_nq<1>(a, grid, smem, st);
      case 2: return launch_nq<2>(a, grid, smem, st);
      case 3: return launch_nq<3>(a, grid, smem, st);
      default: return launch_nq<4>(a, grid, smem, st);
    }
  } else {
    const size_t smem = (a.stage ? bytes : 0) + (h ? kWideBmBytes : 0);
    switch (nq) {
      case 1: return launch_wide_nq<1>(a, grid, smem, st);
      case 2: return launch_wide_nq<2>(a, grid, smem, st);
      case 3: return launch_wide_nq<3>(a, grid, smem, st);
      default: return launch_wide_nq<4>(a, grid, smem, st);
    }
  }
}

template <int NC>
int64_t tgcn_attn_bwd_workspace_bytes(const stmp_plan* plan, int64_t B) {
  if (!plan || B < 0) return 0;
  return (int64_t)B * ((plan->n + kNodesPerBlock - 1) / kNodesPerBlock) * bwd_partial(NC) * 4;
}

template <int NC>
int tgcn_attn_bwd(const stmp_plan* plan, int64_t B, int64_t fin, int64_t periods, const float* x, const float* A, const float* c,
                  const float* probs, const float* gout, void* workspace, float* dA, float* dc, float* dprobs, void* stream) {
  using Nm = TgcnNames<NC>;
  constexpr int CO = 32 * NC, W = bwd_partial(NC);
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: plan is NULL", Nm::bwd);
  STMP_REQUIRE(plan->n_ops >= 1, STMP_EINVAL, "%s: plan has no operator", Nm::bwd);
  STMP_REQUIRE(x && A && c && gout && workspace && dA && dc, STMP_EINVAL, "%s: NULL tensor", Nm::bwd);
  STMP_REQUIRE(B >= 1 && periods >= 1, STMP_EINVAL, "%s: bad B/periods", Nm::bwd);
  if (fin < 1 || fin > 4 || fin * periods > 128)
    return set_error(STMP_EUNSUPPORTED, "fused TGCN-attention backward takes in_channels <= 4 and in_channels*periods <= 128 (got %lld x %lld)",
                     (long long)fin, (long long)periods);
  STMP_REQUIRE(B < 65536, STMP_ESHAPE, "%s: batch too large for one launch", Nm::bwd);
  cudaStream_t st = (cudaStream_t)stream;
  TgcnBwdArgs a;
  a.rowptr = plan->fwd[0].rowptr; a.cv = plan->fwd[0].cv;
  a.N = plan->n; a.FIN = (int)fin; a.P = (int)periods; a.FP = (int)(fin * periods);
  a.x = x; a.A = A; a.c = c; a.probs = probs; a.gout = gout; a.partial = reinterpret_cast<float*>(workspace);
  const size_t bytes = (size_t)a.N * a.FP * 4;
  a.stage = (bytes <= kBwdStageBytes && bytes % 16 == 0 && (reinterpret_cast<uintptr_t>(x) % 16) == 0) ? 1 : 0;
  const size_t smem = a.stage ? bytes : 0;
  dim3 grid((unsigned)((a.N + kNodesPerBlock - 1) / kNodesPerBlock), (unsigned)B);
  STMP_CUDA_OK(cudaMemsetAsync(dA, 0, (size_t)fin * 3 * CO * 4, st));      // the r-gate columns have no gradient when H = 0
  STMP_CUDA_OK(cudaMemsetAsync(dc, 0, 3 * CO * 4, st));
  const int nq = (a.FP + 31) / 32;
#define STMP_TGCN_BWD(NQ)                                                                                                     \
  do {                                                                                                                        \
    STMP_CUDA_OK(cudaFuncSetAttribute(k_tgcn_attn_bwd<NQ, NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));      \
    k_tgcn_attn_bwd<NQ, NC><<<grid, 256, smem, st>>>(a);                                                                      \
  } while (0)
  switch (nq) {
    case 1: STMP_TGCN_BWD(1); break;
    case 2: STMP_TGCN_BWD(2); break;
    case 3: STMP_TGCN_BWD(3); break;
    default: STMP_TGCN_BWD(4); break;
  }
#undef STMP_TGCN_BWD
  STMP_LAUNCH_OK(Nm::k_bwd);
  if (!a.stage) { static const int slotg = path_slot(Nm::k_bwd_global); count_path(slotg); }
  k_tgcn_attn_bwd_reduce<NC><<<(W + 31) / 32, 256, 0, st>>>((int)(grid.x * grid.y), (int)fin, (int)periods, a.partial, dA, dc, dprobs);
  STMP_LAUNCH_OK(Nm::k_bwd_reduce);
  return STMP_OK;
}

// The 64-wide cell backward's workspace, carved at 16-byte offsets from `base`: dp [rows][192] | S1, S2 [rows][kWideLd] | the
// contraction's partials [3][parts][kWideLd * 64 + 64] | dw [192][FIN + 64 <= 68].
struct WideCellWs {
  float *dp, *S1, *S2, *partial, *dw;
  size_t bytes;
};
WideCellWs wide_cell_ws(void* base, long long rows) {
  WideCellWs w;
  size_t off = 0;
  auto take = [&](size_t floats) {
    float* p = reinterpret_cast<float*>(reinterpret_cast<uintptr_t>(base) + off);
    off += (floats * 4 + 15) / 16 * 16;
    return p;
  };
  w.dp = take((size_t)rows * 192);
  w.S1 = take((size_t)rows * kWideLd);
  w.S2 = take((size_t)rows * kWideLd);
  w.partial = take((size_t)3 * wgrad_ffma_max_parts() * (kWideLd * 64 + 64));
  w.dw = take(192 * 68);
  w.bytes = off;
  return w;
}

}  // namespace
}  // namespace stmp

using namespace stmp;

extern "C" int stmp_tgcn_attn_fwd(const stmp_plan* plan, int64_t B, int64_t fin, int64_t periods, const float* x, const float* h,
                                  int64_t h_bstride, const float* A, const float* Bm, const float* c, const float* probs,
                                  float* out, void* stream) {
  return tgcn_attn_fwd<1>(plan, B, fin, periods, x, h, h_bstride, A, Bm, c, probs, out, stream);
}

extern "C" int stmp_tgcn_wide_attn_fwd(const stmp_plan* plan, int64_t B, int64_t fin, int64_t periods, const float* x, const float* h,
                                       int64_t h_bstride, const float* A, const float* Bm, const float* c, const float* probs,
                                       float* out, void* stream) {
  return tgcn_attn_fwd<2>(plan, B, fin, periods, x, h, h_bstride, A, Bm, c, probs, out, stream);
}

extern "C" int64_t stmp_tgcn_attn_bwd_workspace_bytes(const stmp_plan* plan, int64_t B) { return tgcn_attn_bwd_workspace_bytes<1>(plan, B); }

extern "C" int64_t stmp_tgcn_wide_attn_bwd_workspace_bytes(const stmp_plan* plan, int64_t B) {
  return tgcn_attn_bwd_workspace_bytes<2>(plan, B);
}

extern "C" int stmp_tgcn_attn_bwd(const stmp_plan* plan, int64_t B, int64_t fin, int64_t periods, const float* x, const float* A,
                                  const float* c, const float* probs, const float* gout, void* workspace, float* dA, float* dc,
                                  float* dprobs, void* stream) {
  return tgcn_attn_bwd<1>(plan, B, fin, periods, x, A, c, probs, gout, workspace, dA, dc, dprobs, stream);
}

extern "C" int stmp_tgcn_wide_attn_bwd(const stmp_plan* plan, int64_t B, int64_t fin, int64_t periods, const float* x, const float* A,
                                       const float* c, const float* probs, const float* gout, void* workspace, float* dA, float* dc,
                                       float* dprobs, void* stream) {
  return tgcn_attn_bwd<2>(plan, B, fin, periods, x, A, c, probs, gout, workspace, dA, dc, dprobs, stream);
}

extern "C" int64_t stmp_tgcn_cell_bwd_workspace_bytes(const stmp_plan* plan, int64_t B) {
  if (!plan || B < 0) return 0;
  return (int64_t)B * ((plan->n + kNodesPerBlock - 1) / kNodesPerBlock) * kCellPartial * 4;
}

extern "C" int stmp_tgcn_cell_bwd(const stmp_plan* plan, int64_t B, int64_t fin, const float* x, const float* h, int64_t h_bstride,
                                  const float* A, const float* Bm, const float* c, const float* gout, void* workspace, float* dh,
                                  float* dA, float* dBm, float* dc, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_tgcn_cell_bwd: plan is NULL");
  STMP_REQUIRE(plan->n_ops >= 1, STMP_EINVAL, "stmp_tgcn_cell_bwd: plan has no operator");
  if (fin < 1 || fin > 4)
    return set_error(STMP_EUNSUPPORTED, "fused TGCN cell backward takes in_channels <= 4 (got %lld)", (long long)fin);
  STMP_REQUIRE(x && h && A && Bm && c && gout && workspace && dA && dBm && dc, STMP_EINVAL, "stmp_tgcn_cell_bwd: NULL tensor");
  STMP_REQUIRE(B >= 1, STMP_EINVAL, "stmp_tgcn_cell_bwd: bad B");
  STMP_REQUIRE(B < 65536, STMP_ESHAPE, "stmp_tgcn_cell_bwd: batch too large for one launch");
  cudaStream_t st = (cudaStream_t)stream;
  TgcnCellBwdArgs a;
  a.rowptr = plan->fwd[0].rowptr; a.cv = plan->fwd[0].cv;
  a.N = plan->n; a.FIN = (int)fin;
  a.x = x; a.h = h; a.h_bstride = h_bstride; a.A = A; a.Bm = Bm; a.c = c; a.gout = gout; a.dh = dh;
  a.partial = reinterpret_cast<float*>(workspace);
  const size_t bytes = (size_t)a.N * a.FIN * 4;
  a.stage = (bytes <= kBwdStageBytes && bytes % 16 == 0 && (reinterpret_cast<uintptr_t>(x) % 16) == 0) ? 1 : 0;
  const size_t smem = a.stage ? bytes : 0;
  dim3 grid((unsigned)((a.N + kNodesPerBlock - 1) / kNodesPerBlock), (unsigned)B);
  STMP_CUDA_OK(cudaFuncSetAttribute(k_tgcn_cell_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_tgcn_cell_bwd<<<grid, 256, smem, st>>>(a);
  STMP_LAUNCH_OK("k_tgcn_cell_bwd");
  if (!a.stage) { static const int slotg = path_slot("k_tgcn_cell_bwd[x-global]"); count_path(slotg); }
  k_tgcn_cell_bwd_reduce<<<(kCellPartial + 31) / 32, 256, 0, st>>>((int)(grid.x * grid.y), (int)fin, a.partial, dA, dBm, dc);
  STMP_LAUNCH_OK("k_tgcn_cell_bwd_reduce");
  return STMP_OK;
}

extern "C" int64_t stmp_tgcn_wide_cell_bwd_workspace_bytes(const stmp_plan* plan, int64_t B) {
  if (!plan || B < 0) return 0;
  return (int64_t)wide_cell_ws(nullptr, (long long)B * plan->n).bytes;
}

extern "C" int stmp_tgcn_wide_cell_bwd(const stmp_plan* plan, int64_t B, int64_t fin, const float* x, const float* h, int64_t h_bstride,
                                       const float* A, const float* Bm, const float* c, const float* gout, void* workspace, float* dh,
                                       float* dA, float* dBm, float* dc, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_tgcn_wide_cell_bwd: plan is NULL");
  STMP_REQUIRE(plan->n_ops >= 1, STMP_EINVAL, "stmp_tgcn_wide_cell_bwd: plan has no operator");
  if (fin < 1 || fin > 4)
    return set_error(STMP_EUNSUPPORTED, "fused TGCN cell backward takes in_channels <= 4 (got %lld)", (long long)fin);
  STMP_REQUIRE(x && h && A && Bm && c && gout && workspace && dA && dBm && dc, STMP_EINVAL, "stmp_tgcn_wide_cell_bwd: NULL tensor");
  STMP_REQUIRE(B >= 1, STMP_EINVAL, "stmp_tgcn_wide_cell_bwd: bad B");
  STMP_REQUIRE(B < 65536, STMP_ESHAPE, "stmp_tgcn_wide_cell_bwd: batch too large for one launch");
  STMP_REQUIRE(((uintptr_t)workspace & 15u) == 0, STMP_ESHAPE, "stmp_tgcn_wide_cell_bwd: the workspace must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const long long rows = B * (long long)plan->n;
  const WideCellWs ws = wide_cell_ws(workspace, rows);
  TgcnWideCellBwdArgs a;
  a.rowptr = plan->fwd[0].rowptr; a.cv = plan->fwd[0].cv;
  a.N = plan->n; a.FIN = (int)fin;
  a.x = x; a.h = h; a.h_bstride = h_bstride; a.A = A; a.Bm = Bm; a.c = c; a.gout = gout; a.dh = dh;
  a.dp = ws.dp; a.S1 = ws.S1; a.S2 = ws.S2;
  const size_t bytes = (size_t)a.N * a.FIN * 4;
  a.stage = (bytes <= kBwdStageBytes && bytes % 16 == 0 && (reinterpret_cast<uintptr_t>(x) % 16) == 0) ? 1 : 0;
  const size_t smem = (a.stage ? bytes : 0) + kWideBmBytes;
  dim3 grid((unsigned)((a.N + kNodesPerBlock - 1) / kNodesPerBlock), (unsigned)B);
  STMP_CUDA_OK(cudaFuncSetAttribute(k_tgcn_wide_cell_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_tgcn_wide_cell_bwd<<<grid, 256, smem, st>>>(a);
  STMP_LAUNCH_OK("k_tgcn_wide_cell_bwd");
  if (!a.stage) { static const int slotg = path_slot("k_tgcn_wide_cell_bwd[x-global]"); count_path(slotg); }
  const int parts = wide_wgrad_parts(rows), nb = (int)fin + 64;
  const WideWgradOps<3> op = {{ws.S1, ws.S1, ws.S2}, {ws.dp, ws.dp + 64, ws.dp + 128}, {192, 192, 192}};
  k_wide_rows_wgrad<3><<<dim3(parts, 3), kWideWgThreads, 0, st>>>(rows, kWideLd, op, ws.partial);
  STMP_LAUNCH_OK("k_tgcn_wide_wgrad");
  k_wide_rows_wgrad_reduce<3><<<(192 * nb + 192 + 31) / 32, 256, 0, st>>>(parts, kWideLd, nb, ws.partial, 0, 0, nullptr, ws.dw, dc, nullptr);
  STMP_LAUNCH_OK("k_tgcn_wide_wgrad_reduce");
  k_tgcn_wide_wgrad_unpack<<<(nb * 192 + 255) / 256, 256, 0, st>>>((int)fin, ws.dw, dA, dBm);
  STMP_LAUNCH_OK("k_tgcn_wide_wgrad_unpack");
  return STMP_OK;
}
