// dcrnn_wide_rows.cu -- BatchedDCRNN at 64 hidden channels (the DCRNN paper's width), K = 2 or 3, cin 1..4, on graphs of ANY size, split
// over CTAs by destination rows (DESIGN §4m).  The row-split scheme of §4k / §4l -- one launch per all-to-all dependency, every launch
// serving all B windows of a step, the X diffusion hoisted out of the time loop -- with a contraction that no longer fits one lane per
// output channel and all weights staged per CTA ((2K-1)(cin+64) x 192 fp32 is up to 261 KB):
//
//   rows i = b N + n (window-major), scratch blocks (B N, 64) floats; a warp owns kRW = 8 consecutive rows, lane l channels 2l, 2l + 1
//
// Per row the warp gathers the hop vectors (each CSR entry is one 256-byte read of a source row, entries broadcast), writes the row's basis
// into its shared-memory tile in the order [X columns | pad | H columns], and contracts its 8 rows against a weight image in global memory
// (L1 / L2 resident, a float2 per lane per basis column, reused over 8 rows): exact fp32 FFMA, no tensor cores -- the fp16 hi/lo split of
// the wgmma kernels would be the faster route, this one is the exact one.  The image is built at the start of every call from wzrT / whsT
// (one launch): wf (nbp, 192) for the forward, basis column m' -> outputs z | r | h, and its transpose wb (192, nbp) for the backward's
// d W^T.  No atomics and no block barriers: every value depends only on its own row's fixed-order sums, so repeated calls are bit-identical.
//
// The basis of U = [X | H] is [U | P_o U | P_i U | 2 P_o T_1o - U | 2 P_i T_1i - U] (as dcrnn_narrow_rows.cu); block j = 1 + 2 (k - 1) + o
// is hop k of operator o.  Launches (L = K - 1):
//   forward, step t >= 1: L per basis, k_dcrnn_wrows_fwd (hop k of [.. | H] / [.. | H*R]; the last hop of the first basis computes Z, R,
//     H*R and the X part of pre_h, the last hop of the second Ht and H_t).  Step 0 (H = 0) is one rowwise launch, k_dcrnn_wrows_fwd0,
//     unless the plan holds a non-finite operator value: then the full chain runs on a zeroed state, so inf * 0 = NaN spreads as in the
//     reference.
//   backward, reverse time: k_dcrnn_wrows_bwd0 (rowwise start of step T-1), then per step t >= 1 L transposed-gather launches of the
//     adjoint of dS2's H columns and L of dS1's, k_dcrnn_wrows_bwd.  The X columns of dS1 + dS2 are written rowwise; the caller applies
//     the transposed X-basis adjoint to them once, after the loop.
#include "common.cuh"

namespace stmp {
namespace {

constexpr int kThreads = 256, kWarps = kThreads / 32;
constexpr int kRW = 8;                       // rows per warp
constexpr int kCO = 64, kQ = 3 * kCO;        // hidden channels; outputs z | r | h
constexpr int kMaxNbp = 20 + 5 * kCO;        // (2K-1) cin rounded up to 4, + (2K-1) 64, K <= 3, cin <= 4
constexpr int kTP = 344;                     // floats per row of a warp's tile: >= kMaxNbp and >= 2 kQ - kCO (backward: d | gathered)
constexpr int kSmem = kWarps * kRW * kTP * 4;
constexpr long long kImgFloats = 2ll * kMaxNbp * kQ;

// scratch blocks of the forward
constexpr int kHS = 0, kHR = 1, kZB = 2, kPH = 3, kHop0 = 4;            // H | H*R | Z | X part of pre_h | hop 1 of op o at kHop0 + o
// ... and of the backward
constexpr int kG = 0, kDPH = 1, kDPZ = 2, kDPR = 3, kDHP = 4, kSACC = 5, kA0 = 6;   // A(parity p, op o) at kA0 + 2 p + o
constexpr int kBlocks = 10;

// the backward tile of a row: d = dpz | dpr | dph at [0, 192) (q order of the image), the two gathered adjoint vectors at [192, 320)
constexpr int kTGat = kQ;

struct WRows {
  const int* rp[2]; const int2* cv[2];       // P_o, P_i: by destination (forward) or by source (backward, the transposed products)
  int n, B, T, t, cin, K, nbc, w, wp, nbp;   // nbc = (2K-1)(cin+64); w = (2K-1) cin X columns, wp = w rounded up to 4; nbp = wp + (2K-1) 64
  long long rows, blk;                       // B n; floats per scratch block (rows * 64)
  const float* x; long long xbs, xts, xld; int xblk;   // X block j of (t, b, n): x + t xts + b xbs + n xld + j xblk
  const float* wf; const float* wb;          // (nbp, 192), (192, nbp)
  const float* bz; const float* br; const float* bh;   // nullable
  float* out;                                // (B, T, N, 64)
  float* scr;                                // kBlocks scratch blocks
  float* stash;                              // (T, B N, 192): Z | R | Ht, nullable in the forward
  float* S1; float* S2;                      // (T*B, N, nbc), nullable
  const float* gout;                         // (B, T, N, 64)
  float* dph; float* dpzr;                   // (T, B, N, 64), (T, B, N, 128)
  float* dsx; long long dsx_ld;              // (T*B, N, dsx_ld): X columns of dS1 + dS2, block j at j * cin; nullable
  int beta, hop, par;
};

__device__ __forceinline__ float2 ld2(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }
__device__ __forceinline__ float2 ld2s(const float* p) { return *reinterpret_cast<const float2*>(p); }   // own-row scratch, written earlier
__device__ __forceinline__ void st2(float* p, float2 v) { *reinterpret_cast<float2*>(p) = v; }

__device__ __forceinline__ float* sblk(const WRows& a, int k, long long i) { return a.scr + k * a.blk + i * kCO; }
__device__ __forceinline__ long long trow(const WRows& a, int t, long long i) { return (long long)t * a.rows + i; }
__device__ __forceinline__ float* outp(const WRows& a, int b, int t, int n) { return a.out + (((long long)b * a.T + t) * a.n + n) * kCO; }
__device__ __forceinline__ float* stashp(const WRows& a, int t, long long i) { return a.stash + trow(a, t, i) * kQ; }

// sum_e val_e * src[col_e] over CSR row n, in entry order; src = the window's block rows, offset to this lane's two channels
__device__ __forceinline__ float2 gather(const int* __restrict__ rowptr, const int2* __restrict__ cv, int n, const float* __restrict__ src) {
  float2 s = make_float2(0.f, 0.f);
  const int beg = __ldg(rowptr + n), end = __ldg(rowptr + n + 1);
  int k = beg;
  for (; k + 4 <= end; k += 4) {
    int2 e[4];
    float2 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) e[u] = __ldg(cv + k + u);
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = ld2(src + (long long)e[u].x * kCO);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float w = __int_as_float(e[u].y);
      s.x = __fadd_rn(s.x, __fmul_rn(w, v[u].x));
      s.y = __fadd_rn(s.y, __fmul_rn(w, v[u].y));
    }
  }
  for (; k < end; ++k) {
    const int2 e = __ldg(cv + k);
    const float2 v = ld2(src + (long long)e.x * kCO);
    const float w = __int_as_float(e.y);
    s.x = __fadd_rn(s.x, __fmul_rn(w, v.x));
    s.y = __fadd_rn(s.y, __fmul_rn(w, v.y));
  }
  return s;
}

// source pointer of block k for window b, this lane's channels
__device__ __forceinline__ const float* gsrc(const WRows& a, int k, int b, int lane) {
  return a.scr + k * a.blk + (long long)b * a.n * kCO + 2 * lane;
}

__device__ __forceinline__ void fma2(float2& acc, float s, float2 w) {
  acc.x = fmaf(s, w.x, acc.x);
  acc.y = fmaf(s, w.y, acc.y);
}

// the row's X columns into its tile ([0, wp): block j channel c at j cin + c, zero pad) and, in training, into S2
__device__ __forceinline__ void tile_x(const WRows& a, float* tr, int t, int b, int n, long long r, int lane) {
  const float* xr = a.x + t * a.xts + b * a.xbs + n * a.xld;
  const int C = a.cin + kCO;
  for (int m = lane; m < a.wp; m += 32) {
    float s = 0.f;
    if (m < a.w) {
      const int j = m / a.cin, c = m - j * a.cin;
      s = __ldg(xr + j * a.xblk + c);
      if (a.S2) a.S2[r * a.nbc + j * C + c] = s;
    }
    tr[m] = s;
  }
}

// acc[r] += sum_{m in [m0, m1)} tile[r][m] * wf[m][q0 + 2 lane ..]: forward contraction of the warp's rows against one output slice
template <int NS>
__device__ __forceinline__ void fcon(const WRows& a, const float* tile, int m0, int m1, const int* q0, float2 (*acc)[kRW], int lane) {
#pragma unroll 2
  for (int m = m0; m < m1; ++m) {
    float2 w[NS];
#pragma unroll
    for (int s = 0; s < NS; ++s) w[s] = ld2(a.wf + (long long)m * kQ + q0[s] + 2 * lane);
#pragma unroll
    for (int r = 0; r < kRW; ++r) {
      const float v = tile[r * kTP + m];
#pragma unroll
      for (int s = 0; s < NS; ++s) fma2(acc[s][r], v, w[s]);
    }
  }
}

// acc[r] = sum_{q in [q0, q1)} tile[r][q] * wb[q][m0 + 2 lane ..]: a 64-column block of d W^T for the warp's rows
__device__ __forceinline__ void dcon(const WRows& a, const float* tile, int q0, int q1, int m0, float2* acc, int lane) {
#pragma unroll
  for (int r = 0; r < kRW; ++r) acc[r] = make_float2(0.f, 0.f);
#pragma unroll 2
  for (int q = q0; q < q1; ++q) {
    const float2 w = ld2(a.wb + (long long)q * a.nbp + m0 + 2 * lane);
#pragma unroll
    for (int r = 0; r < kRW; ++r) fma2(acc[r], tile[r * kTP + q], w);
  }
}

// X columns of dS1 + dS2 = [dpz | dpr | dph] W^T over the X columns -> dsx rows of step t (lanes own columns)
__device__ __forceinline__ void write_dsx(const WRows& a, const float* tile, int t, long long base, int nr, int lane) {
  for (int m = lane; m < a.w; m += 32) {
    float acc[kRW];
#pragma unroll
    for (int r = 0; r < kRW; ++r) acc[r] = 0.f;
    for (int q = 0; q < kQ; ++q) {
      const float w = __ldg(a.wb + (long long)q * a.nbp + m);
#pragma unroll
      for (int r = 0; r < kRW; ++r) acc[r] = fmaf(tile[r * kTP + q], w, acc[r]);
    }
#pragma unroll
    for (int r = 0; r < kRW; ++r)
      if (r < nr) a.dsx[trow(a, t, base + r) * a.dsx_ld + m] = acc[r];
  }
}

#define WR_FOR(a, base)                                                                                                         \
  for (long long base = ((long long)blockIdx.x * kWarps + (threadIdx.x >> 5)) * kRW; base < (a).rows;                           \
       base += (long long)gridDim.x * kWarps * kRW)

__device__ __forceinline__ float bias(const float* b, int q) { return b ? __ldg(b + q) : 0.f; }

// ---- weight image -----------------------------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kThreads) k_dcrnn_wrows_image(WRows a, const float* __restrict__ wzrT, const float* __restrict__ whsT,
                                                                float* wf, float* wb) {
  const int C = a.cin + kCO, total = a.nbp * kQ;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int mp = idx / kQ, q = idx - mp * kQ;
    int m = -1;
    if (mp < a.w) m = (mp / a.cin) * C + mp % a.cin;
    else if (mp >= a.wp) m = ((mp - a.wp) / kCO) * C + a.cin + (mp - a.wp) % kCO;
    const float v = m < 0 ? 0.f : (q < 2 * kCO ? __ldg(wzrT + (size_t)q * a.nbc + m) : __ldg(whsT + (size_t)(q - 2 * kCO) * a.nbc + m));
    wf[idx] = v;
    wb[(size_t)q * a.nbp + mp] = v;
  }
}

// ---- forward ----------------------------------------------------------------------------------------------------------------------------

// step 0 on a finite plan: H_{-1} = 0, so R is dead and every H column is zero; pre = b + (X columns) W^T
__global__ void __launch_bounds__(kThreads, 2) k_dcrnn_wrows_fwd0(WRows a) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31;
  float* tile = smem + (threadIdx.x >> 5) * kRW * kTP;
  const int nb = 2 * a.K - 1, C = a.cin + kCO;
  WR_FOR(a, base) {
    const int nr = (int)min((long long)kRW, a.rows - base);
    for (int r = 0; r < nr; ++r) {
      const long long i = base + r;
      const int b = (int)(i / a.n), n = (int)(i - (long long)b * a.n);
      tile_x(a, tile + r * kTP, 0, b, n, trow(a, 0, i), lane);
    }
    __syncwarp();
    float2 acc[2][kRW];
    const int q0[2] = {0, 2 * kCO};
#pragma unroll
    for (int r = 0; r < kRW; ++r) {
      acc[0][r] = make_float2(bias(a.bz, 2 * lane), bias(a.bz, 2 * lane + 1));
      acc[1][r] = make_float2(bias(a.bh, 2 * lane), bias(a.bh, 2 * lane + 1));
    }
    fcon<2>(a, tile, 0, a.wp, q0, acc, lane);
#pragma unroll
    for (int r = 0; r < kRW; ++r) {
      if (r >= nr) break;
      const long long i = base + r, rr = trow(a, 0, i);
      const int b = (int)(i / a.n), n = (int)(i - (long long)b * a.n);
      const float2 z = make_float2(sigmoidf_acc(acc[0][r].x), sigmoidf_acc(acc[0][r].y));
      const float2 ht = make_float2(tanhf(acc[1][r].x), tanhf(acc[1][r].y));
      const float2 h = make_float2((1.f - z.x) * ht.x, (1.f - z.y) * ht.y);
      st2(outp(a, b, 0, n) + 2 * lane, h);
      st2(sblk(a, kHS, i) + 2 * lane, h);
      if (a.stash) {
        float* st = stashp(a, 0, i);
        st2(st + 2 * lane, z);
        st2(st + kCO + 2 * lane, make_float2(0.f, 0.f));   // R multiplies a zero state: its gradient term is zero
        st2(st + 2 * kCO + 2 * lane, ht);
      }
      if (a.S1)                              // the H columns of both bases are zero at step 0
        for (int j = 0; j < nb; ++j) {
          float* p1 = a.S1 + rr * a.nbc + j * C + a.cin + 2 * lane;
          float* p2 = a.S2 + rr * a.nbc + j * C + a.cin + 2 * lane;
          p1[0] = p1[1] = p2[0] = p2[1] = 0.f;
        }
    }
    __syncwarp();
  }
}

// hop a.hop of basis a.beta at step a.t; the last hop of each basis also does that basis's contraction and gate math
__global__ void __launch_bounds__(kThreads, 2) k_dcrnn_wrows_fwd(WRows a) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31;
  float* tile = smem + (threadIdx.x >> 5) * kRW * kTP;
  const int cin = a.cin, C = cin + kCO, nb = 2 * a.K - 1, t = a.t, k = a.hop, L = a.K - 1;
  const bool last = k == L;
  const int ub = a.beta == 1 ? kHS : kHR;    // U's H columns: H or H*R
  float* S = a.beta == 1 ? a.S1 : a.S2;
  WR_FOR(a, base) {
    const int nr = (int)min((long long)kRW, a.rows - base);
    for (int r = 0; r < nr; ++r) {
      const long long i = base + r, rr = trow(a, t, i);
      const int b = (int)(i / a.n), n = (int)(i - (long long)b * a.n);
      const float2 u = ld2s(sblk(a, ub, i) + 2 * lane);
      float2 v[2];
#pragma unroll
      for (int o = 0; o < 2; ++o) {
        v[o] = gather(a.rp[o], a.cv[o], n, gsrc(a, k == 1 ? ub : kHop0 + o, b, lane));
        if (k > 1) v[o] = make_float2(__fadd_rn(2.f * v[o].x, -u.x), __fadd_rn(2.f * v[o].y, -u.y));
        if (S) {
          float* p = S + rr * a.nbc + (1 + 2 * (k - 1) + o) * C + cin + 2 * lane;
          p[0] = v[o].x;
          p[1] = v[o].y;
        }
      }
      if (!last) {
#pragma unroll
        for (int o = 0; o < 2; ++o) st2(sblk(a, kHop0 + o, i) + 2 * lane, v[o]);
        continue;
      }
      float* tr = tile + r * kTP;
      for (int j = 0; j < nb; ++j) {         // the row's H-column blocks: U, the earlier hop (scratch) and this launch's hop
        const int kj = (j + 1) >> 1, oj = (j - 1) & 1;
        float2 hv;
        if (j == 0) hv = u;
        else if (kj < k) hv = ld2s(sblk(a, kHop0 + oj, i) + 2 * lane);
        else hv = oj ? v[1] : v[0];
        st2(tr + a.wp + j * kCO + 2 * lane, hv);
      }
      if (a.beta == 1) tile_x(a, tr, t, b, n, rr, lane);
    }
    if (!last) continue;
    __syncwarp();
    if (a.beta == 1) {
      float2 acc[3][kRW];
      const int q0[3] = {0, kCO, 2 * kCO};
#pragma unroll
      for (int r = 0; r < kRW; ++r) {
        acc[0][r] = make_float2(bias(a.bz, 2 * lane), bias(a.bz, 2 * lane + 1));
        acc[1][r] = make_float2(bias(a.br, 2 * lane), bias(a.br, 2 * lane + 1));
        acc[2][r] = make_float2(bias(a.bh, 2 * lane), bias(a.bh, 2 * lane + 1));
      }
      fcon<3>(a, tile, 0, a.wp, q0, acc, lane);
      fcon<2>(a, tile, a.wp, a.nbp, q0, acc, lane);
#pragma unroll
      for (int r = 0; r < kRW; ++r) {
        if (r >= nr) break;
        const long long i = base + r, rr = trow(a, t, i);
        const float2 u = ld2s(tile + r * kTP + a.wp + 2 * lane);
        const float2 z = make_float2(sigmoidf_acc(acc[0][r].x), sigmoidf_acc(acc[0][r].y));
        const float2 rg = make_float2(sigmoidf_acc(acc[1][r].x), sigmoidf_acc(acc[1][r].y));
        const float2 hr = make_float2(u.x * rg.x, u.y * rg.y);
        st2(sblk(a, kHR, i) + 2 * lane, hr);
        st2(sblk(a, kZB, i) + 2 * lane, z);
        st2(sblk(a, kPH, i) + 2 * lane, acc[2][r]);
        if (a.stash) {
          float* st = stashp(a, t, i);
          st2(st + 2 * lane, z);
          st2(st + kCO + 2 * lane, rg);
        }
        if (a.S1) {
          float* p1 = a.S1 + rr * a.nbc + cin + 2 * lane;
          float* p2 = a.S2 + rr * a.nbc + cin + 2 * lane;
          p1[0] = u.x; p1[1] = u.y;
          p2[0] = hr.x; p2[1] = hr.y;
        }
      }
    } else {
      float2 acc[1][kRW];
      const int q0[1] = {2 * kCO};
#pragma unroll
      for (int r = 0; r < kRW; ++r) acc[0][r] = r < nr ? ld2s(sblk(a, kPH, base + r) + 2 * lane) : make_float2(0.f, 0.f);
      fcon<1>(a, tile, a.wp, a.nbp, q0, acc, lane);
#pragma unroll
      for (int r = 0; r < kRW; ++r) {
        if (r >= nr) break;
        const long long i = base + r;
        const int b = (int)(i / a.n), n = (int)(i - (long long)b * a.n);
        const float2 z = ld2s(sblk(a, kZB, i) + 2 * lane), h = ld2s(sblk(a, kHS, i) + 2 * lane);
        const float2 ht = make_float2(tanhf(acc[0][r].x), tanhf(acc[0][r].y));
        const float2 hn = make_float2(z.x * h.x + (1.f - z.x) * ht.x, z.y * h.y + (1.f - z.y) * ht.y);
        st2(outp(a, b, t, n) + 2 * lane, hn);
        st2(sblk(a, kHS, i) + 2 * lane, hn);   // own row only: this launch's gathers read the H*R chain, not H
        if (a.stash) st2(stashp(a, t, i) + 2 * kCO + 2 * lane, ht);
      }
    }
    __syncwarp();
  }
}

// ---- backward ---------------------------------------------------------------------------------------------------------------------------

// elementwise start of step t for row i given g = dL/dH_t: dph, dpz -> dph_all / dpzr_all and the tile (dpr = 0 there); t >= 1: g, dph,
// dpz -> scratch
__device__ __forceinline__ void rowwise_elem(const WRows& a, float* tr, long long i, int t, float2 g, int lane) {
  const int b = (int)(i / a.n), n = (int)(i - (long long)b * a.n);
  const float* st = stashp(a, t, i);
  const float2 z = ld2s(st + 2 * lane), ht = ld2s(st + 2 * kCO + 2 * lane);
  const float2 hp = t ? ld2(outp(a, b, t - 1, n) + 2 * lane) : make_float2(0.f, 0.f);
  const long long r = trow(a, t, i);
  const float2 dph = make_float2(g.x * (1.f - z.x) * (1.f - ht.x * ht.x), g.y * (1.f - z.y) * (1.f - ht.y * ht.y));
  const float2 dpz = make_float2(g.x * (hp.x - ht.x) * z.x * (1.f - z.x), g.y * (hp.y - ht.y) * z.y * (1.f - z.y));
  st2(a.dph + r * kCO + 2 * lane, dph);
  st2(a.dpzr + r * 2 * kCO + 2 * lane, dpz);
  st2(tr + 2 * lane, dpz);
  st2(tr + kCO + 2 * lane, make_float2(0.f, 0.f));
  st2(tr + 2 * kCO + 2 * lane, dph);
  if (t == 0) {
    st2(a.dpzr + r * 2 * kCO + kCO + 2 * lane, make_float2(0.f, 0.f));
    return;
  }
  st2(sblk(a, kG, i) + 2 * lane, g);
  st2(sblk(a, kDPH, i) + 2 * lane, dph);
  st2(sblk(a, kDPZ, i) + 2 * lane, dpz);
}

// the contraction part of the rowwise start (tile holds the warp's d rows): t = 0: the X columns of dS1 + dS2; t >= 1: the top adjoint
// level of dS2's H columns -> A blocks of parity 1 - a.par (and SACC for K = 3)
__device__ __forceinline__ void rowwise_con(const WRows& a, const float* tile, long long base, int nr, int t, int lane) {
  if (t == 0) {
    if (a.dsx) write_dsx(a, tile, 0, base, nr, lane);
    return;
  }
  const int L = a.K - 1, w = 1 - a.par;
  float2 top[2][kRW];
#pragma unroll
  for (int o = 0; o < 2; ++o) dcon(a, tile, 2 * kCO, kQ, a.wp + (1 + 2 * (L - 1) + o) * kCO, top[o], lane);
#pragma unroll
  for (int r = 0; r < kRW; ++r) {
    if (r >= nr) break;
    const long long i = base + r;
#pragma unroll
    for (int o = 0; o < 2; ++o) st2(sblk(a, kA0 + 2 * w + o, i) + 2 * lane, top[o][r]);
    if (L >= 2) st2(sblk(a, kSACC, i) + 2 * lane, make_float2(top[0][r].x + top[1][r].x, top[0][r].y + top[1][r].y));
  }
}

__global__ void __launch_bounds__(kThreads, 2) k_dcrnn_wrows_bwd0(WRows a) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31;
  float* tile = smem + (threadIdx.x >> 5) * kRW * kTP;
  WR_FOR(a, base) {
    const int nr = (int)min((long long)kRW, a.rows - base);
    for (int r = 0; r < nr; ++r) {
      const long long i = base + r;
      const int b = (int)(i / a.n), n = (int)(i - (long long)b * a.n);
      const float2 g = ld2(a.gout + (((long long)b * a.T + a.t) * a.n + n) * kCO + 2 * lane);
      rowwise_elem(a, tile + r * kTP, i, a.t, g, lane);
    }
    __syncwarp();
    rowwise_con(a, tile, base, nr, a.t, lane);
    __syncwarp();
  }
}

// level a.hop of the transposed basis adjoint of dS_beta's H columns at step a.t >= 1:
//   A_{k-1} = D_{k-1} + 2 P^T A_k (k = 2; the -U term of T_2 = 2 P T_1 - U sits in SACC), or, at k = 1, dU = D_0 - SACC + P_o^T A_1o +
//   P_i^T A_1i, after which beta = 2 derives d(H*R), dpr and the top level of dS1, and beta = 1 completes dH_{t-1} and starts t-1.
__global__ void __launch_bounds__(kThreads, 2) k_dcrnn_wrows_bwd(WRows a) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31;
  float* tile = smem + (threadIdx.x >> 5) * kRW * kTP;
  const int t = a.t, k = a.hop, L = a.K - 1, p = a.par, w = 1 - p;
  const int q0 = a.beta == 2 ? 2 * kCO : 0, q1 = a.beta == 2 ? kQ : 2 * kCO;   // dph (h rows) or dpz | dpr (z | r rows)
  WR_FOR(a, base) {
    const int nr = (int)min((long long)kRW, a.rows - base);
    for (int r = 0; r < nr; ++r) {
      const long long i = base + r;
      const int b = (int)(i / a.n), n = (int)(i - (long long)b * a.n);
      float* tr = tile + r * kTP;
#pragma unroll
      for (int o = 0; o < 2; ++o) st2(tr + kTGat + o * kCO + 2 * lane, gather(a.rp[o], a.cv[o], n, gsrc(a, kA0 + 2 * p + o, b, lane)));
      if (a.beta == 2) {
        st2(tr + 2 * lane, ld2s(sblk(a, kDPZ, i) + 2 * lane));
        st2(tr + 2 * kCO + 2 * lane, ld2s(sblk(a, kDPH, i) + 2 * lane));
      } else {
        st2(tr + 2 * lane, ld2s(sblk(a, kDPZ, i) + 2 * lane));
        st2(tr + kCO + 2 * lane, ld2s(sblk(a, kDPR, i) + 2 * lane));
      }
    }
    __syncwarp();
    if (k >= 2) {
#pragma unroll
      for (int o = 0; o < 2; ++o) {
        float2 nv[kRW];
        dcon(a, tile, q0, q1, a.wp + (1 + 2 * (k - 2) + o) * kCO, nv, lane);
#pragma unroll
        for (int r = 0; r < kRW; ++r) {
          if (r >= nr) break;
          const float2 gv = ld2s(tile + r * kTP + kTGat + o * kCO + 2 * lane);
          st2(sblk(a, kA0 + 2 * w + o, base + r) + 2 * lane, make_float2(__fadd_rn(nv[r].x, 2.f * gv.x), __fadd_rn(nv[r].y, 2.f * gv.y)));
        }
      }
      __syncwarp();
      continue;
    }
    float2 du[kRW];
    dcon(a, tile, q0, q1, a.wp, du, lane);
#pragma unroll
    for (int r = 0; r < kRW; ++r) {
      if (r >= nr) break;
      const float* tr = tile + r * kTP;
      const float2 g0 = ld2s(tr + kTGat + 2 * lane), g1 = ld2s(tr + kTGat + kCO + 2 * lane);
      const float2 sacc = L >= 2 ? ld2s(sblk(a, kSACC, base + r) + 2 * lane) : make_float2(0.f, 0.f);
      du[r] = make_float2(du[r].x - sacc.x + g0.x + g1.x, du[r].y - sacc.y + g0.y + g1.y);
    }
    __syncwarp();                            // every lane has read the tile before it is rewritten
    if (a.beta == 2) {                       // du = d(H*R)
#pragma unroll
      for (int r = 0; r < kRW; ++r) {
        if (r >= nr) break;
        const long long i = base + r, rr = trow(a, t, i);
        const int b = (int)(i / a.n), n = (int)(i - (long long)b * a.n);
        const float* st = stashp(a, t, i);
        const float2 z = ld2s(st + 2 * lane), rg = ld2s(st + kCO + 2 * lane), g = ld2s(sblk(a, kG, i) + 2 * lane);
        const float2 hp = ld2(outp(a, b, t - 1, n) + 2 * lane);
        const float2 dpr = make_float2(du[r].x * hp.x * rg.x * (1.f - rg.x), du[r].y * hp.y * rg.y * (1.f - rg.y));
        st2(a.dpzr + rr * 2 * kCO + kCO + 2 * lane, dpr);
        st2(sblk(a, kDPR, i) + 2 * lane, dpr);
        st2(sblk(a, kDHP, i) + 2 * lane, make_float2(g.x * z.x + du[r].x * rg.x, g.y * z.y + du[r].y * rg.y));
        st2(tile + r * kTP + kCO + 2 * lane, dpr);
      }
      __syncwarp();
      if (a.dsx) write_dsx(a, tile, t, base, nr, lane);
      float2 top[2][kRW];
#pragma unroll
      for (int o = 0; o < 2; ++o) dcon(a, tile, 0, 2 * kCO, a.wp + (1 + 2 * (L - 1) + o) * kCO, top[o], lane);
#pragma unroll
      for (int r = 0; r < kRW; ++r) {
        if (r >= nr) break;
        const long long i = base + r;
#pragma unroll
        for (int o = 0; o < 2; ++o) st2(sblk(a, kA0 + 2 * w + o, i) + 2 * lane, top[o][r]);
        if (L >= 2) st2(sblk(a, kSACC, i) + 2 * lane, make_float2(top[0][r].x + top[1][r].x, top[0][r].y + top[1][r].y));
      }
    } else {                                 // du = dS1's share of dH_{t-1}
#pragma unroll
      for (int r = 0; r < kRW; ++r) {
        if (r >= nr) break;
        const long long i = base + r;
        const int b = (int)(i / a.n), n = (int)(i - (long long)b * a.n);
        const float2 dhp = ld2s(sblk(a, kDHP, i) + 2 * lane);
        const float2 go = ld2(a.gout + (((long long)b * a.T + t - 1) * a.n + n) * kCO + 2 * lane);
        rowwise_elem(a, tile + r * kTP, i, t - 1, make_float2(go.x + (dhp.x + du[r].x), go.y + (dhp.y + du[r].y)), lane);
      }
      __syncwarp();
      rowwise_con(a, tile, base, nr, t - 1, lane);
    }
    __syncwarp();
  }
}

}  // namespace
}  // namespace stmp

using namespace stmp;

static bool wrows_envelope(int64_t cin, int64_t cout, int64_t K) { return cin >= 1 && cin <= 4 && cout == kCO && (K == 2 || K == 3); }

extern "C" int stmp_dcrnn_wide_rows_supported(const stmp_plan* plan, int64_t cin, int64_t cout, int64_t K) {
  return plan && plan->flavor == STMP_FLAVOR_DCONV && plan->n_ops == 2 && wrows_envelope(cin, cout, K) ? 1 : 0;
}

extern "C" int64_t stmp_dcrnn_wide_rows_scratch_bytes(const stmp_plan* plan, int64_t B, int64_t cout, int64_t K) {
  if (!plan || B <= 0 || cout != kCO || K < 2 || K > 3) return 0;
  return (kImgFloats + (int64_t)kBlocks * plan->n * B * kCO) * 4;
}

static int wrows_check(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K, const char* who) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: plan is NULL", who);
  STMP_REQUIRE(plan->flavor == STMP_FLAVOR_DCONV && plan->n_ops == 2, STMP_EINVAL, "%s: plan is not a DConv plan", who);
  STMP_REQUIRE(wrows_envelope(cin, cout, K), STMP_EUNSUPPORTED, "%s: cin 1..4, cout = 64 and K 2..3 only (got %lld, %lld, %lld)", who,
               (long long)cin, (long long)cout, (long long)K);
  STMP_REQUIRE(B >= 0 && T >= 0, STMP_EINVAL, "%s: negative B/T", who);
  STMP_REQUIRE(B * plan->n < (1ll << 40) && T < (1ll << 31) && B < (1ll << 31), STMP_ESHAPE, "%s: B * N too large", who);
  return STMP_OK;
}

static WRows wrows_params(const stmp_plan* plan, bool transposed, int64_t B, int64_t T, int64_t cin, int64_t K, float* scratch) {
  WRows a = {};
  for (int op = 0; op < 2; ++op) {
    const Csr& c = transposed ? plan->bwd[op] : plan->fwd[op];
    a.rp[op] = c.rowptr;
    a.cv[op] = c.cv;
  }
  a.n = plan->n; a.B = (int)B; a.T = (int)T; a.cin = (int)cin; a.K = (int)K;
  const int nb = 2 * (int)K - 1;
  a.nbc = nb * (int)(cin + kCO);
  a.w = nb * (int)cin;
  a.wp = (a.w + 3) / 4 * 4;
  a.nbp = a.wp + nb * kCO;
  a.rows = (long long)B * plan->n;
  a.blk = a.rows * kCO;
  a.wf = scratch;
  a.wb = scratch + kImgFloats / 2;
  a.scr = scratch + kImgFloats;
  return a;
}

static int wrows_grid(long long rows) {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long blocks = (rows + kWarps * kRW - 1) / (kWarps * kRW);
  return (int)(blocks < 32ll * sms ? (blocks > 0 ? blocks : 1) : 32ll * sms);
}

static int wrows_image(const WRows& a, const float* wzrT, const float* whsT, cudaStream_t st) {
  const int total = a.nbp * kQ;
  k_dcrnn_wrows_image<<<(total + kThreads - 1) / kThreads, kThreads, 0, st>>>(a, wzrT, whsT, const_cast<float*>(a.wf),
                                                                              const_cast<float*>(a.wb));
  STMP_LAUNCH_OK("k_dcrnn_wrows_image");
  return STMP_OK;
}

// every kernel takes kSmem bytes of dynamic shared memory: the attribute is per device, so it is set on every call (no stream work)
static int wrows_smem() {
  STMP_CUDA_OK(cudaFuncSetAttribute(k_dcrnn_wrows_fwd0, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  STMP_CUDA_OK(cudaFuncSetAttribute(k_dcrnn_wrows_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  STMP_CUDA_OK(cudaFuncSetAttribute(k_dcrnn_wrows_bwd0, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  STMP_CUDA_OK(cudaFuncSetAttribute(k_dcrnn_wrows_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
  return STMP_OK;
}

extern "C" int stmp_dcrnn_wide_rows_fwd(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K, const float* x,
                                        int64_t x_bstride, int64_t x_tstride, int64_t x_ld, int64_t x_blk, const float* wzrT,
                                        const float* whsT, const float* bz, const float* br, const float* bh, float* scratch, float* out,
                                        float* stash, float* S1, float* S2, void* stream) {
  const char* who = "stmp_dcrnn_wide_rows_fwd";
  const int rc = wrows_check(plan, B, T, cin, cout, K, who);
  if (rc != STMP_OK) return rc;
  STMP_REQUIRE(!stash == !S1 && !S1 == !S2, STMP_EINVAL, "%s: give stash, S1 and S2 together or none of them", who);
  STMP_REQUIRE((x || S1) && wzrT && whsT && out && scratch, STMP_EINVAL, "%s: NULL tensor", who);
  const void* ps[] = {x, wzrT, whsT, bz, br, bh, S1, S2};
  for (const void* p : ps) STMP_REQUIRE(((uintptr_t)p & 3u) == 0, STMP_ESHAPE, "%s: misaligned tensor", who);
  STMP_REQUIRE((((uintptr_t)scratch | (uintptr_t)stash | (uintptr_t)out) & 15u) == 0, STMP_ESHAPE,
               "%s: scratch, stash and out must be 16-byte aligned", who);
  if (B == 0 || T == 0) return STMP_OK;
  WRows a = wrows_params(plan, false, B, T, cin, K, scratch);
  if (S1) {                                  // training: the X blocks are S1's X columns
    a.x = S1; a.xld = a.nbc; a.xbs = (long long)plan->n * a.nbc; a.xts = B * a.xbs; a.xblk = (int)(cin + cout);
  } else {
    STMP_REQUIRE(x_ld >= cin && x_blk >= cin && x_bstride >= 0 && x_tstride >= 0, STMP_ESHAPE, "%s: bad X block strides", who);
    a.x = x; a.xld = x_ld; a.xbs = x_bstride; a.xts = x_tstride; a.xblk = (int)x_blk;
  }
  a.bz = bz; a.br = br; a.bh = bh;
  a.out = out; a.stash = stash; a.S1 = S1; a.S2 = S2;
  cudaStream_t st = (cudaStream_t)stream;
  int e = wrows_smem();
  if (e == STMP_OK) e = wrows_image(a, wzrT, whsT, st);
  if (e != STMP_OK) return e;
  const int grid = wrows_grid(a.rows), L = a.K - 1;
  for (int t = 0; t < a.T; ++t) {
    a.t = t;
    if (t == 0 && !plan->nonfinite_vals) {
      k_dcrnn_wrows_fwd0<<<grid, kThreads, kSmem, st>>>(a);
      STMP_LAUNCH_OK("k_dcrnn_wrows_fwd0");
      continue;
    }
    if (t == 0) STMP_CUDA_OK(cudaMemsetAsync(a.scr + kHS * a.blk, 0, a.blk * sizeof(float), st));   // the chain on a zero state
    for (int beta = 1; beta <= 2; ++beta)
      for (int k = 1; k <= L; ++k) {
        a.beta = beta;
        a.hop = k;
        k_dcrnn_wrows_fwd<<<grid, kThreads, kSmem, st>>>(a);
        STMP_LAUNCH_OK("k_dcrnn_wrows_fwd");
      }
  }
  return STMP_OK;
}

extern "C" int stmp_dcrnn_wide_rows_bwd(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K, const float* gout,
                                        const float* out, const float* stash, const float* wzrT, const float* whsT, float* scratch,
                                        float* dph_all, float* dpzr_all, float* dsx, int64_t dsx_ld, void* stream) {
  const char* who = "stmp_dcrnn_wide_rows_bwd";
  const int rc = wrows_check(plan, B, T, cin, cout, K, who);
  if (rc != STMP_OK) return rc;
  STMP_REQUIRE(gout && out && stash && wzrT && whsT && scratch && dph_all && dpzr_all, STMP_EINVAL, "%s: NULL tensor", who);
  const void* ps[] = {wzrT, whsT, dsx};
  for (const void* p : ps) STMP_REQUIRE(((uintptr_t)p & 3u) == 0, STMP_ESHAPE, "%s: misaligned tensor", who);
  STMP_REQUIRE((((uintptr_t)scratch | (uintptr_t)stash | (uintptr_t)gout | (uintptr_t)out | (uintptr_t)dph_all | (uintptr_t)dpzr_all) &
                15u) == 0, STMP_ESHAPE, "%s: scratch, stash, gout, out, dph_all and dpzr_all must be 16-byte aligned", who);
  STMP_REQUIRE(!dsx || dsx_ld >= (2 * K - 1) * cin, STMP_ESHAPE, "%s: the dS row pitch must hold (2K-1) cin columns", who);
  if (B == 0 || T == 0) return STMP_OK;
  WRows a = wrows_params(plan, true, B, T, cin, K, scratch);
  a.out = const_cast<float*>(out); a.gout = gout; a.stash = const_cast<float*>(stash);
  a.dph = dph_all; a.dpzr = dpzr_all; a.dsx = dsx; a.dsx_ld = dsx_ld;
  cudaStream_t st = (cudaStream_t)stream;
  int e = wrows_smem();
  if (e == STMP_OK) e = wrows_image(a, wzrT, whsT, st);
  if (e != STMP_OK) return e;
  const int grid = wrows_grid(a.rows), L = a.K - 1;
  a.t = a.T - 1;
  a.par = 1;                                 // the start writes the A blocks of parity 0
  k_dcrnn_wrows_bwd0<<<grid, kThreads, kSmem, st>>>(a);
  STMP_LAUNCH_OK("k_dcrnn_wrows_bwd0");
  int p = 0;
  for (int t = a.T - 1; t >= 1; --t)
    for (int beta = 2; beta >= 1; --beta)
      for (int k = L; k >= 1; --k) {
        a.t = t;
        a.beta = beta;
        a.hop = k;
        a.par = p;
        k_dcrnn_wrows_bwd<<<grid, kThreads, kSmem, st>>>(a);
        STMP_LAUNCH_OK("k_dcrnn_wrows_bwd");
        p ^= 1;
      }
  return STMP_OK;
}
