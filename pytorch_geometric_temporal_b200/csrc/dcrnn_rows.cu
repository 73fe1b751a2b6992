// dcrnn_rows.cu -- BatchedDCRNN at 32 hidden channels (K = 2, cin 1..4) on graphs of ANY size, split over CTAs by destination rows
// (DESIGN §4k).  All B windows of a step share each launch; a step's two all-to-all dependencies -- P(H*R) in the forward and the
// transposed products in the backward -- split it into a short chain of launches, each a gather + contraction + gate math fused per
// (window, row).  The basis is DConv's [U | P_o U | P_i U] (U = [X | H], C = cin + 32 columns per block, nb = 3C <= 108):
//
//   forward, step t >= 1  k_dcrnn_rows_fwd_a<1>  gather P_o, P_i of [X_t | H_{t-1}]; Z, R, H*R and the X half of pre_h -> scratch
//                         k_dcrnn_rows_fwd_b     gather P_o, P_i of H*R; pre_h, Ht = tanh(pre_h), H_t = Z*H + (1-Z)*Ht -> out[:, t]
//   forward, step 0       k_dcrnn_rows_fwd_a<0>  H_{-1} = 0: R is dead and H*R = 0, so the step is one launch.  A plan whose operators
//                                                hold a non-finite value (DConv's 1/deg = inf at a node of in-degree 0) runs step 0
//                                                as the two launches above on a zero state instead: inf * 0 = NaN then spreads
//                                                through P(H*R) exactly as it does in the reference.
//   backward, reverse time
//     k_dcrnn_rows_bwd_start<T0>  rowwise start of step T-1: dph, dpz, dS2 = dph W_h^T
//     k_dcrnn_rows_bwd_b          P_o^T / P_i^T of dS2's operator blocks -> d(H*R), dpr, dS1 = [dpz | dpr] W_zr^T, own-row dH / dX parts
//     k_dcrnn_rows_bwd_c<T0>      P_o^T / P_i^T of dS1's operator blocks -> dH_{t-1}, dX_t complete; then the rowwise start of step t-1
//     k_dcrnn_rows_bwd_x          step 0's dX (only when asked for): P_o^T / P_i^T of the X columns of dS1 + dS2's operator blocks
//
// Mapping (rows.cuh): one warp per (window, destination row), lane = output channel (and X channel for lane < cin); CTAs own tiles of
// kRowTile consecutive rows of the B*N row space, grid-strided, and stage the weight rows they need once in shared memory at an odd
// pitch (kDPitch = 109 >= 108 columns), so lane-indexed rows and lane-indexed columns are both free of bank conflicts.  Exact fp32 FFMA;
// gathers walk the plan's CSR rows in entry order.  No atomics: every value depends on its own row's fixed-order sums, so repeated
// calls are bit-identical.
#include "rows.cuh"

namespace stmp {
namespace {

using namespace rows;
constexpr int kDPitch = 109;                 // staged weight row: basis columns 0..107 (nb = 3 (cin + 32) <= 108)
constexpr int kFP = 96;                      // forward scratch row: H*R | X half of pre_h | Z
constexpr int kBP = 256;                     // backward scratch row:
constexpr int kQ = 112;                      //   [0, nb) dS2 in basis order | [kQ, kQ + 2C) Q = dS1's operator blocks |
constexpr int kGo = 184, kDH = 216, kDX = 248;   //   g = dL/dH_t | dH_{t-1} own-row part | dX_t own-row part (cin)
constexpr int kStash = 96;                   // stash row: Z | R | Ht

struct DRows {
  const int* rp[2]; const int2* cv[2];       // P_o, P_i: by destination (forward) or by source (backward, the transposed products)
  int n, B, T, t, cin, nb, ld;
  const float* x; const long long* ws;       // X_t of window b at x + (ws ? ws[b] * xt : b * xb) + t * xt
  long long xb, xt;
  const float* wzr; const float* wh;         // (64, nb) z | r rows, (32, nb) h rows: rows are outputs, columns basis columns
  const float* bz; const float* br; const float* bh;   // nullable
  float* out;                                // (B, T, N, 32)
  float* scr;                                // (B*N, kFP) forward / (B*N, kBP) backward
  float* stash;                              // (T, B, N, 96), nullable in the forward
  float* S1; float* S2;                      // (T*B*N, ld), nullable
  const float* gout;                         // (B, T, N, 32)
  float* dph; float* dpzr;                   // (T, B, N, 32), (T, B, N, 64)
  float* dx;                                 // (B, T, N, cin), nullable
};

// rows [0, nr) of w [nr][nb] -> ws [nr][kDPitch] (columns >= nb zero); the caller syncs
__device__ __forceinline__ void stage(float* ws, const float* __restrict__ w, int nb, int nr) {
  for (int i = threadIdx.x; i < nr * kDPitch; i += kRowsThreads) {
    const int r = i / kDPitch, m = i - r * kDPitch;
    ws[i] = m < nb ? __ldg(w + (size_t)r * nb + m) : 0.f;
  }
}

// staged column of basis column lane + 32 q in the 4-chunk contractions: columns past the row's end read the zero padding at kDPitch - 1
// (nb <= 108 < kDPitch), so the chunk q = 3 never leaves the row
__device__ __forceinline__ int wcol(int lane, int q) { return min(lane + 32 * q, kDPitch - 1); }

__device__ __forceinline__ const float* xrow(const DRows& a, int b, int t) {
  return a.x + (a.ws ? __ldg(a.ws + b) * a.xt : (long long)b * a.xb) + (long long)t * a.xt;
}

__device__ __forceinline__ const float* hrow(const DRows& a, int b, int t) {     // out[b, t] as an (N, 32) block
  return a.out + ((size_t)b * a.T + t) * a.n * kCo;
}

// sum_e val_e * 0 over CSR row i in entry order: +0, or NaN where an entry is not finite (P applied to a zero state)
__device__ __forceinline__ float gather_zero(const int* __restrict__ rowptr, const int2* __restrict__ cv, int i) {
  float s = 0.f;
  for (int k = __ldg(rowptr + i), end = __ldg(rowptr + i + 1); k < end; ++k) s = __fadd_rn(s, __fmul_rn(__int_as_float(__ldg(&cv[k].y)), 0.f));
  return s;
}

// HAS_H = 1: launch A of a two-launch step (t = 0: a zero state).  HAS_H = 0: the whole of step 0.
template <bool HAS_H>
__global__ void __launch_bounds__(kRowsThreads, 2) k_dcrnn_rows_fwd_a(DRows a) {
  extern __shared__ float ws[];              // z | r | h rows: [96][kDPitch]
  stage(ws, a.wzr, a.nb, 2 * kCo);
  stage(ws + 2 * kCo * kDPitch, a.wh, a.nb, kCo);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + kCo, t = a.t, rows = a.B * a.n;
  const float bz = a.bz ? __ldg(a.bz + lane) : 0.f, br = a.br ? __ldg(a.br + lane) : 0.f, bh = a.bh ? __ldg(a.bh + lane) : 0.f;
  const bool zero_h = !HAS_H || t == 0;
  for (int t0 = blockIdx.x * kRowTile; t0 < rows; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, rows);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const int b = i / a.n, n = i - b * a.n;
      const float* xb = xrow(a, b, t);
      const float* hb = zero_h ? nullptr : hrow(a, b, t - 1);
      const float xv = lane < cin ? __ldg(xb + (size_t)n * cin + lane) : 0.f;
      const float hv = hb ? __ldg(hb + (size_t)n * kCo + lane) : 0.f;
      float lh[2], lx[2];
#pragma unroll
      for (int op = 0; op < 2; ++op) {
        if (hb) {
          gather_row<true>(a.rp[op], a.cv[op], n, hb, kCo, xb, cin, cin, lane, lh[op], lx[op]);
        } else {
          gather_row<false>(a.rp[op], a.cv[op], n, nullptr, 0, xb, cin, cin, lane, lh[op], lx[op]);
          if (HAS_H) lh[op] = gather_zero(a.rp[op], a.cv[op], n);
        }
      }
      float pz = bz, pr = br, ph = bh;       // pre = b + S W^T in basis order; ph takes the X columns only when H is carried
#pragma unroll
      for (int blk = 0; blk < 3; ++blk) {
        const float sx = blk ? lx[blk - 1] : xv, sh = blk ? lh[blk - 1] : hv;
        const float* wb = ws + blk * C;
        for (int c = 0; c < cin; ++c) {
          const float s = __shfl_sync(0xffffffffu, sx, c);
          pz = fmaf(s, wb[lane * kDPitch + c], pz);
          if (HAS_H) pr = fmaf(s, wb[(kCo + lane) * kDPitch + c], pr);
          ph = fmaf(s, wb[(2 * kCo + lane) * kDPitch + c], ph);
        }
        if (HAS_H) {
#pragma unroll 8
          for (int o = 0; o < kCo; ++o) {
            const float s = __shfl_sync(0xffffffffu, sh, o);
            pz = fmaf(s, wb[lane * kDPitch + cin + o], pz);
            pr = fmaf(s, wb[(kCo + lane) * kDPitch + cin + o], pr);
          }
        }
      }
      const float Z = sigmoidf_acc(pz);
      const size_t ri = ((size_t)t * a.B + b) * a.n + n;         // row of the (T, B, N) training operands
      float* st = a.stash ? a.stash + ri * kStash : nullptr;
      if (HAS_H) {
        const float R = sigmoidf_acc(pr), hr = hv * R;
        float* s = a.scr + (size_t)i * kFP;
        s[lane] = hr;
        s[kCo + lane] = ph;
        s[2 * kCo + lane] = Z;
        if (st) {
          st[lane] = Z;
          st[kCo + lane] = R;
        }
        if (a.S2) a.S2[ri * a.ld + cin + lane] = hr;
      } else {
        const float Ht = tanhf(ph);
        a.out[((size_t)b * a.T + t) * a.n * kCo + (size_t)n * kCo + lane] = (1.f - Z) * Ht;
        if (st) {
          st[lane] = Z;
          st[kCo + lane] = 0.f;              // R multiplies a zero state: its gradient term is zero
          st[2 * kCo + lane] = Ht;
        }
      }
      if (a.S1) {                            // S1 = [X | H | P_o X | P_o H | P_i X | P_i H] (+ zero padding); S2's X columns
        float* r1 = a.S1 + ri * a.ld;
        float* r2 = a.S2 + ri * a.ld;
#pragma unroll
        for (int blk = 0; blk < 3; ++blk) {
          const float sx = blk ? lx[blk - 1] : xv;
          if (lane < cin) r1[blk * C + lane] = r2[blk * C + lane] = sx;
          r1[blk * C + cin + lane] = blk ? lh[blk - 1] : hv;
          if (!HAS_H) r2[blk * C + cin + lane] = 0.f;            // H*R and its diffusions are zero at step 0
        }
        if (a.nb + lane < a.ld) r1[a.nb + lane] = r2[a.nb + lane] = 0.f;
      }
    }
  }
}

__global__ void __launch_bounds__(kRowsThreads, 2) k_dcrnn_rows_fwd_b(DRows a) {
  extern __shared__ float ws[];              // h rows: [32][kDPitch]
  stage(ws, a.wh, a.nb, kCo);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + kCo, t = a.t, rows = a.B * a.n;
  for (int t0 = blockIdx.x * kRowTile; t0 < rows; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, rows);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const int b = i / a.n, n = i - b * a.n;
      const float* sw = a.scr + (size_t)b * a.n * kFP;          // this window's scratch block
      const float* s = sw + (size_t)n * kFP;
      const float hr = s[lane], Z = s[2 * kCo + lane];
      float ph = s[kCo + lane], l[2], unused;
#pragma unroll
      for (int op = 0; op < 2; ++op) gather_row<true>(a.rp[op], a.cv[op], n, sw, kFP, nullptr, 0, 0, lane, l[op], unused);
#pragma unroll
      for (int blk = 0; blk < 3; ++blk) {
        const float sh = blk ? l[blk - 1] : hr;
        const float* wr = ws + lane * kDPitch + blk * C + cin;
#pragma unroll 8
        for (int o = 0; o < kCo; ++o) ph = fmaf(__shfl_sync(0xffffffffu, sh, o), wr[o], ph);
      }
      const float hv = t ? __ldg(hrow(a, b, t - 1) + (size_t)n * kCo + lane) : 0.f;
      const float Ht = tanhf(ph);
      a.out[((size_t)b * a.T + t) * a.n * kCo + (size_t)n * kCo + lane] = Z * hv + (1.f - Z) * Ht;
      const size_t ri = ((size_t)t * a.B + b) * a.n + n;
      if (a.stash) a.stash[ri * kStash + 2 * kCo + lane] = Ht;
      if (a.S2) {
        a.S2[ri * a.ld + C + cin + lane] = l[0];
        a.S2[ri * a.ld + 2 * C + cin + lane] = l[1];
      }
    }
  }
}

// The rowwise start of step t for row (b, n) given g = dL/dH_t: dph, dpz -> dph_all / dpzr_all; dS2 = dph W_h^T -> the scratch row
// (t >= 1, read by k_dcrnn_rows_bwd_b) and g.  T0 (t = 0, H_{-1} = 0): dpr = 0, and with dx the X columns of dS2 + dS1 (dS1 = [dpz | 0]
// W_zr^T): own block -> the dX part, operator blocks -> the scratch row's dS2 slots (read by k_dcrnn_rows_bwd_x).
template <bool T0>
__device__ __forceinline__ void rowwise(const DRows& a, const float* wsh, const float* wsz, int b, int n, int t, float g, int lane) {
  const int cin = a.cin, C = cin + kCo;
  const size_t ri = ((size_t)t * a.B + b) * a.n + n;
  const float* st = a.stash + ri * kStash;
  const float Z = st[lane], Ht = st[2 * kCo + lane];
  const float hp = T0 ? 0.f : hrow(a, b, t - 1)[(size_t)n * kCo + lane];
  const float dph = g * (1.f - Z) * (1.f - Ht * Ht);
  const float dpz = g * (hp - Ht) * Z * (1.f - Z);
  a.dph[ri * kCo + lane] = dph;
  a.dpzr[ri * 2 * kCo + lane] = dpz;
  if (T0) a.dpzr[ri * 2 * kCo + kCo + lane] = 0.f;
  if (T0 && !a.dx) return;
  float* sr = a.scr + ((size_t)b * a.n + n) * kBP;
  float d2[4] = {0.f, 0.f, 0.f, 0.f}, d1[4] = {0.f, 0.f, 0.f, 0.f};          // basis columns m = lane + 32 q
#pragma unroll 4
  for (int o = 0; o < kCo; ++o) {
    const float s2 = __shfl_sync(0xffffffffu, dph, o);
    const float s1 = T0 ? __shfl_sync(0xffffffffu, dpz, o) : 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      d2[q] = fmaf(s2, wsh[o * kDPitch + wcol(lane, q)], d2[q]);
      if (T0) d1[q] = fmaf(s1, wsz[o * kDPitch + wcol(lane, q)], d1[q]);
    }
  }
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int m = lane + 32 * q;
    if (m >= a.nb) continue;
    if (!T0) {
      sr[m] = d2[q];
    } else {                                 // only the X columns carry a gradient at step 0
      const float v = d2[q] + d1[q];
      if (m < cin) sr[kDX + m] = v;
      else if ((m >= C && m < C + cin) || (m >= 2 * C && m < 2 * C + cin)) sr[m] = v;
    }
  }
  if (!T0) sr[kGo + lane] = g;
}

template <bool T0>
__global__ void __launch_bounds__(kRowsThreads, 2) k_dcrnn_rows_bwd_start(DRows a) {
  extern __shared__ float ws[];              // h rows [32][kDPitch], then (T0 with dx) z rows
  stage(ws, a.wh, a.nb, kCo);
  if (T0 && a.dx) stage(ws + kCo * kDPitch, a.wzr, a.nb, kCo);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, t = a.t, rows = a.B * a.n;
  for (int t0 = blockIdx.x * kRowTile; t0 < rows; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, rows);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const int b = i / a.n, n = i - b * a.n;
      const float g = a.gout[((size_t)b * a.T + t) * a.n * kCo + (size_t)n * kCo + lane];
      rowwise<T0>(a, ws, ws + kCo * kDPitch, b, n, t, g, lane);
    }
  }
}

// step t >= 1: gather P_o^T / P_i^T of dS2's operator blocks (H columns; X columns too with dx) -> d(H*R), dpr, dS1 = [dpz | dpr]
// W_zr^T; the own-row parts of dH_{t-1} and dX_t, and Q = dS1's operator blocks for k_dcrnn_rows_bwd_c.
__global__ void __launch_bounds__(kRowsThreads, 2) k_dcrnn_rows_bwd_b(DRows a) {
  extern __shared__ float ws[];              // z | r rows: [64][kDPitch], then one 128-float row buffer per warp
  stage(ws, a.wzr, a.nb, 2 * kCo);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + kCo, t = a.t, rows = a.B * a.n;
  const int nx = a.dx ? cin : 0;
  float* sb = ws + 2 * kCo * kDPitch + warp * 128;
  for (int t0 = blockIdx.x * kRowTile; t0 < rows; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, rows);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const int b = i / a.n, n = i - b * a.n;
      const float* pw = a.scr + (size_t)b * a.n * kBP;          // this window's scratch block
      float* sr = a.scr + (size_t)i * kBP;
      float th[2], tx[2];
#pragma unroll
      for (int op = 0; op < 2; ++op)
        gather_row<true>(a.rp[op], a.cv[op], n, pw + (op + 1) * C + cin, kBP, pw + (op + 1) * C, kBP, nx, lane, th[op], tx[op]);
      const float dhr = sr[cin + lane] + th[0] + th[1];
      const size_t ri = ((size_t)t * a.B + b) * a.n + n;
      const float* st = a.stash + ri * kStash;
      const float Z = st[lane], R = st[kCo + lane], g = sr[kGo + lane];
      const float hp = hrow(a, b, t - 1)[(size_t)n * kCo + lane];
      const float dpr = dhr * hp * R * (1.f - R);
      const float dpz = a.dpzr[ri * 2 * kCo + lane];
      a.dpzr[ri * 2 * kCo + kCo + lane] = dpr;
      float d1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
      for (int o = 0; o < kCo; ++o) {
        const float sz = __shfl_sync(0xffffffffu, dpz, o), sp = __shfl_sync(0xffffffffu, dpr, o);
#pragma unroll
        for (int q = 0; q < 4; ++q)
          d1[q] = fmaf(sp, ws[(kCo + o) * kDPitch + wcol(lane, q)], fmaf(sz, ws[o * kDPitch + wcol(lane, q)], d1[q]));
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) sb[lane + 32 * q] = d1[q];
      __syncwarp();
      sr[kDH + lane] = g * Z + dhr * R + sb[cin + lane];
      if (lane < nx) sr[kDX + lane] = sr[lane] + sb[lane] + tx[0] + tx[1];
      for (int c = lane; c < 2 * C; c += 32) sr[kQ + c] = sb[C + c];
      __syncwarp();
    }
  }
}

// step t >= 1: gather P_o^T / P_i^T of Q -> dH_{t-1} (complete), dX_t (with dx); then the rowwise start of step t - 1 (T0: t - 1 = 0).
template <bool T0>
__global__ void __launch_bounds__(kRowsThreads, 2) k_dcrnn_rows_bwd_c(DRows a) {
  extern __shared__ float ws[];              // h rows [32][kDPitch], then (T0 with dx) z rows
  stage(ws, a.wh, a.nb, kCo);
  if (T0 && a.dx) stage(ws + kCo * kDPitch, a.wzr, a.nb, kCo);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + kCo, t = a.t, rows = a.B * a.n;
  const int nx = a.dx ? cin : 0;
  for (int t0 = blockIdx.x * kRowTile; t0 < rows; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, rows);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const int b = i / a.n, n = i - b * a.n;
      const float* qw = a.scr + (size_t)b * a.n * kBP + kQ;
      const float* sr = a.scr + (size_t)i * kBP;
      float th[2], tx[2];
#pragma unroll
      for (int op = 0; op < 2; ++op) gather_row<true>(a.rp[op], a.cv[op], n, qw + op * C + cin, kBP, qw + op * C, kBP, nx, lane, th[op], tx[op]);
      const float dh = sr[kDH + lane] + th[0] + th[1];
      if (lane < nx) a.dx[(((size_t)b * a.T + t) * a.n + n) * cin + lane] = sr[kDX + lane] + tx[0] + tx[1];
      const float g = a.gout[((size_t)b * a.T + t - 1) * a.n * kCo + (size_t)n * kCo + lane] + dh;
      rowwise<T0>(a, ws, ws + kCo * kDPitch, b, n, t - 1, g, lane);
    }
  }
}

// step 0's dX: own-row part + P_o^T / P_i^T of the X columns that k_dcrnn_rows_bwd_*<T0> left in the dS2 slots
__global__ void __launch_bounds__(kRowsThreads) k_dcrnn_rows_bwd_x(DRows a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + kCo, rows = a.B * a.n;
  for (int t0 = blockIdx.x * kRowTile; t0 < rows; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, rows);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const int b = i / a.n, n = i - b * a.n;
      const float* pw = a.scr + (size_t)b * a.n * kBP;
      float tx[2], unused;
#pragma unroll
      for (int op = 0; op < 2; ++op) gather_row<false>(a.rp[op], a.cv[op], n, nullptr, 0, pw + (op + 1) * C, kBP, cin, lane, unused, tx[op]);
      if (lane < cin) a.dx[((size_t)b * a.T * a.n + n) * cin + lane] = a.scr[(size_t)i * kBP + kDX + lane] + tx[0] + tx[1];
    }
  }
}

}  // namespace
}  // namespace stmp

using namespace stmp;

static bool drows_envelope(int64_t cin, int64_t cout, int64_t K) { return cout == kCo && K == 2 && cin >= 1 && cin <= 4; }

static int drows_ld(int64_t cin) { return (3 * ((int)cin + kCo) + 7) / 8 * 8; }

extern "C" int stmp_dcrnn_rows_supported(const stmp_plan* plan, int64_t cin, int64_t cout, int64_t K) {
  return plan && plan->flavor == STMP_FLAVOR_DCONV && plan->n_ops == 2 && drows_envelope(cin, cout, K) ? 1 : 0;
}

extern "C" int64_t stmp_dcrnn_rows_scratch_bytes(const stmp_plan* plan, int64_t B) {
  return plan && B > 0 ? (int64_t)B * plan->n * kBP * 4 : 0;
}

static int drows_check(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, const char* who) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: plan is NULL", who);
  STMP_REQUIRE(plan->flavor == STMP_FLAVOR_DCONV && plan->n_ops == 2, STMP_EINVAL, "%s: plan is not a DConv plan", who);
  STMP_REQUIRE(drows_envelope(cin, kCo, 2), STMP_EUNSUPPORTED, "%s: cin 1..4 only (got %lld)", who, (long long)cin);
  STMP_REQUIRE(B >= 0 && T >= 0, STMP_EINVAL, "%s: negative B/T", who);
  STMP_REQUIRE(B * plan->n < (1ll << 31) && B * T * plan->n < (1ll << 40), STMP_ESHAPE, "%s: B * N too large for one launch", who);
  return STMP_OK;
}

static DRows drows_params(const stmp_plan* plan, bool transposed, int64_t B, int64_t T, int64_t cin) {
  DRows a = {};
  for (int op = 0; op < 2; ++op) {
    const Csr& c = transposed ? plan->bwd[op] : plan->fwd[op];
    a.rp[op] = c.rowptr;
    a.cv[op] = c.cv;
  }
  a.n = plan->n; a.B = (int)B; a.T = (int)T; a.cin = (int)cin; a.nb = 3 * ((int)cin + kCo); a.ld = drows_ld(cin);
  return a;
}

extern "C" int stmp_dcrnn_rows_fwd(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, const float* x, const int64_t* win_start,
                                   int64_t x_bstride, int64_t x_tstride, const float* wzrT, const float* whsT, const float* bz,
                                   const float* br, const float* bh, float* scratch, float* out, float* stash, float* S1, float* S2,
                                   int64_t ld, void* stream) {
  const int rc = drows_check(plan, B, T, cin, "stmp_dcrnn_rows_fwd");
  if (rc != STMP_OK) return rc;
  STMP_REQUIRE(x && wzrT && whsT && scratch && out, STMP_EINVAL, "stmp_dcrnn_rows_fwd: NULL tensor");
  STMP_REQUIRE(!stash == !S1 && !S1 == !S2, STMP_EINVAL, "stmp_dcrnn_rows_fwd: give stash, S1 and S2 together or none of them");
  STMP_REQUIRE(!S1 || ld == drows_ld(cin), STMP_ESHAPE, "stmp_dcrnn_rows_fwd: the basis row pitch must be 3(cin+32) rounded up to 8");
  const void* ps[] = {x, wzrT, whsT, bz, br, bh, scratch, out, stash};
  for (const void* p : ps) STMP_REQUIRE(al4(p), STMP_ESHAPE, "stmp_dcrnn_rows_fwd: misaligned tensor");
  STMP_REQUIRE((((uintptr_t)S1 | (uintptr_t)S2) & 15u) == 0, STMP_ESHAPE, "stmp_dcrnn_rows_fwd: S1 / S2 must be 16-byte aligned");
  if (B == 0 || T == 0) return STMP_OK;
  DRows a = drows_params(plan, false, B, T, cin);
  a.x = x; a.ws = reinterpret_cast<const long long*>(win_start); a.xb = x_bstride; a.xt = x_tstride;
  a.wzr = wzrT; a.wh = whsT; a.bz = bz; a.br = br; a.bh = bh;
  a.out = out; a.scr = scratch; a.stash = stash; a.S1 = S1; a.S2 = S2;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = rows_grid((int)(B * plan->n)), smem_a = 3 * kCo * kDPitch * 4, smem_b = kCo * kDPitch * 4;
  for (int t = 0; t < (int)T; ++t) {
    a.t = t;
    if (t == 0 && !plan->nonfinite_vals) {
      k_dcrnn_rows_fwd_a<false><<<grid, kRowsThreads, smem_a, st>>>(a);
      STMP_LAUNCH_OK("k_dcrnn_rows_fwd_a");
      continue;
    }
    k_dcrnn_rows_fwd_a<true><<<grid, kRowsThreads, smem_a, st>>>(a);
    STMP_LAUNCH_OK("k_dcrnn_rows_fwd_a");
    k_dcrnn_rows_fwd_b<<<grid, kRowsThreads, smem_b, st>>>(a);
    STMP_LAUNCH_OK("k_dcrnn_rows_fwd_b");
  }
  return STMP_OK;
}

extern "C" int stmp_dcrnn_rows_bwd(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, const float* gout, const float* out,
                                   const float* stash, const float* wzrT, const float* whsT, float* scratch, float* dph_all,
                                   float* dpzr_all, float* dx, void* stream) {
  const int rc = drows_check(plan, B, T, cin, "stmp_dcrnn_rows_bwd");
  if (rc != STMP_OK) return rc;
  STMP_REQUIRE(gout && out && stash && wzrT && whsT && scratch && dph_all && dpzr_all, STMP_EINVAL, "stmp_dcrnn_rows_bwd: NULL tensor");
  const void* ps[] = {gout, out, stash, wzrT, whsT, scratch, dph_all, dpzr_all, dx};
  for (const void* p : ps) STMP_REQUIRE(al4(p), STMP_ESHAPE, "stmp_dcrnn_rows_bwd: misaligned tensor");
  if (B == 0 || T == 0) return STMP_OK;
  DRows a = drows_params(plan, true, B, T, cin);
  a.out = const_cast<float*>(out); a.gout = gout; a.stash = const_cast<float*>(stash); a.wzr = wzrT; a.wh = whsT;
  a.scr = scratch; a.dph = dph_all; a.dpzr = dpzr_all; a.dx = dx;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = rows_grid((int)(B * plan->n));
  const int smem_h = 2 * kCo * kDPitch * 4, smem_b = (2 * kCo * kDPitch + kRowsWarps * 128) * 4;
  STMP_CUDA_OK(cudaFuncSetAttribute(k_dcrnn_rows_bwd_b, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_b));
  a.t = (int)T - 1;
  if (T == 1) {
    k_dcrnn_rows_bwd_start<true><<<grid, kRowsThreads, smem_h, st>>>(a);
  } else {
    k_dcrnn_rows_bwd_start<false><<<grid, kRowsThreads, smem_h, st>>>(a);
  }
  STMP_LAUNCH_OK("k_dcrnn_rows_bwd_start");
  for (int t = (int)T - 1; t >= 1; --t) {
    a.t = t;
    k_dcrnn_rows_bwd_b<<<grid, kRowsThreads, smem_b, st>>>(a);
    STMP_LAUNCH_OK("k_dcrnn_rows_bwd_b");
    if (t == 1) {
      k_dcrnn_rows_bwd_c<true><<<grid, kRowsThreads, smem_h, st>>>(a);
    } else {
      k_dcrnn_rows_bwd_c<false><<<grid, kRowsThreads, smem_h, st>>>(a);
    }
    STMP_LAUNCH_OK("k_dcrnn_rows_bwd_c");
  }
  if (dx) {
    a.t = 0;
    k_dcrnn_rows_bwd_x<<<grid, kRowsThreads, 0, st>>>(a);
    STMP_LAUNCH_OK("k_dcrnn_rows_bwd_x");
  }
  return STMP_OK;
}
