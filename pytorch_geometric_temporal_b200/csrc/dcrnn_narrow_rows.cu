// dcrnn_narrow_rows.cu -- BatchedDCRNN for narrow states (cout 1..4, cin 1..4, K 1..4: the reference's BatchedDCRNN(F, F, K=3)) on
// graphs of ANY size, split over CTAs by destination rows (DESIGN §4l).  The row-split scheme of §4i / §4k -- one launch per all-to-all
// dependency, every launch serving all B windows of a step -- with the state kept node-major, because one window's row (<= 4 floats) is
// too narrow to give a warp a gather:
//
//   scratch blocks (N, B, CP) floats, CP = cout padded to 1, 2 or 4 (one vector load per (row, window)); row (n, b) at (n B + b) CP
//
// Mapping: a lane owns one (destination row, window).  Lane groups of G = min(32, 2^ceil(log2 B)) lanes own one row each and take
// consecutive windows, so all lanes of a group walk the same CSR row (entries are broadcast, trip counts uniform) and each source row's
// gather is one contiguous G * CP read.  B >= 32: a warp is one row and ceil(B / 32) window groups follow each other; B < 32: a warp
// holds 32 / G rows (their trip counts differ, as in any one-row-per-lane-group kernel).  Every multiply-add of a (window, row) happens in
// CSR entry order whatever B is.  Weights ((2K-1)(cin+cout) x 3 cout <= 56 x 12) are staged once per CTA in shared memory and read as
// broadcasts.  Exact fp32; no atomics: every value depends only on its own row's fixed-order sums, so repeated calls are bit-identical.
//
// The basis of U = [X | H] is [U | P_o U | P_i U | 2 P_o T_1o - U | 2 P_i T_1i - U | ...] (T_k = 2 P T_{k-1} - U for k >= 2: the reference
// never advances Tx_0 past U, dcrnn.py:_basis); block j = 1 + 2 (k - 1) + o is hop k of operator o.  The X blocks do not depend on the
// recurrence: the caller builds them for all (t, b) before the time loop (stmp_spmm), and the per-step chain gathers only the H columns.
//
//   forward, K >= 2, step t >= 1: L = K - 1 launches per basis, k_dcrnn_nrows_fwd (hop k of [.. | H] / [.. | H*R]); the last hop of the
//     first basis also computes Z, R, H*R and the X part of pre_h, the last hop of the second Ht and H_t.  Step 0 (H = 0) is one rowwise
//     launch, k_dcrnn_nrows_fwd0, unless the plan holds a non-finite operator value: then step 0 runs the full chain on a zeroed state,
//     so inf * 0 = NaN spreads exactly as in the reference.  K = 1 has no graph coupling: one launch for the sequence, k_dcrnn_nrows_seq1.
//   backward, K >= 2, reverse time: k_dcrnn_nrows_bwd0 (rowwise start of step T-1), then per step t >= 1 L transposed-gather launches of
//     the adjoint of dS2's H columns and L of dS1's, k_dcrnn_nrows_bwd (level k of the adjoint; the last level of dS2 yields d(H*R), dpr
//     and starts dS1, the last level of dS1 completes dH_{t-1} and runs the rowwise start of step t-1).  Step 0 needs no gather: its
//     state had no predecessor.  K = 1: one launch, k_dcrnn_nrows_bseq1.  The X columns of dS1 + dS2 are written rowwise for every (t, b);
//     the caller applies the transposed basis adjoint to them once, after the loop.
#include "common.cuh"

namespace stmp {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxNbc = 7 * 8;               // (2K - 1)(cin + cout) <= 56

// scratch blocks of the forward
constexpr int kHS = 0, kHR = 1, kZB = 2, kPH = 3, kHop0 = 4;            // H | H*R | Z | X part of pre_h | hop k, op o at kHop0 + 2 (k-1) + o
// ... and of the backward
constexpr int kG = 0, kDPH = 1, kDPZ = 2, kDPR = 3, kDHP = 4, kSACC = 5, kA0 = 6;   // A(parity p, op o) at kA0 + 2 p + o
constexpr int kBlocks = 10;                  // the larger of the two (forward: 4 + 2 (K-1) <= 10)

template <int CO> struct Cp { static constexpr int v = CO == 3 ? 4 : CO; };
template <int CP> struct Vf { float v[CP]; };

template <int CP> __device__ __forceinline__ Vf<CP> ldv(const float* p);
template <> __device__ __forceinline__ Vf<1> ldv<1>(const float* p) { return {{__ldg(p)}}; }
template <> __device__ __forceinline__ Vf<2> ldv<2>(const float* p) {
  const float2 t = __ldg(reinterpret_cast<const float2*>(p));
  return {{t.x, t.y}};
}
template <> __device__ __forceinline__ Vf<4> ldv<4>(const float* p) {
  const float4 t = __ldg(reinterpret_cast<const float4*>(p));
  return {{t.x, t.y, t.z, t.w}};
}
template <int CP> __device__ __forceinline__ void stv(float* p, const Vf<CP>& a);
template <> __device__ __forceinline__ void stv<1>(float* p, const Vf<1>& a) { *p = a.v[0]; }
template <> __device__ __forceinline__ void stv<2>(float* p, const Vf<2>& a) { *reinterpret_cast<float2*>(p) = make_float2(a.v[0], a.v[1]); }
template <> __device__ __forceinline__ void stv<4>(float* p, const Vf<4>& a) {
  *reinterpret_cast<float4*>(p) = make_float4(a.v[0], a.v[1], a.v[2], a.v[3]);
}
template <int CP> __device__ __forceinline__ Vf<CP> zv() {
  Vf<CP> r;
#pragma unroll
  for (int c = 0; c < CP; ++c) r.v[c] = 0.f;
  return r;
}

struct NRows {
  const int* rp[2]; const int2* cv[2];       // P_o, P_i: by destination (forward) or by source (backward, the transposed products)
  int n, B, T, t, cin, K, nbc, G, lg, WG;    // nbc = (2K-1)(cin+cout); G = lanes per row group = 1 << lg; WG window groups per row
  int items; long long blk;                  // lanes to visit (n * WG * G < 2^31), floats per scratch block (n * B * CP)
  const float* x; long long xbs, xts, xld; int xblk;   // X block j of (t, b, n): x + t xts + b xbs + n xld + j xblk
  const float* wzr; const float* wh;         // (2 cout, nbc) z | r rows, (cout, nbc) h rows: rows are outputs, columns basis columns
  const float* bz; const float* br; const float* bh;   // nullable
  float* out;                                // (B, T, N, cout)
  float* scr;                                // kBlocks scratch blocks
  float* stash;                              // (T, N, B, 3 CP): Z | R | Ht, nullable in the forward
  float* S1; float* S2;                      // (T*B, N, nbc), nullable
  const float* gout;                         // (B, T, N, cout)
  float* dph; float* dpzr;                   // (T, B, N, cout), (T, B, N, 2 cout)
  float* dsx; long long dsx_ld;              // (T*B, N, dsx_ld): X columns of dS1 + dS2, block j at j * cin; nullable
  int beta, hop, par;                        // this launch: basis (1: [X | H], 2: [X | H*R]), hop / adjoint level, A-block parity read
};

// weights as ws[m][q], q = z outputs | r outputs | h outputs (3 CO floats per basis column m); every lane reads the same word
template <int CO>
__device__ __forceinline__ void stage(float* ws, const NRows& a) {
  constexpr int Q = 3 * CO;
  for (int i = threadIdx.x; i < a.nbc * Q; i += blockDim.x) {
    const int m = i / Q, q = i - m * Q;
    ws[i] = q < 2 * CO ? __ldg(a.wzr + (size_t)q * a.nbc + m) : __ldg(a.wh + (size_t)(q - 2 * CO) * a.nbc + m);
  }
  __syncthreads();
}

// acc[q] += s * w[m][q0 + q] for q < CO
template <int CO>
__device__ __forceinline__ void mac(float* acc, float s, const float* wm) {
#pragma unroll
  for (int q = 0; q < CO; ++q) acc[q] = fmaf(s, wm[q], acc[q]);
}

// sum_q d[q] w[m][q0 + q]: a column of d W^T
template <int CO>
__device__ __forceinline__ float dot(const float* d, const float* wm) {
  float s = 0.f;
#pragma unroll
  for (int q = 0; q < CO; ++q) s = fmaf(d[q], wm[q], s);
  return s;
}

// (row, window) of lane item i; false for the lanes past B in the last window group
__device__ __forceinline__ bool item(const NRows& a, int i, int& n, int& b) {
  const int task = i >> a.lg;               // 32-bit: items < 2^31 (nrows_check)
  n = task / a.WG;
  b = (task - n * a.WG) * a.G + (i & (a.G - 1));
  return b < a.B;
}

#define NR_FOR(a) for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < (a).items; i += gridDim.x * blockDim.x)

template <int CP>
__device__ __forceinline__ float* sblk(const NRows& a, int k, int n, int b) { return a.scr + k * a.blk + ((long long)n * a.B + b) * CP; }

__device__ __forceinline__ long long trow(const NRows& a, int t, int b, int n) { return ((long long)t * a.B + b) * a.n + n; }

__device__ __forceinline__ const float* xrow(const NRows& a, int t, int b, int n) {
  return a.x + t * a.xts + b * a.xbs + n * a.xld;
}

template <int CO>
__device__ __forceinline__ float* outp(const NRows& a, int b, int t, int n) { return a.out + (((long long)b * a.T + t) * a.n + n) * CO; }

template <int CP>
__device__ __forceinline__ float* stashp(const NRows& a, int t, int n, int b) {
  return a.stash + (((long long)t * a.n + n) * a.B + b) * (3 * CP);
}

// sum_e val_e * src[col_e] (window b) over CSR row n, in entry order
template <int CP>
__device__ __forceinline__ Vf<CP> gather(const int* __restrict__ rowptr, const int2* __restrict__ cv, int n, const float* __restrict__ src,
                                         int B, int b) {
  Vf<CP> s = zv<CP>();
  const int beg = __ldg(rowptr + n), end = __ldg(rowptr + n + 1);
  int k = beg;
  for (; k + 4 <= end; k += 4) {
    int2 e[4];
    Vf<CP> v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) e[u] = __ldg(cv + k + u);
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = ldv<CP>(src + ((long long)e[u].x * B + b) * CP);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float w = __int_as_float(e[u].y);
#pragma unroll
      for (int c = 0; c < CP; ++c) s.v[c] = __fadd_rn(s.v[c], __fmul_rn(w, v[u].v[c]));
    }
  }
  for (; k < end; ++k) {
    const int2 e = __ldg(cv + k);
    const Vf<CP> v = ldv<CP>(src + ((long long)e.x * B + b) * CP);
    const float w = __int_as_float(e.y);
#pragma unroll
    for (int c = 0; c < CP; ++c) s.v[c] = __fadd_rn(s.v[c], __fmul_rn(w, v.v[c]));
  }
  return s;
}

// ---- forward ----------------------------------------------------------------------------------------------------------------------------

// step 0 of K >= 2 on a finite plan: H_{-1} = 0, so R is dead and every H column is zero; pre = b + (X columns) W^T
template <int CO>
__global__ void __launch_bounds__(kThreads, 2) k_dcrnn_nrows_fwd0(NRows a) {
  constexpr int CP = Cp<CO>::v, Q = 3 * CO;
  __shared__ float ws[kMaxNbc * Q];
  stage<CO>(ws, a);
  const int cin = a.cin, C = cin + CO, nb = 2 * a.K - 1;
  NR_FOR(a) {
    int n, b;
    if (!item(a, i, n, b)) continue;
    float pz[CO], ph[CO];
#pragma unroll
    for (int q = 0; q < CO; ++q) {
      pz[q] = a.bz ? __ldg(a.bz + q) : 0.f;
      ph[q] = a.bh ? __ldg(a.bh + q) : 0.f;
    }
    const float* xr = xrow(a, 0, b, n);
    const long long r = trow(a, 0, b, n);
    for (int j = 0; j < nb; ++j)
      for (int c = 0; c < cin; ++c) {
        const float s = __ldg(xr + j * a.xblk + c);
        const float* wm = ws + (j * C + c) * Q;
        mac<CO>(pz, s, wm);
        mac<CO>(ph, s, wm + 2 * CO);
        if (a.S2) a.S2[r * a.nbc + j * C + c] = s;
      }
    Vf<CP> h = zv<CP>(), z = zv<CP>(), ht = zv<CP>();
#pragma unroll
    for (int q = 0; q < CO; ++q) {
      z.v[q] = sigmoidf_acc(pz[q]);
      ht.v[q] = tanhf(ph[q]);
      h.v[q] = (1.f - z.v[q]) * ht.v[q];
      outp<CO>(a, b, 0, n)[q] = h.v[q];
    }
    stv<CP>(sblk<CP>(a, kHS, n, b), h);
    if (a.stash) {
      float* st = stashp<CP>(a, 0, n, b);
      stv<CP>(st, z);
      stv<CP>(st + CP, zv<CP>());            // R multiplies a zero state: its gradient term is zero
      stv<CP>(st + 2 * CP, ht);
    }
    if (a.S1)                                // the H columns of both bases are zero at step 0
      for (int j = 0; j < nb; ++j)
#pragma unroll
        for (int q = 0; q < CO; ++q) a.S1[r * a.nbc + j * C + cin + q] = a.S2[r * a.nbc + j * C + cin + q] = 0.f;
  }
}

// hop a.hop of basis a.beta at step a.t (K >= 2); the last hop of each basis also does that basis's contraction and gate math
template <int CO>
__global__ void __launch_bounds__(kThreads, 2) k_dcrnn_nrows_fwd(NRows a) {
  constexpr int CP = Cp<CO>::v, Q = 3 * CO;
  __shared__ float ws[kMaxNbc * Q];
  stage<CO>(ws, a);
  const int cin = a.cin, C = cin + CO, nb = 2 * a.K - 1, t = a.t, k = a.hop, L = a.K - 1;
  const bool last = k == L;
  const int ub = a.beta == 1 ? kHS : kHR;    // U's H columns: H or H*R
  float* S = a.beta == 1 ? a.S1 : a.S2;
  NR_FOR(a) {
    int n, b;
    if (!item(a, i, n, b)) continue;
    const Vf<CP> u = ldv<CP>(sblk<CP>(a, ub, n, b));
    Vf<CP> v[2];
#pragma unroll
    for (int o = 0; o < 2; ++o) {
      const float* src = a.scr + (k == 1 ? ub : kHop0 + 2 * (k - 2) + o) * a.blk;
      v[o] = gather<CP>(a.rp[o], a.cv[o], n, src, a.B, b);
      if (k > 1) {
#pragma unroll
        for (int c = 0; c < CP; ++c) v[o].v[c] = __fadd_rn(2.f * v[o].v[c], -u.v[c]);
      }
    }
    const long long r = trow(a, t, b, n);
    if (S)
#pragma unroll
      for (int o = 0; o < 2; ++o)
#pragma unroll
        for (int q = 0; q < CO; ++q) S[r * a.nbc + (1 + 2 * (k - 1) + o) * C + cin + q] = v[o].v[q];
    if (!last) {
#pragma unroll
      for (int o = 0; o < 2; ++o) stv<CP>(sblk<CP>(a, kHop0 + 2 * (k - 1) + o, n, b), v[o]);
      continue;
    }
    // the row's H-column blocks: U, the earlier hops (scratch) and this launch's hop
    float acc[3 * CO];
    if (a.beta == 1) {
#pragma unroll
      for (int q = 0; q < CO; ++q) {
        acc[q] = a.bz ? __ldg(a.bz + q) : 0.f;
        acc[CO + q] = a.br ? __ldg(a.br + q) : 0.f;
        acc[2 * CO + q] = a.bh ? __ldg(a.bh + q) : 0.f;
      }
      const float* xr = xrow(a, t, b, n);
      for (int j = 0; j < nb; ++j)
        for (int c = 0; c < cin; ++c) {
          const float s = __ldg(xr + j * a.xblk + c);
          mac<3 * CO>(acc, s, ws + (j * C + c) * Q);
          if (a.S2) a.S2[r * a.nbc + j * C + c] = s;
        }
    } else {
      const Vf<CP> p = ldv<CP>(sblk<CP>(a, kPH, n, b));
#pragma unroll
      for (int q = 0; q < CO; ++q) acc[2 * CO + q] = p.v[q];
    }
    for (int j = 0; j < nb; ++j) {
      const int kj = (j + 1) >> 1, oj = (j - 1) & 1;
      Vf<CP> hv;
      if (j == 0) hv = u;
      else if (kj < k) hv = ldv<CP>(sblk<CP>(a, kHop0 + 2 * (kj - 1) + oj, n, b));
      else if (oj) hv = v[1];
      else hv = v[0];
#pragma unroll
      for (int c = 0; c < CO; ++c) {
        const float* wm = ws + (j * C + cin + c) * Q;
        if (a.beta == 1) mac<2 * CO>(acc, hv.v[c], wm);
        else mac<CO>(acc + 2 * CO, hv.v[c], wm + 2 * CO);
      }
    }
    if (a.beta == 1) {
      Vf<CP> z = zv<CP>(), rr = zv<CP>(), hr = zv<CP>(), ph = zv<CP>();
#pragma unroll
      for (int q = 0; q < CO; ++q) {
        z.v[q] = sigmoidf_acc(acc[q]);
        rr.v[q] = sigmoidf_acc(acc[CO + q]);
        hr.v[q] = u.v[q] * rr.v[q];
        ph.v[q] = acc[2 * CO + q];
      }
      stv<CP>(sblk<CP>(a, kHR, n, b), hr);
      stv<CP>(sblk<CP>(a, kZB, n, b), z);
      stv<CP>(sblk<CP>(a, kPH, n, b), ph);
      if (a.stash) {
        float* st = stashp<CP>(a, t, n, b);
        stv<CP>(st, z);
        stv<CP>(st + CP, rr);
      }
      if (a.S1)
#pragma unroll
        for (int q = 0; q < CO; ++q) {
          a.S1[r * a.nbc + cin + q] = u.v[q];
          a.S2[r * a.nbc + cin + q] = hr.v[q];
        }
    } else {
      const Vf<CP> z = ldv<CP>(sblk<CP>(a, kZB, n, b)), h = ldv<CP>(sblk<CP>(a, kHS, n, b));
      Vf<CP> hn = zv<CP>(), ht = zv<CP>();
#pragma unroll
      for (int q = 0; q < CO; ++q) {
        ht.v[q] = tanhf(acc[2 * CO + q]);
        hn.v[q] = z.v[q] * h.v[q] + (1.f - z.v[q]) * ht.v[q];
        outp<CO>(a, b, t, n)[q] = hn.v[q];
      }
      stv<CP>(sblk<CP>(a, kHS, n, b), hn);   // own row only: this launch's gathers read the H*R chain, not H
      if (a.stash) stv<CP>(stashp<CP>(a, t, n, b) + 2 * CP, ht);
    }
  }
}

// K = 1: no graph coupling; each lane runs its (row, window) through every step with H in registers
template <int CO>
__global__ void __launch_bounds__(kThreads, 2) k_dcrnn_nrows_seq1(NRows a) {
  constexpr int CP = Cp<CO>::v, Q = 3 * CO;
  __shared__ float ws[kMaxNbc * Q];
  stage<CO>(ws, a);
  const int cin = a.cin;
  NR_FOR(a) {
    int n, b;
    if (!item(a, i, n, b)) continue;
    float h[CO];
#pragma unroll
    for (int q = 0; q < CO; ++q) h[q] = 0.f;
    for (int t = 0; t < a.T; ++t) {
      float acc[3 * CO];
#pragma unroll
      for (int q = 0; q < CO; ++q) {
        acc[q] = a.bz ? __ldg(a.bz + q) : 0.f;
        acc[CO + q] = a.br ? __ldg(a.br + q) : 0.f;
        acc[2 * CO + q] = a.bh ? __ldg(a.bh + q) : 0.f;
      }
      const float* xr = xrow(a, t, b, n);
      const long long r = trow(a, t, b, n);
      for (int c = 0; c < cin; ++c) {
        const float s = __ldg(xr + c);
        mac<3 * CO>(acc, s, ws + c * Q);
        if (a.S2) a.S2[r * a.nbc + c] = s;
      }
#pragma unroll
      for (int c = 0; c < CO; ++c) mac<2 * CO>(acc, h[c], ws + (cin + c) * Q);
      Vf<CP> z = zv<CP>(), rr = zv<CP>(), ht = zv<CP>();
      float hr[CO];
#pragma unroll
      for (int q = 0; q < CO; ++q) {
        z.v[q] = sigmoidf_acc(acc[q]);
        rr.v[q] = sigmoidf_acc(acc[CO + q]);
        hr[q] = h[q] * rr.v[q];
      }
#pragma unroll
      for (int c = 0; c < CO; ++c) mac<CO>(acc + 2 * CO, hr[c], ws + (cin + c) * Q + 2 * CO);
#pragma unroll
      for (int q = 0; q < CO; ++q) {
        ht.v[q] = tanhf(acc[2 * CO + q]);
        if (a.S1) {
          a.S1[r * a.nbc + cin + q] = h[q];
          a.S2[r * a.nbc + cin + q] = hr[q];
        }
        h[q] = z.v[q] * h[q] + (1.f - z.v[q]) * ht.v[q];
        outp<CO>(a, b, t, n)[q] = h[q];
      }
      if (a.stash) {
        float* st = stashp<CP>(a, t, n, b);
        stv<CP>(st, z);
        stv<CP>(st + CP, rr);
        stv<CP>(st + 2 * CP, ht);
      }
    }
  }
}

// ---- backward ---------------------------------------------------------------------------------------------------------------------------

// X columns of dS1 + dS2 = [dpz | dpr] W_zr^T + dph W_h^T for every block -> dsx row r
template <int CO>
__device__ __forceinline__ void write_dsx(const NRows& a, const float* ws, long long r, const float* dpzr, const float* dph) {
  const int cin = a.cin, C = cin + CO, nb = 2 * a.K - 1;
  float* d = a.dsx + r * a.dsx_ld;
  for (int j = 0; j < nb; ++j)
    for (int c = 0; c < cin; ++c) {
      const float* wm = ws + (j * C + c) * 3 * CO;
      d[j * cin + c] = dot<2 * CO>(dpzr, wm) + dot<CO>(dph, wm + 2 * CO);
    }
}

// D of one H-column block j: d W^T over outputs [q0, q0 + NQ) (dph with the h rows, [dpz | dpr] with the z | r rows)
template <int CO, int NQ>
__device__ __forceinline__ Vf<Cp<CO>::v> dblock(const NRows& a, const float* ws, int j, const float* d, int q0) {
  Vf<Cp<CO>::v> r = zv<Cp<CO>::v>();
  const int C = a.cin + CO;
#pragma unroll
  for (int c = 0; c < CO; ++c) r.v[c] = dot<NQ>(d, ws + (j * C + a.cin + c) * 3 * CO + q0);
  return r;
}

// rowwise start of step t for (n, b) given g = dL/dH_t: dph, dpz -> dph_all / dpzr_all; t >= 1: g, dph, dpz and the top adjoint level
// of dS2's H columns -> scratch (A blocks of parity 1 - a.par); t = 0: dpr = 0 and only the X columns of dS1 + dS2 remain
template <int CO>
__device__ __forceinline__ void rowwise(const NRows& a, const float* ws, int n, int b, int t, const float* g) {
  constexpr int CP = Cp<CO>::v;
  const float* st = stashp<CP>(a, t, n, b);
  const Vf<CP> z = ldv<CP>(st), ht = ldv<CP>(st + 2 * CP);
  const float* hprev = t ? outp<CO>(a, b, t - 1, n) : nullptr;
  const long long r = trow(a, t, b, n);
  float dph[CO], dpzr[2 * CO];
  Vf<CP> vg = zv<CP>(), vh = zv<CP>(), vz = zv<CP>();
#pragma unroll
  for (int q = 0; q < CO; ++q) {
    const float h = hprev ? __ldg(hprev + q) : 0.f;
    dph[q] = g[q] * (1.f - z.v[q]) * (1.f - ht.v[q] * ht.v[q]);
    dpzr[q] = g[q] * (h - ht.v[q]) * z.v[q] * (1.f - z.v[q]);
    dpzr[CO + q] = 0.f;
    a.dph[r * CO + q] = dph[q];
    a.dpzr[r * 2 * CO + q] = dpzr[q];
    vg.v[q] = g[q];
    vh.v[q] = dph[q];
    vz.v[q] = dpzr[q];
  }
  if (t == 0) {
#pragma unroll
    for (int q = 0; q < CO; ++q) a.dpzr[r * 2 * CO + CO + q] = 0.f;
    if (a.dsx) write_dsx<CO>(a, ws, r, dpzr, dph);
    return;
  }
  stv<CP>(sblk<CP>(a, kG, n, b), vg);
  stv<CP>(sblk<CP>(a, kDPH, n, b), vh);
  stv<CP>(sblk<CP>(a, kDPZ, n, b), vz);
  const int L = a.K - 1, w = 1 - a.par;
  Vf<CP> top[2];
#pragma unroll
  for (int o = 0; o < 2; ++o) {
    top[o] = dblock<CO, CO>(a, ws, 1 + 2 * (L - 1) + o, dph, 2 * CO);
    stv<CP>(sblk<CP>(a, kA0 + 2 * w + o, n, b), top[o]);
  }
  if (L >= 2) {
    Vf<CP> s;
#pragma unroll
    for (int c = 0; c < CP; ++c) s.v[c] = top[0].v[c] + top[1].v[c];
    stv<CP>(sblk<CP>(a, kSACC, n, b), s);
  }
}

template <int CO>
__global__ void __launch_bounds__(kThreads, 2) k_dcrnn_nrows_bwd0(NRows a) {
  constexpr int Q = 3 * CO;
  __shared__ float ws[kMaxNbc * Q];
  stage<CO>(ws, a);
  NR_FOR(a) {
    int n, b;
    if (!item(a, i, n, b)) continue;
    float g[CO];
    const float* go = a.gout + (((long long)b * a.T + a.t) * a.n + n) * CO;
#pragma unroll
    for (int q = 0; q < CO; ++q) g[q] = __ldg(go + q);
    rowwise<CO>(a, ws, n, b, a.t, g);
  }
}

// level a.hop of the transposed basis adjoint of dS_beta's H columns at step a.t >= 1:
//   A_{k-1} = D_{k-1} + 2 P^T A_k (k >= 2; the -U terms of T_k = 2 P T_{k-1} - U collect in SACC), or, at k = 1, dU = D_0 - SACC + P_o^T
//   A_1o + P_i^T A_1i, after which beta = 2 derives d(H*R), dpr and the top level of dS1, and beta = 1 completes dH_{t-1} and starts t-1.
template <int CO>
__global__ void __launch_bounds__(kThreads, 2) k_dcrnn_nrows_bwd(NRows a) {
  constexpr int CP = Cp<CO>::v, Q = 3 * CO;
  __shared__ float ws[kMaxNbc * Q];
  stage<CO>(ws, a);
  const int t = a.t, k = a.hop, L = a.K - 1, p = a.par, w = 1 - p;
  NR_FOR(a) {
    int n, b;
    if (!item(a, i, n, b)) continue;
    Vf<CP> gv[2];
#pragma unroll
    for (int o = 0; o < 2; ++o) gv[o] = gather<CP>(a.rp[o], a.cv[o], n, a.scr + (kA0 + 2 * p + o) * a.blk, a.B, b);
    float d[2 * CO];                         // beta = 2: dph (h rows); beta = 1: dpz | dpr (z | r rows)
    {
      const Vf<CP> d0 = ldv<CP>(sblk<CP>(a, a.beta == 2 ? kDPH : kDPZ, n, b));
      Vf<CP> d1 = zv<CP>();
      if (a.beta == 1) d1 = ldv<CP>(sblk<CP>(a, kDPR, n, b));
#pragma unroll
      for (int q = 0; q < CO; ++q) {
        d[q] = d0.v[q];
        d[CO + q] = d1.v[q];
      }
    }
    if (k >= 2) {
      Vf<CP> nv[2];
#pragma unroll
      for (int o = 0; o < 2; ++o) {
        const int j = 1 + 2 * (k - 2) + o;
        if (a.beta == 2) nv[o] = dblock<CO, CO>(a, ws, j, d, 2 * CO);
        else nv[o] = dblock<CO, 2 * CO>(a, ws, j, d, 0);
#pragma unroll
        for (int c = 0; c < CP; ++c) nv[o].v[c] = __fadd_rn(nv[o].v[c], 2.f * gv[o].v[c]);
        stv<CP>(sblk<CP>(a, kA0 + 2 * w + o, n, b), nv[o]);
      }
      if (k - 1 >= 2) {
        Vf<CP> s = ldv<CP>(sblk<CP>(a, kSACC, n, b));
#pragma unroll
        for (int c = 0; c < CP; ++c) s.v[c] = s.v[c] + nv[0].v[c] + nv[1].v[c];
        stv<CP>(sblk<CP>(a, kSACC, n, b), s);
      }
      continue;
    }
    Vf<CP> du, sacc = zv<CP>();
    if (a.beta == 2) du = dblock<CO, CO>(a, ws, 0, d, 2 * CO);
    else du = dblock<CO, 2 * CO>(a, ws, 0, d, 0);
    if (L >= 2) sacc = ldv<CP>(sblk<CP>(a, kSACC, n, b));
#pragma unroll
    for (int c = 0; c < CP; ++c) du.v[c] = du.v[c] - sacc.v[c] + gv[0].v[c] + gv[1].v[c];
    const long long r = trow(a, t, b, n);
    if (a.beta == 2) {                       // du = d(H*R)
      const float* st = stashp<CP>(a, t, n, b);
      const Vf<CP> z = ldv<CP>(st), rr = ldv<CP>(st + CP), g = ldv<CP>(sblk<CP>(a, kG, n, b));
      const Vf<CP> dz = ldv<CP>(sblk<CP>(a, kDPZ, n, b));
      const float* hprev = outp<CO>(a, b, t - 1, n);
      float dpzr[2 * CO];
      Vf<CP> vr = zv<CP>(), dhp = zv<CP>();
#pragma unroll
      for (int q = 0; q < CO; ++q) {
        const float dpr = du.v[q] * __ldg(hprev + q) * rr.v[q] * (1.f - rr.v[q]);
        dpzr[q] = dz.v[q];
        dpzr[CO + q] = dpr;
        vr.v[q] = dpr;
        a.dpzr[r * 2 * CO + CO + q] = dpr;
        dhp.v[q] = g.v[q] * z.v[q] + du.v[q] * rr.v[q];
      }
      stv<CP>(sblk<CP>(a, kDPR, n, b), vr);
      stv<CP>(sblk<CP>(a, kDHP, n, b), dhp);
      if (a.dsx) write_dsx<CO>(a, ws, r, dpzr, d);
      Vf<CP> top[2];
#pragma unroll
      for (int o = 0; o < 2; ++o) {
        top[o] = dblock<CO, 2 * CO>(a, ws, 1 + 2 * (L - 1) + o, dpzr, 0);
        stv<CP>(sblk<CP>(a, kA0 + 2 * w + o, n, b), top[o]);
      }
      if (L >= 2) {
        Vf<CP> s;
#pragma unroll
        for (int c = 0; c < CP; ++c) s.v[c] = top[0].v[c] + top[1].v[c];
        stv<CP>(sblk<CP>(a, kSACC, n, b), s);
      }
    } else {                                 // du = dS1's share of dH_{t-1}
      const Vf<CP> dhp = ldv<CP>(sblk<CP>(a, kDHP, n, b));
      const float* go = a.gout + (((long long)b * a.T + t - 1) * a.n + n) * CO;
      float g[CO];
#pragma unroll
      for (int q = 0; q < CO; ++q) g[q] = __ldg(go + q) + (dhp.v[q] + du.v[q]);
      rowwise<CO>(a, ws, n, b, t - 1, g);
    }
  }
}

// K = 1: the whole reverse recurrence per (row, window), dL/dH in registers
template <int CO>
__global__ void __launch_bounds__(kThreads, 2) k_dcrnn_nrows_bseq1(NRows a) {
  constexpr int CP = Cp<CO>::v, Q = 3 * CO;
  __shared__ float ws[kMaxNbc * Q];
  stage<CO>(ws, a);
  const int cin = a.cin;
  NR_FOR(a) {
    int n, b;
    if (!item(a, i, n, b)) continue;
    float dh[CO];
#pragma unroll
    for (int q = 0; q < CO; ++q) dh[q] = 0.f;
    for (int t = a.T - 1; t >= 0; --t) {
      const float* st = stashp<CP>(a, t, n, b);
      const Vf<CP> z = ldv<CP>(st), rr = ldv<CP>(st + CP), ht = ldv<CP>(st + 2 * CP);
      const float* go = a.gout + (((long long)b * a.T + t) * a.n + n) * CO;
      const float* hprev = t ? outp<CO>(a, b, t - 1, n) : nullptr;
      const long long r = trow(a, t, b, n);
      float g[CO], hp[CO], dph[CO], dpzr[2 * CO];
#pragma unroll
      for (int q = 0; q < CO; ++q) {
        g[q] = __ldg(go + q) + dh[q];
        hp[q] = hprev ? __ldg(hprev + q) : 0.f;
        dph[q] = g[q] * (1.f - z.v[q]) * (1.f - ht.v[q] * ht.v[q]);
        dpzr[q] = g[q] * (hp[q] - ht.v[q]) * z.v[q] * (1.f - z.v[q]);
      }
#pragma unroll
      for (int c = 0; c < CO; ++c) {
        const float dhr = dot<CO>(dph, ws + (cin + c) * Q + 2 * CO);
        dpzr[CO + c] = t ? dhr * hp[c] * rr.v[c] * (1.f - rr.v[c]) : 0.f;
        dh[c] = g[c] * z.v[c] + dhr * rr.v[c];
      }
#pragma unroll
      for (int c = 0; c < CO; ++c) dh[c] += dot<2 * CO>(dpzr, ws + (cin + c) * Q);
#pragma unroll
      for (int q = 0; q < CO; ++q) {
        a.dph[r * CO + q] = dph[q];
        a.dpzr[r * 2 * CO + q] = dpzr[q];
        a.dpzr[r * 2 * CO + CO + q] = dpzr[CO + q];
      }
      if (a.dsx) write_dsx<CO>(a, ws, r, dpzr, dph);
    }
  }
}

}  // namespace
}  // namespace stmp

using namespace stmp;

static bool nrows_envelope(int64_t cin, int64_t cout, int64_t K) {
  return cin >= 1 && cin <= 4 && cout >= 1 && cout <= 4 && K >= 1 && K <= 4;
}

static int nrows_cp(int64_t cout) { return cout == 3 ? 4 : (int)cout; }

extern "C" int stmp_dcrnn_narrow_rows_supported(const stmp_plan* plan, int64_t cin, int64_t cout, int64_t K) {
  return plan && plan->flavor == STMP_FLAVOR_DCONV && plan->n_ops == 2 && nrows_envelope(cin, cout, K) ? 1 : 0;
}

extern "C" int64_t stmp_dcrnn_narrow_rows_scratch_bytes(const stmp_plan* plan, int64_t B, int64_t cout, int64_t K) {
  if (!plan || B <= 0 || cout < 1 || cout > 4 || K < 2 || K > 4) return 0;
  return (int64_t)kBlocks * plan->n * B * nrows_cp(cout) * 4;
}

static int nrows_check(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K, const char* who) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: plan is NULL", who);
  STMP_REQUIRE(plan->flavor == STMP_FLAVOR_DCONV && plan->n_ops == 2, STMP_EINVAL, "%s: plan is not a DConv plan", who);
  STMP_REQUIRE(nrows_envelope(cin, cout, K), STMP_EUNSUPPORTED, "%s: cin, cout and K in 1..4 only (got %lld, %lld, %lld)", who,
               (long long)cin, (long long)cout, (long long)K);
  STMP_REQUIRE(B >= 0 && T >= 0, STMP_EINVAL, "%s: negative B/T", who);
  STMP_REQUIRE((B + 31) * plan->n < (1ll << 31), STMP_ESHAPE, "%s: B * N too large for one launch", who);
  return STMP_OK;
}

static NRows nrows_params(const stmp_plan* plan, bool transposed, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K) {
  NRows a = {};
  for (int op = 0; op < 2; ++op) {
    const Csr& c = transposed ? plan->bwd[op] : plan->fwd[op];
    a.rp[op] = c.rowptr;
    a.cv[op] = c.cv;
  }
  a.n = plan->n; a.B = (int)B; a.T = (int)T; a.cin = (int)cin; a.K = (int)K; a.nbc = (2 * (int)K - 1) * (int)(cin + cout);
  a.lg = 0;
  while ((1 << a.lg) < B && a.lg < 5) ++a.lg;
  a.G = 1 << a.lg;
  a.WG = (int)((B + a.G - 1) / a.G);
  a.items = plan->n * a.WG * a.G;
  a.blk = (long long)plan->n * B * nrows_cp(cout);
  return a;
}

static int nrows_grid(long long items) {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long blocks = (items + kThreads - 1) / kThreads;
  return (int)(blocks < 8ll * sms ? (blocks > 0 ? blocks : 1) : 8ll * sms);
}

template <int CO>
static int nrows_fwd_launch(const stmp_plan* plan, NRows a, cudaStream_t st) {
  const int grid = nrows_grid(a.items), L = a.K - 1;
  if (a.K == 1) {
    k_dcrnn_nrows_seq1<CO><<<grid, kThreads, 0, st>>>(a);
    STMP_LAUNCH_OK("k_dcrnn_nrows_seq1");
    return STMP_OK;
  }
  for (int t = 0; t < a.T; ++t) {
    a.t = t;
    if (t == 0 && !plan->nonfinite_vals) {
      k_dcrnn_nrows_fwd0<CO><<<grid, kThreads, 0, st>>>(a);
      STMP_LAUNCH_OK("k_dcrnn_nrows_fwd0");
      continue;
    }
    if (t == 0) STMP_CUDA_OK(cudaMemsetAsync(a.scr + kHS * a.blk, 0, a.blk * sizeof(float), st));   // the chain on a zero state
    for (int beta = 1; beta <= 2; ++beta)
      for (int k = 1; k <= L; ++k) {
        a.beta = beta;
        a.hop = k;
        k_dcrnn_nrows_fwd<CO><<<grid, kThreads, 0, st>>>(a);
        STMP_LAUNCH_OK("k_dcrnn_nrows_fwd");
      }
  }
  return STMP_OK;
}

template <int CO>
static int nrows_bwd_launch(NRows a, cudaStream_t st) {
  const int grid = nrows_grid(a.items), L = a.K - 1;
  if (a.K == 1) {
    k_dcrnn_nrows_bseq1<CO><<<grid, kThreads, 0, st>>>(a);
    STMP_LAUNCH_OK("k_dcrnn_nrows_bseq1");
    return STMP_OK;
  }
  a.t = a.T - 1;
  a.par = 1;                                 // the start writes the A blocks of parity 0
  k_dcrnn_nrows_bwd0<CO><<<grid, kThreads, 0, st>>>(a);
  STMP_LAUNCH_OK("k_dcrnn_nrows_bwd0");
  int p = 0;
  for (int t = a.T - 1; t >= 1; --t)
    for (int beta = 2; beta >= 1; --beta)
      for (int k = L; k >= 1; --k) {
        a.t = t;
        a.beta = beta;
        a.hop = k;
        a.par = p;
        k_dcrnn_nrows_bwd<CO><<<grid, kThreads, 0, st>>>(a);
        STMP_LAUNCH_OK("k_dcrnn_nrows_bwd");
        p ^= 1;
      }
  return STMP_OK;
}

extern "C" int stmp_dcrnn_narrow_rows_fwd(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K, const float* x,
                                          int64_t x_bstride, int64_t x_tstride, int64_t x_ld, int64_t x_blk, const float* wzrT,
                                          const float* whsT, const float* bz, const float* br, const float* bh, float* scratch, float* out,
                                          float* stash, float* S1, float* S2, void* stream) {
  const char* who = "stmp_dcrnn_narrow_rows_fwd";
  const int rc = nrows_check(plan, B, T, cin, cout, K, who);
  if (rc != STMP_OK) return rc;
  STMP_REQUIRE(!stash == !S1 && !S1 == !S2, STMP_EINVAL, "%s: give stash, S1 and S2 together or none of them", who);
  STMP_REQUIRE((x || S1) && wzrT && whsT && out && (scratch || K == 1), STMP_EINVAL, "%s: NULL tensor", who);
  const void* ps[] = {x, wzrT, whsT, bz, br, bh, out, S1, S2};
  for (const void* p : ps) STMP_REQUIRE(((uintptr_t)p & 3u) == 0, STMP_ESHAPE, "%s: misaligned tensor", who);
  STMP_REQUIRE((((uintptr_t)scratch | (uintptr_t)stash) & 15u) == 0, STMP_ESHAPE, "%s: scratch and stash must be 16-byte aligned", who);
  if (B == 0 || T == 0) return STMP_OK;
  NRows a = nrows_params(plan, false, B, T, cin, cout, K);
  if (S1) {                                  // training: the X blocks are S1's X columns
    a.x = S1; a.xld = a.nbc; a.xbs = (long long)plan->n * a.nbc; a.xts = B * a.xbs; a.xblk = (int)(cin + cout);
  } else {
    STMP_REQUIRE(x_ld >= cin && x_blk >= cin && x_bstride >= 0 && x_tstride >= 0, STMP_ESHAPE, "%s: bad X block strides", who);
    a.x = x; a.xld = x_ld; a.xbs = x_bstride; a.xts = x_tstride; a.xblk = (int)x_blk;
  }
  a.wzr = wzrT; a.wh = whsT; a.bz = bz; a.br = br; a.bh = bh;
  a.out = out; a.scr = scratch; a.stash = stash; a.S1 = S1; a.S2 = S2;
  cudaStream_t st = (cudaStream_t)stream;
  switch (cout) {
    case 1: return nrows_fwd_launch<1>(plan, a, st);
    case 2: return nrows_fwd_launch<2>(plan, a, st);
    case 3: return nrows_fwd_launch<3>(plan, a, st);
    default: return nrows_fwd_launch<4>(plan, a, st);
  }
}

extern "C" int stmp_dcrnn_narrow_rows_bwd(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K, const float* gout,
                                          const float* out, const float* stash, const float* wzrT, const float* whsT, float* scratch,
                                          float* dph_all, float* dpzr_all, float* dsx, int64_t dsx_ld, void* stream) {
  const char* who = "stmp_dcrnn_narrow_rows_bwd";
  const int rc = nrows_check(plan, B, T, cin, cout, K, who);
  if (rc != STMP_OK) return rc;
  STMP_REQUIRE(gout && out && stash && wzrT && whsT && (scratch || K == 1) && dph_all && dpzr_all, STMP_EINVAL, "%s: NULL tensor", who);
  const void* ps[] = {gout, out, wzrT, whsT, dph_all, dpzr_all, dsx};
  for (const void* p : ps) STMP_REQUIRE(((uintptr_t)p & 3u) == 0, STMP_ESHAPE, "%s: misaligned tensor", who);
  STMP_REQUIRE((((uintptr_t)scratch | (uintptr_t)stash) & 15u) == 0, STMP_ESHAPE, "%s: scratch and stash must be 16-byte aligned", who);
  STMP_REQUIRE(!dsx || dsx_ld >= (2 * K - 1) * cin, STMP_ESHAPE, "%s: the dS row pitch must hold (2K-1) cin columns", who);
  if (B == 0 || T == 0) return STMP_OK;
  NRows a = nrows_params(plan, true, B, T, cin, cout, K);
  a.out = const_cast<float*>(out); a.gout = gout; a.stash = const_cast<float*>(stash); a.wzr = wzrT; a.wh = whsT;
  a.scr = scratch; a.dph = dph_all; a.dpzr = dpzr_all; a.dsx = dsx; a.dsx_ld = dsx_ld;
  cudaStream_t st = (cudaStream_t)stream;
  switch (cout) {
    case 1: return nrows_bwd_launch<1>(a, st);
    case 2: return nrows_bwd_launch<2>(a, st);
    case 3: return nrows_bwd_launch<3>(a, st);
    default: return nrows_bwd_launch<4>(a, st);
  }
}
