// gru_rows.cu -- the generic graph-GRU cell (out = 32 or 64, n_ops <= 1: GConvGRU K <= 2) on graphs of ANY size, split over CTAs by
// destination rows (DESIGN §4i, §4n).  One graph, one step per call; the two all-to-all dependencies of a step -- Op(H*R) in the forward and
// Op^T(.) in the backward -- split a cell into a short chain of launches, each a gather + contraction + gate math fused per row:
//
//   forward, H given   k_gru_rows_fwd_a<1>  gather Op[X | H]; Z, R, H*R and the X half of the candidate pre-activation -> scratch
//                      k_gru_rows_fwd_b     gather Op(H*R); pre_h, Ht = tanh(pre_h), H' = Z*H + (1-Z)*Ht
//   forward, H = None  k_gru_rows_fwd_a<0>  gather Op X; Z and H' = (1-Z)*tanh(pre_h) (R is dead: H*R = 0)
//   backward           k_gru_rows_bwd_a     dph, dpz and dS2 = dph W_h^T (rowwise)
//                      k_gru_rows_bwd_b     gather Op^T of dS2's H*R block: d(H*R), dpr, dS1 = [dpz | dpr] W_zr^T, the own-row dH / dX
//                      k_gru_rows_bwd_c     gather Op^T of the operator blocks of dS1 (+ dS2's X columns): dH, dX complete
//
// Mapping: one warp per destination row, lane = output channel (NC = 1, out = 32) or channels lane and lane + 32 (NC = 2, out = 64), and X
// channel for lane < cin; a CTA owns tiles of kRowTile consecutive rows (grid-strided) and stages the weight rows its launch contracts in
// shared memory once.  The contraction is exact fp32 FFMA: every basis value is broadcast with a shuffle and multiplied into the lane's
// columns of the staged weights (odd pitch Wd<NC>::P: the lane-indexed rows and the lane-indexed columns are both free of bank conflicts).
// Gathers walk the plan's CSR rows in entry order with separate multiply and add, as stmp_spmm does.  No atomics anywhere; every result
// depends on its row alone, so repeated calls are bit-identical.  The 64-wide instance (stmp_gru_wide_rows_*) keeps the per-launch staging of
// the 32-wide one: at the graph sizes the cell serves, a step has fewer 16-row tiles than the H100 has SMs, so the one CTA per SM that
// 123 KB of staged weights allows costs nothing there; its weight gradients come from k_wide_rows_wgrad<3> (rows.cuh).
#include "rows.cuh"

namespace stmp {
namespace {

using namespace rows;

// per-width constants: out channels, the widest basis (n_ops = 1, cin = 16), the staged weight pitch, basis columns per lane, the
// backward scratch row (dS2 (NB) | Op^T operand Q (NB)) and the forward scratch row (H*R | X half of pre_h | Z)
template <int NC>
struct Wd {
  static constexpr int CO = 32 * NC, NB = 2 * (kMaxCin + CO), P = NB + 1, NQ = NB / 32, SP = 2 * NB, FP = 3 * CO;
};

struct RowsFwd {
  const int* rowptr; const int2* cv;         // operator 0 by destination (n_ops = 1)
  int n, cin, nops, nb;                      // nb = (nops + 1)(cin + CO) basis columns
  const float* x; const float* h;            // (N, cin), (N, CO) or NULL (H = None)
  const float* w; const float* b;            // packed [3 CO][nb], [3 CO]
  float* out;                                // (N, CO)
  float* scr;                                // (N, 3 CO)  H given
  float* stash;                              // (3, N, CO) Z | R | Ht, nullable
  float* S1; float* S2; int ld;              // (N, ld) weight-gradient bases, nullable
};

// HAS_H = 1: launch A of the two-launch forward.  HAS_H = 0: the whole H = None cell.
template <int NC, bool HAS_H>
__global__ void __launch_bounds__(kRowsThreads, 2) k_gru_rows_fwd_a(RowsFwd a) {
  using D = Wd<NC>;
  constexpr int CO = D::CO, P = D::P;
  extern __shared__ float ws[];              // [3 CO][P]
  stage_w<P>(ws, a.w, a.nb, 0, 3 * CO);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + CO;
  float bz[NC], br[NC], bh[NC];
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    bz[j] = __ldg(a.b + lane + 32 * j); br[j] = __ldg(a.b + CO + lane + 32 * j); bh[j] = __ldg(a.b + 2 * CO + lane + 32 * j);
  }
  const size_t NC_ = (size_t)a.n * CO;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const float xv = lane < cin ? __ldg(a.x + (size_t)i * cin + lane) : 0.f;
      float hv[NC], lh[NC], lx = 0.f;
#pragma unroll
      for (int j = 0; j < NC; ++j) { hv[j] = HAS_H ? __ldg(a.h + (size_t)i * CO + lane + 32 * j) : 0.f; lh[j] = 0.f; }
      if (a.nops) gather_rows<NC, HAS_H>(a.rowptr, a.cv, i, a.h, CO, a.x, cin, cin, lane, lh, lx);
      float pz[NC], pr[NC], ph[NC];          // pre = b + [U | Op U] W^T in basis order; ph takes the X columns only here
#pragma unroll
      for (int j = 0; j < NC; ++j) { pz[j] = bz[j]; pr[j] = br[j]; ph[j] = bh[j]; }
      for (int blk = 0; blk <= a.nops; ++blk) {
        const float sx = blk ? lx : xv;
        const float* wb = ws + blk * C;
        for (int c = 0; c < cin; ++c) {
          const float s = __shfl_sync(0xffffffffu, sx, c);
#pragma unroll
          for (int j = 0; j < NC; ++j) {
            pz[j] = fmaf(s, wb[(lane + 32 * j) * P + c], pz[j]);
            if (HAS_H) pr[j] = fmaf(s, wb[(CO + lane + 32 * j) * P + c], pr[j]);
            ph[j] = fmaf(s, wb[(2 * CO + lane + 32 * j) * P + c], ph[j]);
          }
        }
        if (HAS_H) {
#pragma unroll
          for (int jo = 0; jo < NC; ++jo) {
            const float sh = blk ? lh[jo] : hv[jo];
#pragma unroll 8
            for (int o = 0; o < 32; ++o) {
              const float s = __shfl_sync(0xffffffffu, sh, o);
#pragma unroll
              for (int j = 0; j < NC; ++j) {
                pz[j] = fmaf(s, wb[(lane + 32 * j) * P + cin + 32 * jo + o], pz[j]);
                pr[j] = fmaf(s, wb[(CO + lane + 32 * j) * P + cin + 32 * jo + o], pr[j]);
              }
            }
          }
        }
      }
#pragma unroll
      for (int j = 0; j < NC; ++j) {
        const int ch = lane + 32 * j;
        const float Z = sigmoidf_acc(pz[j]);
        if (HAS_H) {
          const float R = sigmoidf_acc(pr[j]), hr = hv[j] * R;
          float* s = a.scr + (size_t)i * D::FP;
          s[ch] = hr;
          s[CO + ch] = ph[j];
          s[2 * CO + ch] = Z;
          if (a.stash) {
            a.stash[(size_t)i * CO + ch] = Z;
            a.stash[NC_ + (size_t)i * CO + ch] = R;
          }
          if (a.S2) a.S2[(size_t)i * a.ld + cin + ch] = hr;
        } else {
          const float Ht = tanhf(ph[j]), hn = (1.f - Z) * Ht;
          a.out[(size_t)i * CO + ch] = hn;
          if (a.stash) {
            a.stash[(size_t)i * CO + ch] = Z;
            a.stash[2 * NC_ + (size_t)i * CO + ch] = Ht;
          }
        }
      }
      if (a.S1) {                            // [X | H | Op X | Op H] (+ zero padding); H = None: H columns zero
        float* r1 = a.S1 + (size_t)i * a.ld;
        if (lane < cin) r1[lane] = xv;
#pragma unroll
        for (int j = 0; j < NC; ++j) r1[cin + lane + 32 * j] = hv[j];
        if (a.nops) {
          if (lane < cin) r1[C + lane] = lx;
#pragma unroll
          for (int j = 0; j < NC; ++j) r1[C + cin + lane + 32 * j] = lh[j];
        }
        if (a.nb + lane < a.ld) r1[a.nb + lane] = 0.f;
        if (HAS_H && a.S2) {                 // S2's X columns and padding; H*R above, Op(H*R) in launch B
          float* r2 = a.S2 + (size_t)i * a.ld;
          if (lane < cin) r2[lane] = xv;
          if (a.nops && lane < cin) r2[C + lane] = lx;
          if (a.nb + lane < a.ld) r2[a.nb + lane] = 0.f;
        }
      }
    }
  }
}

template <int NC>
__global__ void __launch_bounds__(kRowsThreads, 2) k_gru_rows_fwd_b(RowsFwd a) {
  using D = Wd<NC>;
  constexpr int CO = D::CO, P = D::P, FP = D::FP;
  extern __shared__ float ws[];              // candidate rows of the weights: [CO][P]
  stage_w<P>(ws, a.w, a.nb, 2 * CO, CO);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + CO;
  const size_t NC_ = (size_t)a.n * CO;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const float* s = a.scr + (size_t)i * FP;
      float hr[NC], ph[NC], lhr[NC];
#pragma unroll
      for (int j = 0; j < NC; ++j) { hr[j] = s[lane + 32 * j]; ph[j] = s[CO + lane + 32 * j]; lhr[j] = 0.f; }
      float unused;
      if (a.nops) gather_rows<NC, true>(a.rowptr, a.cv, i, a.scr, FP, a.scr, FP, 0, lane, lhr, unused);
      for (int blk = 0; blk <= a.nops; ++blk) {
#pragma unroll
        for (int jo = 0; jo < NC; ++jo) {
          const float sh = blk ? lhr[jo] : hr[jo];
#pragma unroll 8
          for (int o = 0; o < 32; ++o) {
            const float v = __shfl_sync(0xffffffffu, sh, o);
#pragma unroll
            for (int j = 0; j < NC; ++j) ph[j] = fmaf(v, ws[(lane + 32 * j) * P + blk * C + cin + 32 * jo + o], ph[j]);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < NC; ++j) {
        const int ch = lane + 32 * j;
        const float Z = s[2 * CO + ch], hv = __ldg(a.h + (size_t)i * CO + ch);
        const float Ht = tanhf(ph[j]);
        a.out[(size_t)i * CO + ch] = Z * hv + (1.f - Z) * Ht;
        if (a.stash) a.stash[2 * NC_ + (size_t)i * CO + ch] = Ht;
        if (a.S2 && a.nops) a.S2[(size_t)i * a.ld + C + cin + ch] = lhr[j];
      }
    }
  }
}

struct RowsBwd {
  const int* rowptr; const int2* cv;         // operator 0 by SOURCE (the transposed product)
  int n, cin, nops, nb;
  const float* gout; const float* h;         // (N, CO); h NULL for H = None
  const float* stash; const float* w;        // (3, N, CO), packed [3 CO][nb]
  float* dph; float* dpzr;                   // (N, CO), (N, 2 CO)
  float* scr;                                // (N, SP): dS2 | Q
  float* dx; float* dh;                      // (N, cin), (N, CO), nullable
};

// rowwise: dph, dpz (dpr = 0 when H = None), dS2 = dph W_h^T -> scratch; H = None: also dS1 = [dpz | 0] W_zr^T and the X gradient's own row
// and its Op^T operand (the X columns of both bases).
template <int NC, bool HAS_H>
__global__ void __launch_bounds__(kRowsThreads, 2) k_gru_rows_bwd_a(RowsBwd a) {
  using D = Wd<NC>;
  constexpr int CO = D::CO, P = D::P, NQ = D::NQ, SP = D::SP;
  extern __shared__ float ws[];              // [3 CO][P]
  stage_w<P>(ws, a.w, a.nb, 0, 3 * CO);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + CO;
  const size_t NC_ = (size_t)a.n * CO;
  const bool need_ds = HAS_H || a.dx != nullptr;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      float dph[NC], dpz[NC];
#pragma unroll
      for (int j = 0; j < NC; ++j) {
        const size_t io = (size_t)i * CO + lane + 32 * j;
        const float g = a.gout[io], Z = a.stash[io], Ht = a.stash[2 * NC_ + io];
        const float hp = HAS_H ? a.h[io] : 0.f;
        dph[j] = g * (1.f - Z) * (1.f - Ht * Ht);
        dpz[j] = g * (hp - Ht) * Z * (1.f - Z);
        a.dph[io] = dph[j];
        a.dpzr[(size_t)i * 2 * CO + lane + 32 * j] = dpz[j];
        if (!HAS_H) a.dpzr[(size_t)i * 2 * CO + CO + lane + 32 * j] = 0.f;
      }
      if (!need_ds) continue;
      float d2[NQ], d1[NQ];                  // basis columns m = lane + 32 q
#pragma unroll
      for (int q = 0; q < NQ; ++q) d2[q] = d1[q] = 0.f;
#pragma unroll
      for (int jo = 0; jo < NC; ++jo) {
#pragma unroll 4
        for (int o = 0; o < 32; ++o) {
          const float s2 = __shfl_sync(0xffffffffu, dph[jo], o);
          const float s1 = HAS_H ? 0.f : __shfl_sync(0xffffffffu, dpz[jo], o);
#pragma unroll
          for (int q = 0; q < NQ; ++q) {
            d2[q] = fmaf(s2, ws[(2 * CO + 32 * jo + o) * P + lane + 32 * q], d2[q]);
            if (!HAS_H) d1[q] = fmaf(s1, ws[(32 * jo + o) * P + lane + 32 * q], d1[q]);
          }
        }
      }
      float* sr = a.scr + (size_t)i * SP;
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int m = lane + 32 * q;
        if (m >= a.nb) continue;
        if (HAS_H) {
          sr[m] = d2[q];
        } else {                             // only the X columns carry a gradient
          const float v = d2[q] + d1[q];
          if (m < cin) a.dx[(size_t)i * cin + m] = v;
          else if (m >= C && m < C + cin) sr[SP / 2 + m - C] = v;
        }
      }
    }
  }
}

// H given: gather Op^T of dS2's H*R block -> d(H*R), dpr, dS1 = [dpz | dpr] W_zr^T; the own-row parts of dH and dX; Q = the Op^T operand of
// the final gather (dS1's operator block, plus dS2's operator-block X columns).
template <int NC>
__global__ void __launch_bounds__(kRowsThreads, 2) k_gru_rows_bwd_b(RowsBwd a) {
  using D = Wd<NC>;
  constexpr int CO = D::CO, P = D::P, NQ = D::NQ, SP = D::SP;
  extern __shared__ float ws[];              // z | r rows: [2 CO][P], then one NB-float row buffer per warp
  stage_w<P>(ws, a.w, a.nb, 0, 2 * CO);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + CO;
  float* sb = ws + 2 * CO * P + warp * D::NB;
  const size_t NC_ = (size_t)a.n * CO;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int j = t0 + warp; j < t1; j += kRowsWarps) {
      const float* sr = a.scr + (size_t)j * SP;
      float dhr[NC];
#pragma unroll
      for (int c = 0; c < NC; ++c) dhr[c] = sr[cin + lane + 32 * c];
      if (a.nops) {
        float t[NC], unused;
        gather_rows<NC, true>(a.rowptr, a.cv, j, a.scr + C + cin, SP, a.scr, SP, 0, lane, t, unused);
#pragma unroll
        for (int c = 0; c < NC; ++c) dhr[c] += t[c];
      }
      float dpr[NC], dpz[NC];
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const size_t io = (size_t)j * CO + lane + 32 * c;
        const float R = a.stash[NC_ + io], hp = a.h[io];
        dpr[c] = dhr[c] * hp * R * (1.f - R);
        dpz[c] = a.dpzr[(size_t)j * 2 * CO + lane + 32 * c];
        a.dpzr[(size_t)j * 2 * CO + CO + lane + 32 * c] = dpr[c];
      }
      float d1[NQ];
#pragma unroll
      for (int q = 0; q < NQ; ++q) d1[q] = 0.f;
#pragma unroll
      for (int jo = 0; jo < NC; ++jo) {
#pragma unroll 4
        for (int o = 0; o < 32; ++o) {
          const float sz = __shfl_sync(0xffffffffu, dpz[jo], o), sp = __shfl_sync(0xffffffffu, dpr[jo], o);
#pragma unroll
          for (int q = 0; q < NQ; ++q)
            d1[q] = fmaf(sp, ws[(CO + 32 * jo + o) * P + lane + 32 * q], fmaf(sz, ws[(32 * jo + o) * P + lane + 32 * q], d1[q]));
        }
      }
#pragma unroll
      for (int q = 0; q < NQ; ++q) sb[lane + 32 * q] = d1[q];
      __syncwarp();
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const size_t io = (size_t)j * CO + lane + 32 * c;
        const float g = a.gout[io], Z = a.stash[io], R = a.stash[NC_ + io];
        if (a.dh) a.dh[io] = g * Z + dhr[c] * R + sb[cin + lane + 32 * c];
      }
      if (a.dx && lane < cin) a.dx[(size_t)j * cin + lane] = sr[lane] + sb[lane];
      if (a.nops)
        for (int c = lane; c < C; c += 32) a.scr[(size_t)j * SP + SP / 2 + c] = sb[C + c] + (c < cin ? sr[C + c] : 0.f);
      __syncwarp();
    }
  }
}

// dH += Op^T Q[:, cin:], dX += Op^T Q[:, :cin]  (either nullable)
template <int NC>
__global__ void __launch_bounds__(kRowsThreads) k_gru_rows_bwd_c(RowsBwd a) {
  using D = Wd<NC>;
  constexpr int CO = D::CO, SP = D::SP;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin;
  const float* q = a.scr + SP / 2;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int j = t0 + warp; j < t1; j += kRowsWarps) {
      float th[NC], tx;
      if (a.dh) gather_rows<NC, true>(a.rowptr, a.cv, j, q + cin, SP, q, SP, a.dx ? cin : 0, lane, th, tx);
      else gather_rows<NC, false>(a.rowptr, a.cv, j, q + cin, SP, q, SP, cin, lane, th, tx);
      if (a.dh)
#pragma unroll
        for (int c = 0; c < NC; ++c) a.dh[(size_t)j * CO + lane + 32 * c] += th[c];
      if (a.dx && lane < cin) a.dx[(size_t)j * cin + lane] += tx;
    }
  }
}

// w [3 CO][nb]: row gate*CO + o, column m = blk*(cin+CO) + c of the basis [X | H | Op X | Op H]; b [3 CO] = bx + bh (zeros without biases)
template <int NC>
__global__ void k_gru_rows_pack(int nops, int cin, const float* __restrict__ wx, const float* __restrict__ wh, const float* __restrict__ bx,
                                const float* __restrict__ bh, float* __restrict__ w, float* __restrict__ b) {
  constexpr int CO = Wd<NC>::CO;
  const int C = cin + CO, nbk = nops + 1, nb = nbk * C;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 3 * CO * nb) {
    const int row = i / nb, m = i - row * nb, gate = row / CO, o = row % CO, blk = m / C, c = m - blk * C;
    w[i] = c < cin ? wx[(((size_t)gate * nbk + blk) * CO + o) * cin + c] : wh[(((size_t)gate * nbk + blk) * CO + o) * CO + c - cin];
  } else if (i < 3 * CO * nb + 3 * CO) {
    const int r = i - 3 * CO * nb;
    b[r] = bx ? bx[r] + bh[r] : 0.f;
  }
}

// The fixed-order sums (fixed_order_sum, rows.cuh) of the 32-wide cell's k_dcrnn_wgrad<32> partials [part][ld*96 + 96] into its packed
// layout dw [96][nb] (row gate*32 + o, column m of the basis [X | H | Op X | Op H]) and db [96] (nullable).
__global__ void __launch_bounds__(256) k_gru_rows_wgrad_reduce(int parts, int MG, int nb, const float* __restrict__ partial,
                                                               float* __restrict__ dw, float* __restrict__ db) {
  __shared__ float sub[8][32];
  const int x = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + x;
  const size_t stride = (size_t)MG * 8 * 3 * kCo + 3 * kCo;
  size_t src = 0;
  float* dst = nullptr;
  if (i < 96 * nb) {
    const int row = i / nb, m = i - row * nb, gate = row >> 5, o = row & 31;
    src = gate == 2 ? (size_t)MG * 8 * 2 * kCo + (size_t)m * kCo + o : (size_t)m * 2 * kCo + gate * kCo + o;
    dst = dw + i;
  } else if (i < 96 * nb + 3 * kCo) {
    const int b = i - 96 * nb;                                   // bias sums are stored z | r | h
    src = (size_t)MG * 8 * 3 * kCo + b;
    dst = db ? db + b : nullptr;
  }
  const float t = fixed_order_sum(partial + src, stride, parts, dst != nullptr, sub);
  if (w == 0 && dst) *dst = t;
}

}  // namespace
}  // namespace stmp

using namespace stmp;

static bool rows_supported(const stmp_plan* plan, int n_ops, int64_t cin, int64_t cout) {
  return plan && n_ops >= 0 && n_ops <= 1 && n_ops <= plan->n_ops && (cout == 32 || cout == 64) && cin >= 1 && cin <= kMaxCin;
}

extern "C" int stmp_gru_rows_supported(const stmp_plan* plan, int n_ops, int64_t cin, int64_t cout) {
  return rows_supported(plan, n_ops, cin, cout) ? 1 : 0;
}

// the entry names of one width, for errors and launch accounting
template <int NC> struct Names;
template <> struct Names<1> {
  static constexpr const char* pack = "stmp_gru_rows_pack_weights";
  static constexpr const char* fwd = "stmp_gru_rows_fwd";
  static constexpr const char* bwd = "stmp_gru_rows_bwd";
  static constexpr const char* fwd_a = "k_gru_rows_fwd_a";
  static constexpr const char* fwd_b = "k_gru_rows_fwd_b";
  static constexpr const char* bwd_a = "k_gru_rows_bwd_a";
  static constexpr const char* bwd_b = "k_gru_rows_bwd_b";
  static constexpr const char* bwd_c = "k_gru_rows_bwd_c";
  static constexpr const char* kpack = "k_gru_rows_pack";
  static constexpr const char* wgrad = "stmp_gru_rows_wgrad";
  static constexpr const char* wgrad_reduce = "k_gru_rows_wgrad_reduce";
};
template <> struct Names<2> {
  static constexpr const char* pack = "stmp_gru_wide_rows_pack_weights";
  static constexpr const char* fwd = "stmp_gru_wide_rows_fwd";
  static constexpr const char* bwd = "stmp_gru_wide_rows_bwd";
  static constexpr const char* fwd_a = "k_gru_wide_rows_fwd_a";
  static constexpr const char* fwd_b = "k_gru_wide_rows_fwd_b";
  static constexpr const char* bwd_a = "k_gru_wide_rows_bwd_a";
  static constexpr const char* bwd_b = "k_gru_wide_rows_bwd_b";
  static constexpr const char* bwd_c = "k_gru_wide_rows_bwd_c";
  static constexpr const char* kpack = "k_gru_wide_rows_pack";
  static constexpr const char* wgrad = "stmp_gru_wide_rows_wgrad";
  static constexpr const char* wgrad_reduce = "k_gru_wide_rows_wgrad_reduce";
};

template <int NC>
static int pack_weights(int n_ops, int64_t cin, const float* wx, const float* wh, const float* bx, const float* bh, float* w, float* b,
                        void* stream) {
  using N = Names<NC>;
  constexpr int CO = Wd<NC>::CO;
  STMP_REQUIRE(wx && wh && w && b, STMP_EINVAL, "%s: NULL tensor", N::pack);
  STMP_REQUIRE(!bx == !bh, STMP_EINVAL, "%s: give both bias stacks or neither", N::pack);
  STMP_REQUIRE(n_ops >= 0 && n_ops <= 1 && cin >= 1 && cin <= kMaxCin, STMP_EUNSUPPORTED, "%s: n_ops <= 1, cin 1..16 only", N::pack);
  const int total = 3 * CO * (n_ops + 1) * ((int)cin + CO) + 3 * CO;
  k_gru_rows_pack<NC><<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n_ops, (int)cin, wx, wh, bx, bh, w, b);
  STMP_LAUNCH_OK(N::kpack);
  return STMP_OK;
}

template <int NC>
static int rows_fwd(const stmp_plan* plan, int n_ops, int64_t cin, const float* x, const float* h, const float* w, const float* b,
                    float* scratch, float* out, float* stash, float* S1, float* S2, int64_t ld, void* stream) {
  using N = Names<NC>;
  using D = Wd<NC>;
  constexpr int CO = D::CO;
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: plan is NULL", N::fwd);
  STMP_REQUIRE(rows_supported(plan, n_ops, cin, CO), STMP_EUNSUPPORTED,
               "%s: n_ops <= min(1, plan's operators), cin 1..16 only (n_ops=%d, cin=%lld)", N::fwd, n_ops, (long long)cin);
  STMP_REQUIRE(x && w && b && out && (!h || scratch), STMP_EINVAL, "%s: NULL tensor", N::fwd);
  STMP_REQUIRE(!S2 || (S1 && h), STMP_EINVAL, "%s: S2 needs S1 and h (H = None: S2 = S1)", N::fwd);
  const int nb = (n_ops + 1) * ((int)cin + CO);
  STMP_REQUIRE(!S1 || ld == (nb + 7) / 8 * 8, STMP_ESHAPE, "%s: the basis row pitch must be (n_ops+1)(cin+%d) rounded up to 8", N::fwd, CO);
  const void* ps[] = {x, h, w, b, scratch, out, stash, S1, S2};
  for (const void* p : ps) STMP_REQUIRE(al4(p), STMP_ESHAPE, "%s: misaligned tensor", N::fwd);
  STMP_REQUIRE(!S1 || (((uintptr_t)S1 | (uintptr_t)S2) & 15u) == 0, STMP_ESHAPE, "%s: S1 / S2 must be 16-byte aligned", N::fwd);
  if (plan->n == 0) return STMP_OK;
  RowsFwd a;
  a.rowptr = plan->fwd[0].rowptr; a.cv = plan->fwd[0].cv;
  a.n = plan->n; a.cin = (int)cin; a.nops = n_ops; a.nb = nb;
  a.x = x; a.h = h; a.w = w; a.b = b; a.out = out; a.scr = scratch; a.stash = stash; a.S1 = S1; a.S2 = S2; a.ld = (int)ld;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = rows_grid(plan->n), smem = 3 * CO * D::P * 4, smem_b = CO * D::P * 4;
  if (h) {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_gru_rows_fwd_a<NC, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k_gru_rows_fwd_a<NC, true><<<grid, kRowsThreads, smem, st>>>(a);
    STMP_LAUNCH_OK(N::fwd_a);
    STMP_CUDA_OK(cudaFuncSetAttribute(k_gru_rows_fwd_b<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_b));
    k_gru_rows_fwd_b<NC><<<grid, kRowsThreads, smem_b, st>>>(a);
    STMP_LAUNCH_OK(N::fwd_b);
  } else {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_gru_rows_fwd_a<NC, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k_gru_rows_fwd_a<NC, false><<<grid, kRowsThreads, smem, st>>>(a);
    STMP_LAUNCH_OK(N::fwd_a);
  }
  return STMP_OK;
}

template <int NC>
static int rows_bwd(const stmp_plan* plan, int n_ops, int64_t cin, const float* gout, const float* h, const float* stash, const float* w,
                    float* scratch, float* dph, float* dpzr, float* dx, float* dh, void* stream) {
  using N = Names<NC>;
  using D = Wd<NC>;
  constexpr int CO = D::CO;
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: plan is NULL", N::bwd);
  STMP_REQUIRE(rows_supported(plan, n_ops, cin, CO), STMP_EUNSUPPORTED,
               "%s: n_ops <= min(1, plan's operators), cin 1..16 only (n_ops=%d, cin=%lld)", N::bwd, n_ops, (long long)cin);
  STMP_REQUIRE(gout && stash && w && scratch && dph && dpzr, STMP_EINVAL, "%s: NULL tensor", N::bwd);
  STMP_REQUIRE(h || !dh, STMP_EINVAL, "%s: dh needs h (H = None has no state gradient)", N::bwd);
  const void* ps[] = {gout, h, stash, w, scratch, dph, dpzr, dx, dh};
  for (const void* p : ps) STMP_REQUIRE(al4(p), STMP_ESHAPE, "%s: misaligned tensor", N::bwd);
  if (plan->n == 0) return STMP_OK;
  RowsBwd a;
  a.rowptr = plan->bwd[0].rowptr; a.cv = plan->bwd[0].cv;
  a.n = plan->n; a.cin = (int)cin; a.nops = n_ops; a.nb = (n_ops + 1) * ((int)cin + CO);
  a.gout = gout; a.h = h; a.stash = stash; a.w = w; a.dph = dph; a.dpzr = dpzr; a.scr = scratch; a.dx = dx; a.dh = dh;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = rows_grid(plan->n), smem = 3 * CO * D::P * 4, smem_b = (2 * CO * D::P + kRowsWarps * D::NB) * 4;
  if (h) {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_gru_rows_bwd_a<NC, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k_gru_rows_bwd_a<NC, true><<<grid, kRowsThreads, smem, st>>>(a);
    STMP_LAUNCH_OK(N::bwd_a);
    STMP_CUDA_OK(cudaFuncSetAttribute(k_gru_rows_bwd_b<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_b));
    k_gru_rows_bwd_b<NC><<<grid, kRowsThreads, smem_b, st>>>(a);
    STMP_LAUNCH_OK(N::bwd_b);
  } else {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_gru_rows_bwd_a<NC, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k_gru_rows_bwd_a<NC, false><<<grid, kRowsThreads, smem, st>>>(a);
    STMP_LAUNCH_OK(N::bwd_a);
  }
  if (n_ops && (dh || dx)) {
    k_gru_rows_bwd_c<NC><<<grid, kRowsThreads, 0, st>>>(a);
    STMP_LAUNCH_OK(N::bwd_c);
  }
  return STMP_OK;
}

// the weight-gradient workspace: wgrad_ffma_max_parts() partials of (ld + 1) * 3 CO floats (at 64 wide, one of (ld + 1) * CO per gate)
template <int NC>
static int64_t rows_wgrad_workspace_bytes(int n_ops, int64_t cin) {
  constexpr int CO = Wd<NC>::CO;
  const int64_t ld = ((n_ops + 1) * (cin + CO) + 7) / 8 * 8;
  return (int64_t)wgrad_ffma_max_parts() * (ld + 1) * 3 * CO * 4;
}

// Exact fp32: per-CTA FFMA partials over strided row tiles, then a fixed-order sum into the packed layout dw [3 CO][nb], db [3 CO].  The
// 32-wide cell contracts with train.cu's k_dcrnn_wgrad<32> (16-row tiles), the 64-wide one with k_wide_rows_wgrad<3> (rows.cuh; 32-row tiles,
// one partial per gate and CTA).
template <int NC>
static int rows_wgrad(int n_ops, int64_t cin, int64_t rows, int64_t ld, const float* S1, const float* S2, const float* dpzr, const float* dph,
                      void* workspace, float* dw, float* db, void* stream) {
  using N = Names<NC>;
  constexpr int CO = Wd<NC>::CO;
  STMP_REQUIRE(S1 && S2 && dpzr && dph && workspace && dw && rows >= 0, STMP_EINVAL, "%s: bad argument", N::wgrad);
  STMP_REQUIRE(n_ops >= 0 && n_ops <= 1 && cin >= 1 && cin <= kMaxCin, STMP_EUNSUPPORTED, "%s: n_ops <= 1, cin 1..16 only", N::wgrad);
  const int nb = (n_ops + 1) * ((int)cin + CO);
  STMP_REQUIRE(ld == (nb + 7) / 8 * 8, STMP_ESHAPE, "%s: the basis row pitch must be (n_ops+1)(cin+%d) rounded up to 8", N::wgrad, CO);
  STMP_REQUIRE((((uintptr_t)S1 | (uintptr_t)S2 | (uintptr_t)dpzr | (uintptr_t)dph | (uintptr_t)workspace) & 15u) == 0, STMP_ESHAPE,
               "%s: S1, S2, dpzr, dph and the workspace must be 16-byte aligned", N::wgrad);
  cudaStream_t st = (cudaStream_t)stream;
  if (rows == 0) {
    STMP_CUDA_OK(cudaMemsetAsync(dw, 0, (size_t)3 * CO * nb * 4, st));
    if (db) STMP_CUDA_OK(cudaMemsetAsync(db, 0, (size_t)3 * CO * 4, st));
    return STMP_OK;
  }
  float* partial = reinterpret_cast<float*>(workspace);
  const int reduce_grid = (3 * CO * nb + 3 * CO + 31) / 32;
  if constexpr (NC == 1) {
    int parts = 0;
    const int rc = wgrad_ffma_launch(CO, rows, (int)ld, S1, S2, dpzr, dph, partial, st, &parts);
    if (rc != STMP_OK) return rc;
    k_gru_rows_wgrad_reduce<<<reduce_grid, 256, 0, st>>>(parts, (int)ld / 8, nb, partial, dw, db);
  } else {
    const int parts = wide_wgrad_parts(rows);
    const WideWgradOps<3> op = {{S1, S1, S2}, {dpzr, dpzr + CO, dph}, {2 * CO, 2 * CO, CO}};
    k_wide_rows_wgrad<3><<<dim3(parts, 3), kWideWgThreads, 0, st>>>(rows, (int)ld, op, partial);
    STMP_LAUNCH_OK("k_gru_wide_rows_wgrad");
    k_wide_rows_wgrad_reduce<3><<<reduce_grid, 256, 0, st>>>(parts, (int)ld, nb, partial, 0, 0, nullptr, dw, db, nullptr);
  }
  STMP_LAUNCH_OK(N::wgrad_reduce);
  return STMP_OK;
}

extern "C" int stmp_gru_rows_pack_weights(int n_ops, int64_t cin, const float* wx, const float* wh, const float* bx, const float* bh,
                                          float* w, float* b, void* stream) {
  return pack_weights<1>(n_ops, cin, wx, wh, bx, bh, w, b, stream);
}

extern "C" int stmp_gru_rows_fwd(const stmp_plan* plan, int n_ops, int64_t cin, const float* x, const float* h, const float* w, const float* b,
                                 float* scratch, float* out, float* stash, float* S1, float* S2, int64_t ld, void* stream) {
  return rows_fwd<1>(plan, n_ops, cin, x, h, w, b, scratch, out, stash, S1, S2, ld, stream);
}

extern "C" int64_t stmp_gru_rows_scratch_bytes(const stmp_plan* plan) {
  return plan ? (int64_t)plan->n * Wd<1>::SP * 4 : 0;
}

extern "C" int stmp_gru_rows_bwd(const stmp_plan* plan, int n_ops, int64_t cin, const float* gout, const float* h, const float* stash,
                                 const float* w, float* scratch, float* dph, float* dpzr, float* dx, float* dh, void* stream) {
  return rows_bwd<1>(plan, n_ops, cin, gout, h, stash, w, scratch, dph, dpzr, dx, dh, stream);
}

extern "C" int64_t stmp_gru_rows_wgrad_workspace_bytes(int n_ops, int64_t cin) { return rows_wgrad_workspace_bytes<1>(n_ops, cin); }

extern "C" int stmp_gru_rows_wgrad(int n_ops, int64_t cin, int64_t rows, int64_t ld, const float* S1, const float* S2, const float* dpzr,
                                   const float* dph, void* workspace, float* dw, float* db, void* stream) {
  return rows_wgrad<1>(n_ops, cin, rows, ld, S1, S2, dpzr, dph, workspace, dw, db, stream);
}

extern "C" int stmp_gru_wide_rows_pack_weights(int n_ops, int64_t cin, const float* wx, const float* wh, const float* bx, const float* bh,
                                               float* w, float* b, void* stream) {
  return pack_weights<2>(n_ops, cin, wx, wh, bx, bh, w, b, stream);
}

extern "C" int stmp_gru_wide_rows_fwd(const stmp_plan* plan, int n_ops, int64_t cin, const float* x, const float* h, const float* w,
                                      const float* b, float* scratch, float* out, float* stash, float* S1, float* S2, int64_t ld, void* stream) {
  return rows_fwd<2>(plan, n_ops, cin, x, h, w, b, scratch, out, stash, S1, S2, ld, stream);
}

extern "C" int64_t stmp_gru_wide_rows_scratch_bytes(const stmp_plan* plan) {
  return plan ? (int64_t)plan->n * Wd<2>::SP * 4 : 0;
}

extern "C" int stmp_gru_wide_rows_bwd(const stmp_plan* plan, int n_ops, int64_t cin, const float* gout, const float* h, const float* stash,
                                      const float* w, float* scratch, float* dph, float* dpzr, float* dx, float* dh, void* stream) {
  return rows_bwd<2>(plan, n_ops, cin, gout, h, stash, w, scratch, dph, dpzr, dx, dh, stream);
}

extern "C" int64_t stmp_gru_wide_rows_wgrad_workspace_bytes(int n_ops, int64_t cin) { return rows_wgrad_workspace_bytes<2>(n_ops, cin); }

extern "C" int stmp_gru_wide_rows_wgrad(int n_ops, int64_t cin, int64_t rows, int64_t ld, const float* S1, const float* S2, const float* dpzr,
                                        const float* dph, void* workspace, float* dw, float* db, void* stream) {
  return rows_wgrad<2>(n_ops, cin, rows, ld, S1, S2, dpzr, dph, workspace, dw, db, stream);
}
