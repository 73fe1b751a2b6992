// lstm_rows.cu -- the peephole graph-LSTM cell (out = 32 or 64, n_ops <= 1: GConvLSTM and GCLSTM at K <= 2) on graphs of ANY size, split
// over CTAs by destination rows (DESIGN §4j, §4o).  One graph, one step per call.  An LSTM step has a single all-to-all dependency -- the
// diffusion of [X | H] (GConvLSTM) or of H (GCLSTM) -- so the forward is one launch and the backward a rowwise launch plus one transposed
// gather:
//
//   forward            k_lstm_rows_fwd<NC, GC, HAS_H>  gather Op[X | H] (Op H); pre = S W^T + b; I, F, T, C', O, H'
//   backward           k_lstm_rows_bwd_a<NC, GC>       dpre = (dpi, dpf, dpc, dpo), dC, dS = dpre W: the own-row block -> dX, dH, the
//                                                      operator block -> Q; per-CTA partials of the peephole sums
//                      k_lstm_rows_bwd_b<NC, GC>       gather Op^T Q: dH (and dX for GConvLSTM) complete
//   weight gradients   out = 32: k_dcrnn_wgrad<64> (train.cu) + k_lstm_rows_wgrad_reduce; out = 64: k_wide_rows_wgrad<4> +
//                      k_wide_rows_wgrad_reduce<4> (rows.cuh): dw = dpre^T S, db = 1^T dpre, the peephole sums
//
// Basis per row (X channels first): GConvLSTM [X | H | Op X | Op H], GCLSTM [X | H | Op H] (X is not diffused, gc_lstm.py:139-165).  With
// n_ops = 0 both are [X | H].  Mapping as gru_rows.cu: one warp per destination row, lane = output channel (NC = 1, out = 32) or channels
// lane and lane + 32 (NC = 2, out = 64), and X channel for lane < cin; weights staged once per CTA at pitch LWd<NC>::P, exact fp32 FFMA,
// gathers in the plan's CSR entry order.  Every per-channel sum keeps the order of the 32-wide kernels.  No atomics anywhere.  The 64-wide
// instance (stmp_lstm_wide_rows_*) stages all 256 gate rows per CTA (161 KB): one CTA per SM, which costs nothing at the graph sizes
// the cell serves (DESIGN §4o).
#include "rows.cuh"

namespace stmp {
namespace {

using namespace rows;

// per-width constants: out channels, gate rows of the packed weights (i | f | c | o), the widest basis (GConvLSTM with NO operators,
// cin = 16), the staged weight pitch, basis columns per lane, the backward scratch row (the operator blocks of dS: per operator Op X
// columns for GConvLSTM, then Op H) and the peephole sums (w_c_i | w_c_f | w_c_o).  NO = 2 is the two-operator GConvLSTM basis of LRGCN's
// two relations, served at 32 channels only (DESIGN §4q).
template <int NC, int NO = 1>
struct LWd {
  static constexpr int CO = 32 * NC, G = 4 * CO, NB = (NO + 1) * (kMaxCin + CO), P = NB + 1, NQ = (NB + 31) / 32, QP = NO * (kMaxCin + CO),
                       PEEP = 3 * CO;
};

struct LstmFwd {
  const int* rowptr; const int2* cv;         // operator 0 by destination (n_ops = 1)
  int n, cin, nops, nb, ld;
  const float* x; const float* h; const float* c;        // (N, cin), (N, CO) or NULL, (N, CO) or NULL
  const float* w; const float* b; const float* peep;     // packed [4 CO][nb], [4 CO], (3, CO) or NULL
  float* hout; float* cout;                  // (N, CO) each
  float* stash;                              // (4, N, CO) I | F | T | O, nullable
  float* S;                                  // (N, ld) weight-gradient basis, nullable
};

// the arguments of an NO-operator instance: operator 1's CSR (by destination in the forward, by source in the backward) follows the
// one-operator arguments, which keep their layout
struct Op1 { const int* rowptr1; const int2* cv1; };
template <class A, int NO> struct WithOps : A {};
template <class A> struct WithOps<A, 2> : A, Op1 {};

template <int NC, bool GC, bool HAS_H, int NO = 1>
__global__ void __launch_bounds__(kRowsThreads, 2) k_lstm_rows_fwd(WithOps<LstmFwd, NO> a) {
  using D = LWd<NC, NO>;
  constexpr int CO = D::CO, P = D::P;
  extern __shared__ float ws[];              // [4 CO][P]
  stage_w<P>(ws, a.w, a.nb, 0, D::G);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + CO, xo = GC ? 0 : cin;
  float bias[4][NC], wci[NC], wcf[NC], wco[NC];
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    const int ch = lane + 32 * j;
#pragma unroll
    for (int g = 0; g < 4; ++g) bias[g][j] = __ldg(a.b + g * CO + ch);
    wci[j] = a.peep ? __ldg(a.peep + ch) : 0.f;
    wcf[j] = a.peep ? __ldg(a.peep + CO + ch) : 0.f;
    wco[j] = a.peep ? __ldg(a.peep + 2 * CO + ch) : 0.f;
  }
  const size_t NCn = (size_t)a.n * CO;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const float xv = lane < cin ? __ldg(a.x + (size_t)i * cin + lane) : 0.f;
      float hv[NC], lh[NC], lx = 0.f, lh1[NC], lx1 = 0.f;   // lh1, lx1: operator 1 (NO = 2)
#pragma unroll
      for (int j = 0; j < NC; ++j) { hv[j] = HAS_H ? __ldg(a.h + (size_t)i * CO + lane + 32 * j) : 0.f; lh[j] = 0.f; lh1[j] = 0.f; }
      if (a.nops && (HAS_H || !GC)) gather_rows<NC, HAS_H>(a.rowptr, a.cv, i, a.h, CO, a.x, cin, xo, lane, lh, lx);
      if constexpr (NO > 1) gather_rows<NC, HAS_H>(a.rowptr1, a.cv1, i, a.h, CO, a.x, cin, xo, lane, lh1, lx1);
      float p[4][NC];                        // pre = b + S W^T, S's columns in basis order
#pragma unroll
      for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int j = 0; j < NC; ++j) p[g][j] = bias[g][j];
      auto col = [&](float s, int m) {
#pragma unroll
        for (int g = 0; g < 4; ++g)
#pragma unroll
          for (int j = 0; j < NC; ++j) p[g][j] = fmaf(s, ws[(g * CO + lane + 32 * j) * P + m], p[g][j]);
      };
      for (int c = 0; c < cin; ++c) col(__shfl_sync(0xffffffffu, xv, c), c);
      if (HAS_H) {
#pragma unroll
        for (int jo = 0; jo < NC; ++jo) {
#pragma unroll 8
          for (int o = 0; o < 32; ++o) col(__shfl_sync(0xffffffffu, hv[jo], o), cin + 32 * jo + o);
        }
      }
      if (a.nops) {
        if (!GC)
          for (int c = 0; c < cin; ++c) col(__shfl_sync(0xffffffffu, lx, c), C + c);
        if (HAS_H) {
#pragma unroll
          for (int jo = 0; jo < NC; ++jo) {
#pragma unroll 8
            for (int o = 0; o < 32; ++o) col(__shfl_sync(0xffffffffu, lh[jo], o), C + xo + 32 * jo + o);
          }
        }
      }
      if constexpr (NO > 1) {                  // operator 1's block [Op1 X | Op1 H] at column 2 C (GConvLSTM basis only)
        for (int c = 0; c < cin; ++c) col(__shfl_sync(0xffffffffu, lx1, c), 2 * C + c);
        if (HAS_H) {
#pragma unroll
          for (int jo = 0; jo < NC; ++jo) {
#pragma unroll 8
            for (int o = 0; o < 32; ++o) col(__shfl_sync(0xffffffffu, lh1[jo], o), 2 * C + cin + 32 * jo + o);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < NC; ++j) {
        const size_t io = (size_t)i * CO + lane + 32 * j;
        const float cp = a.c ? __ldg(a.c + io) : 0.f;
        const float I = sigmoidf_acc(p[0][j] + wci[j] * cp), F = sigmoidf_acc(p[1][j] + wcf[j] * cp), T = tanhf(p[2][j]);
        const float cn = F * cp + I * T;
        const float O = sigmoidf_acc(p[3][j] + wco[j] * cn);   // the output gate sees the NEW cell state (gconv_lstm.py:235-236)
        a.hout[io] = O * tanhf(cn);
        a.cout[io] = cn;
        if (a.stash) {
          a.stash[io] = I;
          a.stash[NCn + io] = F;
          a.stash[2 * NCn + io] = T;
          a.stash[3 * NCn + io] = O;
        }
      }
      if (a.S) {                             // the basis row (+ zero padding); H = None: H columns zero
        float* r = a.S + (size_t)i * a.ld;
        if (lane < cin) r[lane] = xv;
#pragma unroll
        for (int j = 0; j < NC; ++j) r[cin + lane + 32 * j] = hv[j];
        if (a.nops) {
          if (!GC && lane < cin) r[C + lane] = lx;
#pragma unroll
          for (int j = 0; j < NC; ++j) r[C + xo + lane + 32 * j] = lh[j];
        }
        if constexpr (NO > 1) {
          if (lane < cin) r[2 * C + lane] = lx1;
#pragma unroll
          for (int j = 0; j < NC; ++j) r[2 * C + cin + lane + 32 * j] = lh1[j];
        }
        if (a.nb + lane < a.ld) r[a.nb + lane] = 0.f;
      }
    }
  }
}

struct LstmBwd {
  const int* rowptr; const int2* cv;         // operator 0 by SOURCE (the transposed product)
  int n, cin, nops, nb;
  const float* gh; const float* gc;          // dL/dH', dL/dC' (N, CO), either nullable
  const float* c; const float* cn;           // C (nullable: C = None) and C' of the forward
  const float* stash; const float* w; const float* peep;  // (4, N, CO), packed [4 CO][nb], (3, CO) or NULL
  float* dpre;                               // (2, N, 2 CO): [dpi | dpf], [dpc | dpo]
  float* q;                                  // (N, QP): the operator block of dS
  float* pp;                                 // [grid][3 CO] per-CTA peephole sums, nullable
  float* dx; float* dh; float* dc;           // (N, cin), (N, CO), (N, CO), nullable
};

template <int NC, bool GC, int NO = 1>
__global__ void __launch_bounds__(kRowsThreads, 2) k_lstm_rows_bwd_a(WithOps<LstmBwd, NO> a) {
  using D = LWd<NC, NO>;
  constexpr int CO = D::CO, P = D::P, NQ = D::NQ, QP = D::QP, PEEP = D::PEEP;
  extern __shared__ float ws[];              // [4 CO][P], then [kRowsWarps][3 CO] for the peephole sums
  const bool need_ds = a.dx != nullptr || a.dh != nullptr;
  if (need_ds) stage_w<P>(ws, a.w, a.nb, 0, D::G);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + CO;
  float wci[NC], wcf[NC], wco[NC], si[NC], sf[NC], so[NC];
#pragma unroll
  for (int j = 0; j < NC; ++j) {
    const int ch = lane + 32 * j;
    wci[j] = a.peep ? __ldg(a.peep + ch) : 0.f;
    wcf[j] = a.peep ? __ldg(a.peep + CO + ch) : 0.f;
    wco[j] = a.peep ? __ldg(a.peep + 2 * CO + ch) : 0.f;
    si[j] = sf[j] = so[j] = 0.f;
  }
  const size_t NCn = (size_t)a.n * CO;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int r = t0 + warp; r < t1; r += kRowsWarps) {
      float dp[4][NC];                       // dpi | dpf | dpc | dpo
#pragma unroll
      for (int j = 0; j < NC; ++j) {
        const int ch = lane + 32 * j;
        const size_t io = (size_t)r * CO + ch;
        const float I = a.stash[io], F = a.stash[NCn + io], T = a.stash[2 * NCn + io], O = a.stash[3 * NCn + io];
        const float cp = a.c ? a.c[io] : 0.f, cn = a.cn[io];
        const float g = a.gh ? a.gh[io] : 0.f, gcv = a.gc ? a.gc[io] : 0.f;
        const float tc = tanhf(cn);
        const float dpo = g * tc * O * (1.f - O);
        const float dcn = gcv + g * O * (1.f - tc * tc) + dpo * wco[j];
        const float dpi = dcn * T * I * (1.f - I), dpf = dcn * cp * F * (1.f - F), dpc = dcn * I * (1.f - T * T);
        if (a.dc) a.dc[io] = dcn * F + dpi * wci[j] + dpf * wcf[j];
        float* d0 = a.dpre + (size_t)r * 2 * CO;
        float* d1 = a.dpre + 2 * NCn + (size_t)r * 2 * CO;
        d0[ch] = dpi;
        d0[CO + ch] = dpf;
        d1[ch] = dpc;
        d1[CO + ch] = dpo;
        si[j] += dpi * cp;
        sf[j] += dpf * cp;
        so[j] += dpo * cn;
        dp[0][j] = dpi; dp[1][j] = dpf; dp[2][j] = dpc; dp[3][j] = dpo;
      }
      if (!need_ds) continue;
      float d[NQ];                           // dS = dpre W: basis columns m = lane + 32 q
#pragma unroll
      for (int q = 0; q < NQ; ++q) d[q] = 0.f;
#pragma unroll
      for (int gt = 0; gt < 4; ++gt) {
#pragma unroll
        for (int jo = 0; jo < NC; ++jo) {
          const float* wg = ws + (gt * CO + 32 * jo) * P + lane;
#pragma unroll 4
          for (int o = 0; o < 32; ++o) {
            const float s = __shfl_sync(0xffffffffu, dp[gt][jo], o);
#pragma unroll
            for (int q = 0; q < NQ; ++q)             // a last group past the widest basis (NB % 32 != 0) reads no column beyond it
              if (32 * (q + 1) <= D::NB || lane + 32 * q < D::NB) d[q] = fmaf(s, wg[o * P + 32 * q], d[q]);
          }
        }
      }
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int m = lane + 32 * q;
        if (m >= a.nb) continue;
        if (m < cin) {
          if (a.dx) a.dx[(size_t)r * cin + m] = d[q];
        } else if (m < C) {
          if (a.dh) a.dh[(size_t)r * CO + m - cin] = d[q];
        } else {
          a.q[(size_t)r * QP + m - C] = d[q];
        }
      }
    }
  }
  if (a.pp) {                                // the CTA's peephole sums: its warps' lane sums, added in warp order
    float* red = ws + D::G * P;
#pragma unroll
    for (int j = 0; j < NC; ++j) {
      red[warp * PEEP + lane + 32 * j] = si[j];
      red[warp * PEEP + CO + lane + 32 * j] = sf[j];
      red[warp * PEEP + 2 * CO + lane + 32 * j] = so[j];
    }
    __syncthreads();
    if (warp == 0) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
#pragma unroll
        for (int j = 0; j < NC; ++j) {
          const int e = k * CO + lane + 32 * j;
          float t = red[e];
          for (int w = 1; w < kRowsWarps; ++w) t += red[w * PEEP + e];
          a.pp[(size_t)blockIdx.x * PEEP + e] = t;
        }
      }
    }
  }
}

// dH += Op^T Q[:, xo:], and for GConvLSTM dX += Op^T Q[:, :cin]  (either nullable); with NO = 2 both operators in one pass,
// dH += Op0^T Q0 + Op1^T Q1 (Q1 at column C of the scratch row)
template <int NC, bool GC, int NO = 1>
__global__ void __launch_bounds__(kRowsThreads) k_lstm_rows_bwd_b(WithOps<LstmBwd, NO> a) {
  constexpr int CO = LWd<NC, NO>::CO, QP = LWd<NC, NO>::QP;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, xo = GC ? 0 : cin;
  const int nx = (!GC && a.dx) ? cin : 0;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int j = t0 + warp; j < t1; j += kRowsWarps) {
      float th[NC], tx, th1[NC], tx1 = 0.f;
      auto gather = [&](const int* rp, const int2* cv, const float* qk, float (&h)[NC], float& x) {
        if (a.dh) gather_rows<NC, true>(rp, cv, j, qk + xo, QP, qk, QP, nx, lane, h, x);
        else gather_rows<NC, false>(rp, cv, j, qk + xo, QP, qk, QP, nx, lane, h, x);
      };
      gather(a.rowptr, a.cv, a.q, th, tx);
      if (NO > 1) {
        if constexpr (NO > 1) gather(a.rowptr1, a.cv1, a.q + cin + CO, th1, tx1);
#pragma unroll
        for (int c = 0; c < NC; ++c) th[c] += th1[c];
        tx += tx1;
      }
      if (a.dh)
#pragma unroll
        for (int c = 0; c < NC; ++c) a.dh[(size_t)j * CO + lane + 32 * c] += th[c];
      if (lane < nx) a.dx[(size_t)j * cin + lane] += tx;
    }
  }
}

// w [4 CO][nb]: row gate*CO + o (gates i | f | c | o), column m of the basis; b [4 CO] = (bx + bh) + bg.
//   GConvLSTM: wx [4][n_ops+1][CO][cin], wh [4][n_ops+1][CO][CO] (gate, Chebyshev order or operator, out, in), bx / bh [4][CO] or NULL
//   GCLSTM:    wx [4][cin][CO] (the dense W_g, in x out), wh [4][n_ops+1][CO][CO], bx NULL, bh [4][CO] or NULL
template <int NC, bool GC>
__global__ void k_lstm_rows_pack(int nops, int cin, const float* __restrict__ wx, const float* __restrict__ wh, const float* __restrict__ bx,
                                 const float* __restrict__ bh, const float* __restrict__ bg, float* __restrict__ w, float* __restrict__ b) {
  constexpr int CO = LWd<NC>::CO, G = LWd<NC>::G;
  const int C = cin + CO, nbk = nops + 1, nb = GC ? cin + nbk * CO : nbk * C;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < G * nb) {
    const int row = i / nb, m = i - row * nb, gate = row / CO, o = row - gate * CO;
    if (GC) {
      const int hm = m - cin, blk = hm / CO, c = hm - blk * CO;
      w[i] = m < cin ? wx[((size_t)gate * cin + m) * CO + o] : wh[(((size_t)gate * nbk + blk) * CO + o) * CO + c];
    } else {
      const int blk = m / C, c = m - blk * C;
      w[i] = c < cin ? wx[(((size_t)gate * nbk + blk) * CO + o) * cin + c] : wh[(((size_t)gate * nbk + blk) * CO + o) * CO + c - cin];
    }
  } else if (i < G * nb + G) {
    const int r = i - G * nb;
    const float cb = (bx ? bx[r] : 0.f) + (bh ? bh[r] : 0.f);
    b[r] = cb + bg[r];
  }
}

constexpr int kG = LWd<1>::G, kPeep = LWd<1>::PEEP;

// Fixed-order sums (fixed_order_sum, rows.cuh) of the 32-wide cell's per-CTA partials into dw [128][nb] (the packed layout), db [128] and
// dpeep [96] (both nullable).  The weight partials are k_dcrnn_wgrad<64>'s: S^T [dpi | dpf] (m*64 + row), then S^T [dpc | dpo], then the
// column sums of dpre; the peephole partials are k_lstm_rows_bwd_a's, with their own base, stride and count.
__global__ void __launch_bounds__(256) k_lstm_rows_wgrad_reduce(int parts, int MG, int nb, const float* __restrict__ partial, int pparts,
                                                                const float* __restrict__ pp, float* __restrict__ dw, float* __restrict__ db,
                                                                float* __restrict__ dpeep) {
  __shared__ float sub[8][32];
  const int x = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + x;
  const size_t wstride = (size_t)MG * 8 * kG + kG;
  const float* base = partial;
  size_t src = 0, stride = wstride;
  int n = parts;
  float* dst = nullptr;
  if (i < kG * nb) {
    const int row = i / nb, m = i - row * nb;
    src = row < 2 * kCo ? (size_t)m * 2 * kCo + row : (size_t)MG * 8 * 2 * kCo + (size_t)m * 2 * kCo + row - 2 * kCo;
    dst = dw + i;
  } else if (i < kG * nb + kG) {
    const int r = i - kG * nb;
    src = (size_t)MG * 8 * kG + r;
    dst = db ? db + r : nullptr;
  } else if (i < kG * nb + kG + kPeep) {
    src = i - kG * nb - kG;
    base = pp;
    stride = kPeep;
    n = pparts;
    dst = dpeep ? dpeep + src : nullptr;
  }
  const float t = fixed_order_sum(base + src, stride, n, dst != nullptr, sub);
  if (w == 0 && dst) *dst = t;
}

}  // namespace
}  // namespace stmp

using namespace stmp;
using namespace stmp::rows;

static int lstm_nb(int variant, int n_ops, int cin, int cout) {
  return variant == STMP_LSTM_GC ? cin + (n_ops + 1) * cout : (n_ops + 1) * (cin + cout);
}

// n_ops <= 1 for both bases at 32 and 64 channels; n_ops = 2 (two independent one-hop operators, LRGCN's two relations) for the
// GConvLSTM basis at 32 channels only: at 64 its 256 staged gate rows would not fit in shared memory
static bool lstm_envelope(int variant, int n_ops, int64_t cin, int64_t cout) {
  return (variant == STMP_LSTM_GCONV || variant == STMP_LSTM_GC) && n_ops >= 0 &&
         (n_ops <= 1 || (n_ops == 2 && variant == STMP_LSTM_GCONV && cout == 32)) && cin >= 1 && cin <= kMaxCin;
}

static bool lstm_supported(const stmp_plan* plan, int variant, int n_ops, int64_t cin, int64_t cout) {
  return plan && (cout == 32 || cout == 64) && lstm_envelope(variant, n_ops, cin, cout) && n_ops <= plan->n_ops;
}

static int64_t lstm_ld(int variant, int n_ops, int64_t cin, int cout) { return (lstm_nb(variant, n_ops, (int)cin, cout) + 7) / 8 * 8; }

extern "C" int stmp_lstm_rows_supported(const stmp_plan* plan, int variant, int n_ops, int64_t cin, int64_t cout) {
  return lstm_supported(plan, variant, n_ops, cin, cout) ? 1 : 0;
}

// the entry and kernel names of one width, for errors and launch accounting
template <int NC> struct LNames;
template <> struct LNames<1> {
  static constexpr const char* pack = "stmp_lstm_rows_pack_weights";
  static constexpr const char* fwd = "stmp_lstm_rows_fwd";
  static constexpr const char* bwd = "stmp_lstm_rows_bwd";
  static constexpr const char* wgrad = "stmp_lstm_rows_wgrad";
  static constexpr const char* kpack = "k_lstm_rows_pack";
  static constexpr const char* kfwd = "k_lstm_rows_fwd";
  static constexpr const char* bwd_a = "k_lstm_rows_bwd_a";
  static constexpr const char* bwd_b = "k_lstm_rows_bwd_b";
  static constexpr const char* wgrad_reduce = "k_lstm_rows_wgrad_reduce";
};
template <> struct LNames<2> {
  static constexpr const char* pack = "stmp_lstm_wide_rows_pack_weights";
  static constexpr const char* fwd = "stmp_lstm_wide_rows_fwd";
  static constexpr const char* bwd = "stmp_lstm_wide_rows_bwd";
  static constexpr const char* wgrad = "stmp_lstm_wide_rows_wgrad";
  static constexpr const char* kpack = "k_lstm_wide_rows_pack";
  static constexpr const char* kfwd = "k_lstm_wide_rows_fwd";
  static constexpr const char* bwd_a = "k_lstm_wide_rows_bwd_a";
  static constexpr const char* bwd_b = "k_lstm_wide_rows_bwd_b";
  static constexpr const char* wgrad_reduce = "k_lstm_wide_rows_wgrad_reduce";
};

template <int NC>
static int lstm_pack_weights(int variant, int n_ops, int64_t cin, const float* wx, const float* wh, const float* bx, const float* bh,
                             const float* bg, float* w, float* b, void* stream) {
  using N = LNames<NC>;
  constexpr int CO = LWd<NC>::CO, G = LWd<NC>::G;
  STMP_REQUIRE(variant == STMP_LSTM_GCONV || variant == STMP_LSTM_GC, STMP_EINVAL, "%s: unknown variant %d", N::pack, variant);
  STMP_REQUIRE(wx && wh && bg && w && b, STMP_EINVAL, "%s: NULL tensor", N::pack);
  STMP_REQUIRE(variant == STMP_LSTM_GC ? bx == nullptr : !bx == !bh, STMP_EINVAL,
               "%s: GConvLSTM takes both ChebConv bias stacks or neither, GCLSTM no bx", N::pack);
  STMP_REQUIRE(lstm_envelope(variant, n_ops, cin, CO), STMP_EUNSUPPORTED, "%s: n_ops <= 1 (2 for GConvLSTM at 32 channels), cin 1..16 only",
               N::pack);
  const int total = G * lstm_nb(variant, n_ops, (int)cin, CO) + G;
  cudaStream_t st = (cudaStream_t)stream;
  if (variant == STMP_LSTM_GC) k_lstm_rows_pack<NC, true><<<(total + 255) / 256, 256, 0, st>>>(n_ops, (int)cin, wx, wh, bx, bh, bg, w, b);
  else k_lstm_rows_pack<NC, false><<<(total + 255) / 256, 256, 0, st>>>(n_ops, (int)cin, wx, wh, bx, bh, bg, w, b);
  STMP_LAUNCH_OK(N::kpack);
  return STMP_OK;
}

template <int NC, bool GC, bool HAS_H, int NO = 1>
static int launch_fwd(const WithOps<LstmFwd, NO>& a, int grid, cudaStream_t st) {
  const int smem = LWd<NC, NO>::G * LWd<NC, NO>::P * 4;
  STMP_CUDA_OK(cudaFuncSetAttribute(k_lstm_rows_fwd<NC, GC, HAS_H, NO>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_lstm_rows_fwd<NC, GC, HAS_H, NO><<<grid, kRowsThreads, smem, st>>>(a);
  STMP_LAUNCH_OK(LNames<NC>::kfwd);
  return STMP_OK;
}

template <int NC>
static int lstm_fwd(const stmp_plan* plan, int variant, int n_ops, int64_t cin, const float* x, const float* h, const float* c, const float* w,
                    const float* b, const float* peep, float* hout, float* cout, float* stash, float* S, int64_t ld, void* stream) {
  using N = LNames<NC>;
  constexpr int CO = LWd<NC>::CO;
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: plan is NULL", N::fwd);
  STMP_REQUIRE(variant == STMP_LSTM_GCONV || variant == STMP_LSTM_GC, STMP_EINVAL, "%s: unknown variant %d", N::fwd, variant);
  STMP_REQUIRE(lstm_supported(plan, variant, n_ops, cin, CO), STMP_EUNSUPPORTED,
               "%s: n_ops <= the plan's operators and 1 (2 for GConvLSTM at 32 channels), cin 1..16 only (n_ops=%d, cin=%lld)", N::fwd, n_ops,
               (long long)cin);
  STMP_REQUIRE(x && w && b && hout && cout, STMP_EINVAL, "%s: NULL tensor", N::fwd);
  STMP_REQUIRE(!S || ld == lstm_ld(variant, n_ops, cin, CO), STMP_ESHAPE, "%s: the basis row pitch must be nb rounded up to 8", N::fwd);
  const void* ps[] = {x, h, c, w, b, peep, hout, cout, stash, S};
  for (const void* p : ps) STMP_REQUIRE(al4(p), STMP_ESHAPE, "%s: misaligned tensor", N::fwd);
  STMP_REQUIRE(((uintptr_t)S & 15u) == 0, STMP_ESHAPE, "%s: S must be 16-byte aligned", N::fwd);
  if (plan->n == 0) return STMP_OK;
  WithOps<LstmFwd, 1> a;
  a.rowptr = plan->fwd[0].rowptr; a.cv = plan->fwd[0].cv;
  a.n = plan->n; a.cin = (int)cin; a.nops = n_ops; a.nb = lstm_nb(variant, n_ops, (int)cin, CO); a.ld = (int)ld;
  a.x = x; a.h = h; a.c = c; a.w = w; a.b = b; a.peep = peep; a.hout = hout; a.cout = cout; a.stash = stash; a.S = S;
  const int grid = rows_grid(plan->n);
  cudaStream_t st = (cudaStream_t)stream;
  if constexpr (NC == 1) {
    if (n_ops == 2) {
      WithOps<LstmFwd, 2> a2;
      static_cast<LstmFwd&>(a2) = a;
      a2.rowptr1 = plan->fwd[1].rowptr; a2.cv1 = plan->fwd[1].cv;
      return h ? launch_fwd<NC, false, true, 2>(a2, grid, st) : launch_fwd<NC, false, false, 2>(a2, grid, st);
    }
  }
  if (variant == STMP_LSTM_GC) return h ? launch_fwd<NC, true, true>(a, grid, st) : launch_fwd<NC, true, false>(a, grid, st);
  return h ? launch_fwd<NC, false, true>(a, grid, st) : launch_fwd<NC, false, false>(a, grid, st);
}

// the backward scratch row: the operator blocks of dS, one per operator of the widest basis the plan serves (two on a two-operator plan
// at 32 channels)
template <int NC>
static int lstm_qp(int n_ops) { return NC == 1 && n_ops >= 2 ? LWd<1, 2>::QP : LWd<NC>::QP; }

// the backward scratch: N scratch rows, then the per-CTA peephole sums
template <int NC>
static int64_t lstm_scratch_bytes(const stmp_plan* plan) {
  return plan ? ((int64_t)plan->n * lstm_qp<NC>(plan->n_ops) + (int64_t)rows_grid(plan->n) * LWd<NC>::PEEP) * 4 : 0;
}

template <int NC, bool GC, int NO = 1>
static int launch_bwd(const WithOps<LstmBwd, NO>& a, int grid, bool gather, cudaStream_t st) {
  using D = LWd<NC, NO>;
  const int smem = (D::G * D::P + kRowsWarps * D::PEEP) * 4;
  STMP_CUDA_OK(cudaFuncSetAttribute(k_lstm_rows_bwd_a<NC, GC, NO>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_lstm_rows_bwd_a<NC, GC, NO><<<grid, kRowsThreads, smem, st>>>(a);
  STMP_LAUNCH_OK(LNames<NC>::bwd_a);
  if (gather) {
    k_lstm_rows_bwd_b<NC, GC, NO><<<grid, kRowsThreads, 0, st>>>(a);
    STMP_LAUNCH_OK(LNames<NC>::bwd_b);
  }
  return STMP_OK;
}

template <int NC>
static int lstm_bwd(const stmp_plan* plan, int variant, int n_ops, int64_t cin, const float* gh, const float* gc, const float* c,
                    const float* cn, const float* stash, const float* w, const float* peep, float* scratch, float* dpre, float* dx, float* dh,
                    float* dc, void* stream) {
  using N = LNames<NC>;
  constexpr int CO = LWd<NC>::CO;
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: plan is NULL", N::bwd);
  STMP_REQUIRE(variant == STMP_LSTM_GCONV || variant == STMP_LSTM_GC, STMP_EINVAL, "%s: unknown variant %d", N::bwd, variant);
  STMP_REQUIRE(lstm_supported(plan, variant, n_ops, cin, CO), STMP_EUNSUPPORTED,
               "%s: n_ops <= the plan's operators and 1 (2 for GConvLSTM at 32 channels), cin 1..16 only (n_ops=%d, cin=%lld)", N::bwd, n_ops,
               (long long)cin);
  STMP_REQUIRE(cn && stash && w && scratch && dpre, STMP_EINVAL, "%s: NULL tensor", N::bwd);
  STMP_REQUIRE(c || !dc, STMP_EINVAL, "%s: dc needs c (C = None has no state gradient)", N::bwd);
  const void* ps[] = {gh, gc, c, cn, stash, w, peep, scratch, dx, dh, dc};
  for (const void* p : ps) STMP_REQUIRE(al4(p), STMP_ESHAPE, "%s: misaligned tensor", N::bwd);
  STMP_REQUIRE(((uintptr_t)dpre & 15u) == 0, STMP_ESHAPE, "%s: dpre must be 16-byte aligned", N::bwd);
  if (plan->n == 0) return STMP_OK;
  WithOps<LstmBwd, 1> a;
  a.rowptr = plan->bwd[0].rowptr; a.cv = plan->bwd[0].cv;
  a.n = plan->n; a.cin = (int)cin; a.nops = n_ops; a.nb = lstm_nb(variant, n_ops, (int)cin, CO);
  a.gh = gh; a.gc = gc; a.c = c; a.cn = cn; a.stash = stash; a.w = w; a.peep = peep; a.dpre = dpre;
  a.q = scratch; a.pp = peep ? scratch + (size_t)plan->n * lstm_qp<NC>(n_ops) : nullptr; a.dx = dx; a.dh = dh; a.dc = dc;
  const int grid = rows_grid(plan->n);
  const bool gc_basis = variant == STMP_LSTM_GC;
  const bool gather = n_ops >= 1 && (dh != nullptr || (!gc_basis && dx != nullptr));      // GCLSTM: X is not diffused
  cudaStream_t st = (cudaStream_t)stream;
  if constexpr (NC == 1) {
    if (n_ops == 2) {
      WithOps<LstmBwd, 2> a2;
      static_cast<LstmBwd&>(a2) = a;
      a2.rowptr1 = plan->bwd[1].rowptr; a2.cv1 = plan->bwd[1].cv;
      return launch_bwd<NC, false, 2>(a2, grid, gather, st);
    }
  }
  return gc_basis ? launch_bwd<NC, true>(a, grid, gather, st) : launch_bwd<NC, false>(a, grid, gather, st);
}

// the weight-gradient workspace: wgrad_ffma_max_parts() partials of (ld + 1) * 4 CO floats (at 64 wide, one of (ld + 1) * CO per gate)
template <int NC>
static int64_t lstm_wgrad_workspace_bytes(int variant, int n_ops, int64_t cin) {
  if (n_ops > 1 || !lstm_envelope(variant, n_ops, cin, LWd<NC>::CO)) return 0;
  return (int64_t)wgrad_ffma_max_parts() * (lstm_ld(variant, n_ops, cin, LWd<NC>::CO) + 1) * LWd<NC>::G * 4;
}

// Exact fp32: per-CTA FFMA partials over strided row tiles, then a fixed-order sum into the packed layout dw [4 CO][nb], db [4 CO] and the
// peephole sums dpeep [3 CO].  The 32-wide cell contracts with train.cu's k_dcrnn_wgrad<64> (16-row tiles), the 64-wide one with
// k_wide_rows_wgrad<4> (32-row tiles, one partial per gate and CTA).
template <int NC>
static int lstm_wgrad(int variant, int n_ops, int64_t cin, int64_t rows, int64_t ld, const float* S, const float* dpre, const float* scratch,
                      void* workspace, float* dw, float* db, float* dpeep, void* stream) {
  using N = LNames<NC>;
  using D = LWd<NC>;
  constexpr int CO = D::CO, G = D::G;
  STMP_REQUIRE(variant == STMP_LSTM_GCONV || variant == STMP_LSTM_GC, STMP_EINVAL, "%s: unknown variant %d", N::wgrad, variant);
  STMP_REQUIRE(S && dpre && workspace && dw && rows >= 0 && (scratch || !dpeep), STMP_EINVAL, "%s: bad argument", N::wgrad);
  STMP_REQUIRE(n_ops <= 1 && lstm_envelope(variant, n_ops, cin, CO), STMP_EUNSUPPORTED, "%s: n_ops <= 1, cin 1..16 only", N::wgrad);
  const int nb = lstm_nb(variant, n_ops, (int)cin, CO);
  STMP_REQUIRE(ld == lstm_ld(variant, n_ops, cin, CO), STMP_ESHAPE, "%s: the basis row pitch must be nb rounded up to 8", N::wgrad);
  STMP_REQUIRE((((uintptr_t)S | (uintptr_t)dpre | (uintptr_t)workspace) & 15u) == 0, STMP_ESHAPE,
               "%s: S, dpre and the workspace must be 16-byte aligned", N::wgrad);
  STMP_REQUIRE(al4(scratch) && al4(dw) && al4(db) && al4(dpeep), STMP_ESHAPE, "%s: misaligned tensor", N::wgrad);
  cudaStream_t st = (cudaStream_t)stream;
  if (rows == 0) {
    STMP_CUDA_OK(cudaMemsetAsync(dw, 0, (size_t)G * nb * 4, st));
    if (db) STMP_CUDA_OK(cudaMemsetAsync(db, 0, (size_t)G * 4, st));
    if (dpeep) STMP_CUDA_OK(cudaMemsetAsync(dpeep, 0, (size_t)D::PEEP * 4, st));
    return STMP_OK;
  }
  float* partial = reinterpret_cast<float*>(workspace);
  const float* pp = dpeep ? scratch + (size_t)rows * D::QP : nullptr;
  const int pparts = rows_grid((int)rows), reduce_grid = (G * nb + G + D::PEEP + 31) / 32;
  if constexpr (NC == 1) {
    int parts = 0;
    const int rc = wgrad_ffma_launch(2 * CO, rows, (int)ld, S, S, dpre, dpre + (size_t)rows * 2 * CO, partial, st, &parts);
    if (rc != STMP_OK) return rc;
    k_lstm_rows_wgrad_reduce<<<reduce_grid, 256, 0, st>>>(parts, (int)ld / 8, nb, partial, pparts, pp, dw, db, dpeep);
  } else {
    const int parts = wide_wgrad_parts(rows);
    const float* d1 = dpre + (size_t)rows * 2 * CO;          // [dpc | dpo]
    const WideWgradOps<4> op = {{S, S, S, S}, {dpre, dpre + CO, d1, d1 + CO}, {2 * CO, 2 * CO, 2 * CO, 2 * CO}};
    k_wide_rows_wgrad<4><<<dim3(parts, 4), kWideWgThreads, 0, st>>>(rows, (int)ld, op, partial);
    STMP_LAUNCH_OK("k_lstm_wide_rows_wgrad");
    k_wide_rows_wgrad_reduce<4><<<reduce_grid, 256, 0, st>>>(parts, (int)ld, nb, partial, D::PEEP, pparts, pp, dw, db, dpeep);
  }
  STMP_LAUNCH_OK(N::wgrad_reduce);
  return STMP_OK;
}

extern "C" int stmp_lstm_rows_pack_weights(int variant, int n_ops, int64_t cin, const float* wx, const float* wh, const float* bx,
                                           const float* bh, const float* bg, float* w, float* b, void* stream) {
  return lstm_pack_weights<1>(variant, n_ops, cin, wx, wh, bx, bh, bg, w, b, stream);
}

extern "C" int stmp_lstm_rows_fwd(const stmp_plan* plan, int variant, int n_ops, int64_t cin, const float* x, const float* h, const float* c,
                                  const float* w, const float* b, const float* peep, float* hout, float* cout, float* stash, float* S,
                                  int64_t ld, void* stream) {
  return lstm_fwd<1>(plan, variant, n_ops, cin, x, h, c, w, b, peep, hout, cout, stash, S, ld, stream);
}

extern "C" int64_t stmp_lstm_rows_scratch_bytes(const stmp_plan* plan) { return lstm_scratch_bytes<1>(plan); }

extern "C" int stmp_lstm_rows_bwd(const stmp_plan* plan, int variant, int n_ops, int64_t cin, const float* gh, const float* gc,
                                  const float* c, const float* cn, const float* stash, const float* w, const float* peep, float* scratch,
                                  float* dpre, float* dx, float* dh, float* dc, void* stream) {
  return lstm_bwd<1>(plan, variant, n_ops, cin, gh, gc, c, cn, stash, w, peep, scratch, dpre, dx, dh, dc, stream);
}

extern "C" int64_t stmp_lstm_rows_wgrad_workspace_bytes(int variant, int n_ops, int64_t cin) {
  return lstm_wgrad_workspace_bytes<1>(variant, n_ops, cin);
}

extern "C" int stmp_lstm_rows_wgrad(int variant, int n_ops, int64_t cin, int64_t rows, int64_t ld, const float* S, const float* dpre,
                                    const float* scratch, void* workspace, float* dw, float* db, float* dpeep, void* stream) {
  return lstm_wgrad<1>(variant, n_ops, cin, rows, ld, S, dpre, scratch, workspace, dw, db, dpeep, stream);
}

extern "C" int stmp_lstm_wide_rows_pack_weights(int variant, int n_ops, int64_t cin, const float* wx, const float* wh, const float* bx,
                                                const float* bh, const float* bg, float* w, float* b, void* stream) {
  return lstm_pack_weights<2>(variant, n_ops, cin, wx, wh, bx, bh, bg, w, b, stream);
}

extern "C" int stmp_lstm_wide_rows_fwd(const stmp_plan* plan, int variant, int n_ops, int64_t cin, const float* x, const float* h,
                                       const float* c, const float* w, const float* b, const float* peep, float* hout, float* cout,
                                       float* stash, float* S, int64_t ld, void* stream) {
  return lstm_fwd<2>(plan, variant, n_ops, cin, x, h, c, w, b, peep, hout, cout, stash, S, ld, stream);
}

extern "C" int64_t stmp_lstm_wide_rows_scratch_bytes(const stmp_plan* plan) { return lstm_scratch_bytes<2>(plan); }

extern "C" int stmp_lstm_wide_rows_bwd(const stmp_plan* plan, int variant, int n_ops, int64_t cin, const float* gh, const float* gc,
                                       const float* c, const float* cn, const float* stash, const float* w, const float* peep,
                                       float* scratch, float* dpre, float* dx, float* dh, float* dc, void* stream) {
  return lstm_bwd<2>(plan, variant, n_ops, cin, gh, gc, c, cn, stash, w, peep, scratch, dpre, dx, dh, dc, stream);
}

extern "C" int64_t stmp_lstm_wide_rows_wgrad_workspace_bytes(int variant, int n_ops, int64_t cin) {
  return lstm_wgrad_workspace_bytes<2>(variant, n_ops, cin);
}

extern "C" int stmp_lstm_wide_rows_wgrad(int variant, int n_ops, int64_t cin, int64_t rows, int64_t ld, const float* S, const float* dpre,
                                         const float* scratch, void* workspace, float* dw, float* db, float* dpeep, void* stream) {
  return lstm_wgrad<2>(variant, n_ops, cin, rows, ld, S, dpre, scratch, workspace, dw, db, dpeep, stream);
}

// The two-operator GConvLSTM basis at 32 channels (nb = 3 (cin + 32) <= 144): the 64-wide cells' per-gate contraction with the packed rows
// taken as two 64-row halves, [dpi | dpf] and [dpc | dpo] (k_wide_rows_wgrad<2>, 32-row tiles), then its fixed-order reduce into dw [128][nb]
// and db [128].  No peepholes (LRGCN has none).
extern "C" int64_t stmp_lstm_rows_wgrad2_workspace_bytes(int64_t cin) {
  if (!lstm_envelope(STMP_LSTM_GCONV, 2, cin, kCo)) return 0;
  return (int64_t)wgrad_ffma_max_parts() * (lstm_ld(STMP_LSTM_GCONV, 2, cin, kCo) + 1) * kG * 4;
}

extern "C" int stmp_lstm_rows_wgrad2(int64_t cin, int64_t rows, int64_t ld, const float* S, const float* dpre, void* workspace, float* dw,
                                     float* db, void* stream) {
  STMP_REQUIRE(S && dpre && workspace && dw && rows >= 0, STMP_EINVAL, "stmp_lstm_rows_wgrad2: bad argument");
  STMP_REQUIRE(lstm_envelope(STMP_LSTM_GCONV, 2, cin, kCo), STMP_EUNSUPPORTED, "stmp_lstm_rows_wgrad2: cin 1..16 only");
  const int nb = lstm_nb(STMP_LSTM_GCONV, 2, (int)cin, kCo);
  STMP_REQUIRE(ld == lstm_ld(STMP_LSTM_GCONV, 2, cin, kCo), STMP_ESHAPE, "stmp_lstm_rows_wgrad2: the basis row pitch must be nb rounded up to 8");
  STMP_REQUIRE((((uintptr_t)S | (uintptr_t)dpre | (uintptr_t)workspace) & 15u) == 0, STMP_ESHAPE,
               "stmp_lstm_rows_wgrad2: S, dpre and the workspace must be 16-byte aligned");
  STMP_REQUIRE(al4(dw) && al4(db), STMP_ESHAPE, "stmp_lstm_rows_wgrad2: misaligned tensor");
  cudaStream_t st = (cudaStream_t)stream;
  if (rows == 0) {
    STMP_CUDA_OK(cudaMemsetAsync(dw, 0, (size_t)kG * nb * 4, st));
    if (db) STMP_CUDA_OK(cudaMemsetAsync(db, 0, (size_t)kG * 4, st));
    return STMP_OK;
  }
  const int parts = wide_wgrad_parts(rows);
  const WideWgradOps<2> op = {{S, S}, {dpre, dpre + (size_t)rows * 2 * kCo}, {2 * kCo, 2 * kCo}};
  k_wide_rows_wgrad<2><<<dim3(parts, 2), kWideWgThreads, 0, st>>>(rows, (int)ld, op, reinterpret_cast<float*>(workspace));
  STMP_LAUNCH_OK("k_lstm_rows_wgrad2");
  k_wide_rows_wgrad_reduce<2><<<(kG * nb + kG + 31) / 32, 256, 0, st>>>(parts, (int)ld, nb, reinterpret_cast<const float*>(workspace), 0, 0,
                                                                         nullptr, dw, db, nullptr);
  STMP_LAUNCH_OK("k_lstm_rows_wgrad2_reduce");
  return STMP_OK;
}
