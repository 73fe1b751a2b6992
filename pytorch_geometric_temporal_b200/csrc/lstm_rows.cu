// lstm_rows.cu -- the peephole graph-LSTM cell (out = 32, n_ops <= 1: GConvLSTM and GCLSTM at K <= 2) on graphs of ANY size, split over
// CTAs by destination rows (DESIGN §4j).  One graph, one step per call.  An LSTM step has a single all-to-all dependency -- the diffusion
// of [X | H] (GConvLSTM) or of H (GCLSTM) -- so the forward is one launch and the backward a rowwise launch plus one transposed gather:
//
//   forward            k_lstm_rows_fwd<GC, HAS_H>  gather Op[X | H] (Op H); pre = S W^T + b; I, F, T, C', O, H'
//   backward           k_lstm_rows_bwd_a<GC>       dpre = (dpi, dpf, dpc, dpo), dC, dS = dpre W: the own-row block -> dX, dH, the
//                                                  operator block -> Q; per-CTA partials of the peephole sums
//                      k_lstm_rows_bwd_b<GC>       gather Op^T Q: dH (and dX for GConvLSTM) complete
//   weight gradients   k_dcrnn_wgrad<64> (train.cu) + k_lstm_rows_wgrad_reduce: dw = dpre^T S, db = 1^T dpre, the peephole sums
//
// Basis per row (X channels first): GConvLSTM [X | H | Op X | Op H], GCLSTM [X | H | Op H] (X is not diffused, gc_lstm.py:139-165).  With
// n_ops = 0 both are [X | H].  Mapping as gru_rows.cu: one warp per destination row, lane = output channel (and X channel for lane < cin),
// weights staged once per CTA at pitch 97, exact fp32 FFMA, gathers in the plan's CSR entry order.  No atomics anywhere.
#include "rows.cuh"

namespace stmp {
namespace {

using namespace rows;
constexpr int kG = 4 * kCo;                  // gate rows of the packed weights: i | f | c | o
constexpr int kQPitch = 48;                  // backward scratch row: the operator block of dS (Op X columns for GConvLSTM, then Op H)
constexpr int kPeep = 3 * kCo;               // peephole sums w_c_i | w_c_f | w_c_o

struct LstmFwd {
  const int* rowptr; const int2* cv;         // operator 0 by destination (n_ops = 1)
  int n, cin, nops, nb, ld;
  const float* x; const float* h; const float* c;        // (N, cin), (N, 32) or NULL, (N, 32) or NULL
  const float* w; const float* b; const float* peep;     // packed [128][nb], [128], (3, 32) or NULL
  float* hout; float* cout;                  // (N, 32) each
  float* stash;                              // (4, N, 32) I | F | T | O, nullable
  float* S;                                  // (N, ld) weight-gradient basis, nullable
};

template <bool GC, bool HAS_H>
__global__ void __launch_bounds__(kRowsThreads, 2) k_lstm_rows_fwd(LstmFwd a) {
  extern __shared__ float ws[];              // [128][kWPitch]
  stage_w(ws, a.w, a.nb, 0, kG);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + kCo, xo = GC ? 0 : cin;
  float bias[4];
#pragma unroll
  for (int g = 0; g < 4; ++g) bias[g] = __ldg(a.b + g * kCo + lane);
  const float wci = a.peep ? __ldg(a.peep + lane) : 0.f, wcf = a.peep ? __ldg(a.peep + kCo + lane) : 0.f;
  const float wco = a.peep ? __ldg(a.peep + 2 * kCo + lane) : 0.f;
  const float* wr = ws + lane * kWPitch;     // this lane's row of gate i; gate g at + g * 32 * kWPitch
  const size_t NC = (size_t)a.n * kCo;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const size_t io = (size_t)i * kCo + lane;
      const float xv = lane < cin ? __ldg(a.x + (size_t)i * cin + lane) : 0.f;
      const float hv = HAS_H ? __ldg(a.h + io) : 0.f;
      float lh = 0.f, lx = 0.f;
      if (a.nops && (HAS_H || !GC)) gather_row<HAS_H>(a.rowptr, a.cv, i, a.h, kCo, a.x, cin, xo, lane, lh, lx);
      float p[4] = {bias[0], bias[1], bias[2], bias[3]};   // pre = b + S W^T, S's columns in basis order
      auto col = [&](float s, int m) {
#pragma unroll
        for (int g = 0; g < 4; ++g) p[g] = fmaf(s, wr[g * kCo * kWPitch + m], p[g]);
      };
      for (int c = 0; c < cin; ++c) col(__shfl_sync(0xffffffffu, xv, c), c);
      if (HAS_H) {
#pragma unroll 8
        for (int o = 0; o < kCo; ++o) col(__shfl_sync(0xffffffffu, hv, o), cin + o);
      }
      if (a.nops) {
        if (!GC)
          for (int c = 0; c < cin; ++c) col(__shfl_sync(0xffffffffu, lx, c), C + c);
        if (HAS_H) {
#pragma unroll 8
          for (int o = 0; o < kCo; ++o) col(__shfl_sync(0xffffffffu, lh, o), C + xo + o);
        }
      }
      const float cp = a.c ? __ldg(a.c + io) : 0.f;
      const float I = sigmoidf_acc(p[0] + wci * cp), F = sigmoidf_acc(p[1] + wcf * cp), T = tanhf(p[2]);
      const float cn = F * cp + I * T;
      const float O = sigmoidf_acc(p[3] + wco * cn);         // the output gate sees the NEW cell state (gconv_lstm.py:235-236)
      a.hout[io] = O * tanhf(cn);
      a.cout[io] = cn;
      if (a.stash) {
        a.stash[io] = I;
        a.stash[NC + io] = F;
        a.stash[2 * NC + io] = T;
        a.stash[3 * NC + io] = O;
      }
      if (a.S) {                             // the basis row (+ zero padding); H = None: H columns zero
        float* r = a.S + (size_t)i * a.ld;
        if (lane < cin) r[lane] = xv;
        r[cin + lane] = hv;
        if (a.nops) {
          if (!GC && lane < cin) r[C + lane] = lx;
          r[C + xo + lane] = lh;
        }
        if (a.nb + lane < a.ld) r[a.nb + lane] = 0.f;
      }
    }
  }
}

struct LstmBwd {
  const int* rowptr; const int2* cv;         // operator 0 by SOURCE (the transposed product)
  int n, cin, nops, nb;
  const float* gh; const float* gc;          // dL/dH', dL/dC' (N, 32), either nullable
  const float* c; const float* cn;           // C (nullable: C = None) and C' of the forward
  const float* stash; const float* w; const float* peep;  // (4, N, 32), packed [128][nb], (3, 32) or NULL
  float* dpre;                               // (2, N, 64): [dpi | dpf], [dpc | dpo]
  float* q;                                  // (N, kQPitch): the operator block of dS
  float* pp;                                 // [grid][96] per-CTA peephole sums, nullable
  float* dx; float* dh; float* dc;           // (N, cin), (N, 32), (N, 32), nullable
};

template <bool GC>
__global__ void __launch_bounds__(kRowsThreads, 2) k_lstm_rows_bwd_a(LstmBwd a) {
  extern __shared__ float ws[];              // [128][kWPitch], then [kRowsWarps][96] for the peephole sums
  const bool need_ds = a.dx != nullptr || a.dh != nullptr;
  if (need_ds) stage_w(ws, a.w, a.nb, 0, kG);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + kCo;
  const float wci = a.peep ? __ldg(a.peep + lane) : 0.f, wcf = a.peep ? __ldg(a.peep + kCo + lane) : 0.f;
  const float wco = a.peep ? __ldg(a.peep + 2 * kCo + lane) : 0.f;
  const size_t NC = (size_t)a.n * kCo;
  float si = 0.f, sf = 0.f, so = 0.f;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int j = t0 + warp; j < t1; j += kRowsWarps) {
      const size_t io = (size_t)j * kCo + lane;
      const float I = a.stash[io], F = a.stash[NC + io], T = a.stash[2 * NC + io], O = a.stash[3 * NC + io];
      const float cp = a.c ? a.c[io] : 0.f, cn = a.cn[io];
      const float g = a.gh ? a.gh[io] : 0.f, gcv = a.gc ? a.gc[io] : 0.f;
      const float tc = tanhf(cn);
      const float dpo = g * tc * O * (1.f - O);
      const float dcn = gcv + g * O * (1.f - tc * tc) + dpo * wco;
      const float dpi = dcn * T * I * (1.f - I), dpf = dcn * cp * F * (1.f - F), dpc = dcn * I * (1.f - T * T);
      if (a.dc) a.dc[io] = dcn * F + dpi * wci + dpf * wcf;
      float* d0 = a.dpre + (size_t)j * 2 * kCo;
      float* d1 = a.dpre + 2 * NC + (size_t)j * 2 * kCo;
      d0[lane] = dpi;
      d0[kCo + lane] = dpf;
      d1[lane] = dpc;
      d1[kCo + lane] = dpo;
      si += dpi * cp;
      sf += dpf * cp;
      so += dpo * cn;
      if (!need_ds) continue;
      float d[3] = {0.f, 0.f, 0.f};          // dS = dpre W: basis columns m = lane + 32 q
#pragma unroll
      for (int gt = 0; gt < 4; ++gt) {
        const float dv = gt == 0 ? dpi : gt == 1 ? dpf : gt == 2 ? dpc : dpo;
        const float* wg = ws + gt * kCo * kWPitch + lane;
#pragma unroll 4
        for (int o = 0; o < kCo; ++o) {
          const float s = __shfl_sync(0xffffffffu, dv, o);
#pragma unroll
          for (int qq = 0; qq < 3; ++qq) d[qq] = fmaf(s, wg[o * kWPitch + 32 * qq], d[qq]);
        }
      }
#pragma unroll
      for (int qq = 0; qq < 3; ++qq) {
        const int m = lane + 32 * qq;
        if (m >= a.nb) continue;
        if (m < cin) {
          if (a.dx) a.dx[(size_t)j * cin + m] = d[qq];
        } else if (m < C) {
          if (a.dh) a.dh[(size_t)j * kCo + m - cin] = d[qq];
        } else {
          a.q[(size_t)j * kQPitch + m - C] = d[qq];
        }
      }
    }
  }
  if (a.pp) {                                // the CTA's peephole sums: its warps' lane sums, added in warp order
    float* red = ws + kG * kWPitch;
    red[warp * kPeep + lane] = si;
    red[warp * kPeep + kCo + lane] = sf;
    red[warp * kPeep + 2 * kCo + lane] = so;
    __syncthreads();
    if (warp == 0) {
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        float t = red[k * kCo + lane];
        for (int w = 1; w < kRowsWarps; ++w) t += red[w * kPeep + k * kCo + lane];
        a.pp[(size_t)blockIdx.x * kPeep + k * kCo + lane] = t;
      }
    }
  }
}

// dH += Op^T Q[:, xo:], and for GConvLSTM dX += Op^T Q[:, :cin]  (either nullable)
template <bool GC>
__global__ void __launch_bounds__(kRowsThreads) k_lstm_rows_bwd_b(LstmBwd a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, xo = GC ? 0 : cin;
  const int nx = (!GC && a.dx) ? cin : 0;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int j = t0 + warp; j < t1; j += kRowsWarps) {
      float th, tx;
      if (a.dh) gather_row<true>(a.rowptr, a.cv, j, a.q + xo, kQPitch, a.q, kQPitch, nx, lane, th, tx);
      else gather_row<false>(a.rowptr, a.cv, j, a.q + xo, kQPitch, a.q, kQPitch, nx, lane, th, tx);
      if (a.dh) a.dh[(size_t)j * kCo + lane] += th;
      if (lane < nx) a.dx[(size_t)j * cin + lane] += tx;
    }
  }
}

// w [128][nb]: row gate*32 + o (gates i | f | c | o), column m of the basis; b [128] = (bx + bh) + bg.
//   GConvLSTM: wx [4][n_ops+1][32][cin], wh [4][n_ops+1][32][32] (gate, Chebyshev order, out, in), bx / bh [4][32] or NULL
//   GCLSTM:    wx [4][cin][32] (the dense W_g, in x out), wh [4][n_ops+1][32][32], bx NULL, bh [4][32] or NULL
template <bool GC>
__global__ void k_lstm_rows_pack(int nops, int cin, const float* __restrict__ wx, const float* __restrict__ wh, const float* __restrict__ bx,
                                 const float* __restrict__ bh, const float* __restrict__ bg, float* __restrict__ w, float* __restrict__ b) {
  const int C = cin + kCo, nbk = nops + 1, nb = GC ? cin + nbk * kCo : nbk * C;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < kG * nb) {
    const int row = i / nb, m = i - row * nb, gate = row >> 5, o = row & 31;
    if (GC) {
      const int hm = m - cin, blk = hm >> 5, c = hm & 31;
      w[i] = m < cin ? wx[((size_t)gate * cin + m) * kCo + o] : wh[(((size_t)gate * nbk + blk) * kCo + o) * kCo + c];
    } else {
      const int blk = m / C, c = m - blk * C;
      w[i] = c < cin ? wx[(((size_t)gate * nbk + blk) * kCo + o) * cin + c] : wh[(((size_t)gate * nbk + blk) * kCo + o) * kCo + c - cin];
    }
  } else if (i < kG * nb + kG) {
    const int r = i - kG * nb;
    const float cb = (bx ? bx[r] : 0.f) + (bh ? bh[r] : 0.f);
    b[r] = cb + bg[r];
  }
}

// Fixed-order sums (fixed_order_sum, rows.cuh) of the per-CTA partials into dw [128][nb] (the packed layout), db [128] and dpeep [96]
// (both nullable).  The weight partials are k_dcrnn_wgrad<64>'s: S^T [dpi | dpf] (m*64 + row), then S^T [dpc | dpo], then the column sums
// of dpre; the peephole partials are k_lstm_rows_bwd_a's, with their own base, stride and count.
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

static int lstm_nb(int variant, int n_ops, int cin) {
  return variant == STMP_LSTM_GC ? cin + (n_ops + 1) * kCo : (n_ops + 1) * (cin + kCo);
}

static bool lstm_envelope(int variant, int n_ops, int64_t cin) {
  return (variant == STMP_LSTM_GCONV || variant == STMP_LSTM_GC) && n_ops >= 0 && n_ops <= 1 && cin >= 1 && cin <= kMaxCin;
}

static bool lstm_supported(const stmp_plan* plan, int variant, int n_ops, int64_t cin, int64_t cout) {
  return plan && lstm_envelope(variant, n_ops, cin) && n_ops <= plan->n_ops && cout == kCo;
}

static int64_t lstm_ld(int variant, int n_ops, int64_t cin) { return (lstm_nb(variant, n_ops, (int)cin) + 7) / 8 * 8; }

extern "C" int stmp_lstm_rows_supported(const stmp_plan* plan, int variant, int n_ops, int64_t cin, int64_t cout) {
  return lstm_supported(plan, variant, n_ops, cin, cout) ? 1 : 0;
}

extern "C" int stmp_lstm_rows_pack_weights(int variant, int n_ops, int64_t cin, const float* wx, const float* wh, const float* bx,
                                           const float* bh, const float* bg, float* w, float* b, void* stream) {
  STMP_REQUIRE(variant == STMP_LSTM_GCONV || variant == STMP_LSTM_GC, STMP_EINVAL, "stmp_lstm_rows_pack_weights: unknown variant %d", variant);
  STMP_REQUIRE(wx && wh && bg && w && b, STMP_EINVAL, "stmp_lstm_rows_pack_weights: NULL tensor");
  STMP_REQUIRE(variant == STMP_LSTM_GC ? bx == nullptr : !bx == !bh, STMP_EINVAL,
               "stmp_lstm_rows_pack_weights: GConvLSTM takes both ChebConv bias stacks or neither, GCLSTM no bx");
  STMP_REQUIRE(lstm_envelope(variant, n_ops, cin), STMP_EUNSUPPORTED, "stmp_lstm_rows_pack_weights: n_ops <= 1, cin 1..16 only");
  const int total = kG * lstm_nb(variant, n_ops, (int)cin) + kG;
  cudaStream_t st = (cudaStream_t)stream;
  if (variant == STMP_LSTM_GC) k_lstm_rows_pack<true><<<(total + 255) / 256, 256, 0, st>>>(n_ops, (int)cin, wx, wh, bx, bh, bg, w, b);
  else k_lstm_rows_pack<false><<<(total + 255) / 256, 256, 0, st>>>(n_ops, (int)cin, wx, wh, bx, bh, bg, w, b);
  STMP_LAUNCH_OK("k_lstm_rows_pack");
  return STMP_OK;
}

template <bool GC, bool HAS_H>
static int launch_fwd(const LstmFwd& a, int grid, cudaStream_t st) {
  const int smem = kG * kWPitch * 4;
  STMP_CUDA_OK(cudaFuncSetAttribute(k_lstm_rows_fwd<GC, HAS_H>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_lstm_rows_fwd<GC, HAS_H><<<grid, kRowsThreads, smem, st>>>(a);
  STMP_LAUNCH_OK("k_lstm_rows_fwd");
  return STMP_OK;
}

extern "C" int stmp_lstm_rows_fwd(const stmp_plan* plan, int variant, int n_ops, int64_t cin, const float* x, const float* h, const float* c,
                                  const float* w, const float* b, const float* peep, float* hout, float* cout, float* stash, float* S,
                                  int64_t ld, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_lstm_rows_fwd: plan is NULL");
  STMP_REQUIRE(variant == STMP_LSTM_GCONV || variant == STMP_LSTM_GC, STMP_EINVAL, "stmp_lstm_rows_fwd: unknown variant %d", variant);
  STMP_REQUIRE(lstm_supported(plan, variant, n_ops, cin, kCo), STMP_EUNSUPPORTED,
               "stmp_lstm_rows_fwd: n_ops <= min(1, plan's operators), cin 1..16 only (n_ops=%d, cin=%lld)", n_ops, (long long)cin);
  STMP_REQUIRE(x && w && b && hout && cout, STMP_EINVAL, "stmp_lstm_rows_fwd: NULL tensor");
  STMP_REQUIRE(!S || ld == lstm_ld(variant, n_ops, cin), STMP_ESHAPE, "stmp_lstm_rows_fwd: the basis row pitch must be nb rounded up to 8");
  const void* ps[] = {x, h, c, w, b, peep, hout, cout, stash, S};
  for (const void* p : ps) STMP_REQUIRE(al4(p), STMP_ESHAPE, "stmp_lstm_rows_fwd: misaligned tensor");
  STMP_REQUIRE(((uintptr_t)S & 15u) == 0, STMP_ESHAPE, "stmp_lstm_rows_fwd: S must be 16-byte aligned");
  if (plan->n == 0) return STMP_OK;
  LstmFwd a;
  a.rowptr = plan->fwd[0].rowptr; a.cv = plan->fwd[0].cv;
  a.n = plan->n; a.cin = (int)cin; a.nops = n_ops; a.nb = lstm_nb(variant, n_ops, (int)cin); a.ld = (int)ld;
  a.x = x; a.h = h; a.c = c; a.w = w; a.b = b; a.peep = peep; a.hout = hout; a.cout = cout; a.stash = stash; a.S = S;
  const int grid = rows_grid(plan->n);
  cudaStream_t st = (cudaStream_t)stream;
  if (variant == STMP_LSTM_GC) return h ? launch_fwd<true, true>(a, grid, st) : launch_fwd<true, false>(a, grid, st);
  return h ? launch_fwd<false, true>(a, grid, st) : launch_fwd<false, false>(a, grid, st);
}

extern "C" int64_t stmp_lstm_rows_scratch_bytes(const stmp_plan* plan) {
  return plan ? ((int64_t)plan->n * kQPitch + (int64_t)rows_grid(plan->n) * kPeep) * 4 : 0;
}

template <bool GC>
static int launch_bwd(const LstmBwd& a, int grid, bool gather, cudaStream_t st) {
  const int smem = (kG * kWPitch + kRowsWarps * kPeep) * 4;
  STMP_CUDA_OK(cudaFuncSetAttribute(k_lstm_rows_bwd_a<GC>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_lstm_rows_bwd_a<GC><<<grid, kRowsThreads, smem, st>>>(a);
  STMP_LAUNCH_OK("k_lstm_rows_bwd_a");
  if (gather) {
    k_lstm_rows_bwd_b<GC><<<grid, kRowsThreads, 0, st>>>(a);
    STMP_LAUNCH_OK("k_lstm_rows_bwd_b");
  }
  return STMP_OK;
}

extern "C" int stmp_lstm_rows_bwd(const stmp_plan* plan, int variant, int n_ops, int64_t cin, const float* gh, const float* gc,
                                  const float* c, const float* cn, const float* stash, const float* w, const float* peep, float* scratch,
                                  float* dpre, float* dx, float* dh, float* dc, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_lstm_rows_bwd: plan is NULL");
  STMP_REQUIRE(variant == STMP_LSTM_GCONV || variant == STMP_LSTM_GC, STMP_EINVAL, "stmp_lstm_rows_bwd: unknown variant %d", variant);
  STMP_REQUIRE(lstm_supported(plan, variant, n_ops, cin, kCo), STMP_EUNSUPPORTED,
               "stmp_lstm_rows_bwd: n_ops <= min(1, plan's operators), cin 1..16 only (n_ops=%d, cin=%lld)", n_ops, (long long)cin);
  STMP_REQUIRE(cn && stash && w && scratch && dpre, STMP_EINVAL, "stmp_lstm_rows_bwd: NULL tensor");
  STMP_REQUIRE(c || !dc, STMP_EINVAL, "stmp_lstm_rows_bwd: dc needs c (C = None has no state gradient)");
  const void* ps[] = {gh, gc, c, cn, stash, w, peep, scratch, dx, dh, dc};
  for (const void* p : ps) STMP_REQUIRE(al4(p), STMP_ESHAPE, "stmp_lstm_rows_bwd: misaligned tensor");
  STMP_REQUIRE(((uintptr_t)dpre & 15u) == 0, STMP_ESHAPE, "stmp_lstm_rows_bwd: dpre must be 16-byte aligned");
  if (plan->n == 0) return STMP_OK;
  LstmBwd a;
  a.rowptr = plan->bwd[0].rowptr; a.cv = plan->bwd[0].cv;
  a.n = plan->n; a.cin = (int)cin; a.nops = n_ops; a.nb = lstm_nb(variant, n_ops, (int)cin);
  a.gh = gh; a.gc = gc; a.c = c; a.cn = cn; a.stash = stash; a.w = w; a.peep = peep; a.dpre = dpre;
  a.q = scratch; a.pp = peep ? scratch + (size_t)plan->n * kQPitch : nullptr; a.dx = dx; a.dh = dh; a.dc = dc;
  const int grid = rows_grid(plan->n);
  const bool gc_basis = variant == STMP_LSTM_GC;
  const bool gather = n_ops == 1 && (dh != nullptr || (!gc_basis && dx != nullptr));      // GCLSTM: X is not diffused
  cudaStream_t st = (cudaStream_t)stream;
  return gc_basis ? launch_bwd<true>(a, grid, gather, st) : launch_bwd<false>(a, grid, gather, st);
}

extern "C" int64_t stmp_lstm_rows_wgrad_workspace_bytes(int variant, int n_ops, int64_t cin) {
  if (!lstm_envelope(variant, n_ops, cin)) return 0;
  return (int64_t)wgrad_ffma_max_parts() * (lstm_ld(variant, n_ops, cin) * kG + kG) * 4;
}

extern "C" int stmp_lstm_rows_wgrad(int variant, int n_ops, int64_t cin, int64_t rows, int64_t ld, const float* S, const float* dpre,
                                    const float* scratch, void* workspace, float* dw, float* db, float* dpeep, void* stream) {
  STMP_REQUIRE(variant == STMP_LSTM_GCONV || variant == STMP_LSTM_GC, STMP_EINVAL, "stmp_lstm_rows_wgrad: unknown variant %d", variant);
  STMP_REQUIRE(S && dpre && workspace && dw && rows >= 0 && (scratch || !dpeep), STMP_EINVAL, "stmp_lstm_rows_wgrad: bad argument");
  STMP_REQUIRE(lstm_envelope(variant, n_ops, cin), STMP_EUNSUPPORTED, "stmp_lstm_rows_wgrad: n_ops <= 1, cin 1..16 only");
  const int nb = lstm_nb(variant, n_ops, (int)cin);
  STMP_REQUIRE(ld == lstm_ld(variant, n_ops, cin), STMP_ESHAPE, "stmp_lstm_rows_wgrad: the basis row pitch must be nb rounded up to 8");
  STMP_REQUIRE((((uintptr_t)S | (uintptr_t)dpre | (uintptr_t)workspace) & 15u) == 0, STMP_ESHAPE,
               "stmp_lstm_rows_wgrad: S, dpre and the workspace must be 16-byte aligned");
  STMP_REQUIRE(al4(scratch) && al4(dw) && al4(db) && al4(dpeep), STMP_ESHAPE, "stmp_lstm_rows_wgrad: misaligned tensor");
  cudaStream_t st = (cudaStream_t)stream;
  if (rows == 0) {
    STMP_CUDA_OK(cudaMemsetAsync(dw, 0, (size_t)kG * nb * 4, st));
    if (db) STMP_CUDA_OK(cudaMemsetAsync(db, 0, (size_t)kG * 4, st));
    if (dpeep) STMP_CUDA_OK(cudaMemsetAsync(dpeep, 0, (size_t)kPeep * 4, st));
    return STMP_OK;
  }
  float* partial = reinterpret_cast<float*>(workspace);
  int parts = 0;
  const int rc = wgrad_ffma_launch(2 * kCo, rows, (int)ld, S, S, dpre, dpre + (size_t)rows * 2 * kCo, partial, st, &parts);
  if (rc != STMP_OK) return rc;
  const float* pp = dpeep ? scratch + (size_t)rows * kQPitch : nullptr;
  const int total = kG * nb + kG + kPeep;
  k_lstm_rows_wgrad_reduce<<<(total + 31) / 32, 256, 0, st>>>(parts, (int)ld / 8, nb, partial, rows_grid((int)rows), pp, dw, db, dpeep);
  STMP_LAUNCH_OK("k_lstm_rows_wgrad_reduce");
  return STMP_OK;
}
