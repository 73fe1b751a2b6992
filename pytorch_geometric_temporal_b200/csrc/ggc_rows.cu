// ggc_rows.cu -- PyG GatedGraphConv (the convolution of DyGrEncoder) on graphs of ANY size, split over CTAs by destination rows
// (DESIGN §4r).  A layer is m = x W_l, an aggregation over the in-edges (add, mean or max) and a GRUCell whose one weight set every
// layer shares; each layer's all-to-all dependency (the gather) makes it one launch:
//
//   forward, add / mean   k_ggc_rows_fwd<0> x L    gather a = Op x^l; m = a W_l; x^{l+1} = GRUCell(m, x^l)
//   forward, max          k_ggc_rows_msg           m^0 = x^0 W_0 for every row
//                         k_ggc_rows_fwd<1> x L    gather agg = max_e w_e m^l_j; x^{l+1} = GRUCell(agg, x^l); m^{l+1} = x^{l+1} W_{l+1}
//   backward              k_ggc_rows_bwd<.> x L    (l < L-1) gather Op^T of layer l + 1 -> dx^{l+1}; GRUCell backward of layer l -> dG, the
//                                                  gradient at the GRU input and the direct part of dx^l
//                         k_ggc_rows_bwd<.>        (l = -1) the transposed gather of layer 0 -> dX (and max's message gradient of layer 0)
//   weight gradients      k_ggc_rows_wgrad + k_ggc_rows_wgrad_reduce
//
// Mapping: one warp per destination row, lane = channel (C <= 32), CTAs owning grid-strided tiles of kRowTile rows, the layer's C x C
// weight, W_ih, W_hh and both biases staged once per CTA (30 KB at C = 32).  Gathers walk the plan's CSR rows in entry order with separate
// multiply and add (rows::gather_row); contractions are fp32 FFMA over shuffled operands.  No atomics: every result depends on its row
// alone, so repeated calls are bit-identical.
#include "rows.cuh"

namespace stmp {
namespace {

using namespace rows;

constexpr int kGgcMaxC = kGruMaxC;
constexpr int kGP = kGruPitch;               // the staged pitch of the GRUCell and row products (rows.cuh)
constexpr int kGgcMaxLayers = 1024;         // the weight-gradient grid holds one row of CTAs per layer
constexpr int kSlots = 8;                    // stash slots per layer
enum Slot { kX = 0, kPre = 1, kIn = 2, kR = 3, kZ = 4, kN = 5, kHn = 6, kCnt = 7 };

struct GgcW {
  const float* W; const float* wih; const float* whh; const float* bih; const float* bhh;
};

// W_l (C x C, nullable) at pitch kGP, W_ih and W_hh rows (3C x C) at pitch kGP, both biases
struct GgcSmem {
  float w[kGgcMaxC * kGP];
  float ih[3 * kGgcMaxC * kGP];
  float hh[3 * kGgcMaxC * kGP];
  float bi[3 * kGgcMaxC];
  float bh[3 * kGgcMaxC];
};

__device__ __forceinline__ void stage(GgcSmem& s, const float* __restrict__ Wl, const GgcW& g, int C, bool gru) {
  if (Wl)
    for (int i = threadIdx.x; i < C * C; i += kRowsThreads) s.w[(i / C) * kGP + i % C] = __ldg(Wl + i);
  if (gru) {
    for (int i = threadIdx.x; i < 3 * C * C; i += kRowsThreads) {
      const int r = i / C, k = i - r * C;
      s.ih[r * kGP + k] = __ldg(g.wih + i);
      s.hh[r * kGP + k] = __ldg(g.whh + i);
    }
    if (g.bih)                               // the forward's biases (the backward needs none)
      for (int i = threadIdx.x; i < 3 * C; i += kRowsThreads) {
        s.bi[i] = __ldg(g.bih + i);
        s.bh[i] = __ldg(g.bhh + i);
      }
  }
  __syncthreads();
}

struct GgcFwd {
  const int* rowptr; const int2* cv;         // the plan's operator by destination
  int n, C, cin, L;
  const float* x;                            // (N, cin)
  GgcW g;
  float* out;                                // (N, C)
  float* scr;                                // inference: x ping-pong (2 N C) | m ping-pong (2 N C)
  float* stash;                              // training: (L, kSlots, N, C), nullable
};

__device__ __forceinline__ float* slot(float* stash, int l, int s, int n, int C) {
  return stash + ((size_t)l * kSlots + s) * n * C;
}

// x^l of layer l (l >= 1) and where layer l writes x^{l+1}; m^l of the max aggregation
__device__ __forceinline__ const float* x_in(const GgcFwd& a, int l) {
  return l == 0 ? a.x : a.stash ? slot(a.stash, l, kX, a.n, a.C) : a.scr + (size_t)((l - 1) & 1) * a.n * a.C;
}
__device__ __forceinline__ float* x_out(const GgcFwd& a, int l) {
  return l == a.L - 1 ? a.out : a.stash ? slot(a.stash, l + 1, kX, a.n, a.C) : a.scr + (size_t)(l & 1) * a.n * a.C;
}
__device__ __forceinline__ float* m_buf(const GgcFwd& a, int l) {
  return a.stash ? slot(a.stash, l, kPre, a.n, a.C) : a.scr + (size_t)(2 + (l & 1)) * a.n * a.C;
}

// m^0 = x^0 W_0 (max): one warp per row
__global__ void __launch_bounds__(kRowsThreads) k_ggc_rows_msg(GgcFwd a) {
  __shared__ float w[kGgcMaxC * kGP];
  for (int i = threadIdx.x; i < a.C * a.C; i += kRowsThreads) w[(i / a.C) * kGP + i % a.C] = __ldg(a.g.W + i);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, C = a.C, lc = lane < C ? lane : 0;
  float* m = m_buf(a, 0);
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const float xv = lane < a.cin ? __ldg(a.x + (size_t)i * a.cin + lane) : 0.f;
      const float y = row_times_w(w, xv, a.cin, lc);
      if (lane < C) m[(size_t)i * C + lane] = y;
    }
  }
}

// agg = max_e (w_e * m[src_e][lane]) over CSR row i in entry order, 0 for an empty row; cnt = the number of entries equal to it, plus one
// when it is exactly 0 (the zero-initialised output of scatter_reduce(include_self=False) compares equal too)
__device__ __forceinline__ void gather_max(const int* __restrict__ rowptr, const int2* __restrict__ cv, int i, const float* __restrict__ m,
                                           int C, int lane, float& agg, float& cnt) {
  const int beg = __ldg(rowptr + i), end = __ldg(rowptr + i + 1);
  const bool on = lane < C;
  float best = 0.f, n = 0.f;
  int k = beg;
  for (; k + 4 <= end; k += 4) {
    int2 e[4];
    float v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) e[u] = __ldg(cv + k + u);
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = on ? __fmul_rn(__int_as_float(e[u].y), __ldg(m + (size_t)e[u].x * C + lane)) : 0.f;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (n == 0.f || v[u] > best) { best = v[u]; n = 1.f; }
      else if (v[u] == best) n += 1.f;
    }
  }
  for (; k < end; ++k) {
    const int2 e = __ldg(cv + k);
    const float v = on ? __fmul_rn(__int_as_float(e.y), __ldg(m + (size_t)e.x * C + lane)) : 0.f;
    if (n == 0.f || v > best) { best = v; n = 1.f; }
    else if (v == best) n += 1.f;
  }
  if (n > 0.f && best == 0.f) n += 1.f;
  agg = best;
  cnt = n;
}

// one layer: aggregate, GRUCell; MAX also writes the next layer's messages
template <bool MAX>
__global__ void __launch_bounds__(kRowsThreads) k_ggc_rows_fwd(GgcFwd a, int l) {
  __shared__ GgcSmem s;
  const int C = a.C, n = a.n;
  const bool next = l + 1 < a.L;
  stage(s, MAX ? (next ? a.g.W + (size_t)(l + 1) * C * C : nullptr) : a.g.W + (size_t)l * C * C, a.g, C, true);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, lc = lane < C ? lane : 0;
  const int kin = l == 0 ? a.cin : C;          // valid channels of x^l as stored (layer 0 reads X itself)
  const float* xl = x_in(a, l);
  float* xo = x_out(a, l);
  const float* mi = MAX ? m_buf(a, l) : nullptr;
  float* mo = MAX && next ? m_buf(a, l + 1) : nullptr;
  float* st = a.stash ? slot(a.stash, l, 0, n, C) : nullptr;
  const size_t NC = (size_t)n * C;
  float bir = 0.f, biz = 0.f, bin = 0.f, bhr = 0.f, bhz = 0.f, bhn = 0.f;
  if (lane < C) {
    bir = s.bi[lane]; biz = s.bi[C + lane]; bin = s.bi[2 * C + lane];
    bhr = s.bh[lane]; bhz = s.bh[C + lane]; bhn = s.bh[2 * C + lane];
  }
  for (int t0 = blockIdx.x * kRowTile; t0 < n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const float hv = lane < kin ? __ldg(xl + (size_t)i * kin + lane) : 0.f;
      float pre = 0.f, gin, cnt = 0.f;
      if (MAX) {
        gather_max(a.rowptr, a.cv, i, mi, C, lane, gin, cnt);
      } else {
        float unused;
        gather_row<false>(a.rowptr, a.cv, i, nullptr, 0, xl, kin, kin, lane, unused, pre);
        gin = row_times_w(s.w, pre, kin, lc);
      }
      const GruFwd g = gru_cell_fwd(s.ih, s.hh, gin, hv, bir, biz, bin, bhr, bhz, bhn, C, lc);
      const float r = g.r, z = g.z, nn = g.n, hn = g.hn, h1 = g.h;
      if (mo) {
        const float y = row_times_w(s.w, h1, C, lc);
        if (lane < C) mo[(size_t)i * C + lane] = y;
      }
      if (lane < C) {
        const size_t io = (size_t)i * C + lane;
        xo[io] = h1;
        if (st) {
          if (l == 0) st[kX * NC + io] = hv;
          if (!MAX) st[kPre * NC + io] = pre;
          st[kIn * NC + io] = gin;
          st[kR * NC + io] = r;
          st[kZ * NC + io] = z;
          st[kN * NC + io] = nn;
          st[kHn * NC + io] = hn;
          if (MAX) st[kCnt * NC + io] = cnt;
        }
      }
    }
  }
}

struct GgcBwd {
  const int* rowptr; const int2* cv;         // the plan's operator by SOURCE (the transposed product)
  int n, C, cin, L;
  const float* gout;                         // (N, C)
  const float* stash;                        // (L, kSlots, N, C)
  GgcW g;
  float* dG;                                 // (L, N, 4C): dr | dz | dn | r dn (pre-activation gradients; the last is W_hn's)
  float* dM;                                 // (L, N, C)
  float* scr;                                // the gathered operand ping-pong (2 N C) | the direct part of dx (N C)
  float* dx;                                 // (N, cin), nullable
};

// l >= 0: (l < L - 1) the transposed gather of layer l + 1 completes dx^{l+1}, then the GRUCell backward of layer l.  l = -1: the
// transposed gather of layer 0, then dX.  The operand gathered for layer q is da^q = dm^q W_q^T (add, mean) or dagg^q (max).
template <bool MAX>
__global__ void __launch_bounds__(kRowsThreads) k_ggc_rows_bwd(GgcBwd a, int l) {
  __shared__ GgcSmem s;
  const int C = a.C, n = a.n, q = l + 1;       // q: the layer whose transposed gather this launch runs (q < L)
  const bool gather = q < a.L, gru = l >= 0;
  const float* Wq = MAX ? (gather ? a.g.W + (size_t)q * C * C : nullptr) : (gru ? a.g.W + (size_t)l * C * C : nullptr);
  stage(s, Wq, a.g, C, gru);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, lc = lane < C ? lane : 0;
  const size_t NC = (size_t)n * C;
  float* dxd = a.scr + 2 * NC;
  const float* op_in = a.scr + (size_t)(q & 1) * NC;         // written by the launch of layer q
  float* op_out = a.scr + (size_t)(l & 1) * NC;              // l >= 0 only
  const float* sq = gather ? a.stash + (size_t)q * kSlots * NC : nullptr;
  const float* sl = gru ? a.stash + (size_t)l * kSlots * NC : nullptr;
  for (int t0 = blockIdx.x * kRowTile; t0 < n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, n);
    for (int j = t0 + warp; j < t1; j += kRowsWarps) {
      const size_t jo = (size_t)j * C + lc;
      float dx;                                // dL/dx^{q}_j
      if (!gather) {
        dx = lane < C ? a.gout[jo] : 0.f;
      } else if (MAX) {                        // dm_j = sum_e w_e [w_e m_j == agg_i] dagg_i / cnt_i, then dx = dxd + dm_j W_q^T
        const int beg = __ldg(a.rowptr + j), end = __ldg(a.rowptr + j + 1);
        const float mj = lane < C ? sq[kPre * NC + jo] : 0.f;
        float dm = 0.f;
        for (int k = beg; k < end; ++k) {
          const int2 e = __ldg(a.cv + k);
          const float w = __int_as_float(e.y);
          if (lane < C) {
            const size_t io = (size_t)e.x * C + lane;
            if (__fmul_rn(w, mj) == sq[kIn * NC + io]) dm = __fadd_rn(dm, __fmul_rn(w, __fdiv_rn(op_in[io], sq[kCnt * NC + io])));
          }
        }
        if (lane < C) a.dM[(size_t)q * NC + jo] = dm;
        dx = (lane < C ? dxd[jo] : 0.f) + row_times_wt(s.w, dm, C, lc);
      } else {
        float unused, t;
        gather_row<false>(a.rowptr, a.cv, j, nullptr, 0, op_in, C, C, lane, unused, t);
        dx = (lane < C ? dxd[jo] : 0.f) + t;
      }
      if (!gru) {
        if (a.dx && lane < a.cin) a.dx[(size_t)j * a.cin + lane] = dx;
        continue;
      }
      float r = 0.f, z = 0.f, nn = 0.f, hn = 0.f, hv = 0.f;
      if (lane < C) {
        r = sl[kR * NC + jo]; z = sl[kZ * NC + jo]; nn = sl[kN * NC + jo]; hn = sl[kHn * NC + jo]; hv = sl[kX * NC + jo];
      }
      const GruGrad gg = gru_cell_bwd_gates(dx, r, z, nn, hn, hv);
      if (lane < C) {
        float* g = a.dG + ((size_t)l * n + j) * 4 * C;
        g[lane] = gg.dr; g[C + lane] = gg.dz; g[2 * C + lane] = gg.dn; g[3 * C + lane] = gg.dhn;
      }
      float din = 0.f, dh = dx * z;              // the gradients at the GRU input and (direct) at x^l
      gru_cell_bwd_inputs(s.ih, s.hh, gg, C, lc, din, dh);
      float opv = din;                           // max: dagg is the operand; add / mean: dm is dW_l's, da = dm W_l^T the operand
      if (!MAX) {
        opv = row_times_wt(s.w, din, C, lc);
        if (lane < C) a.dM[(size_t)l * NC + jo] = din;
      }
      if (lane < C) {
        op_out[jo] = opv;
        dxd[jo] = dh;
      }
    }
  }
}

// ---- weight gradients -------------------------------------------------------------------------------------------------------------------
// job 0: dW_ih [3C][C] = sum over the L N rows of dgi^T gin, db_ih = sum dgi; job 1: dW_hh = sum dgh^T x^l, db_hh = sum dgh (dgi = dG's
// columns [0, 3C), dgh = [0, 2C) and [3C, 4C)); job 2 + l: dW_l [C][C] = sum over layer l's N rows of P^T dM^l, P = a^l (add, mean) or x^l
// (max).  Per-CTA partials over strided tiles of kWgRows rows, summed by k_ggc_rows_wgrad_reduce in a fixed order.
constexpr int kWgRows = 32;
constexpr int kWgOut = 3 * kGgcMaxC * kGgcMaxC;           // the largest product of a job
constexpr int kWgPart = kWgOut + 3 * kGgcMaxC;             // a partial: the product, then the column sums of A
constexpr int kWgPer = kWgOut / kRowsThreads;              // products per thread

struct GgcWg {
  int n, C, L, max_aggr;
  const float* stash; const float* dG; const float* dM;
};

__global__ void __launch_bounds__(kRowsThreads) k_ggc_rows_wgrad(GgcWg a, float* __restrict__ partial) {
  __shared__ float sa[kWgRows][3 * kGgcMaxC + 1];
  __shared__ float sb[kWgRows][kGgcMaxC + 1];
  const int job = blockIdx.y, C = a.C, tid = threadIdx.x;
  const bool gru = job < 2;
  const int ka = gru ? 3 * C : C, nout = ka * C;
  const size_t NC = (size_t)a.n * C;
  const long long rows = gru ? (long long)a.L * a.n : a.n;
  const int l0 = gru ? 0 : job - 2;
  float acc[kWgPer], cs = 0.f;
  int ar[kWgPer], bc[kWgPer];                // output o = tid + q 256: row ar of A's columns, column bc of B's
#pragma unroll
  for (int q = 0; q < kWgPer; ++q) {
    const int o = min(tid + q * kRowsThreads, nout - 1);
    acc[q] = 0.f;
    ar[q] = o / C;
    bc[q] = o - ar[q] * C;
  }
  const long long tiles = (rows + kWgRows - 1) / kWgRows;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long r0 = tile * kWgRows;
    const int nr = (int)min((long long)kWgRows, rows - r0);
    for (int e = tid; e < nr * ka; e += kRowsThreads) {
      const int rr = e / ka, c = e - rr * ka;
      const long long r = r0 + rr;
      float v;
      if (gru) {
        const long long l = r / a.n, i = r - l * a.n;
        v = a.dG[(size_t)(l * a.n + i) * 4 * C + (job == 1 && c >= 2 * C ? c + C : c)];
      } else {
        v = a.stash[((size_t)l0 * kSlots + (a.max_aggr ? kX : kPre)) * NC + (size_t)r * C + c];
      }
      sa[rr][c] = v;
    }
    for (int e = tid; e < nr * C; e += kRowsThreads) {
      const int rr = e / C, c = e - rr * C;
      const long long r = r0 + rr;
      float v;
      if (gru) {
        const long long l = r / a.n, i = r - l * a.n;
        v = a.stash[((size_t)l * kSlots + (job == 0 ? kIn : kX)) * NC + (size_t)i * C + c];
      } else {
        v = a.dM[(size_t)l0 * NC + (size_t)r * C + c];
      }
      sb[rr][c] = v;
    }
    __syncthreads();
    for (int rr = 0; rr < nr; ++rr) {
#pragma unroll
      for (int q = 0; q < kWgPer; ++q) acc[q] = fmaf(sa[rr][ar[q]], sb[rr][bc[q]], acc[q]);
      if (gru && tid < ka) cs += sa[rr][tid];
    }
    __syncthreads();
  }
  float* out = partial + ((size_t)job * gridDim.x + blockIdx.x) * kWgPart;
#pragma unroll
  for (int q = 0; q < kWgPer; ++q) {
    const int o = tid + q * kRowsThreads;
    if (o < nout) out[o] = acc[q];
  }
  if (gru && tid < ka) out[kWgOut + tid] = cs;
}

// the fixed-order sums (fixed_order_sum, rows.cuh) of the partials into dW_ih | db_ih | dW_hh | db_hh | dW (one output per lane)
__global__ void __launch_bounds__(256) k_ggc_rows_wgrad_reduce(int parts, int C, int L, const float* __restrict__ partial, float* __restrict__ dW,
                                                               float* __restrict__ dwih, float* __restrict__ dwhh, float* __restrict__ dbih,
                                                               float* __restrict__ dbhh) {
  __shared__ float sub[8][32];
  const int x = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int gw = 3 * C * C, gb = 3 * C;
  long long i = (long long)blockIdx.x * 32 + x;
  int job = -1, o = 0;
  float* dst = nullptr;
  if (i < 2 * (gw + gb)) {
    job = (int)(i / (gw + gb));
    const int k = (int)(i - (long long)job * (gw + gb));
    o = k < gw ? k : kWgOut + k - gw;
    dst = k < gw ? (job ? dwhh : dwih) + k : (job ? dbhh : dbih) + k - gw;
  } else if (i < 2 * (gw + gb) + (long long)L * C * C) {
    const long long k = i - 2 * (gw + gb);
    job = 2 + (int)(k / (C * C));
    o = (int)(k % (C * C));
    dst = dW + k;
  }
  const float* src = partial + (job >= 0 ? ((size_t)job * parts) * kWgPart + o : 0);
  const float t = fixed_order_sum(src, kWgPart, parts, dst != nullptr, sub);
  if (w == 0 && dst) *dst = t;
}

inline int wgrad_parts(long long rows) {
  const long long tiles = (rows + kWgRows - 1) / kWgRows, max_parts = wgrad_ffma_max_parts();
  return (int)(tiles < max_parts ? (tiles > 0 ? tiles : 1) : max_parts);
}

}  // namespace
}  // namespace stmp

using namespace stmp;

static bool ggc_supported(const stmp_plan* plan, int64_t L, int64_t cin, int64_t C) {
  return plan && plan->flavor == STMP_FLAVOR_GATED && plan->n_ops == 1 && L >= 1 && L <= kGgcMaxLayers && C >= 1 && C <= kGgcMaxC &&
         cin >= 1 && cin <= C;
}

extern "C" int stmp_ggc_rows_supported(const stmp_plan* plan, int64_t num_layers, int64_t cin, int64_t channels) {
  return ggc_supported(plan, num_layers, cin, channels) ? 1 : 0;
}

extern "C" int64_t stmp_ggc_rows_scratch_bytes(const stmp_plan* plan, int64_t channels) {
  return plan && channels >= 1 && channels <= kGgcMaxC ? (int64_t)4 * plan->n * channels * 4 : 0;
}

static int ggc_check(const char* fn, const stmp_plan* plan, int64_t L, int64_t cin, int64_t C) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: plan is NULL", fn);
  STMP_REQUIRE(plan->flavor == STMP_FLAVOR_GATED, STMP_EINVAL, "%s: the plan is not a GatedGraphConv plan (flavor %d)", fn, plan->flavor);
  STMP_REQUIRE(ggc_supported(plan, L, cin, C), STMP_EUNSUPPORTED, "%s: channels 1..32, cin 1..channels, num_layers 1..1024 only "
               "(num_layers=%lld, cin=%lld, channels=%lld)", fn, (long long)L, (long long)cin, (long long)C);
  return STMP_OK;
}

extern "C" int stmp_ggc_rows_fwd(const stmp_plan* plan, int64_t num_layers, int64_t cin, int64_t channels, const float* x, const float* W,
                                 const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, float* scratch, float* out,
                                 float* stash, void* stream) {
  const char* fn = "stmp_ggc_rows_fwd";
  if (int rc = ggc_check(fn, plan, num_layers, cin, channels)) return rc;
  STMP_REQUIRE(x && W && w_ih && w_hh && b_ih && b_hh && out && (stash || scratch), STMP_EINVAL, "%s: NULL tensor", fn);
  const void* ps[] = {x, W, w_ih, w_hh, b_ih, b_hh, scratch, out, stash};
  for (const void* p : ps) STMP_REQUIRE(al4(p), STMP_ESHAPE, "%s: misaligned tensor", fn);
  GgcFwd a;
  a.rowptr = plan->fwd[0].rowptr; a.cv = plan->fwd[0].cv;
  a.n = plan->n; a.C = (int)channels; a.cin = (int)cin; a.L = (int)num_layers;
  a.x = x; a.g = {W, w_ih, w_hh, b_ih, b_hh}; a.out = out; a.scr = scratch; a.stash = stash;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = rows_grid(plan->n);
  const bool mx = plan->aggr == STMP_AGGR_MAX;
  if (mx) {
    k_ggc_rows_msg<<<grid, kRowsThreads, 0, st>>>(a);
    STMP_LAUNCH_OK("k_ggc_rows_msg");
  }
  for (int l = 0; l < a.L; ++l) {
    if (mx) {
      k_ggc_rows_fwd<true><<<grid, kRowsThreads, 0, st>>>(a, l);
      STMP_LAUNCH_OK("k_ggc_rows_fwd_max");
    } else {
      k_ggc_rows_fwd<false><<<grid, kRowsThreads, 0, st>>>(a, l);
      STMP_LAUNCH_OK("k_ggc_rows_fwd");
    }
  }
  return STMP_OK;
}

extern "C" int stmp_ggc_rows_bwd(const stmp_plan* plan, int64_t num_layers, int64_t cin, int64_t channels, const float* gout,
                                 const float* stash, const float* W, const float* w_ih, const float* w_hh, float* scratch, float* dG, float* dM,
                                 float* dx, void* stream) {
  const char* fn = "stmp_ggc_rows_bwd";
  if (int rc = ggc_check(fn, plan, num_layers, cin, channels)) return rc;
  STMP_REQUIRE(gout && stash && W && w_ih && w_hh && scratch && dG && dM, STMP_EINVAL, "%s: NULL tensor", fn);
  const void* ps[] = {gout, stash, W, w_ih, w_hh, scratch, dG, dM, dx};
  for (const void* p : ps) STMP_REQUIRE(al4(p), STMP_ESHAPE, "%s: misaligned tensor", fn);
  GgcBwd a;
  a.rowptr = plan->bwd[0].rowptr; a.cv = plan->bwd[0].cv;
  a.n = plan->n; a.C = (int)channels; a.cin = (int)cin; a.L = (int)num_layers;
  a.gout = gout; a.stash = stash; a.g = {W, w_ih, w_hh, nullptr, nullptr}; a.dG = dG; a.dM = dM; a.scr = scratch; a.dx = dx;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = rows_grid(plan->n);
  const bool mx = plan->aggr == STMP_AGGR_MAX;
  for (int l = a.L - 1; l >= (mx || dx ? -1 : 0); --l) {
    if (mx) {
      k_ggc_rows_bwd<true><<<grid, kRowsThreads, 0, st>>>(a, l);
      STMP_LAUNCH_OK("k_ggc_rows_bwd_max");
    } else {
      k_ggc_rows_bwd<false><<<grid, kRowsThreads, 0, st>>>(a, l);
      STMP_LAUNCH_OK("k_ggc_rows_bwd");
    }
  }
  return STMP_OK;
}

extern "C" int64_t stmp_ggc_rows_wgrad_workspace_bytes(int64_t num_layers, int64_t channels) {
  if (num_layers < 1 || num_layers > kGgcMaxLayers || channels < 1 || channels > kGgcMaxC) return 0;
  return (int64_t)wgrad_ffma_max_parts() * (2 + num_layers) * kWgPart * 4;
}

extern "C" int stmp_ggc_rows_wgrad(const stmp_plan* plan, int64_t num_layers, int64_t channels, const float* stash, const float* dG,
                                   const float* dM, void* workspace, float* dW, float* dw_ih, float* dw_hh, float* db_ih, float* db_hh,
                                   void* stream) {
  const char* fn = "stmp_ggc_rows_wgrad";
  if (int rc = ggc_check(fn, plan, num_layers, 1, channels)) return rc;
  STMP_REQUIRE(stash && dG && dM && workspace && dW && dw_ih && dw_hh && db_ih && db_hh, STMP_EINVAL, "%s: NULL tensor", fn);
  const void* ps[] = {stash, dG, dM, workspace, dW, dw_ih, dw_hh, db_ih, db_hh};
  for (const void* p : ps) STMP_REQUIRE(al4(p), STMP_ESHAPE, "%s: misaligned tensor", fn);
  const int L = (int)num_layers, C = (int)channels;
  GgcWg a = {plan->n, C, L, plan->aggr == STMP_AGGR_MAX, stash, dG, dM};
  cudaStream_t st = (cudaStream_t)stream;
  const int parts = wgrad_parts((long long)L * plan->n);
  float* partial = reinterpret_cast<float*>(workspace);
  k_ggc_rows_wgrad<<<dim3(parts, 2 + L), kRowsThreads, 0, st>>>(a, partial);
  STMP_LAUNCH_OK("k_ggc_rows_wgrad");
  const long long outs = 2LL * (3 * C * C + 3 * C) + (long long)L * C * C;
  k_ggc_rows_wgrad_reduce<<<(unsigned)((outs + 31) / 32), 256, 0, st>>>(parts, C, L, partial, dW, dw_ih, dw_hh, db_ih, db_hh);
  STMP_LAUNCH_OK("k_ggc_rows_wgrad_reduce");
  return STMP_OK;
}
