// evolvegcn_rows.cu -- EvolveGCN-O and EvolveGCN-H (DESIGN §4s) on graphs of ANY size, split over CTAs by destination rows.  One call
// evolves the C x C weight with a torch GRU step over its C rows (batch C, features C) and then applies GCNConv_Fixed_W: out = Op (X W_t),
// computed as (Op X) W_t.  Op is the plan's operator: gcn_norm (STMP_FLAVOR_GCN) or the raw edge weights (STMP_FLAVOR_GATED, add).
//
//   forward, -O     k_egcn_fwd<false>     W_t = GRU(W_{t-1}, W_{t-1}) in every CTA; a = Op x; out = a W_t
//   forward, -H     k_egcn_score          s = tanh((x p) / |p|) per node; per-CTA top-C candidates (score desc, lower index on ties)
//                   k_egcn_fwd<true>      every CTA merges the candidates -> perm; X~ = X[perm] s[perm]; W_t = GRU(X~, W_{t-1}); as -O
//   backward        k_egcn_bwd_rows       dX = Op^T (dOut) W_t^T; per-CTA partials of a^T dOut (a stashed by the training forward)
//                   k_egcn_wgrad          (one CTA) dW_t = the fixed-order sum of the partials + the incoming dW_t; the GRU recomputed and
//                                         its backward over the C rows; -H: the TopK backward into dX[perm] and dp
//
// Every CTA of a forward launch stages W_{t-1}, W_ih, W_hh and both biases and runs the same GRU on the same operands, so its W_t is
// bit-identical everywhere and no grid-wide synchronisation is needed; CTA 0 writes it (and -H's selection) out.  The gathers walk the
// plan's CSR rows in entry order with separate multiply and add (rows::gather_row); contractions are fp32 FFMA; no atomics, so repeated
// calls are bit-identical.
#include "rows.cuh"

namespace stmp {
namespace {

using namespace rows;

constexpr int kEgMaxC = kGruMaxC;
constexpr int kP = kGruPitch;
constexpr int kSelParts = 256;               // the most CTAs of k_egcn_score: the merge gives each list one thread of the 256

struct EgGru {
  const float* wprev; const float* wih; const float* whh; const float* bih; const float* bhh;
};

struct EgSmem {
  float w[kEgMaxC * kP];                     // W_{t-1}, then W_t in place (row r is read and rewritten by the warp that owns it)
  float ih[3 * kEgMaxC * kP];
  float hh[3 * kEgMaxC * kP];
  float bi[3 * kEgMaxC];
  float bh[3 * kEgMaxC];
  float xt[kEgMaxC * kP];                    // -H: the GRU input X~ = X[perm] s[perm]
  float sc[kEgMaxC];                         // -H: s[perm]
  int perm[kEgMaxC];
};

__device__ __forceinline__ void stage(EgSmem& s, const EgGru& g, int C) {
  for (int i = threadIdx.x; i < C * C; i += kRowsThreads) s.w[(i / C) * kP + i % C] = __ldg(g.wprev + i);
  for (int i = threadIdx.x; i < 3 * C * C; i += kRowsThreads) {
    const int r = i / C, k = i - r * C;
    s.ih[r * kP + k] = __ldg(g.wih + i);
    s.hh[r * kP + k] = __ldg(g.whh + i);
  }
  for (int i = threadIdx.x; i < 3 * C; i += kRowsThreads) {
    s.bi[i] = __ldg(g.bih + i);
    s.bh[i] = __ldg(g.bhh + i);
  }
  __syncthreads();
}

// GRU row r of the shared operands (input X~ row r for -H, W_{t-1} row r for -O; hidden W_{t-1} row r)
__device__ __forceinline__ GruFwd gru_row(const EgSmem& s, bool topk, int r, int C, int lane, int lc) {
  const float hv = lane < C ? s.w[r * kP + lane] : 0.f;
  const float gin = topk ? (lane < C ? s.xt[r * kP + lane] : 0.f) : hv;
  float bir = 0.f, biz = 0.f, bin = 0.f, bhr = 0.f, bhz = 0.f, bhn = 0.f;
  if (lane < C) {
    bir = s.bi[lane]; biz = s.bi[C + lane]; bin = s.bi[2 * C + lane];
    bhr = s.bh[lane]; bhz = s.bh[C + lane]; bhn = s.bh[2 * C + lane];
  }
  return gru_cell_fwd(s.ih, s.hh, gin, hv, bir, biz, bin, bhr, bhz, bhn, C, lc);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- the TopK order: a higher score first, the lower node index on equal scores; index -1 is "none" and comes last -------------------
struct Cand {
  float s;
  int i, tag;                                // tag: the candidate list a merge took it from
};

__device__ __forceinline__ bool before(const Cand& a, const Cand& b) {
  if (a.i < 0) return false;
  if (b.i < 0) return true;
  return a.s > b.s || (a.s == b.s && a.i < b.i);
}

// The first of every thread's candidate in the TopK order, returned to every thread.  The order is total on distinct indices, so the
// result does not depend on the reduction's association.  Holds two __syncthreads; `red` is 8 entries of shared memory.
__device__ __forceinline__ Cand block_first(Cand c, Cand* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Cand d;
    d.s = __shfl_xor_sync(0xffffffffu, c.s, o);
    d.i = __shfl_xor_sync(0xffffffffu, c.i, o);
    d.tag = __shfl_xor_sync(0xffffffffu, c.tag, o);
    if (before(d, c)) c = d;
  }
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = c;
  __syncthreads();
  Cand b = red[0];
  for (int w = 1; w < kRowsWarps; ++w)
    if (before(red[w], b)) b = red[w];
  __syncthreads();
  return b;
}

// |p| from lanes < C of one warp
__device__ __forceinline__ float pnorm(const float* __restrict__ p, int C, int lane) {
  const float v = lane < C ? __ldg(p + lane) : 0.f;
  return sqrtf(warp_sum(v * v));
}

// ---- -H, launch 1: scores and per-CTA candidates ------------------------------------------------------------------------------------
struct EgScore {
  int n, C;
  const float* x; const float* p;
  float* score;                              // (N)
  float* cand_s; int* cand_i;                // (gridDim.x, C): this CTA's first C nodes in the TopK order (index -1 past its rows)
};

__global__ void __launch_bounds__(kRowsThreads) k_egcn_score(EgScore a) {
  __shared__ Cand red[kRowsWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, C = a.C, n = a.n;
  const float norm = pnorm(a.p, C, lane);
  const float pv = lane < C ? __ldg(a.p + lane) : 0.f;
  for (int t0 = blockIdx.x * kRowTile; t0 < n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const float u = warp_sum(lane < C ? __fmul_rn(__ldg(a.x + (size_t)i * C + lane), pv) : 0.f);
      if (lane == 0) a.score[i] = tanhf(__fdiv_rn(u, norm));
    }
  }
  __syncthreads();                           // this CTA's scores, read back below (plain loads: written by this launch)
  const long long stride = (long long)gridDim.x * kRowTile;
  Cand last = {0.f, -1, 0};
  for (int r = 0; r < C; ++r) {
    Cand best = {0.f, -1, 0};
    for (long long t = blockIdx.x * kRowTile + (threadIdx.x >> 4) * stride; t < n; t += 16 * stride) {
      const int i = (int)t + (threadIdx.x & 15);
      if (i >= n) continue;
      const Cand c = {a.score[i], i, 0};
      if ((r == 0 || before(last, c)) && before(c, best)) best = c;
    }
    best = block_first(best, red);
    if (threadIdx.x == 0) {
      a.cand_s[(size_t)blockIdx.x * C + r] = best.s;
      a.cand_i[(size_t)blockIdx.x * C + r] = best.i;
    }
    last = best;
    if (best.i < 0) {                         // this CTA's rows are exhausted (uniform across the block)
      for (int q = r + 1 + (int)threadIdx.x; q < C; q += kRowsThreads) a.cand_i[(size_t)blockIdx.x * C + q] = -1;
      break;
    }
  }
}

// ---- forward ------------------------------------------------------------------------------------------------------------------------
struct EgFwd {
  const int* rowptr; const int2* cv;         // the plan's operator by destination
  int n, C;
  const float* x;                            // (N, C)
  EgGru g;
  float* out;                                // (N, C)
  float* wnew;                               // (C, C)
  float* stash;                              // training: a = Op x (N, C), nullable
  // -H
  const float* cand_s; const int* cand_i; int parts;
  int* perm; float* sc;                      // (C): the selection, written by CTA 0
};

template <bool TOPK>
__global__ void __launch_bounds__(kRowsThreads, 2) k_egcn_fwd(EgFwd a) {
  __shared__ EgSmem s;
  __shared__ Cand red[kRowsWarps];
  __shared__ int head[kSelParts];
  const int C = a.C, n = a.n, tid = threadIdx.x;
  stage(s, a.g, C);
  const int lane = tid & 31, warp = tid >> 5, lc = lane < C ? lane : 0;
  if (TOPK) {                                // merge the per-CTA lists: C rounds, each takes the first head in the TopK order
    for (int q = tid; q < kSelParts; q += kRowsThreads) head[q] = 0;
    __syncthreads();
    for (int r = 0; r < C; ++r) {
      Cand c = {0.f, -1, tid};
      if (tid < a.parts) {
        const int h = head[tid];
        if (h < C) c = {__ldg(a.cand_s + (size_t)tid * C + h), __ldg(a.cand_i + (size_t)tid * C + h), tid};
      }
      const Cand b = block_first(c, red);    // the host guarantees N >= C, so b.i >= 0
      if (tid == 0) {
        s.perm[r] = b.i;
        s.sc[r] = b.s;
        head[b.tag] += 1;
      }
      __syncthreads();
    }
    for (int e = tid; e < C * C; e += kRowsThreads) {
      const int r = e / C, c = e - r * C;
      s.xt[r * kP + c] = __fmul_rn(__ldg(a.x + (size_t)s.perm[r] * C + c), s.sc[r]);
    }
    if (blockIdx.x == 0 && tid < C) {
      a.perm[tid] = s.perm[tid];
      a.sc[tid] = s.sc[tid];
    }
    __syncthreads();
  }
  for (int r = warp; r < C; r += kRowsWarps) {
    const GruFwd g = gru_row(s, TOPK, r, C, lane, lc);
    if (lane < C) {
      s.w[r * kP + lane] = g.h;
      if (blockIdx.x == 0) a.wnew[r * C + lane] = g.h;
    }
  }
  __syncthreads();
  for (int t0 = blockIdx.x * kRowTile; t0 < n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      float unused, ax;
      gather_row<false>(a.rowptr, a.cv, i, nullptr, 0, a.x, C, C, lane, unused, ax);
      const float y = row_times_w(s.w, ax, C, lc);
      if (lane < C) {
        a.out[(size_t)i * C + lane] = y;
        if (a.stash) a.stash[(size_t)i * C + lane] = ax;
      }
    }
  }
}

// ---- backward, launch 1: dX = Op^T dOut W_t^T and the per-CTA partials of a^T dOut --------------------------------------------------
struct EgBwd {
  const int* rowptr; const int2* cv;         // the plan's operator by SOURCE
  int n, C;
  const float* gout;                         // (N, C)
  const float* stash;                        // a (N, C)
  const float* wnew;                         // W_t (C, C)
  float* dx;                                 // (N, C), nullable
  float* partial;                            // (gridDim.x, C, C)
};

__global__ void __launch_bounds__(kRowsThreads, 2) k_egcn_bwd_rows(EgBwd a) {
  __shared__ float w[kEgMaxC * kP];
  __shared__ float red[kRowsWarps][kEgMaxC * kEgMaxC];
  const int C = a.C, n = a.n, tid = threadIdx.x;
  for (int i = tid; i < C * C; i += kRowsThreads) w[(i / C) * kP + i % C] = __ldg(a.wnew + i);
  __syncthreads();
  const int lane = tid & 31, warp = tid >> 5, lc = lane < C ? lane : 0;
  float acc[kEgMaxC];
#pragma unroll
  for (int k = 0; k < kEgMaxC; ++k) acc[k] = 0.f;
  for (int t0 = blockIdx.x * kRowTile; t0 < n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, n);
    for (int j = t0 + warp; j < t1; j += kRowsWarps) {
      if (a.dx) {
        float unused, t;
        gather_row<false>(a.rowptr, a.cv, j, nullptr, 0, a.gout, C, C, lane, unused, t);
        const float d = row_times_wt(w, t, C, lc);
        if (lane < C) a.dx[(size_t)j * C + lane] = d;
      }
      const size_t jo = (size_t)j * C + lane;
      const float av = lane < C ? __ldg(a.stash + jo) : 0.f, gv = lane < C ? __ldg(a.gout + jo) : 0.f;
#pragma unroll
      for (int k = 0; k < kEgMaxC; ++k)
        if (k < C) acc[k] = fmaf(__shfl_sync(0xffffffffu, av, k), gv, acc[k]);
    }
  }
#pragma unroll
  for (int k = 0; k < kEgMaxC; ++k)
    if (k < C) red[warp][k * kEgMaxC + lane] = acc[k];
  __syncthreads();
  for (int o = tid; o < C * C; o += kRowsThreads) {
    const int k = o / C, c = o - k * C;
    float v = red[0][k * kEgMaxC + c];
    for (int q = 1; q < kRowsWarps; ++q) v += red[q][k * kEgMaxC + c];
    a.partial[(size_t)blockIdx.x * C * C + o] = v;
  }
}

// ---- backward, launch 2 (one CTA): dW_t, the GRU backward and -H's TopK backward ---------------------------------------------------------
struct EgWg {
  int parts, C;
  const float* partial;                      // (parts, C, C), then dG (C, 4C) as this launch's scratch
  const float* gwnew;                        // the incoming dL/dW_t (C, C), nullable
  EgGru g;
  const float* x; const float* p; const int* perm; const float* sc;    // -H (p non-NULL)
  float* dwprev; float* dwih; float* dwhh; float* dbih; float* dbhh;
  float* dp;                                 // -H: (C)
  float* dx;                                 // -H: (N, C), nullable; the TopK term is added to the rows perm
};

template <bool TOPK>
__global__ void __launch_bounds__(kRowsThreads) k_egcn_wgrad(EgWg a) {
  __shared__ EgSmem s;
  __shared__ float dw[kEgMaxC * kP];         // dL/dW_t, then dL/dX~ (-H)
  __shared__ float sub[8][32];
  __shared__ float du[kEgMaxC], uu[kEgMaxC];
  const int C = a.C, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, lc = lane < C ? lane : 0;
  float* dG = const_cast<float*>(a.partial) + (size_t)a.parts * C * C;
  stage(s, a.g, C);
  if (TOPK) {
    if (tid < C) {
      s.perm[tid] = __ldg(a.perm + tid);
      s.sc[tid] = __ldg(a.sc + tid);
    }
    __syncthreads();
    for (int e = tid; e < C * C; e += kRowsThreads) {
      const int r = e / C, c = e - r * C;
      s.xt[r * kP + c] = __fmul_rn(__ldg(a.x + (size_t)s.perm[r] * C + c), s.sc[r]);
    }
  }
  for (int o0 = 0; o0 < C * C; o0 += 32) {   // dW_t: 32 outputs per pass, one per lane
    const int o = o0 + lane;
    const bool live = o < C * C;
    const float t = fixed_order_sum(a.partial + (live ? o : 0), (size_t)C * C, a.parts, live, sub);
    if (warp == 0 && live) dw[(o / C) * kP + o % C] = t + (a.gwnew ? __ldg(a.gwnew + o) : 0.f);
    __syncthreads();
  }
  for (int r = warp; r < C; r += kRowsWarps) {
    const GruFwd f = gru_row(s, TOPK, r, C, lane, lc);
    const float hv = lane < C ? s.w[r * kP + lane] : 0.f;
    const GruGrad gg = gru_cell_bwd_gates(lane < C ? dw[r * kP + lane] : 0.f, f.r, f.z, f.n, f.hn, hv);
    float din = 0.f, dh = (lane < C ? dw[r * kP + lane] : 0.f) * f.z;
    gru_cell_bwd_inputs(s.ih, s.hh, gg, C, lc, din, dh);
    __syncwarp();
    if (lane < C) {
      float* q = dG + (size_t)r * 4 * C;
      q[lane] = gg.dr; q[C + lane] = gg.dz; q[2 * C + lane] = gg.dn; q[3 * C + lane] = gg.dhn;
      a.dwprev[r * C + lane] = TOPK ? dh : din + dh;
      if (TOPK) dw[r * kP + lane] = din;      // dL/dX~ row r (this warp alone reads and writes row r)
    }
  }
  __syncthreads();
  // dW_ih [3C][C] = sum_r dgi_r^T gin_r, dW_hh = sum_r dgh_r^T h_r; db_ih = sum_r dgi_r, db_hh = sum_r dgh_r (dgi = [dr dz dn],
  // dgh = [dr dz dhn]), every sum over the C rows in row order
  for (int o = tid; o < 3 * C * C; o += kRowsThreads) {
    const int j = o / C, k = o - j * C, jh = j < 2 * C ? j : j + C;
    float si = 0.f, sh = 0.f;
    for (int r = 0; r < C; ++r) {
      const float h = s.w[r * kP + k], in = TOPK ? s.xt[r * kP + k] : h;
      si = fmaf(dG[(size_t)r * 4 * C + j], in, si);
      sh = fmaf(dG[(size_t)r * 4 * C + jh], h, sh);
    }
    a.dwih[o] = si;
    a.dwhh[o] = sh;
  }
  for (int j = tid; j < 3 * C; j += kRowsThreads) {
    const int jh = j < 2 * C ? j : j + C;
    float bi = 0.f, bh = 0.f;
    for (int r = 0; r < C; ++r) {
      bi += dG[(size_t)r * 4 * C + j];
      bh += dG[(size_t)r * 4 * C + jh];
    }
    a.dbih[j] = bi;
    a.dbhh[j] = bh;
  }
  if (!TOPK) return;
  // X~_r = X[perm_r] s_r, s = tanh(v), v = (x p) / |p|: dX[perm_r] += dX~_r s_r + dv_r p / |p|, dp = sum_r dv_r (x_r / |p| - u_r p / |p|^3)
  const float norm = pnorm(a.p, C, lane);
  const float pv = lane < C ? __ldg(a.p + lane) : 0.f;
  for (int r = warp; r < C; r += kRowsWarps) {
    const int i = s.perm[r];
    const float xv = lane < C ? __ldg(a.x + (size_t)i * C + lane) : 0.f, dxt = lane < C ? dw[r * kP + lane] : 0.f;
    const float ds = warp_sum(dxt * xv), u = warp_sum(__fmul_rn(xv, pv));
    const float dv = ds * (1.f - s.sc[r] * s.sc[r]);
    if (lane == 0) { du[r] = dv; uu[r] = u; }
    if (a.dx && lane < C) {
      float* d = a.dx + (size_t)i * C + lane;
      *d = *d + dxt * s.sc[r] + dv * pv / norm;
    }
  }
  __syncthreads();
  if (tid < C) {
    const float pc = __ldg(a.p + tid), n3 = norm * norm * norm;
    float acc = 0.f;
    for (int r = 0; r < C; ++r) acc += du[r] * (__ldg(a.x + (size_t)s.perm[r] * C + tid) / norm - uu[r] * pc / n3);
    a.dp[tid] = acc;
  }
}

}  // namespace
}  // namespace stmp

using namespace stmp;

static bool egcn_supported(const stmp_plan* plan, int64_t C) {
  if (!plan || plan->n_ops < 1 || C < 1 || C > kEgMaxC) return false;
  return plan->flavor == STMP_FLAVOR_GCN || (plan->flavor == STMP_FLAVOR_GATED && plan->aggr == STMP_AGGR_ADD);
}

static int egcn_check(const char* fn, const stmp_plan* plan, int64_t C) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: plan is NULL", fn);
  STMP_REQUIRE(plan->flavor == STMP_FLAVOR_GCN || plan->flavor == STMP_FLAVOR_GATED, STMP_EINVAL,
               "%s: the plan is neither a GCN nor a GatedGraphConv plan (flavor %d)", fn, plan->flavor);
  STMP_REQUIRE(egcn_supported(plan, C), STMP_EUNSUPPORTED, "%s: channels 1..32 on a GCN plan or an add GatedGraphConv plan only "
               "(channels=%lld)", fn, (long long)C);
  return STMP_OK;
}

static int score_grid(int n) { const int g = rows_grid(n); return g < kSelParts ? g : kSelParts; }

extern "C" int stmp_evolvegcn_rows_supported(const stmp_plan* plan, int64_t channels) {
  return egcn_supported(plan, channels) ? 1 : 0;
}

extern "C" int64_t stmp_evolvegcn_rows_scratch_bytes(const stmp_plan* plan, int64_t channels) {
  if (!egcn_supported(plan, channels)) return 0;
  return (int64_t)4 * plan->n + (int64_t)8 * kSelParts * channels;
}

extern "C" int stmp_evolvegcn_rows_fwd(const stmp_plan* plan, int64_t channels, const float* x, const float* w_prev, const float* w_ih,
                                       const float* w_hh, const float* b_ih, const float* b_hh, const float* p, void* scratch, float* out,
                                       float* w_new, int32_t* perm, float* score, float* stash, void* stream) {
  const char* fn = "stmp_evolvegcn_rows_fwd";
  if (int rc = egcn_check(fn, plan, channels)) return rc;
  STMP_REQUIRE(x && w_prev && w_ih && w_hh && b_ih && b_hh && out && w_new, STMP_EINVAL, "%s: NULL tensor", fn);
  STMP_REQUIRE(!p || (scratch && perm && score), STMP_EINVAL, "%s: -H (p given) needs scratch, perm and score", fn);
  STMP_REQUIRE(!p || plan->n >= channels, STMP_EUNSUPPORTED, "%s: -H selects channels=%lld of %d nodes", fn, (long long)channels,
               plan->n);
  const void* ps[] = {x, w_prev, w_ih, w_hh, b_ih, b_hh, p, scratch, out, w_new, perm, score, stash};
  for (const void* q : ps) STMP_REQUIRE(al4(q), STMP_ESHAPE, "%s: misaligned tensor", fn);
  const int C = (int)channels, n = plan->n;
  cudaStream_t st = (cudaStream_t)stream;
  EgFwd a = {};
  a.rowptr = plan->fwd[0].rowptr; a.cv = plan->fwd[0].cv;
  a.n = n; a.C = C; a.x = x; a.g = {w_prev, w_ih, w_hh, b_ih, b_hh};
  a.out = out; a.wnew = w_new; a.stash = stash;
  if (!p) {
    k_egcn_fwd<false><<<rows_grid(n), kRowsThreads, 0, st>>>(a);
    STMP_LAUNCH_OK("k_egcn_fwd");
    return STMP_OK;
  }
  const int parts = score_grid(n);
  float* sscore = reinterpret_cast<float*>(scratch);
  float* cand_s = sscore + n;
  int* cand_i = reinterpret_cast<int*>(cand_s + (size_t)kSelParts * C);
  k_egcn_score<<<parts, kRowsThreads, 0, st>>>(EgScore{n, C, x, p, sscore, cand_s, cand_i});
  STMP_LAUNCH_OK("k_egcn_score");
  a.cand_s = cand_s; a.cand_i = cand_i; a.parts = parts; a.perm = perm; a.sc = score;
  k_egcn_fwd<true><<<rows_grid(n), kRowsThreads, 0, st>>>(a);
  STMP_LAUNCH_OK("k_egcn_fwd_topk");
  return STMP_OK;
}

extern "C" int64_t stmp_evolvegcn_rows_workspace_bytes(const stmp_plan* plan, int64_t channels) {
  if (!egcn_supported(plan, channels)) return 0;
  return ((int64_t)rows_grid(plan->n) * channels * channels + 4 * channels * channels) * 4;
}

extern "C" int stmp_evolvegcn_rows_bwd(const stmp_plan* plan, int64_t channels, const float* gout, const float* stash, const float* w_new,
                                       void* workspace, float* dx, void* stream) {
  const char* fn = "stmp_evolvegcn_rows_bwd";
  if (int rc = egcn_check(fn, plan, channels)) return rc;
  STMP_REQUIRE(gout && stash && w_new && workspace, STMP_EINVAL, "%s: NULL tensor", fn);
  const void* ps[] = {gout, stash, w_new, workspace, dx};
  for (const void* q : ps) STMP_REQUIRE(al4(q), STMP_ESHAPE, "%s: misaligned tensor", fn);
  EgBwd a = {plan->bwd[0].rowptr, plan->bwd[0].cv, plan->n, (int)channels, gout, stash, w_new, dx, reinterpret_cast<float*>(workspace)};
  k_egcn_bwd_rows<<<rows_grid(plan->n), kRowsThreads, 0, (cudaStream_t)stream>>>(a);
  STMP_LAUNCH_OK("k_egcn_bwd_rows");
  return STMP_OK;
}

extern "C" int stmp_evolvegcn_rows_wgrad(const stmp_plan* plan, int64_t channels, void* workspace, const float* g_wnew, const float* x,
                                         const float* w_prev, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                                         const float* p, const int32_t* perm, const float* score, float* dw_prev, float* dw_ih,
                                         float* dw_hh, float* db_ih, float* db_hh, float* dp, float* dx, void* stream) {
  const char* fn = "stmp_evolvegcn_rows_wgrad";
  if (int rc = egcn_check(fn, plan, channels)) return rc;
  STMP_REQUIRE(workspace && w_prev && w_ih && w_hh && b_ih && b_hh && dw_prev && dw_ih && dw_hh && db_ih && db_hh, STMP_EINVAL,
               "%s: NULL tensor", fn);
  STMP_REQUIRE(!p || (x && perm && score && dp), STMP_EINVAL, "%s: -H (p given) needs x, perm, score and dp", fn);
  const void* ps[] = {workspace, g_wnew, x, w_prev, w_ih, w_hh, b_ih, b_hh, p, perm, score, dw_prev, dw_ih, dw_hh, db_ih, db_hh, dp, dx};
  for (const void* q : ps) STMP_REQUIRE(al4(q), STMP_ESHAPE, "%s: misaligned tensor", fn);
  EgWg a = {rows_grid(plan->n), (int)channels, reinterpret_cast<const float*>(workspace), g_wnew, {w_prev, w_ih, w_hh, b_ih, b_hh},
            x, p, perm, score, dw_prev, dw_ih, dw_hh, db_ih, db_hh, dp, dx};
  cudaStream_t st = (cudaStream_t)stream;
  if (p) {
    k_egcn_wgrad<true><<<1, kRowsThreads, 0, st>>>(a);
    STMP_LAUNCH_OK("k_egcn_wgrad_topk");
  } else {
    k_egcn_wgrad<false><<<1, kRowsThreads, 0, st>>>(a);
    STMP_LAUNCH_OK("k_egcn_wgrad");
  }
  return STMP_OK;
}
