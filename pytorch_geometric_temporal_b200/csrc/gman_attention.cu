// gman_attention.cu -- GMAN's multi-head attention (DESIGN §4w), in exact fp32.  One family serves the reference's three attentions
// (nn/attention/gman.py: SpatialAttention, TemporalAttention, TransformAttention) straight from the channels-last (B, T, N, D)
// activations: a problem is one (p0, p1) pair, `heads` heads of width W sit side by side in the channels (head h = channels
// [h W, (h + 1) W)), and each of Q, K, V, O has its own outer strides s0, s1 and sequence stride sl, so no call copies or permutes.
//
//   S = scale Q K^T (scale = 1/sqrt(heads), the reference's 1/sqrt(d)), masked: S[i][j] = -32767 for j > i (kept in the softmax sum)
//   O = softmax(S) V,  lse[i] = log sum_j exp(S[i][j])  (the training stash, (p0, p1, heads, Lq) floats)
//
//   long  kernels (any Lq, Lk, no mask; the spatial attention)      one thread per query row, online softmax over 64-key tiles staged in
//         k_gman_attn_long_fwd                                       shared memory, 16 keys per rescale (each chunk summed on its own)
//         k_gman_attn_long_bwd_q                                     one thread per query row: D = rowsum(dO . O) into the workspace, and dQ
//         k_gman_attn_long_bwd_kv                                    one thread per key row: dK, dV over 64-query tiles (P from lse)
//   short kernels (Lq, Lk <= 64; the temporal and transform ones)   one warp per (problem, head), lanes own rows lane and lane + 32
//         k_gman_attn_short_fwd                                      exact two-pass softmax in registers
//         k_gman_attn_short_bwd                                      one launch: dQ and D per query row, then dK, dV per key row
//
// The long kernels' sums over thousands of rows are two-level (per 16-key chunk or 64-row tile, then across them), which keeps their
// rounding error near that of a blocked GEMM.  Head widths 1..16 run in the instances W = 8 and 16 with the missing channels zero in registers (exact).  Every sum runs in one fixed
// order, there are no atomics and no tensor cores: repeated calls and backwards are bit-identical, and the training forward is the
// inference forward plus the lse store.
#include <math.h>

#include "common.cuh"

namespace stmp {
namespace {

constexpr int kLongThreads = 128;            // query (or key) rows per CTA of the long kernels
constexpr int kTile = 64;                    // keys (or queries) per shared-memory tile
constexpr int kChunk = 16;                   // keys per online-softmax rescale
constexpr int kShortFwdWarps = 4, kShortBwdWarps = 2;
constexpr int kMaxShort = 64, kMaxWidth = 16;
constexpr float kMasked = -32767.f;          // the reference's -(2 ** 15) + 1

struct View {
  const float* p;
  int64_t s0, s1, sl;
};

struct Args {
  int64_t p1, heads, width;                  // problems (p0, p1) flattened as p0 * p1 + p1_index
  int lq, lk, mask;
  float scale;
  View q, k, v, o, dout;                     // dout has O's strides
  float *out, *lse, *delta;                  // O (O's strides), the stash and the long backward's D
  float *dq, *dk, *dv;                       // Q's, K's and V's strides; each NULL when not asked for
};

__device__ __forceinline__ int64_t base_of(const View& t, const Args& a, int64_t prob, int64_t h) {
  const int64_t i0 = prob / a.p1, i1 = prob - i0 * a.p1;
  return i0 * t.s0 + i1 * t.s1 + h * a.width;
}

template <int W>
__device__ __forceinline__ void load_row(float (&r)[W], const float* __restrict__ p, int width) {
#pragma unroll
  for (int c = 0; c < W; ++c) r[c] = c < width ? __ldg(p + c) : 0.f;
}

template <int W>
__device__ __forceinline__ float dot(const float (&a)[W], const float* b) {
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < W; ++c) s = fmaf(a[c], b[c], s);
  return s;
}

template <int W>
__device__ __forceinline__ float dot_rr(const float (&a)[W], const float (&b)[W]) {
  float s = 0.f;
#pragma unroll
  for (int c = 0; c < W; ++c) s = fmaf(a[c], b[c], s);
  return s;
}

// rows [r0, r0 + n) of a (p, h) slice of t -> sm[kTile][W] (rows >= n and channels >= width zero), by all threads of the CTA
template <int W>
__device__ __forceinline__ void stage(float* sm, const View& t, int64_t base, int r0, int n, int width, int nthreads) {
  for (int e = threadIdx.x; e < kTile * W; e += nthreads) {
    const int r = e / W, c = e - r * W;
    sm[e] = (r < n && c < width) ? __ldg(t.p + base + (int64_t)(r0 + r) * t.sl + c) : 0.f;
  }
}

// ---- long kernels ---------------------------------------------------------------------------------------------------------------------
template <int W>
__global__ void __launch_bounds__(kLongThreads) k_gman_attn_long_fwd(const Args a) {
  __shared__ __align__(16) float Ks[kTile * W];
  __shared__ __align__(16) float Vs[kTile * W];
  const int nqb = (a.lq + kLongThreads - 1) / kLongThreads;
  const int64_t ph = blockIdx.x / nqb, prob = ph / a.heads, h = ph - prob * a.heads;
  const int i = (int)(blockIdx.x - ph * nqb) * kLongThreads + threadIdx.x;
  const bool live = i < a.lq;
  const int64_t bq = base_of(a.q, a, prob, h), bk = base_of(a.k, a, prob, h), bv = base_of(a.v, a, prob, h);
  float q[W], o[W];
  if (live) load_row<W>(q, a.q.p + bq + (int64_t)i * a.q.sl, (int)a.width);
  else
#pragma unroll
    for (int c = 0; c < W; ++c) q[c] = 0.f;
#pragma unroll
  for (int c = 0; c < W; ++c) o[c] = 0.f;
  float m = -INFINITY, l = 0.f;
  for (int j0 = 0; j0 < a.lk; j0 += kTile) {
    const int nt = min(kTile, a.lk - j0);
    stage<W>(Ks, a.k, bk, j0, nt, (int)a.width, kLongThreads);
    stage<W>(Vs, a.v, bv, j0, nt, (int)a.width, kLongThreads);
    __syncthreads();
    for (int jj = 0; jj < nt; jj += kChunk) {
      float s[kChunk];
      float cm = -INFINITY;
#pragma unroll
      for (int u = 0; u < kChunk; ++u) {
        s[u] = jj + u < nt ? dot<W>(q, Ks + (jj + u) * W) * a.scale : -INFINITY;
        cm = fmaxf(cm, s[u]);
      }
      const float mn = fmaxf(m, cm);
      const float corr = expf(m - mn);
      float cl = 0.f, oc[W];                 // the chunk's own sums, added to the running ones once: a two-level sum over the keys
#pragma unroll
      for (int c = 0; c < W; ++c) oc[c] = 0.f;
#pragma unroll
      for (int u = 0; u < kChunk; ++u) {
        if (jj + u < nt) {
          const float p = expf(s[u] - mn);
          cl += p;
          const float* vr = Vs + (jj + u) * W;
#pragma unroll
          for (int c = 0; c < W; ++c) oc[c] = fmaf(p, vr[c], oc[c]);
        }
      }
      l = fmaf(l, corr, cl);
#pragma unroll
      for (int c = 0; c < W; ++c) o[c] = fmaf(o[c], corr, oc[c]);
      m = mn;
    }
    __syncthreads();
  }
  if (!live) return;
  float* orow = a.out + base_of(a.o, a, prob, h) + (int64_t)i * a.o.sl;
#pragma unroll
  for (int c = 0; c < W; ++c)
    if (c < a.width) orow[c] = o[c] / l;
  if (a.lse) a.lse[ph * a.lq + i] = m + logf(l);
}

// D[i] = dO[i] . O[i] and, with dq, dQ[i] = scale sum_j P[i][j] (dO[i] . V[j] - D[i]) K[j]
template <int W>
__global__ void __launch_bounds__(kLongThreads) k_gman_attn_long_bwd_q(const Args a) {
  __shared__ __align__(16) float Ks[kTile * W];
  __shared__ __align__(16) float Vs[kTile * W];
  const int nqb = (a.lq + kLongThreads - 1) / kLongThreads;
  const int64_t ph = blockIdx.x / nqb, prob = ph / a.heads, h = ph - prob * a.heads;
  const int i = (int)(blockIdx.x - ph * nqb) * kLongThreads + threadIdx.x;
  const bool live = i < a.lq;
  float q[W], g[W], dq[W];
  float D = 0.f, lse = 0.f;
#pragma unroll
  for (int c = 0; c < W; ++c) q[c] = g[c] = dq[c] = 0.f;
  if (live) {
    float o[W];
    load_row<W>(q, a.q.p + base_of(a.q, a, prob, h) + (int64_t)i * a.q.sl, (int)a.width);
    load_row<W>(g, a.dout.p + base_of(a.dout, a, prob, h) + (int64_t)i * a.dout.sl, (int)a.width);
    load_row<W>(o, a.o.p + base_of(a.o, a, prob, h) + (int64_t)i * a.o.sl, (int)a.width);
    D = dot_rr<W>(g, o);
    lse = a.lse[ph * a.lq + i];
    a.delta[ph * a.lq + i] = D;
  }
  if (!a.dq) return;                         // grid-uniform
  const int64_t bk = base_of(a.k, a, prob, h), bv = base_of(a.v, a, prob, h);
  for (int j0 = 0; j0 < a.lk; j0 += kTile) {
    const int nt = min(kTile, a.lk - j0);
    stage<W>(Ks, a.k, bk, j0, nt, (int)a.width, kLongThreads);
    stage<W>(Vs, a.v, bv, j0, nt, (int)a.width, kLongThreads);
    __syncthreads();
    float tq[W];                             // the tile's own sum, added once: a two-level sum over the keys
#pragma unroll
    for (int c = 0; c < W; ++c) tq[c] = 0.f;
    for (int j = 0; j < nt; ++j) {
      const float* kr = Ks + j * W;
      const float p = expf(dot<W>(q, kr) * a.scale - lse);
      const float ds = p * (dot<W>(g, Vs + j * W) - D);
#pragma unroll
      for (int c = 0; c < W; ++c) tq[c] = fmaf(ds, kr[c], tq[c]);
    }
#pragma unroll
    for (int c = 0; c < W; ++c) dq[c] += tq[c];
    __syncthreads();
  }
  if (!live) return;
  float* r = a.dq + base_of(a.q, a, prob, h) + (int64_t)i * a.q.sl;
#pragma unroll
  for (int c = 0; c < W; ++c)
    if (c < a.width) r[c] = dq[c] * a.scale;
}

// dV[j] = sum_i P[i][j] dO[i],  dK[j] = scale sum_i P[i][j] (dO[i] . V[j] - D[i]) Q[i]
template <int W>
__global__ void __launch_bounds__(kLongThreads) k_gman_attn_long_bwd_kv(const Args a) {
  __shared__ __align__(16) float Qs[kTile * W];
  __shared__ __align__(16) float Gs[kTile * W];
  __shared__ float Ls[kTile], Ds[kTile];
  const int nkb = (a.lk + kLongThreads - 1) / kLongThreads;
  const int64_t ph = blockIdx.x / nkb, prob = ph / a.heads, h = ph - prob * a.heads;
  const int j = (int)(blockIdx.x - ph * nkb) * kLongThreads + threadIdx.x;
  const bool live = j < a.lk;
  float kr[W], vr[W], dk[W], dv[W];
#pragma unroll
  for (int c = 0; c < W; ++c) kr[c] = vr[c] = dk[c] = dv[c] = 0.f;
  if (live) {
    load_row<W>(kr, a.k.p + base_of(a.k, a, prob, h) + (int64_t)j * a.k.sl, (int)a.width);
    load_row<W>(vr, a.v.p + base_of(a.v, a, prob, h) + (int64_t)j * a.v.sl, (int)a.width);
  }
  const int64_t bq = base_of(a.q, a, prob, h), bg = base_of(a.dout, a, prob, h);
  for (int i0 = 0; i0 < a.lq; i0 += kTile) {
    const int nt = min(kTile, a.lq - i0);
    stage<W>(Qs, a.q, bq, i0, nt, (int)a.width, kLongThreads);
    stage<W>(Gs, a.dout, bg, i0, nt, (int)a.width, kLongThreads);
    for (int e = threadIdx.x; e < nt; e += kLongThreads) {
      Ls[e] = a.lse[ph * a.lq + i0 + e];
      Ds[e] = a.delta[ph * a.lq + i0 + e];
    }
    __syncthreads();
    float tk[W], tv[W];                      // the tile's own sums, added once: a two-level sum over the queries
#pragma unroll
    for (int c = 0; c < W; ++c) tk[c] = tv[c] = 0.f;
    for (int i = 0; i < nt; ++i) {
      const float* qr = Qs + i * W;
      const float* gr = Gs + i * W;
      const float p = expf(dot<W>(kr, qr) * a.scale - Ls[i]);
      const float ds = p * (dot<W>(vr, gr) - Ds[i]);
#pragma unroll
      for (int c = 0; c < W; ++c) {
        tv[c] = fmaf(p, gr[c], tv[c]);
        tk[c] = fmaf(ds, qr[c], tk[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < W; ++c) {
      dv[c] += tv[c];
      dk[c] += tk[c];
    }
    __syncthreads();
  }
  if (!live) return;
  if (a.dk) {
    float* r = a.dk + base_of(a.k, a, prob, h) + (int64_t)j * a.k.sl;
#pragma unroll
    for (int c = 0; c < W; ++c)
      if (c < a.width) r[c] = dk[c] * a.scale;
  }
  if (a.dv) {
    float* r = a.dv + base_of(a.v, a, prob, h) + (int64_t)j * a.v.sl;
#pragma unroll
    for (int c = 0; c < W; ++c)
      if (c < a.width) r[c] = dv[c];
  }
}

// ---- short kernels --------------------------------------------------------------------------------------------------------------------
// the (masked) logit of query row qi against the staged key row kr
template <int W>
__device__ __forceinline__ float logit(const Args& a, const float (&q)[W], const float* kr, int qi, int kj) {
  return (a.mask && kj > qi) ? kMasked : dot<W>(q, kr) * a.scale;
}

// rows [0, n) of a (p, h) slice of t -> sm[n][W], by the 32 lanes of one warp
template <int W>
__device__ __forceinline__ void stage_warp(float* sm, const View& t, int64_t base, int n, int width, int lane) {
  for (int e = lane; e < n * W; e += 32) {
    const int r = e / W, c = e - r * W;
    sm[e] = c < width ? __ldg(t.p + base + (int64_t)r * t.sl + c) : 0.f;
  }
}

template <int W>
__global__ void __launch_bounds__(kShortFwdWarps * 32) k_gman_attn_short_fwd(const Args a, int64_t n_ph) {
  extern __shared__ __align__(16) float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t ph = (int64_t)blockIdx.x * kShortFwdWarps + warp;
  if (ph >= n_ph) return;                    // warp-uniform; no CTA-wide barrier below
  const int64_t prob = ph / a.heads, h = ph - prob * a.heads;
  float* Ks = sm + (size_t)warp * 2 * a.lk * W;
  float* Vs = Ks + a.lk * W;
  stage_warp<W>(Ks, a.k, base_of(a.k, a, prob, h), a.lk, (int)a.width, lane);
  stage_warp<W>(Vs, a.v, base_of(a.v, a, prob, h), a.lk, (int)a.width, lane);
  __syncwarp();
  const int64_t bq = base_of(a.q, a, prob, h), bo = base_of(a.o, a, prob, h);
  for (int i = lane; i < a.lq; i += 32) {
    float q[W], o[W];
    load_row<W>(q, a.q.p + bq + (int64_t)i * a.q.sl, (int)a.width);
    float m = -INFINITY;
    for (int j = 0; j < a.lk; ++j) m = fmaxf(m, logit<W>(a, q, Ks + j * W, i, j));
#pragma unroll
    for (int c = 0; c < W; ++c) o[c] = 0.f;
    float l = 0.f;
    for (int j = 0; j < a.lk; ++j) {
      const float p = expf(logit<W>(a, q, Ks + j * W, i, j) - m);
      l += p;
      const float* vr = Vs + j * W;
#pragma unroll
      for (int c = 0; c < W; ++c) o[c] = fmaf(p, vr[c], o[c]);
    }
    float* orow = a.out + bo + (int64_t)i * a.o.sl;
#pragma unroll
    for (int c = 0; c < W; ++c)
      if (c < a.width) orow[c] = o[c] / l;
    if (a.lse) a.lse[ph * a.lq + i] = m + logf(l);
  }
}

// one warp per (problem, head): dQ and D per query row (lanes own queries), then dK and dV per key row (lanes own keys).  A masked
// logit has zero gradient, but its probability still feeds O, D and dV.
template <int W>
__global__ void __launch_bounds__(kShortBwdWarps * 32) k_gman_attn_short_bwd(const Args a, int64_t n_ph) {
  extern __shared__ __align__(16) float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t ph = (int64_t)blockIdx.x * kShortBwdWarps + warp;
  if (ph >= n_ph) return;
  const int64_t prob = ph / a.heads, h = ph - prob * a.heads;
  float* Qs = sm + (size_t)warp * ((2 * a.lq + 2 * a.lk) * W + 2 * a.lq);
  float* Gs = Qs + a.lq * W;
  float* Ks = Gs + a.lq * W;
  float* Vs = Ks + a.lk * W;
  float* Ls = Vs + a.lk * W;
  float* Ds = Ls + a.lq;
  stage_warp<W>(Qs, a.q, base_of(a.q, a, prob, h), a.lq, (int)a.width, lane);
  stage_warp<W>(Gs, a.dout, base_of(a.dout, a, prob, h), a.lq, (int)a.width, lane);
  stage_warp<W>(Ks, a.k, base_of(a.k, a, prob, h), a.lk, (int)a.width, lane);
  stage_warp<W>(Vs, a.v, base_of(a.v, a, prob, h), a.lk, (int)a.width, lane);
  __syncwarp();
  const int64_t bo = base_of(a.o, a, prob, h);
  for (int i = lane; i < a.lq; i += 32) {
    float q[W], g[W], o[W], dq[W];
#pragma unroll
    for (int c = 0; c < W; ++c) {
      q[c] = Qs[i * W + c];
      g[c] = Gs[i * W + c];
      dq[c] = 0.f;
    }
    load_row<W>(o, a.o.p + bo + (int64_t)i * a.o.sl, (int)a.width);
    const float D = dot_rr<W>(g, o), lse = a.lse[ph * a.lq + i];
    Ls[i] = lse;
    Ds[i] = D;
    if (!a.dq) continue;
    for (int j = 0; j < a.lk; ++j) {
      if (a.mask && j > i) continue;         // zero logit gradient
      const float* kr = Ks + j * W;
      const float p = expf(dot<W>(q, kr) * a.scale - lse);
      const float ds = p * (dot<W>(g, Vs + j * W) - D);
#pragma unroll
      for (int c = 0; c < W; ++c) dq[c] = fmaf(ds, kr[c], dq[c]);
    }
    float* r = a.dq + base_of(a.q, a, prob, h) + (int64_t)i * a.q.sl;
#pragma unroll
    for (int c = 0; c < W; ++c)
      if (c < a.width) r[c] = dq[c] * a.scale;
  }
  __syncwarp();
  if (!a.dk && !a.dv) return;
  for (int j = lane; j < a.lk; j += 32) {
    float kr[W], vr[W], dk[W], dv[W];
#pragma unroll
    for (int c = 0; c < W; ++c) {
      kr[c] = Ks[j * W + c];
      vr[c] = Vs[j * W + c];
      dk[c] = dv[c] = 0.f;
    }
    for (int i = 0; i < a.lq; ++i) {
      const float* qr = Qs + i * W;
      const float* gr = Gs + i * W;
      const bool masked = a.mask && j > i;
      const float p = expf((masked ? kMasked : dot<W>(kr, qr) * a.scale) - Ls[i]);
      const float ds = masked ? 0.f : p * (dot<W>(vr, gr) - Ds[i]);
#pragma unroll
      for (int c = 0; c < W; ++c) {
        dv[c] = fmaf(p, gr[c], dv[c]);
        dk[c] = fmaf(ds, qr[c], dk[c]);
      }
    }
    if (a.dk) {
      float* r = a.dk + base_of(a.k, a, prob, h) + (int64_t)j * a.k.sl;
#pragma unroll
      for (int c = 0; c < W; ++c)
        if (c < a.width) r[c] = dk[c] * a.scale;
    }
    if (a.dv) {
      float* r = a.dv + base_of(a.v, a, prob, h) + (int64_t)j * a.v.sl;
#pragma unroll
      for (int c = 0; c < W; ++c)
        if (c < a.width) r[c] = dv[c];
    }
  }
}

// ---- host ---------------------------------------------------------------------------------------------------------------------------
constexpr int64_t kMaxGrid = 2147483647;

size_t short_fwd_smem(int lk, int W) { return (size_t)kShortFwdWarps * 2 * lk * W * 4; }
size_t short_bwd_smem(int lq, int lk, int W) { return (size_t)kShortBwdWarps * ((2 * lq + 2 * lk) * W + 2 * lq) * 4; }

// CTAs of a launch (0 when the grid does not fit)
int64_t grid_of(int64_t p0, int64_t p1, int64_t heads, int64_t rows, int long_kernel, int per_cta) {
  const int64_t ph = p0 * p1 * heads;
  const int64_t n = long_kernel ? ph * ((rows + kLongThreads - 1) / kLongThreads) : (ph + per_cta - 1) / per_cta;
  return n <= kMaxGrid ? n : 0;
}

bool supported(int64_t p0, int64_t p1, int64_t heads, int64_t width, int64_t lq, int64_t lk, int mask, int long_kernel) {
  if (p0 < 0 || p1 < 0 || heads < 1 || width < 1 || width > kMaxWidth || lq < 1 || lk < 1) return false;
  if (p0 > kMaxGrid || p1 > kMaxGrid || heads > kMaxGrid || p0 * p1 > kMaxGrid / heads) return false;   // no int64 overflow below
  if (long_kernel) {
    if (mask || lq > kMaxGrid || lk > kMaxGrid) return false;
    if (p0 * p1 == 0) return true;
    return grid_of(p0, p1, heads, lq, 1, 0) && grid_of(p0, p1, heads, lk, 1, 0);
  }
  if (lq > kMaxShort || lk > kMaxShort || (mask && lq != lk)) return false;
  return p0 * p1 == 0 || grid_of(p0, p1, heads, 0, 0, kShortBwdWarps);
}

int prepare(const char* fn, Args& a, int64_t p0, int64_t p1, int64_t heads, int64_t width, int64_t lq, int64_t lk, int mask,
            int long_kernel, float scale, const int64_t* strides, const float* q, const float* k, const float* v, const float* o) {
  STMP_REQUIRE(p0 >= 0 && p1 >= 0, STMP_EINVAL, "%s: negative problem count (%lld, %lld)", fn, (long long)p0, (long long)p1);
  STMP_REQUIRE(supported(p0, p1, heads, width, lq, lk, mask, long_kernel), STMP_EUNSUPPORTED,
               "%s: p=(%lld, %lld) heads=%lld width=%lld Lq=%lld Lk=%lld mask=%d long=%d outside the envelope (width 1..16; short: Lq, "
               "Lk <= 64, a mask needs Lq == Lk; long: no mask; every grid below 2^31 CTAs)", fn, (long long)p0, (long long)p1,
               (long long)heads, (long long)width, (long long)lq, (long long)lk, mask, long_kernel);
  STMP_REQUIRE(strides && (p0 * p1 == 0 || (q && k && v && o)), STMP_EINVAL, "%s: NULL tensor or stride table", fn);
  a = Args{};
  a.p1 = p1 > 0 ? p1 : 1; a.heads = heads; a.width = width; a.lq = (int)lq; a.lk = (int)lk; a.mask = mask ? 1 : 0; a.scale = scale;
  a.q = View{q, strides[0], strides[1], strides[2]};
  a.k = View{k, strides[3], strides[4], strides[5]};
  a.v = View{v, strides[6], strides[7], strides[8]};
  a.o = View{o, strides[9], strides[10], strides[11]};
  return STMP_OK;
}

template <int W>
int launch_fwd(const Args& a, int64_t p0, int long_kernel, cudaStream_t st) {
  const int64_t n_ph = p0 * a.p1 * a.heads;
  if (long_kernel) {
    k_gman_attn_long_fwd<W><<<(unsigned)grid_of(p0, a.p1, a.heads, a.lq, 1, 0), kLongThreads, 0, st>>>(a);
    STMP_LAUNCH_OK("k_gman_attn_long_fwd");
    return STMP_OK;
  }
  k_gman_attn_short_fwd<W><<<(unsigned)grid_of(p0, a.p1, a.heads, 0, 0, kShortFwdWarps), kShortFwdWarps * 32, short_fwd_smem(a.lk, W),
                             st>>>(a, n_ph);
  STMP_LAUNCH_OK("k_gman_attn_short_fwd");
  return STMP_OK;
}

template <int W>
int launch_bwd(const Args& a, int64_t p0, int long_kernel, cudaStream_t st) {
  const int64_t n_ph = p0 * a.p1 * a.heads;
  if (long_kernel) {
    if (a.dq || a.dk || a.dv) {
      k_gman_attn_long_bwd_q<W><<<(unsigned)grid_of(p0, a.p1, a.heads, a.lq, 1, 0), kLongThreads, 0, st>>>(a);
      STMP_LAUNCH_OK("k_gman_attn_long_bwd_q");
    }
    if (a.dk || a.dv) {
      k_gman_attn_long_bwd_kv<W><<<(unsigned)grid_of(p0, a.p1, a.heads, a.lk, 1, 0), kLongThreads, 0, st>>>(a);
      STMP_LAUNCH_OK("k_gman_attn_long_bwd_kv");
    }
    return STMP_OK;
  }
  if (!a.dq && !a.dk && !a.dv) return STMP_OK;
  k_gman_attn_short_bwd<W><<<(unsigned)grid_of(p0, a.p1, a.heads, 0, 0, kShortBwdWarps), kShortBwdWarps * 32,
                             short_bwd_smem(a.lq, a.lk, W), st>>>(a, n_ph);
  STMP_LAUNCH_OK("k_gman_attn_short_bwd");
  return STMP_OK;
}

}  // namespace
}  // namespace stmp

using namespace stmp;

extern "C" int stmp_gman_attn_supported(int64_t p0, int64_t p1, int64_t heads, int64_t width, int64_t lq, int64_t lk, int mask,
                                        int long_kernel) {
  return supported(p0, p1, heads, width, lq, lk, mask, long_kernel) ? 1 : 0;
}

extern "C" int64_t stmp_gman_attn_stash_bytes(int64_t p0, int64_t p1, int64_t heads, int64_t lq) {
  if (p0 < 0 || p1 < 0 || heads < 1 || lq < 1) return 0;
  return 4 * p0 * p1 * heads * lq;
}

extern "C" int64_t stmp_gman_attn_workspace_bytes(int64_t p0, int64_t p1, int64_t heads, int64_t lq, int long_kernel) {
  return long_kernel ? stmp_gman_attn_stash_bytes(p0, p1, heads, lq) : 0;
}

extern "C" int stmp_gman_attn_fwd(int64_t p0, int64_t p1, int64_t heads, int64_t width, int64_t lq, int64_t lk, int mask,
                                  int long_kernel, float scale, const int64_t* strides, const float* q, const float* k, const float* v,
                                  float* o, float* stash, void* stream) {
  const char* fn = "stmp_gman_attn_fwd";
  Args a;
  if (int rc = prepare(fn, a, p0, p1, heads, width, lq, lk, mask, long_kernel, scale, strides, q, k, v, o)) return rc;
  if (p0 * p1 == 0) return STMP_OK;
  a.out = o;
  a.lse = stash;
  cudaStream_t st = (cudaStream_t)stream;
  return width <= 8 ? launch_fwd<8>(a, p0, long_kernel, st) : launch_fwd<16>(a, p0, long_kernel, st);
}

extern "C" int stmp_gman_attn_bwd(int64_t p0, int64_t p1, int64_t heads, int64_t width, int64_t lq, int64_t lk, int mask,
                                  int long_kernel, float scale, const int64_t* strides, const float* q, const float* k, const float* v,
                                  const float* o, const float* stash, const float* dout, void* workspace, float* dq, float* dk, float* dv,
                                  void* stream) {
  const char* fn = "stmp_gman_attn_bwd";
  Args a;
  if (int rc = prepare(fn, a, p0, p1, heads, width, lq, lk, mask, long_kernel, scale, strides, q, k, v, o)) return rc;
  if (p0 * p1 == 0 || (!dq && !dk && !dv)) return STMP_OK;
  STMP_REQUIRE(stash && dout && (workspace || !long_kernel), STMP_EINVAL, "%s: NULL stash, gradient or workspace", fn);
  a.lse = const_cast<float*>(stash);
  a.dout = a.o;
  a.dout.p = dout;
  a.delta = reinterpret_cast<float*>(workspace);
  a.dq = dq; a.dk = dk; a.dv = dv;
  cudaStream_t st = (cudaStream_t)stream;
  return width <= 8 ? launch_bwd<8>(a, p0, long_kernel, st) : launch_bwd<16>(a, p0, long_kernel, st);
}
