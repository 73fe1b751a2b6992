// rows.cuh -- the pieces shared by the row-split recurrent cells (gru_rows.cu, lstm_rows.cu): one warp per destination row, lane = output
// channel (lane + 32 j for j < NC in the 64-wide instances), CTAs owning grid-strided tiles of kRowTile rows, weights staged once per CTA at pitch kWPitch, and the entry-order CSR gather.
// Also the lane-level torch GRUCell and C x C row products of ggc_rows.cu and evolvegcn_rows.cu, and the weight-gradient pieces of train.cu, gru_rows.cu and lstm_rows.cu: the FFMA contraction's launch, the part count of every
// weight-gradient contraction, the fixed-order sum every reduce kernel adds the partials with, and the per-gate contraction and reduce of
// the 64-wide cells.
#pragma once
#include "common.cuh"

namespace stmp {
namespace rows {

constexpr int kCo = 32;
constexpr int kRowsThreads = 256;
constexpr int kRowsWarps = kRowsThreads / 32;
constexpr int kRowTile = 16;                 // destination rows per CTA tile: two per warp
constexpr int kWPitch = 97;                  // shared-memory pitch of a staged weight row (basis columns 0..95)
constexpr int kMaxCin = 16;

// rows [r0, r0 + nr) of packed weights w [..][nb] -> ws [nr][P] (columns >= nb zero)
template <int P = kWPitch>
__device__ __forceinline__ void stage_w(float* ws, const float* __restrict__ w, int nb, int r0, int nr) {
  for (int i = threadIdx.x; i < nr * P; i += kRowsThreads) {
    const int r = i / P, m = i - r * P;
    ws[i] = m < nb ? __ldg(w + (size_t)(r0 + r) * nb + m) : 0.f;
  }
  __syncthreads();
}

// ah[j] = sum_e val_e * A[col_e][lane + 32 j] (pitch lda, j < NC), ax = sum_e val_e * B[col_e][lane] (pitch ldb, lanes < nx) over CSR row
// i, in entry order.
template <int NC, bool WITH_A>
__device__ __forceinline__ void gather_rows(const int* __restrict__ rowptr, const int2* __restrict__ cv, int i, const float* __restrict__ A,
                                            int lda, const float* __restrict__ Bx, int ldb, int nx, int lane, float (&ah)[NC], float& ax) {
  const int beg = __ldg(rowptr + i), end = __ldg(rowptr + i + 1);
  const bool xl = lane < nx;
#pragma unroll
  for (int j = 0; j < NC; ++j) ah[j] = 0.f;
  ax = 0.f;
  int k = beg;
  for (; k + 4 <= end; k += 4) {
    int2 e[4];
    float av[4][NC], bv[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) e[u] = __ldg(cv + k + u);
#pragma unroll
    for (int u = 0; u < 4; ++u) {
#pragma unroll
      for (int j = 0; j < NC; ++j) av[u][j] = WITH_A ? __ldg(A + (size_t)e[u].x * lda + lane + 32 * j) : 0.f;
      bv[u] = xl ? __ldg(Bx + (size_t)e[u].x * ldb + lane) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float w = __int_as_float(e[u].y);
#pragma unroll
      for (int j = 0; j < NC; ++j)
        if (WITH_A) ah[j] = __fadd_rn(ah[j], __fmul_rn(w, av[u][j]));
      if (xl) ax = __fadd_rn(ax, __fmul_rn(w, bv[u]));
    }
  }
  for (; k < end; ++k) {
    const int2 e = __ldg(cv + k);
    const float w = __int_as_float(e.y);
#pragma unroll
    for (int j = 0; j < NC; ++j)
      if (WITH_A) ah[j] = __fadd_rn(ah[j], __fmul_rn(w, __ldg(A + (size_t)e.x * lda + lane + 32 * j)));
    if (xl) ax = __fadd_rn(ax, __fmul_rn(w, __ldg(Bx + (size_t)e.x * ldb + lane)));
  }
}

// gather_rows for one channel per lane
template <bool WITH_A>
__device__ __forceinline__ void gather_row(const int* __restrict__ rowptr, const int2* __restrict__ cv, int i, const float* __restrict__ A,
                                           int lda, const float* __restrict__ Bx, int ldb, int nx, int lane, float& ah, float& ax) {
  float a[1];
  gather_rows<1, WITH_A>(rowptr, cv, i, A, lda, Bx, ldb, nx, lane, a, ax);
  ah = a[0];
}

// CTAs of a row-split launch over n rows: one per 16-row tile, at most two per SM (the tiles are grid-strided beyond that)
inline int rows_grid(int n) {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int tiles = (n + kRowTile - 1) / kRowTile;
  return tiles < 2 * sms ? (tiles > 0 ? tiles : 1) : 2 * sms;
}

inline bool al4(const void* p) { return ((uintptr_t)p & 3u) == 0; }

// ---- the lane-level torch GRUCell of ggc_rows.cu and evolvegcn_rows.cu: one warp per row, lane = channel (C <= 32), weights staged in
// shared memory at pitch kGruPitch, W_ih / W_hh rows in gate order r | z | n ------------------------------------------------------------
constexpr int kGruMaxC = 32;
constexpr int kGruPitch = kGruMaxC + 1;     // staged pitch: lane-indexed rows and lane-indexed columns are both conflict-free

// y[c] = sum_{k < K} v[k] W[k][c]: lane c, W staged at pitch kGruPitch
__device__ __forceinline__ float row_times_w(const float* __restrict__ w, float v, int K, int lc) {
  float y = 0.f;
  for (int k = 0; k < K; ++k) y = fmaf(__shfl_sync(0xffffffffu, v, k), w[k * kGruPitch + lc], y);
  return y;
}

// y[k] = sum_{c < C} v[c] W[k][c] (v W^T): lane k
__device__ __forceinline__ float row_times_wt(const float* __restrict__ w, float v, int C, int lc) {
  float y = 0.f;
  for (int c = 0; c < C; ++c) y = fmaf(__shfl_sync(0xffffffffu, v, c), w[lc * kGruPitch + c], y);
  return y;
}

struct GruFwd {
  float r, z, n, hn, h;                      // the gates, W_hn h + b_hn, and the new state
};

// h' = GRUCell(x, h) of one row: lane c holds x[c] (gin) and h[c] (hv), bi* / bh* its channel's biases
__device__ __forceinline__ GruFwd gru_cell_fwd(const float* __restrict__ ih, const float* __restrict__ hh, float gin, float hv, float bir,
                                               float biz, float bin, float bhr, float bhz, float bhn, int C, int lc) {
  float gr = bir, gz = biz, gn = bin, hr = bhr, hz = bhz, hn = bhn;
  for (int k = 0; k < C; ++k) {
    const float u = __shfl_sync(0xffffffffu, gin, k), v = __shfl_sync(0xffffffffu, hv, k);
    gr = fmaf(u, ih[lc * kGruPitch + k], gr);
    gz = fmaf(u, ih[(C + lc) * kGruPitch + k], gz);
    gn = fmaf(u, ih[(2 * C + lc) * kGruPitch + k], gn);
    hr = fmaf(v, hh[lc * kGruPitch + k], hr);
    hz = fmaf(v, hh[(C + lc) * kGruPitch + k], hz);
    hn = fmaf(v, hh[(2 * C + lc) * kGruPitch + k], hn);
  }
  const float r = sigmoidf_acc(gr + hr), z = sigmoidf_acc(gz + hz);
  const float nn = tanhf(gn + r * hn);
  return {r, z, nn, hn, (1.f - z) * nn + z * hv};
}

struct GruGrad {
  float dr, dz, dn, dhn;                     // pre-activation gradients of r, z and n, and dhn = r dn (W_hn's)
};

// the pre-activation gradients of one row from dL/dh' (dh1) and the forward's gates
__device__ __forceinline__ GruGrad gru_cell_bwd_gates(float dh1, float r, float z, float nn, float hn, float hv) {
  const float dn = dh1 * (1.f - z);
  const float dzp = dh1 * (hv - nn) * z * (1.f - z);
  const float dnp = dn * (1.f - nn * nn);
  const float dhn = dnp * r;
  const float drp = dnp * hn * r * (1.f - r);
  return {drp, dzp, dnp, dhn};
}

// din += [dr dz dn] W_ih (the gradient at the GRU input), dh += [dr dz dhn] W_hh (at h; enters as its direct part dh' z)
__device__ __forceinline__ void gru_cell_bwd_inputs(const float* __restrict__ ih, const float* __restrict__ hh, const GruGrad& g, int C,
                                                    int lc, float& din, float& dh) {
  for (int c = 0; c < C; ++c) {
    const float ur = __shfl_sync(0xffffffffu, g.dr, c), uz = __shfl_sync(0xffffffffu, g.dz, c);
    const float un = __shfl_sync(0xffffffffu, g.dn, c), uh = __shfl_sync(0xffffffffu, g.dhn, c);
    din = fmaf(ur, ih[c * kGruPitch + lc], din);
    din = fmaf(uz, ih[(C + c) * kGruPitch + lc], din);
    din = fmaf(un, ih[(2 * C + c) * kGruPitch + lc], din);
    dh = fmaf(ur, hh[c * kGruPitch + lc], dh);
    dh = fmaf(uz, hh[(C + c) * kGruPitch + lc], dh);
    dh = fmaf(uh, hh[(2 * C + c) * kGruPitch + lc], dh);
  }
}

}  // namespace rows

// The FFMA weight-gradient contraction of train.cu (k_dcrnn_wgrad<N2>): per-CTA partials [parts][MG*8*(64+N2) + 64+N2] of
// S1^T A (A: rows x 64) and S2^T B (B: rows x N2, N2 = 32 or 64) and the column sums of A and B, over strided 16-row tiles.
int wgrad_ffma_launch(int n2, long long rows, int ld, const float* S1, const float* S2, const float* A, const float* B, float* partial,
                      cudaStream_t st, int* parts);
// 2 x SMs: the most partials any weight-gradient contraction writes (per gate in gru_rows.cu's 64-wide one), which sizes every workspace
int wgrad_ffma_max_parts();

// The sum of p[q * stride] over the n parts q < n in the one fixed association every weight-gradient reduce kernel uses: warp w of the
// 256-thread block adds the contiguous parts [w per, (w + 1) per), per = ceil(n / 8), in two interleaved accumulators (the odd tail into
// the first), and the 8 warp sums are added in warp order.  The association depends on n alone, never on the launch, so the gradients are
// bit-reproducible.  Lane x of each warp sums its own output in column x of `sub`; a thread with nothing to sum passes live = false.
// It holds a __syncthreads, so every thread of the block must call it.  The result is valid in warp 0 only.
__device__ __forceinline__ float fixed_order_sum(const float* p, size_t stride, int n, bool live, float (&sub)[8][32]) {
  const int x = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int per = (n + 7) / 8, q0 = w * per, q1 = (q0 + per < n) ? q0 + per : n;
  float s0 = 0.f, s1 = 0.f;
  if (live) {
    int q = q0;
    for (; q + 2 <= q1; q += 2) {
      s0 += p[(size_t)q * stride];
      s1 += p[(size_t)(q + 1) * stride];
    }
    if (q < q1) s0 += p[(size_t)q * stride];
  }
  sub[w][x] = s0 + s1;
  __syncthreads();
  float t = 0.f;
  if (w == 0) {
    t = sub[0][x];
#pragma unroll
    for (int k = 1; k < 8; ++k) t += sub[k][x];
  }
  return t;
}

// ---- weight gradients of the 64-wide row-split cells (gru_rows.cu: G = 3 gates, lstm_rows.cu: G = 4) -------------------------------------
// Per-CTA partials of one gate's product over strided tiles of kWideWgRows rows: blockIdx.y = gate g, partial [g][part][ld*64 + 64] =
// S_g^T A_g and the column sums of A_g, A_g = the gate's 64 columns of its pre-activation gradient at pitch apitch_g.  Thread (mg, ng) owns
// the 8 x 8 register tile of basis columns 8 mg.. and gate channels 8 ng..; a second launch sums the partials in a fixed order.
constexpr int kWideWgRows = 32, kWideMaxLd = 160;          // the widest basis of either cell: 2 (16 + 64) columns
constexpr int kWideWgThreads = kWideMaxLd;                 // 8 * ceil(kWideMaxLd / 8) tiles

template <int G>
struct WideWgradOps {
  const float* S[G];                         // (rows, ld) basis of gate g
  const float* A[G];                         // (rows, apitch[g]): gate g's 64 columns
  int apitch[G];
};

// partials of the contraction over `rows` rows: one per 32-row tile, at most wgrad_ffma_max_parts()
inline int wide_wgrad_parts(long long rows) {
  const long long tiles = (rows + kWideWgRows - 1) / kWideWgRows, max_parts = wgrad_ffma_max_parts();
  return (int)(tiles < max_parts ? tiles : max_parts);
}

template <int G>
__global__ void __launch_bounds__(kWideWgThreads, 1) k_wide_rows_wgrad(long long rows, int ld, WideWgradOps<G> op, float* __restrict__ partial) {
  __shared__ __align__(16) float ss[kWideWgRows * kWideMaxLd];
  __shared__ __align__(16) float sa[kWideWgRows * 64];
  const int g = blockIdx.y, tid = threadIdx.x, MG = ld / 8;
  const float* S = op.S[0];                  // gate g's operands, selected without indexing the parameter arrays (no local copy)
  const float* A = op.A[0];
  int apitch = op.apitch[0];
#pragma unroll
  for (int k = 1; k < G; ++k)
    if (g == k) { S = op.S[k]; A = op.A[k]; apitch = op.apitch[k]; }
  const bool active = tid < 8 * MG;
  const int mg = tid >> 3, ng = tid & 7;
  float acc[8][8], cs[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    cs[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  }
  const long long n_tiles = (rows + kWideWgRows - 1) / kWideWgRows;
  for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const long long r0 = tile * kWideWgRows;
    const int nr = (int)min((long long)kWideWgRows, rows - r0);
    for (int e = tid; e < nr * (ld / 4); e += kWideWgThreads) {
      const int r = e / (ld / 4), c4 = e - r * (ld / 4);
      reinterpret_cast<float4*>(ss + r * ld)[c4] = __ldg(reinterpret_cast<const float4*>(S + (r0 + r) * ld) + c4);
    }
    for (int e = tid; e < nr * 16; e += kWideWgThreads) {
      const int r = e >> 4, c4 = e & 15;
      reinterpret_cast<float4*>(sa + r * 64)[c4] = __ldg(reinterpret_cast<const float4*>(A + (r0 + r) * apitch) + c4);
    }
    __syncthreads();
    if (active) {
#pragma unroll 4
      for (int k = 0; k < nr; ++k) {
        const float4 a0 = *reinterpret_cast<const float4*>(ss + k * ld + 8 * mg), a1 = *reinterpret_cast<const float4*>(ss + k * ld + 8 * mg + 4);
        const float4 b0 = *reinterpret_cast<const float4*>(sa + k * 64 + 8 * ng), b1 = *reinterpret_cast<const float4*>(sa + k * 64 + 8 * ng + 4);
        const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) acc[i][jj] = fmaf(av[i], bv[jj], acc[i][jj]);
        if (mg == 0) {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) cs[jj] += bv[jj];
        }
      }
    }
    __syncthreads();
  }
  if (!active) return;
  float* out = partial + ((size_t)g * gridDim.x + blockIdx.x) * ((size_t)ld * 64 + 64);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float4* q = reinterpret_cast<float4*>(out + (size_t)(8 * mg + i) * 64 + 8 * ng);
    q[0] = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    q[1] = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
  }
  if (mg == 0) {
    float4* q = reinterpret_cast<float4*>(out + (size_t)ld * 64 + 8 * ng);
    q[0] = make_float4(cs[0], cs[1], cs[2], cs[3]);
    q[1] = make_float4(cs[4], cs[5], cs[6], cs[7]);
  }
}

// The fixed-order sums of k_wide_rows_wgrad<G>'s partials [gate][part][ld*64 + 64] into dw [64 G][nb] (row g*64 + o, column m of the basis)
// and db [64 G] (nullable), and of `pparts` per-CTA partials pp [pparts][npeep] into dpeep [npeep] (the LSTM's peephole sums; npeep = 0
// without them, dpeep nullable).
template <int G>
__global__ void __launch_bounds__(256) k_wide_rows_wgrad_reduce(int parts, int ld, int nb, const float* __restrict__ partial, int npeep,
                                                                int pparts, const float* __restrict__ pp, float* __restrict__ dw,
                                                                float* __restrict__ db, float* __restrict__ dpeep) {
  constexpr int R = 64 * G;
  __shared__ float sub[8][32];
  const int x = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + x;
  const size_t wstride = (size_t)ld * 64 + 64;
  const float* base = partial;
  size_t src = 0, stride = wstride;
  int n = parts;
  float* dst = nullptr;
  if (i < R * nb) {
    const int row = i / nb, m = i - row * nb;
    src = (size_t)(row >> 6) * parts * wstride + (size_t)m * 64 + (row & 63);
    dst = dw + i;
  } else if (i < R * nb + R) {
    const int r = i - R * nb;
    src = (size_t)(r >> 6) * parts * wstride + (size_t)ld * 64 + (r & 63);
    dst = db ? db + r : nullptr;
  } else if (i < R * nb + R + npeep) {
    src = i - R * nb - R;
    base = pp;
    stride = npeep;
    n = pparts;
    dst = dpeep ? dpeep + src : nullptr;
  }
  const float t = fixed_order_sum(base + src, stride, n, dst != nullptr, sub);
  if (w == 0 && dst) *dst = t;
}

}  // namespace stmp
