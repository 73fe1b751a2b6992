// rows.cuh -- the pieces shared by the row-split recurrent cells (gru_rows.cu, lstm_rows.cu): one warp per destination row, lane = output
// channel (lane + 32 j for j < NC in gru_rows.cu's 64-wide instance), CTAs owning grid-strided tiles of kRowTile rows, weights staged once per CTA at pitch kWPitch, and the entry-order CSR gather.
// Also the weight-gradient pieces of train.cu, gru_rows.cu and lstm_rows.cu: the FFMA contraction's launch, the part count of every
// weight-gradient contraction, and the fixed-order sum every reduce kernel adds the partials with.
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

}  // namespace stmp
