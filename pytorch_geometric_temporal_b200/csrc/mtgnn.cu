// mtgnn.cu -- MTGNN's graph work (DESIGN §4x), in exact fp32: the top-k graph of GraphConstructor, the two mix-hop operators of
// MixProp (A and A^T) and their backward, on sparse structures built without atomics.
//
// Graph (learned, GraphConstructor): z = M1 M2^T - M2 M1^T, A = relu(tanh(alpha z)) with only the k largest entries of each row kept
// (among equal values the lower column wins; zeros are dropped, they add nothing and relu passes no gradient at 0).
//   pattern (int32):  col1 [N W] | cnt1 [N] | ptr2 [N + 1] | row2 [N W] | pos2 [N W]
//     row i of A holds col1[i W + s], s < cnt1[i] (W = k, or the widest row of a predefined A); column j of A holds the rows
//     row2[p], p in [ptr2[j], ptr2[j + 1]), ascending, whose entry sits at pos2[p] in the row arrays
//   state   (fp32):   a [N W] (the raw entries of A) | d1 [N] | d2 [N]    d1 = 1 + row sums, d2 = 1 + column sums
//   values  (fp32):   v1 [N W] | v2 [N W] | diag1 [N] | diag2 [N]
//     operator 1 = (A + I) / d1 (rows):    entry (i, j) = v1[e] = a[e] / d1[i], diagonal diag1[i] = 1 / d1[i]
//     operator 2 = (A^T + I) / d2 (rows):  entry (j, i) = v2[e] = a[e] / d2[j], diagonal diag2[j] = 1 / d2[j]     (e = entry (i, j) of A)
//   Operator 1's transpose has operator 2's pattern and vice versa, so these two index sets serve both directions.
//
// Propagation (MixProp, both operators): X (B, C, N, T) contiguous; hops (B, 2 D C, N, T): channel block o D + k - 1 holds hop k of
// operator o, H_k = alpha X + (1 - alpha) S_o H_{k-1}, H_0 = X.  One launch per hop (k_mtgnn_hop), one thread per element.
// Backward: the adjoint chains (k_mtgnn_hop_adjoint, one launch per hop, dX accumulated in place in a fixed order) and, when asked
// for, the sampled products dS = (1 - alpha) sum_k G_k H_{k-1}^T on the pattern and the diagonals (k_mtgnn_dvals: one warp per entry,
// each lane summing one (hop, batch) block at a time before the block sums are added, then a fixed butterfly).
// Graph backward: through both normalisations (k_mtgnn_graph_dd), then the top-k mask, relu and tanh per entry and
// dM1 = (dz - dz^T) M2, dM2 = (dz^T - dz) M1 over the pattern (k_mtgnn_graph_dm).
//
// Everything is FFMA with every sum in one fixed order and no atomics: repeated calls are bit-identical.  The library allocates
// nothing and never synchronises the host; the bitmap workspace (stmp_mtgnn_graph_workspace_bytes) is written in full by each build.
#include <math.h>

#include "common.cuh"

namespace stmp {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxNodes = 4096, kMaxK = 64, kMaxDim = 64, kMaxChannels = 64, kMaxDepth = 4;
constexpr int64_t kMaxGrid = 2147483647;

struct Pattern {
  int n, w;
  const int *col1, *cnt1, *ptr2, *row2, *pos2;
};

// The same arrays, writable: the view of the graph-build kernels.
struct PatternOut {
  int n, w;
  int *col1, *cnt1, *ptr2, *row2, *pos2;
};

__host__ __device__ inline PatternOut pattern_out(int* p, int n, int w) {
  PatternOut q;
  q.n = n; q.w = w;
  q.col1 = p;
  q.cnt1 = p + (int64_t)n * w;
  q.ptr2 = q.cnt1 + n;
  q.row2 = q.ptr2 + n + 1;
  q.pos2 = q.row2 + (int64_t)n * w;
  return q;
}

__host__ __device__ inline Pattern pattern_of(const int* p, int n, int w) {
  const int64_t nw = (int64_t)n * w;
  return Pattern{n, w, p, p + nw, p + nw + n, p + nw + 2 * n + 1, p + 2 * nw + 2 * n + 1};
}

// One sparse operator as a gather: row r sums val[vidx ? vidx[e] : e] * H[nbr[e]] over its entries, plus diag[r] * H[r].  Rows come
// either from the row arrays (ptr == NULL: entries r W .. r W + cnt[r]) or from the column arrays (ptr2).
struct Op {
  const int *ptr, *cnt, *nbr, *vidx;
  int w;
  const float *val, *diag;
};

__device__ __forceinline__ void row_range(const Op& op, int r, int& b, int& e) {
  if (op.ptr) { b = __ldg(op.ptr + r); e = __ldg(op.ptr + r + 1); }
  else { b = r * op.w; e = b + __ldg(op.cnt + r); }
}

__device__ __forceinline__ float gather_row(const Op& op, int r, const float* __restrict__ h, int64_t T, int64_t t) {
  int b, e;
  row_range(op, r, b, e);
  float acc = __ldg(op.diag + r) * __ldg(h + r * T + t);
  for (int p = b; p < e; ++p) {
    const int j = __ldg(op.nbr + p);
    const float v = __ldg(op.val + (op.vidx ? __ldg(op.vidx + p) : p));
    acc = fmaf(v, __ldg(h + j * T + t), acc);
  }
  return acc;
}

// ---- graph build ---------------------------------------------------------------------------------------------------------------
// One CTA per row i: the row of A in shared memory, then k rounds of a block arg-max (value descending, column ascending).
__global__ void __launch_bounds__(kThreads) k_mtgnn_topk(int n, int k, int dim, float alpha, const float* __restrict__ m1,
                                                         const float* __restrict__ m2, PatternOut pat, float* a, float* d1, float* v1,
                                                         float* v2, float* diag1, uint32_t* bits) {
  extern __shared__ float sm[];
  float* row = sm;                                 // [n]
  float* mi = row + n;                             // m1[i], m2[i]: [2 dim]
  uint32_t* word = reinterpret_cast<uint32_t*>(mi + 2 * kMaxDim);   // [ceil(n / 32)]
  __shared__ float red_v[kThreads / 32], sel_v[kMaxK];
  __shared__ int red_j[kThreads / 32], sel_j[kMaxK], n_sel;
  const int i = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int wpr = (n + 31) / 32;
  for (int c = tid; c < dim; c += kThreads) { mi[c] = m1[(int64_t)i * dim + c]; mi[kMaxDim + c] = m2[(int64_t)i * dim + c]; }
  for (int q = tid; q < wpr; q += kThreads) word[q] = 0u;
  __syncthreads();
  for (int j = tid; j < n; j += kThreads) {
    const float* p1 = m1 + (int64_t)j * dim;
    const float* p2 = m2 + (int64_t)j * dim;
    float s = 0.f, u = 0.f;
    for (int c = 0; c < dim; ++c) { s = fmaf(mi[c], __ldg(p2 + c), s); u = fmaf(mi[kMaxDim + c], __ldg(p1 + c), u); }
    const float z = s - u;                         // exactly 0 on the diagonal
    row[j] = fmaxf(tanhf(alpha * z), 0.f);
  }
  if (tid == 0) n_sel = 0;
  __syncthreads();
  for (int round = 0; round < k; ++round) {
    float bv = 0.f;
    int bj = n;
    for (int j = tid; j < n; j += kThreads) {      // ascending j: a later equal value never replaces an earlier one
      const float v = row[j];
      if (v > bv) { bv = v; bj = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
      if (ov > bv || (ov == bv && oj < bj)) { bv = ov; bj = oj; }
    }
    if (lane == 0) { red_v[wid] = bv; red_j[wid] = bj; }
    __syncthreads();
    if (tid == 0) {
      float v = red_v[0];
      int j = red_j[0];
      for (int w2 = 1; w2 < kThreads / 32; ++w2)
        if (red_v[w2] > v || (red_v[w2] == v && red_j[w2] < j)) { v = red_v[w2]; j = red_j[w2]; }
      if (j < n) { sel_v[n_sel] = v; sel_j[n_sel] = j; ++n_sel; row[j] = -1.f; }
    }
    __syncthreads();
    if (n_sel <= round) break;                     // no positive value left: the remaining top-k entries are zeros
  }
  if (tid == 0) {
    const int cnt = n_sel;
    float s = 0.f;
    for (int q = 0; q < cnt; ++q) s += sel_v[q];
    const float d = 1.f + s;
    const int64_t base = (int64_t)i * k;
    for (int q = 0; q < cnt; ++q) {
      pat.col1[base + q] = sel_j[q];
      a[base + q] = sel_v[q];
      v1[base + q] = sel_v[q] / d;
      word[sel_j[q] >> 5] |= 1u << (sel_j[q] & 31);
    }
    for (int q = cnt; q < k; ++q) {                // unused slots: zero values, so every slot of the value arrays is defined
      pat.col1[base + q] = i;
      a[base + q] = 0.f; v1[base + q] = 0.f; v2[base + q] = 0.f;
    }
    pat.cnt1[i] = cnt;
    d1[i] = d;
    diag1[i] = 1.f / d;
  }
  __syncthreads();
  for (int q = tid; q < wpr; q += kThreads) bits[(int64_t)i * wpr + q] = word[q];
}

// Predefined A (dense, N x N): one warp per row, its nonzeros in ascending column order; the row sum adds each 32-column chunk's
// butterfly sum in column order.
__global__ void __launch_bounds__(kThreads) k_mtgnn_dense_rows(int n, int w, const float* __restrict__ A, PatternOut pat, float* a,
                                                               float* d1, float* v1, float* v2, float* diag1, uint32_t* bits) {
  const int i = blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (i >= n) return;
  const int wpr = (n + 31) / 32;
  const int64_t base = (int64_t)i * w;
  int cnt = 0;
  float s = 0.f;
  for (int q = 0; q < wpr; ++q) {
    const int j = q * 32 + lane;
    const float a0 = j < n ? __ldg(A + (int64_t)i * n + j) : 0.f;
    const uint32_t nz = __ballot_sync(0xffffffffu, a0 != 0.f);
    const int slot = cnt + __popc(nz & ((1u << lane) - 1u));
    // only the first w nonzeros of a row are kept: W comes from the host's count, and a row that has grown since (A changed in
    // place without a version bump) must not write past its slots; entry, bit and sum stay consistent
    const bool keep = a0 != 0.f && slot < w;
    const float v = keep ? a0 : 0.f;
    const uint32_t ball = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      pat.col1[base + slot] = j;
      a[base + slot] = v;
    }
    float cs = v;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cs += __shfl_xor_sync(0xffffffffu, cs, o);
    s += cs;
    if (lane == 0) bits[(int64_t)i * wpr + q] = ball;
    cnt += __popc(ball);
  }
  const float d = 1.f + s;
  __syncwarp();
  for (int q = lane; q < cnt; q += 32) v1[base + q] = a[base + q] / d;
  for (int q = cnt + lane; q < w; q += 32) {
    pat.col1[base + q] = i;
    a[base + q] = 0.f; v1[base + q] = 0.f; v2[base + q] = 0.f;
  }
  if (lane == 0) { pat.cnt1[i] = cnt; d1[i] = d; diag1[i] = 1.f / d; }
}

// Columns: one warp per column, 32 columns (one bitmap word column) per CTA of 1024 threads.  Pass 1 counts each column into
// ptr2[j + 1]; pass 2 (after the scan) lists its rows in ascending order with their entry positions, sums the column and
// normalises operator 2's values.
__global__ void __launch_bounds__(1024) k_mtgnn_col_count(int n, PatternOut pat, const uint32_t* __restrict__ bits) {
  const int lane = threadIdx.x & 31, c = threadIdx.x >> 5, j = blockIdx.x * 32 + c;
  if (j >= n) return;
  const int wpr = (n + 31) / 32;
  int cnt = 0;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    const bool on = i < n && ((__ldg(bits + (int64_t)i * wpr + blockIdx.x) >> c) & 1u);
    cnt += __popc(__ballot_sync(0xffffffffu, on));
  }
  if (lane == 0) pat.ptr2[j + 1] = cnt;
}

__global__ void __launch_bounds__(1024) k_mtgnn_col_scan(int n, PatternOut pat) {
  __shared__ int part[1024];
  int* p = pat.ptr2;
  const int per = (n + 1023) / 1024, b = threadIdx.x * per;
  int s = 0;
  for (int q = b; q < b + per && q < n; ++q) s += p[q + 1];
  part[threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    int run = 0;
    for (int q = 0; q < 1024; ++q) { const int v = part[q]; part[q] = run; run += v; }
    p[0] = 0;
  }
  __syncthreads();
  int run = part[threadIdx.x];
  for (int q = b; q < b + per && q < n; ++q) { run += p[q + 1]; p[q + 1] = run; }
}

__global__ void __launch_bounds__(1024) k_mtgnn_col_fill(int n, PatternOut pat, const uint32_t* __restrict__ bits,
                                                         const float* __restrict__ a, float* d2, float* v2, float* diag2) {
  const int lane = threadIdx.x & 31, c = threadIdx.x >> 5, j = blockIdx.x * 32 + c;
  if (j >= n) return;
  const int wpr = (n + 31) / 32;
  const int p0 = __ldg(pat.ptr2 + j);
  int p = p0;
  float s = 0.f;
  for (int i0 = 0; i0 < n; i0 += 32) {
    const int i = i0 + lane;
    const bool on = i < n && ((__ldg(bits + (int64_t)i * wpr + blockIdx.x) >> c) & 1u);
    const uint32_t ball = __ballot_sync(0xffffffffu, on);
    float v = 0.f;
    if (on) {
      const int64_t base = (int64_t)i * pat.w;
      const int cnt = __ldg(pat.cnt1 + i);
      int slot = 0;
      while (slot < cnt && __ldg(pat.col1 + base + slot) != j) ++slot;
      const int q = p + __popc(ball & ((1u << lane) - 1u));
      pat.row2[q] = i;
      pat.pos2[q] = (int)(base + slot);
      v = __ldg(a + base + slot);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    s += v;
    p += __popc(ball);
  }
  const float d = 1.f + s;
  __syncwarp();
  for (int q = p0 + lane; q < p; q += 32) {
    const int e = pat.pos2[q];
    v2[e] = a[e] / d;
  }
  if (lane == 0) { d2[j] = d; diag2[j] = 1.f / d; }
}

// ---- propagation ---------------------------------------------------------------------------------------------------------------
struct Prop {
  int64_t B, C, N, T, depth;
  float alpha;
  int64_t x_bs, h_bs;                               // batch strides of X (C N T) and of the hop buffers (2 D C N T)
};

// out = alpha X + (1 - alpha) S hprev, element (b, c, i, t); hprev and out are channel blocks of the hop buffer (or X)
__global__ void __launch_bounds__(kThreads) k_mtgnn_hop(Prop pr, Op op, const float* __restrict__ x, const float* __restrict__ hprev,
                                                        int64_t hprev_bs, float* __restrict__ out) {
  const int64_t per_b = pr.C * pr.N * pr.T;
  const int64_t idx = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (idx >= pr.B * per_b) return;
  const int64_t b = idx / per_b, r = idx - b * per_b;
  const int64_t c = r / (pr.N * pr.T), r2 = r - c * pr.N * pr.T;
  const int i = (int)(r2 / pr.T);
  const int64_t t = r2 - (int64_t)i * pr.T;
  const float* h = hprev + b * hprev_bs + c * pr.N * pr.T;
  const float acc = gather_row(op, i, h, pr.T, t);
  const float xv = __ldg(x + b * pr.x_bs + r);
  out[b * pr.h_bs + r] = __fadd_rn(__fmul_rn(pr.alpha, xv), __fmul_rn(1.f - pr.alpha, acc));
}

// Adjoint of hop k with S^T: G_{k-1} += (1 - alpha) S^T G_k (first: into dX), and dX += alpha G_k
__global__ void __launch_bounds__(kThreads) k_mtgnn_hop_adjoint(Prop pr, Op op, const float* __restrict__ gk, float* gprev,
                                                                float* dx, int first) {
  const int64_t per_b = pr.C * pr.N * pr.T;
  const int64_t idx = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  if (idx >= pr.B * per_b) return;
  const int64_t b = idx / per_b, r = idx - b * per_b;
  const int64_t c = r / (pr.N * pr.T), r2 = r - c * pr.N * pr.T;
  const int i = (int)(r2 / pr.T);
  const int64_t t = r2 - (int64_t)i * pr.T;
  const float* g = gk + b * pr.h_bs + c * pr.N * pr.T;
  const float acc = __fmul_rn(1.f - pr.alpha, gather_row(op, i, g, pr.T, t));
  const float ag = __fmul_rn(pr.alpha, g[(int64_t)i * pr.T + t]);
  float* dxp = dx + b * pr.x_bs + r;
  if (first) {
    *dxp = __fadd_rn(__fadd_rn(*dxp, ag), acc);
  } else {
    float* gp = gprev + b * pr.h_bs + r;
    *gp = __fadd_rn(*gp, acc);
    *dxp = __fadd_rn(*dxp, ag);
  }
}

// sum over hops k, batches b, channels c and steps t of G_k[b, c, u, t] H_{k-1}[b, c, v, t] for operator o, by one warp: the lanes
// cover (c, t) of one (k, b) block, which is summed on its own before it is added to the lane's total; then a fixed butterfly.
__device__ float sampled(const Prop& pr, int o, const float* __restrict__ x, const float* __restrict__ hops, const float* __restrict__ g,
                         int u, int v, int lane) {
  const int64_t NT = pr.N * pr.T;
  float total = 0.f;
  for (int64_t k = 1; k <= pr.depth; ++k) {
    const int64_t gblk = (o * pr.depth + k - 1) * pr.C;
    const int64_t hblk = (o * pr.depth + k - 2) * pr.C;
    for (int64_t b = 0; b < pr.B; ++b) {
      const float* gb = g + b * pr.h_bs + gblk * NT + (int64_t)u * pr.T;
      const float* hb = k == 1 ? x + b * pr.x_bs + (int64_t)v * pr.T : hops + b * pr.h_bs + hblk * NT + (int64_t)v * pr.T;
      float part = 0.f;
      if (pr.T >= 32) {
        for (int64_t c = 0; c < pr.C; ++c)
          for (int64_t t = lane; t < pr.T; t += 32) part = fmaf(__ldg(gb + c * NT + t), __ldg(hb + c * NT + t), part);
      } else {
        const int per = 32 / (int)pr.T, lc = lane / (int)pr.T;
        const int64_t t = lane - (int64_t)lc * pr.T;
        if (lc < per)
          for (int64_t c = lc; c < pr.C; c += per) part = fmaf(__ldg(gb + c * NT + t), __ldg(hb + c * NT + t), part);
      }
      total += part;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) total += __shfl_xor_sync(0xffffffffu, total, off);
  return __fmul_rn(1.f - pr.alpha, total);
}

// dvals = [dv1 | dv2 | ddiag1 | ddiag2]: tasks 0 .. N W - 1 the entries (i, j) of A (both operators), N W .. N W + N - 1 the diagonals
__global__ void __launch_bounds__(kThreads) k_mtgnn_dvals(Prop pr, Pattern pat, const float* __restrict__ x, const float* __restrict__ hops,
                                                          const float* __restrict__ g, float* dvals) {
  const int64_t task = ((int64_t)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int64_t nw = (int64_t)pat.n * pat.w;
  if (task >= nw + pat.n) return;
  if (task < nw) {
    const int i = (int)(task / pat.w), s = (int)(task - (int64_t)i * pat.w);
    float d1v = 0.f, d2v = 0.f;
    if (s < __ldg(pat.cnt1 + i)) {
      const int j = __ldg(pat.col1 + task);
      d1v = sampled(pr, 0, x, hops, g, i, j, lane);
      d2v = sampled(pr, 1, x, hops, g, j, i, lane);
    }
    if (lane == 0) { dvals[task] = d1v; dvals[nw + task] = d2v; }
  } else {
    const int i = (int)(task - nw);
    const float a = sampled(pr, 0, x, hops, g, i, i, lane);
    const float b = sampled(pr, 1, x, hops, g, i, i, lane);
    if (lane == 0) { dvals[2 * nw + i] = a; dvals[2 * nw + pat.n + i] = b; }
  }
}

// ---- graph backward ------------------------------------------------------------------------------------------------------------
// dd1[r] = dL/dd1[r] = -(sum_row dv1 v1 + ddiag1 diag1) / d1[r], dd2[r] likewise over column r
__global__ void __launch_bounds__(kThreads) k_mtgnn_graph_dd(Pattern pat, const float* __restrict__ state, const float* __restrict__ vals,
                                                             const float* __restrict__ dvals, float* dd) {
  const int r = blockIdx.x * kThreads + threadIdx.x;
  const int n = pat.n;
  if (r >= n) return;
  const int64_t nw = (int64_t)n * pat.w;
  const float *d1 = state + nw, *d2 = d1 + n;
  const float *v1 = vals, *v2 = vals + nw, *diag1 = vals + 2 * nw, *diag2 = diag1 + n;
  const float *dv1 = dvals, *dv2 = dvals + nw, *ddiag1 = dvals + 2 * nw, *ddiag2 = ddiag1 + n;
  float s = 0.f;
  const int64_t base = (int64_t)r * pat.w;
  for (int q = 0; q < pat.cnt1[r]; ++q) s = fmaf(dv1[base + q], v1[base + q], s);
  s = fmaf(ddiag1[r], diag1[r], s);
  dd[r] = -s / d1[r];
  s = 0.f;
  for (int p = pat.ptr2[r]; p < pat.ptr2[r + 1]; ++p) { const int e = pat.pos2[p]; s = fmaf(dv2[e], v2[e], s); }
  s = fmaf(ddiag2[r], diag2[r], s);
  dd[n + r] = -s / d2[r];
}

// one CTA of 64 threads per node r, thread = embedding channel: row r's entries, then column r's, in their stored order
__global__ void __launch_bounds__(kMaxDim) k_mtgnn_graph_dm(Pattern pat, int dim, float alpha, const float* __restrict__ m1,
                                                            const float* __restrict__ m2, const float* __restrict__ state,
                                                            const float* __restrict__ dvals, const float* __restrict__ dd, float* dm1,
                                                            float* dm2) {
  const int r = blockIdx.x, c = threadIdx.x, n = pat.n;
  if (c >= dim) return;
  const int64_t nw = (int64_t)n * pat.w;
  const float *a = state, *d1 = state + nw, *d2 = d1 + n;
  const float *dv1 = dvals, *dv2 = dvals + nw;
  const float* ddc = dd + n;   // column (operator 2) terms
  float g1 = 0.f, g2 = 0.f;
  const int64_t base = (int64_t)r * pat.w;
  for (int q = 0; q < pat.cnt1[r]; ++q) {
    const int j = pat.col1[base + q];
    const float av = a[base + q];
    const float da = ((dv1[base + q] / d1[r] + dv2[base + q] / d2[j]) + dd[r]) + ddc[j];
    const float dz = da * (alpha * fmaf(-av, av, 1.f));
    g1 = fmaf(dz, m2[(int64_t)j * dim + c], g1);
    g2 = fmaf(-dz, m1[(int64_t)j * dim + c], g2);
  }
  for (int p = pat.ptr2[r]; p < pat.ptr2[r + 1]; ++p) {
    const int i = pat.row2[p];
    const int e = pat.pos2[p];
    const float av = a[e];
    const float da = ((dv1[e] / d1[i] + dv2[e] / d2[r]) + dd[i]) + ddc[r];
    const float dz = da * (alpha * fmaf(-av, av, 1.f));
    g1 = fmaf(-dz, m2[(int64_t)i * dim + c], g1);
    g2 = fmaf(dz, m1[(int64_t)i * dim + c], g2);
  }
  dm1[(int64_t)r * dim + c] = g1;
  dm2[(int64_t)r * dim + c] = g2;
}

// ---- host --------------------------------------------------------------------------------------------------------------------------
bool graph_ok(int64_t n, int64_t w) { return n >= 1 && n <= kMaxNodes && w >= 1 && w <= n; }

bool elems_fit(int64_t B, int64_t C, int64_t N, int64_t T) {
  return (double)B * (double)C * (double)N * (double)T <= (double)kMaxGrid * kThreads;
}

int64_t elems_grid(const Prop& pr) {
  const int64_t n = pr.B * pr.C * pr.N * pr.T;
  const int64_t g = (n + kThreads - 1) / kThreads;
  return g <= kMaxGrid ? g : -1;
}

int graph_columns(int n, PatternOut pat, const uint32_t* bits, const float* a, float* d2, float* v2, float* diag2,
                  cudaStream_t st) {
  const int wc = (n + 31) / 32;
  k_mtgnn_col_count<<<wc, 1024, 0, st>>>(n, pat, bits);
  STMP_LAUNCH_OK("k_mtgnn_col_count");
  k_mtgnn_col_scan<<<1, 1024, 0, st>>>(n, pat);
  STMP_LAUNCH_OK("k_mtgnn_col_scan");
  k_mtgnn_col_fill<<<wc, 1024, 0, st>>>(n, pat, bits, a, d2, v2, diag2);
  STMP_LAUNCH_OK("k_mtgnn_col_fill");
  return STMP_OK;
}

Op op_rows(const Pattern& p, const float* val, const float* diag) { return Op{nullptr, p.cnt1, p.col1, nullptr, p.w, val, diag}; }
Op op_cols(const Pattern& p, const float* val, const float* diag) { return Op{p.ptr2, nullptr, p.row2, p.pos2, p.w, val, diag}; }

int prop_prepare(const char* fn, Prop& pr, int64_t B, int64_t C, int64_t N, int64_t T, int64_t W, int64_t depth, float alpha) {
  STMP_REQUIRE(B >= 0 && C >= 1 && T >= 1 && graph_ok(N, W), STMP_EINVAL, "%s: B=%lld C=%lld N=%lld T=%lld W=%lld", fn, (long long)B,
               (long long)C, (long long)N, (long long)T, (long long)W);
  STMP_REQUIRE(C <= kMaxChannels && depth >= 1 && depth <= kMaxDepth, STMP_EUNSUPPORTED,
               "%s: C=%lld depth=%lld outside the envelope (C <= 64, depth 1..4)", fn, (long long)C, (long long)depth);
  STMP_REQUIRE(elems_fit(B, C, N, T), STMP_EUNSUPPORTED, "%s: B=%lld C=%lld N=%lld T=%lld: the grid exceeds 2^31 - 1 CTAs", fn,
               (long long)B, (long long)C, (long long)N, (long long)T);
  pr = Prop{B, C, N, T, depth, alpha, C * N * T, 2 * depth * C * N * T};
  STMP_REQUIRE(elems_grid(pr) >= 0 && (N * W + N) * 32 / kThreads + 1 <= kMaxGrid, STMP_EUNSUPPORTED,
               "%s: B=%lld C=%lld N=%lld T=%lld: a grid exceeds 2^31 - 1 CTAs", fn, (long long)B, (long long)C, (long long)N, (long long)T);
  return STMP_OK;
}

}  // namespace
}  // namespace stmp

using namespace stmp;

extern "C" int stmp_mtgnn_supported(int64_t n, int64_t k, int64_t dim, int64_t channels, int64_t depth, int64_t batch, int64_t steps) {
  if (!graph_ok(n, k) || k > kMaxK || dim < 1 || dim > kMaxDim || channels < 1 || channels > kMaxChannels || depth < 1 ||
      depth > kMaxDepth || batch < 0 || steps < 1)
    return STMP_EUNSUPPORTED;
  if (!elems_fit(batch, channels, n, steps)) return STMP_EUNSUPPORTED;
  return STMP_OK;
}

extern "C" int64_t stmp_mtgnn_graph_workspace_bytes(int64_t n) {
  if (n < 1 || n > kMaxNodes) return 0;
  return 4 * n * ((n + 31) / 32);
}

extern "C" int stmp_mtgnn_graph_fwd(int64_t n, int64_t k, int64_t dim, float alpha, const float* m1, const float* m2, void* workspace,
                                    int* pattern, float* state, float* vals, void* stream) {
  const char* fn = "stmp_mtgnn_graph_fwd";
  STMP_REQUIRE(graph_ok(n, k) && k <= kMaxK && dim >= 1 && dim <= kMaxDim, STMP_EUNSUPPORTED,
               "%s: N=%lld k=%lld dim=%lld outside the envelope (N <= 4096, 1 <= k <= min(N, 64), 1 <= dim <= 64)", fn, (long long)n,
               (long long)k, (long long)dim);
  STMP_REQUIRE(m1 && m2 && workspace && pattern && state && vals, STMP_EINVAL, "%s: NULL argument", fn);
  cudaStream_t st = (cudaStream_t)stream;
  const PatternOut pat = pattern_out(pattern, (int)n, (int)k);
  const int64_t nw = n * k;
  float *a = state, *d1 = state + nw, *d2 = d1 + n;
  float *v1 = vals, *v2 = vals + nw, *diag1 = vals + 2 * nw, *diag2 = diag1 + n;
  uint32_t* bits = reinterpret_cast<uint32_t*>(workspace);
  const size_t smem = sizeof(float) * (n + 2 * kMaxDim) + sizeof(uint32_t) * ((n + 31) / 32);
  k_mtgnn_topk<<<(unsigned)n, kThreads, smem, st>>>((int)n, (int)k, (int)dim, alpha, m1, m2, pat, a, d1, v1, v2, diag1, bits);
  STMP_LAUNCH_OK("k_mtgnn_topk");
  return graph_columns((int)n, pat, bits, a, d2, v2, diag2, st);
}

extern "C" int stmp_mtgnn_graph_dense(int64_t n, int64_t w, const float* A, void* workspace, int* pattern, float* state, float* vals,
                                      void* stream) {
  const char* fn = "stmp_mtgnn_graph_dense";
  STMP_REQUIRE(graph_ok(n, w), STMP_EUNSUPPORTED, "%s: N=%lld W=%lld outside the envelope (N <= 4096, 1 <= W <= N)", fn,
               (long long)n, (long long)w);
  STMP_REQUIRE(A && workspace && pattern && state && vals, STMP_EINVAL, "%s: NULL argument", fn);
  cudaStream_t st = (cudaStream_t)stream;
  const PatternOut pat = pattern_out(pattern, (int)n, (int)w);
  const int64_t nw = n * w;
  float *a = state, *d1 = state + nw, *d2 = d1 + n;
  float *v1 = vals, *v2 = vals + nw, *diag1 = vals + 2 * nw, *diag2 = diag1 + n;
  uint32_t* bits = reinterpret_cast<uint32_t*>(workspace);
  k_mtgnn_dense_rows<<<(unsigned)((n + kThreads / 32 - 1) / (kThreads / 32)), kThreads, 0, st>>>((int)n, (int)w, A, pat, a, d1, v1,
                                                                                               v2, diag1, bits);
  STMP_LAUNCH_OK("k_mtgnn_dense_rows");
  return graph_columns((int)n, pat, bits, a, d2, v2, diag2, st);
}

extern "C" int64_t stmp_mtgnn_graph_bwd_workspace_bytes(int64_t n) { return n >= 1 && n <= kMaxNodes ? 8 * n : 0; }

extern "C" int stmp_mtgnn_graph_bwd(int64_t n, int64_t k, int64_t dim, float alpha, const float* m1, const float* m2, const int* pattern,
                                    const float* state, const float* vals, const float* dvals, void* workspace, float* dm1, float* dm2,
                                    void* stream) {
  const char* fn = "stmp_mtgnn_graph_bwd";
  STMP_REQUIRE(graph_ok(n, k) && k <= kMaxK && dim >= 1 && dim <= kMaxDim, STMP_EUNSUPPORTED,
               "%s: N=%lld k=%lld dim=%lld outside the envelope", fn, (long long)n, (long long)k, (long long)dim);
  STMP_REQUIRE(m1 && m2 && pattern && state && vals && dvals && workspace && dm1 && dm2, STMP_EINVAL, "%s: NULL argument", fn);
  cudaStream_t st = (cudaStream_t)stream;
  const Pattern pat = pattern_of(pattern, (int)n, (int)k);
  float* dd = reinterpret_cast<float*>(workspace);
  k_mtgnn_graph_dd<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, st>>>(pat, state, vals, dvals, dd);
  STMP_LAUNCH_OK("k_mtgnn_graph_dd");
  k_mtgnn_graph_dm<<<(unsigned)n, kMaxDim, 0, st>>>(pat, (int)dim, alpha, m1, m2, state, dvals, dd, dm1, dm2);
  STMP_LAUNCH_OK("k_mtgnn_graph_dm");
  return STMP_OK;
}

extern "C" int stmp_mtgnn_prop_fwd(int64_t B, int64_t C, int64_t N, int64_t T, int64_t W, int64_t depth, float alpha, const float* x,
                                   const int* pattern, const float* vals, float* hops, void* stream) {
  const char* fn = "stmp_mtgnn_prop_fwd";
  Prop pr;
  if (int rc = prop_prepare(fn, pr, B, C, N, T, W, depth, alpha)) return rc;
  if (B == 0) return STMP_OK;
  STMP_REQUIRE(x && pattern && vals && hops, STMP_EINVAL, "%s: NULL argument", fn);
  cudaStream_t st = (cudaStream_t)stream;
  const Pattern pat = pattern_of(pattern, (int)N, (int)W);
  const int64_t nw = N * W;
  const Op ops[2] = {op_rows(pat, vals, vals + 2 * nw), op_cols(pat, vals + nw, vals + 2 * nw + N)};
  const unsigned grid = (unsigned)elems_grid(pr);
  for (int o = 0; o < 2; ++o)
    for (int64_t k = 1; k <= depth; ++k) {
      const float* hprev = k == 1 ? x : hops + (o * depth + k - 2) * C * N * T;
      k_mtgnn_hop<<<grid, kThreads, 0, st>>>(pr, ops[o], x, hprev, k == 1 ? pr.x_bs : pr.h_bs, hops + (o * depth + k - 1) * C * N * T);
      STMP_LAUNCH_OK("k_mtgnn_hop");
    }
  return STMP_OK;
}

extern "C" int stmp_mtgnn_prop_bwd(int64_t B, int64_t C, int64_t N, int64_t T, int64_t W, int64_t depth, float alpha, const float* x,
                                   const int* pattern, const float* vals, const float* hops, float* dhops, float* dx, float* dvals,
                                   void* stream) {
  const char* fn = "stmp_mtgnn_prop_bwd";
  Prop pr;
  if (int rc = prop_prepare(fn, pr, B, C, N, T, W, depth, alpha)) return rc;
  STMP_REQUIRE(pattern && vals, STMP_EINVAL, "%s: NULL pattern or values", fn);
  cudaStream_t st = (cudaStream_t)stream;
  const Pattern pat = pattern_of(pattern, (int)N, (int)W);
  const int64_t nw = N * W;
  if (B == 0) {
    if (dvals) STMP_CUDA_OK(cudaMemsetAsync(dvals, 0, sizeof(float) * (2 * nw + 2 * N), st));
    return STMP_OK;
  }
  STMP_REQUIRE(x && hops && dhops && dx, STMP_EINVAL, "%s: NULL argument", fn);
  // S1^T gathers over the column arrays with operator 1's values, S2^T over the row arrays with operator 2's
  const Op adj[2] = {op_cols(pat, vals, vals + 2 * nw), op_rows(pat, vals + nw, vals + 2 * nw + N)};
  const unsigned grid = (unsigned)elems_grid(pr);
  for (int o = 0; o < 2; ++o)
    for (int64_t k = depth; k >= 1; --k) {
      float* gk = dhops + (o * depth + k - 1) * C * N * T;
      float* gprev = k == 1 ? nullptr : dhops + (o * depth + k - 2) * C * N * T;
      k_mtgnn_hop_adjoint<<<grid, kThreads, 0, st>>>(pr, adj[o], gk, gprev, dx, k == 1 ? 1 : 0);
      STMP_LAUNCH_OK("k_mtgnn_hop_adjoint");
    }
  if (dvals) {
    const int64_t tasks = nw + N;
    k_mtgnn_dvals<<<(unsigned)((tasks * 32 + kThreads - 1) / kThreads), kThreads, 0, st>>>(pr, pat, x, hops, dhops, dvals);
    STMP_LAUNCH_OK("k_mtgnn_dvals");
  }
  return STMP_OK;
}
