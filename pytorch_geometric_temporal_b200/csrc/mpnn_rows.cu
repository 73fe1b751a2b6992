// mpnn_rows.cu -- MPNN-LSTM (DESIGN §4t) on graphs of ANY size, split over CTAs by destination rows.  One call is the
// reference's whole forward: two GCNConvs (gcn_norm's operator Op of the plan, which both share) each followed by ReLU, BatchNorm1d and
// dropout, then two stacked LSTMs over `window` steps and the output [h1 | h2 | S].  X has R = B * window * num_nodes rows (row
// r = (b window + t) num_nodes + n); the LSTMs run over M = B num_nodes sequences (m = b num_nodes + n).
//
//   k_mpnn_conv1   a1 = Op x (one warp per row, two input channels per lane above 32); r1 = relu(a1 W1^T + b1); dropout-1 bits; per-CTA
//                  BatchNorm-1 partials (count, mean, M2 per channel: Welford per lane, Chan's merge across warps)
//   k_mpnn_conv2   every CTA merges the BN-1 partials in the same fixed order (bit-identical statistics everywhere, no grid sync; CTA 0
//                  updates the running statistics); a2 = Op z1 with z1 = dropout(BN1(r1)) applied on the fly; z1 of the CTA's own rows;
//                  r2 = relu(a2 W2^T + b2); dropout-2 bits; BN-2 partials
//   k_mpnn_lstm    BN-2 as above; per sequence (four per warp, sharing every staged weight load) `window` steps of LSTM-1 (64 -> 32) and
//                  LSTM-2 (32 -> 32), states in registers, weights staged once per CTA; out = [h1 | h2 | S]
//
// BatchNorm: training mode normalises with the batch mean and biased variance and updates running_mean / running_var (unbiased variance)
// and num_batches_tracked on the device; a negative momentum stands for None (the cumulative average 1 / num_batches_tracked).  Eval mode
// uses the running statistics.  Dropout keeps an element where the caller's uniform u >= p and scales it by 1 / (1 - p); the kept bits
// are packed to one word per row and layer.  The gathers walk the plan's CSR rows in entry order with separate multiply and add; the
// contractions are fp32 FFMA; no atomics, so repeated calls are bit-identical.
#include "rows.cuh"

namespace stmp {
namespace {

using namespace rows;

constexpr int kH = 32;                       // hidden width
constexpr int kMpMaxCin = 64;
constexpr int kBnPart = 1 + 2 * kH;          // a BN partial: count, mean[32], M2[32]
constexpr int kP1 = 100, kP2 = 68;           // staged LSTM weight pitches: = 4 mod 32, so a warp's float4 row loads are conflict-free
constexpr int kLR = 4;                       // sequences per warp in k_mpnn_lstm
constexpr int kLTile = kRowsWarps * kLR;
constexpr int kLd = 3 * kH;                  // width of every weight-gradient basis (rows of the stash's `a`, both LSTM bases)
constexpr int kW1P = kMpMaxCin + 1;          // staged W1 pitch: odd, so lane-indexed rows are conflict-free

struct BnArgs {
  const float* gamma; const float* beta;
  float* rmean; float* rvar; long long* nbt; // running statistics (updated in training mode by CTA 0)
  float eps, momentum;                       // momentum < 0: None
};

// Training: the operands of the backward, written by the forward (rows r of X)
struct MpStash {
  float* a;                                  // (R, kLd): the convolutions' gathers, a1 = Op x at columns [0, ld1), a2 = Op z1 at [ld1, ld1 + 32)
  float* gates1; float* gates2;              // (R, 128): the LSTMs' activated gates i | f | g | o at step t of row r
  float* c1; float* c2;                      // (R, 32): their cell states
  float* z2;                                 // (R, 32): dropout(BN2(r2)), the second half of LSTM-1's input
  float* stats;                              // (2, 2, 32): per layer the mean and 1 / std BatchNorm normalised with
};

// Chan's merge of (nb, mb, m2b) into (n, mean, m2)
__device__ __forceinline__ void chan(float& n, float& mean, float& m2, float nb, float mb, float m2b) {
  if (nb == 0.f) return;
  const float nn = n + nb, d = mb - mean, f = nb / nn;
  mean = fmaf(d, f, mean);
  m2 = m2 + m2b + d * d * n * f;
  n = nn;
}

// The CTA's Welford states of its 8 warps (lane = channel) merged in warp order and written as its BN partial.  Every thread calls it.
__device__ __forceinline__ void bn_write_partial(float n, float mean, float m2, float* __restrict__ part, float (&red)[3][kRowsWarps][32]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  red[0][warp][lane] = n; red[1][warp][lane] = mean; red[2][warp][lane] = m2;
  __syncthreads();
  if (warp == 0) {
    float cn = 0.f, cm = 0.f, c2 = 0.f;
    for (int w = 0; w < kRowsWarps; ++w) chan(cn, cm, c2, red[0][w][lane], red[1][w][lane], red[2][w][lane]);
    float* q = part + (size_t)blockIdx.x * kBnPart;
    if (lane == 0) q[0] = cn;
    q[1 + lane] = cm;
    q[1 + kH + lane] = c2;
  }
}

// The BatchNorm affine map y = x s + t of channel `lane`, the same in every CTA: training mode merges the `parts` partials in one fixed
// order (warp w the contiguous parts [w per, (w + 1) per), then the 8 warp results in warp order) and CTA 0 updates the running
// statistics; eval mode reads them.  Holds two __syncthreads: every thread calls it.
__device__ __forceinline__ void bn_affine(const BnArgs& bn, bool training, const float* __restrict__ part, int parts,
                                          float (&red)[3][kRowsWarps][32], float& s, float& t, float* stats) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float g = __ldg(bn.gamma + lane), b = __ldg(bn.beta + lane);
  if (!training) {
    const float rm = bn.rmean[lane], rv = bn.rvar[lane];
    s = g / sqrtf(rv + bn.eps);
    t = fmaf(-rm, s, b);
    if (stats && blockIdx.x == 0 && warp == 0) {
      stats[lane] = rm;
      stats[kH + lane] = 1.f / sqrtf(rv + bn.eps);
    }
    return;
  }
  const int per = (parts + kRowsWarps - 1) / kRowsWarps, q0 = warp * per, q1 = min(q0 + per, parts);
  float n = 0.f, mean = 0.f, m2 = 0.f;
  for (int q = q0; q < q1; ++q) {
    const float* p = part + (size_t)q * kBnPart;
    chan(n, mean, m2, p[0], p[1 + lane], p[1 + kH + lane]);
  }
  __syncthreads();                           // red may still be read by a previous bn_write_partial
  red[0][warp][lane] = n; red[1][warp][lane] = mean; red[2][warp][lane] = m2;
  __syncthreads();
  n = mean = m2 = 0.f;
  for (int w = 0; w < kRowsWarps; ++w) chan(n, mean, m2, red[0][w][lane], red[1][w][lane], red[2][w][lane]);
  s = g / sqrtf(m2 / n + bn.eps);
  t = fmaf(-mean, s, b);
  if (blockIdx.x == 0 && warp == 0) {
    if (stats) {
      stats[lane] = mean;
      stats[kH + lane] = 1.f / sqrtf(m2 / n + bn.eps);
    }
    const long long cnt = *bn.nbt + 1;
    const float mom = bn.momentum < 0.f ? 1.f / (float)cnt : bn.momentum;
    bn.rmean[lane] = (1.f - mom) * bn.rmean[lane] + mom * mean;
    bn.rvar[lane] = (1.f - mom) * bn.rvar[lane] + mom * (m2 / (n - 1.f));
    __syncwarp();
    if (lane == 0) *bn.nbt = cnt;
  }
}

__device__ __forceinline__ void welford(float& n, float& mean, float& m2, float x) {
  n += 1.f;
  const float d = x - mean;
  mean += d / n;
  m2 = fmaf(d, x - mean, m2);
}

// y[c] = b[c] + sum_{k < K} v[k] W[c][k], lane c, v[k] on lane k (k < 32) or k - 32 of vhi; W staged [32][ldw]
__device__ __forceinline__ float lin_row(const float* __restrict__ w, int ldw, float bias, float vlo, float vhi, int K, int lane) {
  float y = bias;
  const int k1 = min(K, 32);
  for (int k = 0; k < k1; ++k) y = fmaf(__shfl_sync(0xffffffffu, vlo, k), w[lane * ldw + k], y);
  for (int k = 32; k < K; ++k) y = fmaf(__shfl_sync(0xffffffffu, vhi, k - 32), w[lane * ldw + k], y);
  return y;
}

struct MpLayer {
  const float* w; const float* b;            // W (32, K), b (32)
  const float* u;                            // (R, 32) uniforms of this layer's dropout, NULL for none
  unsigned* mask;                            // (R) kept bits (scratch)
  float* r;                                  // (R, 32) relu(y)
  float* part;                               // (grid, kBnPart) BN partials of r
};

struct MpConv {
  const int* rowptr; const int2* cv;         // Op by destination
  int n, cin;
  float p, scale;                            // dropout probability and 1 / (1 - p)
  const float* x;                            // (R, cin)
  MpLayer l;
  // k_mpnn_conv2: the first layer's output and BatchNorm
  const float* r1; const unsigned* mask1; const float* part1; int parts1;
  BnArgs bn1; int training;
  float* z1;                                 // (R, 32) dropout(BN1(r1))
  MpStash st; int ld1;                       // training (st.a non-NULL): a1 / a2 into st.a, ld1 = cin rounded up to 8
};

__device__ __forceinline__ float drop(float v, unsigned word, int lane, float scale) {
  return (word >> lane) & 1u ? v * scale : 0.f;
}

// r = relu(y) of row i, its dropout bits, and the lane's Welford state
__device__ __forceinline__ void finish_row(const MpConv& a, int i, float y, int lane, float& n, float& mean, float& m2) {
  const float r = fmaxf(y, 0.f);
  a.l.r[(size_t)i * kH + lane] = r;
  if (a.l.u) {
    const unsigned word = __ballot_sync(0xffffffffu, __ldg(a.l.u + (size_t)i * kH + lane) >= a.p);
    if (lane == 0) a.l.mask[i] = word;
  }
  welford(n, mean, m2, r);
}

__global__ void __launch_bounds__(kRowsThreads, 2) k_mpnn_conv1(MpConv a) {
  __shared__ float w[kH * kW1P];
  __shared__ float bias[kH];
  __shared__ float red[3][kRowsWarps][32];
  const int cin = a.cin, ldw = kW1P, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int e = tid; e < kH * cin; e += kRowsThreads) w[(e / cin) * ldw + e % cin] = __ldg(a.l.w + e);
  if (tid < kH) bias[tid] = __ldg(a.l.b + tid);
  __syncthreads();
  float n = 0.f, mean = 0.f, m2 = 0.f;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      float unused, lo, hi = 0.f;
      gather_row<false>(a.rowptr, a.cv, i, nullptr, 0, a.x, cin, min(cin, 32), lane, unused, lo);
      if (cin > 32) gather_row<false>(a.rowptr, a.cv, i, nullptr, 0, a.x + 32, cin, cin - 32, lane, unused, hi);
      if (a.st.a) {
        if (lane < a.ld1) a.st.a[(size_t)i * kLd + lane] = lo;
        if (32 + lane < a.ld1) a.st.a[(size_t)i * kLd + 32 + lane] = hi;
      }
      finish_row(a, i, lin_row(w, ldw, bias[lane], lo, hi, cin, lane), lane, n, mean, m2);
    }
  }
  bn_write_partial(n, mean, m2, a.l.part, red);
}

__global__ void __launch_bounds__(kRowsThreads, 2) k_mpnn_conv2(MpConv a) {
  __shared__ float w[kH * (kH + 1)];
  __shared__ float bias[kH];
  __shared__ float red[3][kRowsWarps][32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int e = tid; e < kH * kH; e += kRowsThreads) w[(e / kH) * (kH + 1) + e % kH] = __ldg(a.l.w + e);
  if (tid < kH) bias[tid] = __ldg(a.l.b + tid);
  float s, t;
  bn_affine(a.bn1, a.training, a.part1, a.parts1, red, s, t, a.st.stats);
  __syncthreads();                           // w, bias, and red free for bn_write_partial
  const bool dropped = a.mask1 != nullptr;
  float n = 0.f, mean = 0.f, m2 = 0.f;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const int beg = __ldg(a.rowptr + i), end = __ldg(a.rowptr + i + 1);
      float acc = 0.f;
      int k = beg;
      for (; k + 4 <= end; k += 4) {
        int2 e[4];
        float v[4];
        unsigned m[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) e[q] = __ldg(a.cv + k + q);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          v[q] = a.r1[(size_t)e[q].x * kH + lane];
          m[q] = dropped ? a.mask1[e[q].x] : 0xffffffffu;
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) acc = __fadd_rn(acc, __fmul_rn(__int_as_float(e[q].y), drop(fmaf(v[q], s, t), m[q], lane, a.scale)));
      }
      for (; k < end; ++k) {
        const int2 e = __ldg(a.cv + k);
        const float z = drop(fmaf(a.r1[(size_t)e.x * kH + lane], s, t), dropped ? a.mask1[e.x] : 0xffffffffu, lane, a.scale);
        acc = __fadd_rn(acc, __fmul_rn(__int_as_float(e.y), z));
      }
      if (a.st.a) {
        a.st.a[(size_t)i * kLd + a.ld1 + lane] = acc;
        if (a.ld1 + 32 + lane < kLd) a.st.a[(size_t)i * kLd + a.ld1 + 32 + lane] = 0.f;
      }
      a.z1[(size_t)i * kH + lane] = drop(fmaf(a.r1[(size_t)i * kH + lane], s, t), dropped ? a.mask1[i] : 0xffffffffu, lane, a.scale);
      finish_row(a, i, lin_row(w, kH + 1, bias[lane], acc, 0.f, kH, lane), lane, n, mean, m2);
    }
  }
  bn_write_partial(n, mean, m2, a.l.part, red);
}

struct MpLstm {
  int nodes, window, seqs, cin;              // seqs = M = R / window
  const float* x;                            // (R, cin): S's source
  const float* z1; const float* r2; const unsigned* mask2;        // mask2 NULL: no dropout
  const float* part2; int parts2;
  BnArgs bn2; int training;
  float scale;
  const float* wih1; const float* whh1; const float* bih1; const float* bhh1;   // (128, 64), (128, 32), (128), (128)
  const float* wih2; const float* whh2; const float* bih2; const float* bhh2;   // (128, 32), (128, 32), (128), (128)
  float* out;                                // (M, 64 + cin + window - 1)
  MpStash st;                                // training: gates, cell states, z2 and BN-2's statistics (st.gates1 non-NULL)
};

struct LstmSmem {
  float w1[4 * kH * kP1];                    // gate row j: [W_ih1[j] (64) | W_hh1[j] (32)]
  float w2[4 * kH * kP2];                    // [W_ih2[j] (32) | W_hh2[j] (32)]
  float xin[kRowsWarps][kLR][3 * kH];        // per warp and sequence: the step's input row
  float red[3][kRowsWarps][32];
};

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float dot4(float4 a, float4 b, float y) { return fmaf(a.w, b.w, fmaf(a.z, b.z, fmaf(a.y, b.y, fmaf(a.x, b.x, y)))); }

// one LSTM step of the warp's kLR sequences: the gate pre-activations of channel `lane` (gate order i | f | g | o) from the staged
// weights w [128][P] and the inputs xin [kLR][K], then c and h updated in place
template <int K, int P>
__device__ __forceinline__ void lstm_step(const float* __restrict__ w, const float (*xin)[3 * kH], const float (&b)[4], float (&c)[kLR],
                                          float (&h)[kLR], int lane, float* gs, float* cs, const size_t (&row)[kLR]) {
  float g[kLR][4];
#pragma unroll
  for (int s = 0; s < kLR; ++s)
#pragma unroll
    for (int q = 0; q < 4; ++q) g[s][q] = b[q];
#pragma unroll 2
  for (int k = 0; k < K; k += 4) {
    float4 wq[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) wq[q] = ld4(w + (q * kH + lane) * P + k);
#pragma unroll
    for (int s = 0; s < kLR; ++s) {
      const float4 xv = ld4(&xin[s][k]);
#pragma unroll
      for (int q = 0; q < 4; ++q) g[s][q] = dot4(wq[q], xv, g[s][q]);
    }
  }
#pragma unroll
  for (int s = 0; s < kLR; ++s) {
    const float ig = sigmoidf_acc(g[s][0]), fg = sigmoidf_acc(g[s][1]), gg = tanhf(g[s][2]), og = sigmoidf_acc(g[s][3]);
    c[s] = fmaf(fg, c[s], ig * gg);
    h[s] = og * tanhf(c[s]);
    if (gs) {                                // training stash (a copy of the last sequence writes the same values twice)
      float* q = gs + row[s] * 4 * kH + lane;
      q[0] = ig; q[kH] = fg; q[2 * kH] = gg; q[3 * kH] = og;
      cs[row[s] * kH + lane] = c[s];
    }
  }
}

__global__ void __launch_bounds__(kRowsThreads, 2) k_mpnn_lstm(MpLstm a) {
  extern __shared__ __align__(16) unsigned char smraw[];
  LstmSmem& sm = *reinterpret_cast<LstmSmem*>(smraw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int e = tid; e < 4 * kH * 3 * kH; e += kRowsThreads) {
    const int j = e / (3 * kH), k = e - j * 3 * kH;
    sm.w1[j * kP1 + k] = k < 2 * kH ? __ldg(a.wih1 + j * 2 * kH + k) : __ldg(a.whh1 + j * kH + k - 2 * kH);
  }
  for (int e = tid; e < 4 * kH * 2 * kH; e += kRowsThreads) {
    const int j = e / (2 * kH), k = e - j * 2 * kH;
    sm.w2[j * kP2 + k] = k < kH ? __ldg(a.wih2 + j * kH + k) : __ldg(a.whh2 + j * kH + k - kH);
  }
  float b1[4], b2[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    b1[q] = __ldg(a.bih1 + q * kH + lane) + __ldg(a.bhh1 + q * kH + lane);
    b2[q] = __ldg(a.bih2 + q * kH + lane) + __ldg(a.bhh2 + q * kH + lane);
  }
  float s, t;
  bn_affine(a.bn2, a.training, a.part2, a.parts2, sm.red, s, t, a.st.stats ? a.st.stats + 2 * kH : nullptr);
  __syncthreads();                           // the staged weights
  const int N = a.nodes, T = a.window, M = a.seqs, cin = a.cin, W = 2 * kH + cin + T - 1;
  float (*xin)[3 * kH] = sm.xin[warp];
  for (int t0 = blockIdx.x * kLTile; t0 < M; t0 += gridDim.x * kLTile) {
    const int m0 = t0 + warp * kLR;
    float h1[kLR], c1[kLR], h2[kLR], c2[kLR];
    long long base[kLR];                     // row of step 0: b T N + n
#pragma unroll
    for (int q = 0; q < kLR; ++q) {
      h1[q] = c1[q] = h2[q] = c2[q] = 0.f;
      const int m = min(m0 + q, M - 1);      // sequences past M compute a copy of the last one and are not written
      base[q] = (long long)(m / N) * T * N + m % N;
    }
    for (int st = 0; st < T; ++st) {
      size_t row[kLR];
#pragma unroll
      for (int q = 0; q < kLR; ++q) {
        const size_t r = (size_t)(base[q] + (long long)st * N);
        row[q] = r;
        const float r2 = a.r2[r * kH + lane];
        const float z2 = drop(fmaf(r2, s, t), a.mask2 ? a.mask2[r] : 0xffffffffu, lane, a.scale);
        xin[q][lane] = a.z1[r * kH + lane];
        xin[q][kH + lane] = z2;
        xin[q][2 * kH + lane] = h1[q];
        if (a.st.z2) a.st.z2[r * kH + lane] = z2;
      }
      __syncwarp();
      lstm_step<3 * kH, kP1>(sm.w1, xin, b1, c1, h1, lane, a.st.gates1, a.st.c1, row);
      __syncwarp();
#pragma unroll
      for (int q = 0; q < kLR; ++q) {
        xin[q][lane] = h1[q];
        xin[q][kH + lane] = h2[q];
      }
      __syncwarp();
      lstm_step<2 * kH, kP2>(sm.w2, xin, b2, c2, h2, lane, a.st.gates2, a.st.c2, row);
      __syncwarp();
    }
#pragma unroll
    for (int q = 0; q < kLR; ++q) {
      if (m0 + q >= M) break;
      float* o = a.out + (size_t)(m0 + q) * W;
      o[lane] = h1[q];
      o[kH + lane] = h2[q];
      for (int k = lane; k < cin + T - 1; k += 32) {
        const long long r = k < cin ? base[q] : base[q] + (long long)(k - cin + 1) * N;
        o[2 * kH + k] = __ldg(a.x + (size_t)r * cin + (k < cin ? k : cin - 1));
      }
    }
  }
}


// ---- backward --------------------------------------------------------------------------------------------------------------------------
//   k_mpnn_lstm_bwd    per sequence (one per warp) BPTT through LSTM-2 then LSTM-1 at each step, newest first: the gates' pre-activation
//                      gradients dpre (R, 128) and the weight-gradient bases [z1 | z2 | h1_{t-1}], [h1_t | h2_{t-1} | 0] (R, 96) of
//                      both LSTMs; dz1 and g2 = dL/d BN2-output (dz2 through the dropout); per-CTA partials of sum g2, sum g2 xhat2
//   k_mpnn_bn_bwd      (per layer) every CTA sums the partials in one fixed order; CTA 0 writes dbeta, dgamma; dY = relu'(y) gamma / std
//                      (g - [training] (mean g + xhat mean(g xhat))) into its half of dY (R, 64) = [dY1 | dY2]
//   k_mpnn_conv2_bwd   dZ1 = dz1 + (Op^T dY2) W2 (transposed gather by source); g1 = dZ1 through the dropout; BN-1 partials
//   k_mpnn_dx          dX = (Op^T dY1) W1 + the gradient of S's columns
//   k_wide_rows_wgrad<5> + _reduce<5> (rows.cuh): dW = dpre^T basis, db = 1^T dpre of both LSTMs and [dY1 | dY2]^T [a1 | a2] of the
//                      convolutions, as five 64-column gates on 96-wide bases: rows 0..127 LSTM-1 ([W_ih | W_hh] over the basis), 128..255
//                      LSTM-2, 256..287 W1 (columns < cin), 288..319 W2 (columns ld1 ..)
struct MpBwdBuf {
  const float* r1; const float* z1; const float* r2; const unsigned* mask1; const unsigned* mask2;   // forward scratch
  MpStash st;
  float* dz1; float* g2; float* g1;          // (R, 32)
  float* dY;                                 // (R, 64) [dY1 | dY2]
  float* dpre1; float* dpre2;                // (R, 128)
  float* basis1; float* basis2;              // (R, 96)
  float* part_l; float* part_c;              // (grid, 64) BN partials [sum g | sum g xhat] of k_mpnn_lstm_bwd (BN-2), k_mpnn_conv2_bwd (BN-1)
};

struct MpLstmBwd {
  int nodes, window, seqs, cin;
  float scale;                               // 1 / (1 - p), masks present when the forward had dropout
  const float* gout;                         // (M, 64 + cin + window - 1)
  const float* wih1; const float* whh1; const float* wih2; const float* whh2;
  MpBwdBuf b;
};

struct LstmBwdSmem {
  float w1[4 * kH * kP1];
  float w2[4 * kH * kP2];
  float dp[kRowsWarps][4 * kH];
  float red[2][kRowsWarps][32];
};

__device__ __forceinline__ void stage_lstm(float* w1, float* w2, const float* wih1, const float* whh1, const float* wih2, const float* whh2) {
  for (int e = threadIdx.x; e < 4 * kH * 3 * kH; e += kRowsThreads) {
    const int j = e / (3 * kH), k = e - j * 3 * kH;
    w1[j * kP1 + k] = k < 2 * kH ? __ldg(wih1 + j * 2 * kH + k) : __ldg(whh1 + j * kH + k - 2 * kH);
  }
  for (int e = threadIdx.x; e < 4 * kH * 2 * kH; e += kRowsThreads) {
    const int j = e / (2 * kH), k = e - j * 2 * kH;
    w2[j * kP2 + k] = k < kH ? __ldg(wih2 + j * kH + k) : __ldg(whh2 + j * kH + k - kH);
  }
}

// one LSTM cell's backward at channel `lane`: dh (total), dc (carried from the later step, replaced by the earlier step's), the activated
// gates and c_t, c_{t-1} -> the pre-activation gradients d[4] (i | f | g | o), also written to dp (the warp's shared row) and dpre
__device__ __forceinline__ void cell_bwd(float dh, float& dc, const float* __restrict__ G, float c, float cp, float* dp, float* dpre,
                                         int lane) {
  const float i = G[lane], f = G[kH + lane], g = G[2 * kH + lane], o = G[3 * kH + lane];
  const float tc = tanhf(c);
  const float dct = fmaf(dh * o, 1.f - tc * tc, dc);
  const float d[4] = {dct * g * i * (1.f - i), dct * cp * f * (1.f - f), dct * i * (1.f - g * g), dh * tc * o * (1.f - o)};
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    dp[q * kH + lane] = d[q];
    dpre[q * kH + lane] = d[q];
  }
  dc = dct * f;
}

__global__ void __launch_bounds__(kRowsThreads, 2) k_mpnn_lstm_bwd(MpLstmBwd a) {
  extern __shared__ __align__(16) unsigned char smraw[];
  LstmBwdSmem& sm = *reinterpret_cast<LstmBwdSmem*>(smraw);
  stage_lstm(sm.w1, sm.w2, a.wih1, a.whh1, a.wih2, a.whh2);
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int N = a.nodes, T = a.window, M = a.seqs, W = 2 * kH + a.cin + T - 1;
  const MpBwdBuf& b = a.b;
  const float mean2 = b.st.stats[2 * kH + lane], inv2 = b.st.stats[3 * kH + lane];
  float* dp = sm.dp[warp];
  float sg = 0.f, sgx = 0.f;
  for (int m = blockIdx.x * kRowsWarps + warp; m < M; m += gridDim.x * kRowsWarps) {
    const long long base = (long long)(m / N) * T * N + m % N;
    float dh1 = a.gout[(size_t)m * W + lane], dh2 = a.gout[(size_t)m * W + kH + lane], dc1 = 0.f, dc2 = 0.f;
    for (int t = T - 1; t >= 0; --t) {
      const size_t r = (size_t)(base + (long long)t * N), rp = t ? r - N : 0;
      const float* G1 = b.st.gates1 + r * 4 * kH;
      const float* G2 = b.st.gates2 + r * 4 * kH;
      const float c1 = b.st.c1[r * kH + lane], c2 = b.st.c2[r * kH + lane];
      const float c1p = t ? b.st.c1[rp * kH + lane] : 0.f, c2p = t ? b.st.c2[rp * kH + lane] : 0.f;
      const float h1 = G1[3 * kH + lane] * tanhf(c1);
      const float h1p = t ? b.st.gates1[rp * 4 * kH + 3 * kH + lane] * tanhf(c1p) : 0.f;
      const float h2p = t ? b.st.gates2[rp * 4 * kH + 3 * kH + lane] * tanhf(c2p) : 0.f;
      cell_bwd(dh2, dc2, G2, c2, c2p, dp, b.dpre2 + r * 4 * kH, lane);
      __syncwarp();
      float dx = 0.f, dhp = 0.f;
      for (int j = 0; j < 4 * kH; ++j) {
        const float v = dp[j];
        dx = fmaf(v, sm.w2[j * kP2 + lane], dx);
        dhp = fmaf(v, sm.w2[j * kP2 + kH + lane], dhp);
      }
      __syncwarp();
      dh2 = dhp;
      dh1 += dx;
      cell_bwd(dh1, dc1, G1, c1, c1p, dp, b.dpre1 + r * 4 * kH, lane);
      __syncwarp();
      float dz1 = 0.f, dz2 = 0.f;
      dhp = 0.f;
      for (int j = 0; j < 4 * kH; ++j) {
        const float v = dp[j];
        dz1 = fmaf(v, sm.w1[j * kP1 + lane], dz1);
        dz2 = fmaf(v, sm.w1[j * kP1 + kH + lane], dz2);
        dhp = fmaf(v, sm.w1[j * kP1 + 2 * kH + lane], dhp);
      }
      __syncwarp();
      dh1 = dhp;
      const float g2 = drop(dz2, b.mask2 ? b.mask2[r] : 0xffffffffu, lane, a.scale);
      b.dz1[r * kH + lane] = dz1;
      b.g2[r * kH + lane] = g2;
      sg += g2;
      sgx = fmaf(g2, (b.r2[r * kH + lane] - mean2) * inv2, sgx);
      float* s1 = b.basis1 + r * kLd;
      s1[lane] = b.z1[r * kH + lane];
      s1[kH + lane] = b.st.z2[r * kH + lane];
      s1[2 * kH + lane] = h1p;
      float* s2 = b.basis2 + r * kLd;
      s2[lane] = h1;
      s2[kH + lane] = h2p;
      s2[2 * kH + lane] = 0.f;
    }
  }
  sm.red[0][warp][lane] = sg;
  sm.red[1][warp][lane] = sgx;
  __syncthreads();
  if (warp == 0) {
    float u = 0.f, v = 0.f;
    for (int w = 0; w < kRowsWarps; ++w) {
      u += sm.red[0][w][lane];
      v += sm.red[1][w][lane];
    }
    b.part_l[(size_t)blockIdx.x * 2 * kH + lane] = u;
    b.part_l[(size_t)blockIdx.x * 2 * kH + kH + lane] = v;
  }
}

struct MpBnBwd {
  int n, parts, training;
  const float* part;                         // (parts, 64) [sum g | sum g xhat]
  const float* r; const float* g;            // (R, 32) relu output and dL/d BN output
  const float* gamma; const float* stats;    // stats: mean | 1 / std
  float* dY; int col;                        // (R, 64): this layer's 32 columns at `col`
  float* dbeta; float* dgamma;
};

__global__ void __launch_bounds__(kRowsThreads) k_mpnn_bn_bwd(MpBnBwd a) {
  __shared__ float sub[8][32];
  __shared__ float tot[2 * kH];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int h = 0; h < 2; ++h) {
    const float v = fixed_order_sum(a.part + h * kH + lane, 2 * kH, a.parts, true, sub);
    if (warp == 0) tot[h * kH + lane] = v;
    __syncthreads();
  }
  if (blockIdx.x == 0 && warp == 0) {
    a.dbeta[lane] = tot[lane];
    a.dgamma[lane] = tot[kH + lane];
  }
  const float mean = a.stats[lane], inv = a.stats[kH + lane], k = __ldg(a.gamma + lane) * inv;
  const float m1 = tot[lane] / (float)a.n, m2 = tot[kH + lane] / (float)a.n;
  for (int i = blockIdx.x * kRowsWarps + warp; i < a.n; i += gridDim.x * kRowsWarps) {
    const size_t e = (size_t)i * kH + lane;
    const float r = a.r[e], g = a.g[e];
    const float d = a.training ? k * (g - m1 - (r - mean) * inv * m2) : k * g;
    a.dY[(size_t)i * 2 * kH + a.col + lane] = r > 0.f ? d : 0.f;
  }
}

struct MpGatherBwd {
  const int* rowptr; const int2* cv;         // Op by SOURCE
  int n, cin, nodes, window;
  float scale;
  const float* w;                            // conv2: W2 (32, 32); dx: W1 (32, cin)
  const float* dY;
  const float* stats;                        // conv2: BN-1's
  MpBwdBuf b;
  const float* gout; float* dx;              // dx: the output's gradient (S's columns) and dX (R, cin)
};

__global__ void __launch_bounds__(kRowsThreads, 2) k_mpnn_conv2_bwd(MpGatherBwd a) {
  __shared__ float w[kH * kGruPitch];
  __shared__ float red[2][kRowsWarps][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int e = threadIdx.x; e < kH * kH; e += kRowsThreads) w[(e / kH) * kGruPitch + e % kH] = __ldg(a.w + e);
  __syncthreads();
  const MpBwdBuf& b = a.b;
  const float mean = a.stats[lane], inv = a.stats[kH + lane];
  float sg = 0.f, sgx = 0.f;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int j = t0 + warp; j < t1; j += kRowsWarps) {
      float unused, t;
      gather_row<false>(a.rowptr, a.cv, j, nullptr, 0, a.dY + kH, 2 * kH, kH, lane, unused, t);
      const size_t e = (size_t)j * kH + lane;
      const float g1 = drop(b.dz1[e] + row_times_w(w, t, kH, lane), b.mask1 ? b.mask1[j] : 0xffffffffu, lane, a.scale);
      b.g1[e] = g1;
      sg += g1;
      sgx = fmaf(g1, (b.r1[e] - mean) * inv, sgx);
    }
  }
  red[0][warp][lane] = sg;
  red[1][warp][lane] = sgx;
  __syncthreads();
  if (warp == 0) {
    float u = 0.f, v = 0.f;
    for (int q = 0; q < kRowsWarps; ++q) {
      u += red[0][q][lane];
      v += red[1][q][lane];
    }
    b.part_c[(size_t)blockIdx.x * 2 * kH + lane] = u;
    b.part_c[(size_t)blockIdx.x * 2 * kH + kH + lane] = v;
  }
}

__global__ void __launch_bounds__(kRowsThreads, 2) k_mpnn_dx(MpGatherBwd a) {
  __shared__ float w[kH * kW1P];
  const int cin = a.cin, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int e = threadIdx.x; e < kH * cin; e += kRowsThreads) w[(e / cin) * kW1P + e % cin] = __ldg(a.w + e);
  __syncthreads();
  const int N = a.nodes, T = a.window, W = 2 * kH + cin + T - 1;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int j = t0 + warp; j < t1; j += kRowsWarps) {
      float unused, t;
      gather_row<false>(a.rowptr, a.cv, j, nullptr, 0, a.dY, 2 * kH, kH, lane, unused, t);
      float lo = 0.f, hi = 0.f;
      for (int c = 0; c < kH; ++c) {
        const float v = __shfl_sync(0xffffffffu, t, c);
        lo = fmaf(v, w[c * kW1P + lane], lo);
        hi = fmaf(v, w[c * kW1P + kH + lane], hi);
      }
      const int step = (j / N) % T;          // S: every feature of step 0, the last feature of steps 1 .. T-1
      const float* go = a.gout + (size_t)((j / N / T) * N + j % N) * W + 2 * kH;
      if (step == 0) {
        if (lane < cin) lo += go[lane];
        if (kH + lane < cin) hi += go[kH + lane];
      } else {
        if (lane == cin - 1) lo += go[cin + step - 1];
        if (kH + lane == cin - 1) hi += go[cin + step - 1];
      }
      if (lane < cin) a.dx[(size_t)j * cin + lane] = lo;
      if (kH + lane < cin) a.dx[(size_t)j * cin + kH + lane] = hi;
    }
  }
}
}  // namespace
}  // namespace stmp

using namespace stmp;

static int lstm_grid(long long seqs) {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long tiles = (seqs + kLTile - 1) / kLTile;
  return (int)(tiles < 2 * sms ? (tiles > 0 ? tiles : 1) : 2 * sms);
}

static int ld1_of(int64_t cin) { return (int)((cin + 7) / 8 * 8); }

// the training stash: a (R, 96), gates1 / gates2 (R, 128), c1 / c2 / z2 (R, 32), the BatchNorm statistics (2, 2, 32); NULL: none
static MpStash stash_of(void* p, int64_t R) {
  MpStash s = {};
  if (!p) return s;
  float* f = reinterpret_cast<float*>(p);
  s.a = f; f += R * kLd;
  s.gates1 = f; f += R * 4 * kH;
  s.gates2 = f; f += R * 4 * kH;
  s.c1 = f; f += R * kH;
  s.c2 = f; f += R * kH;
  s.z2 = f; f += R * kH;
  s.stats = f;
  return s;
}

static bool mpnn_supported(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window) {
  return plan && plan->flavor == STMP_FLAVOR_GCN && plan->flags == 0 && plan->n_ops >= 1 && hidden == kH && cin >= 1 &&
         cin <= kMpMaxCin && window >= 1 && plan->n % window == 0;
}

extern "C" int stmp_mpnn_rows_supported(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window) {
  return mpnn_supported(plan, cin, hidden, window) ? 1 : 0;
}

// r1, z1, r2 (R, 32); mask1, mask2 (R); the BN partials of both layers (grid, kBnPart)
extern "C" int64_t stmp_mpnn_rows_scratch_bytes(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window) {
  if (!mpnn_supported(plan, cin, hidden, window)) return 0;
  const int64_t R = plan->n;
  return (3 * R * kH + 2 * R + 2 * (int64_t)rows_grid(plan->n) * kBnPart) * 4;
}

extern "C" int stmp_mpnn_rows_fwd(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window, int64_t num_nodes, const float* x,
                                  const float* w1,
                                  const float* b1, const float* w2, const float* b2, const float* bn1_weight, const float* bn1_bias,
                                  float* bn1_mean, float* bn1_var, int64_t* bn1_count, float bn1_eps, float bn1_momentum,
                                  const float* bn2_weight, const float* bn2_bias, float* bn2_mean, float* bn2_var, int64_t* bn2_count,
                                  float bn2_eps, float bn2_momentum, const float* w_ih1, const float* w_hh1, const float* b_ih1,
                                  const float* b_hh1, const float* w_ih2, const float* w_hh2, const float* b_ih2, const float* b_hh2,
                                  int training, float p, const float* u, void* scratch, void* stash, float* out, void* stream) {
  const char* fn = "stmp_mpnn_rows_fwd";
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: plan is NULL", fn);
  STMP_REQUIRE(plan->flavor == STMP_FLAVOR_GCN, STMP_EINVAL, "%s: the plan is not a GCN plan (flavor %d)", fn, plan->flavor);
  STMP_REQUIRE(mpnn_supported(plan, cin, hidden, window), STMP_EUNSUPPORTED, "%s: hidden 32, in_channels 1..64, window >= 1 dividing "
               "the %d nodes, and a GCN plan without flags only (in_channels=%lld, hidden=%lld, window=%lld, flags=%u)", fn, plan->n,
               (long long)cin, (long long)hidden, (long long)window, plan->flags);
  STMP_REQUIRE(x && w1 && b1 && w2 && b2 && bn1_weight && bn1_bias && bn1_mean && bn1_var && bn1_count && bn2_weight && bn2_bias && bn2_mean &&
               bn2_var && bn2_count && w_ih1 && w_hh1 && b_ih1 && b_hh1 && w_ih2 && w_hh2 && b_ih2 && b_hh2 && scratch && out,
               STMP_EINVAL, "%s: NULL tensor", fn);
  STMP_REQUIRE(!u || (p > 0.f && p < 1.f), STMP_EINVAL, "%s: dropout uniforms need 0 < p < 1 (p=%g)", fn, (double)p);
  STMP_REQUIRE(num_nodes >= 1 && plan->n % (window * num_nodes) == 0, STMP_ESHAPE, "%s: %d rows are not B x window=%lld x num_nodes=%lld",
               fn, plan->n, (long long)window, (long long)num_nodes);
  STMP_REQUIRE(plan->n >= 2 || !training, STMP_EINVAL, "%s: training-mode BatchNorm needs more than one row", fn);
  const void* ps[] = {x, w1, b1, w2, b2, bn1_weight, bn1_bias, bn1_mean, bn1_var, bn2_weight, bn2_bias, bn2_mean, bn2_var, w_ih1, w_hh1,
                      b_ih1, b_hh1, w_ih2, w_hh2, b_ih2, b_hh2, u, scratch, stash, out};
  for (const void* q : ps) STMP_REQUIRE(al4(q), STMP_ESHAPE, "%s: misaligned tensor", fn);
  STMP_REQUIRE(((uintptr_t)bn1_count & 7u) == 0 && ((uintptr_t)bn2_count & 7u) == 0, STMP_ESHAPE, "%s: misaligned count", fn);
  const int R = plan->n, grid = rows_grid(R);
  float* f = reinterpret_cast<float*>(scratch);
  float* r1 = f; float* z1 = r1 + (size_t)R * kH; float* r2 = z1 + (size_t)R * kH;
  unsigned* m1 = reinterpret_cast<unsigned*>(r2 + (size_t)R * kH); unsigned* m2 = m1 + R;
  float* part1 = reinterpret_cast<float*>(m2 + R); float* part2 = part1 + (size_t)grid * kBnPart;
  const float scale = u ? 1.f / (1.f - p) : 1.f;
  const BnArgs bn1 = {bn1_weight, bn1_bias, bn1_mean, bn1_var, reinterpret_cast<long long*>(bn1_count), bn1_eps, bn1_momentum};
  const BnArgs bn2 = {bn2_weight, bn2_bias, bn2_mean, bn2_var, reinterpret_cast<long long*>(bn2_count), bn2_eps, bn2_momentum};
  cudaStream_t st = (cudaStream_t)stream;
  const MpStash sh = stash_of(stash, R);
  MpConv c = {};
  c.st = sh; c.ld1 = ld1_of(cin);
  c.rowptr = plan->fwd[0].rowptr; c.cv = plan->fwd[0].cv; c.n = R; c.cin = (int)cin; c.p = p; c.scale = scale; c.x = x;
  c.l = {w1, b1, u, m1, r1, part1};
  k_mpnn_conv1<<<grid, kRowsThreads, 0, st>>>(c);
  STMP_LAUNCH_OK("k_mpnn_conv1");
  c.l = {w2, b2, u ? u + (size_t)R * kH : nullptr, m2, r2, part2};
  c.r1 = r1; c.mask1 = u ? m1 : nullptr; c.part1 = part1; c.parts1 = grid; c.bn1 = bn1; c.training = training; c.z1 = z1;
  k_mpnn_conv2<<<grid, kRowsThreads, 0, st>>>(c);
  STMP_LAUNCH_OK("k_mpnn_conv2");
  MpLstm l = {};
  l.nodes = (int)num_nodes; l.window = (int)window; l.seqs = R / (int)window; l.cin = (int)cin; l.x = x;
  l.z1 = z1; l.r2 = r2; l.mask2 = u ? m2 : nullptr; l.part2 = part2; l.parts2 = grid; l.bn2 = bn2; l.training = training; l.scale = scale;
  l.wih1 = w_ih1; l.whh1 = w_hh1; l.bih1 = b_ih1; l.bhh1 = b_hh1; l.wih2 = w_ih2; l.whh2 = w_hh2; l.bih2 = b_ih2; l.bhh2 = b_hh2;
  l.out = out; l.st = sh;
  const int smem = (int)sizeof(LstmSmem);
  STMP_CUDA_OK(cudaFuncSetAttribute(k_mpnn_lstm, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_mpnn_lstm<<<lstm_grid(l.seqs), kRowsThreads, smem, st>>>(l);
  STMP_LAUNCH_OK("k_mpnn_lstm");
  return STMP_OK;
}

extern "C" int64_t stmp_mpnn_rows_stash_bytes(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window) {
  if (!mpnn_supported(plan, cin, hidden, window)) return 0;
  return ((int64_t)plan->n * (kLd + 8 * kH + 3 * kH) + 4 * kH) * 4;
}

static int lstm_bwd_grid(long long seqs) {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const long long tiles = (seqs + kRowsWarps - 1) / kRowsWarps;
  return (int)(tiles < 2 * sms ? (tiles > 0 ? tiles : 1) : 2 * sms);
}

// dz1, g2, g1 (R, 32); dY (R, 64); dpre1, dpre2 (R, 128); basis1, basis2 (R, 96); the BN partials of both layers; the weight-gradient
// partials of k_wide_rows_wgrad<5>
static MpBwdBuf bwd_buf(void* ws, int64_t R, int parts_l, int parts_c, float** wpartial) {
  MpBwdBuf b = {};
  float* f = reinterpret_cast<float*>(ws);
  b.dz1 = f; f += R * kH;
  b.g2 = f; f += R * kH;
  b.g1 = f; f += R * kH;
  b.dY = f; f += R * 2 * kH;
  b.dpre1 = f; f += R * 4 * kH;
  b.dpre2 = f; f += R * 4 * kH;
  b.basis1 = f; f += R * kLd;
  b.basis2 = f; f += R * kLd;
  b.part_l = f; f += (int64_t)parts_l * 2 * kH;
  b.part_c = f; f += (int64_t)parts_c * 2 * kH;
  *wpartial = f;
  return b;
}

extern "C" int64_t stmp_mpnn_rows_workspace_bytes(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window) {
  if (!mpnn_supported(plan, cin, hidden, window)) return 0;
  const int64_t R = plan->n;
  return (R * (5 * kH + 8 * kH + 2 * kLd) + (int64_t)(2 * wgrad_ffma_max_parts() + rows_grid(plan->n)) * 2 * kH +
          (int64_t)5 * wide_wgrad_parts(R) * (kLd * 64 + 64)) * 4;
}

extern "C" int stmp_mpnn_rows_bwd(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window, int64_t num_nodes, const float* gout,
                                  const float* w1, const float* w2, const float* bn1_weight, const float* bn2_weight, const float* w_ih1,
                                  const float* w_hh1, const float* w_ih2, const float* w_hh2, int training, float p, void* scratch,
                                  void* stash, void* workspace, float* dx, float* dbn, void* stream) {
  const char* fn = "stmp_mpnn_rows_bwd";
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: plan is NULL", fn);
  STMP_REQUIRE(mpnn_supported(plan, cin, hidden, window), STMP_EUNSUPPORTED, "%s: outside the envelope of stmp_mpnn_rows_supported", fn);
  STMP_REQUIRE(gout && w1 && w2 && bn1_weight && bn2_weight && w_ih1 && w_hh1 && w_ih2 && w_hh2 && scratch && stash && workspace && dbn,
               STMP_EINVAL, "%s: NULL tensor", fn);
  STMP_REQUIRE(p >= 0.f && p < 1.f, STMP_EINVAL, "%s: p=%g outside [0, 1)", fn, (double)p);
  STMP_REQUIRE(num_nodes >= 1 && plan->n % (window * num_nodes) == 0, STMP_ESHAPE, "%s: %d rows are not B x window=%lld x num_nodes=%lld",
               fn, plan->n, (long long)window, (long long)num_nodes);
  const void* ps[] = {gout, w1, w2, bn1_weight, bn2_weight, w_ih1, w_hh1, w_ih2, w_hh2, scratch, dx, dbn};
  for (const void* q : ps) STMP_REQUIRE(al4(q), STMP_ESHAPE, "%s: misaligned tensor", fn);
  STMP_REQUIRE(((uintptr_t)stash & 15u) == 0 && ((uintptr_t)workspace & 15u) == 0, STMP_ESHAPE, "%s: stash or workspace not 16-byte "
               "aligned", fn);
  const int R = plan->n, grid = rows_grid(R), T = (int)window, M = R / T, lgrid = lstm_bwd_grid(M);
  float* f = reinterpret_cast<float*>(scratch);
  const float* r1 = f; const float* z1 = r1 + (size_t)R * kH; const float* r2 = z1 + (size_t)R * kH;
  const unsigned* m1 = reinterpret_cast<const unsigned*>(r2 + (size_t)R * kH); const unsigned* m2 = m1 + R;
  float* wpart;
  MpBwdBuf b = bwd_buf(workspace, R, lgrid, grid, &wpart);
  b.r1 = r1; b.z1 = z1; b.r2 = r2; b.mask1 = p > 0.f ? m1 : nullptr; b.mask2 = p > 0.f ? m2 : nullptr;
  b.st = stash_of(stash, R);
  const float scale = p > 0.f ? 1.f / (1.f - p) : 1.f;
  cudaStream_t st = (cudaStream_t)stream;
  MpLstmBwd l = {(int)num_nodes, T, M, (int)cin, scale, gout, w_ih1, w_hh1, w_ih2, w_hh2, b};
  const int smem = (int)sizeof(LstmBwdSmem);
  STMP_CUDA_OK(cudaFuncSetAttribute(k_mpnn_lstm_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_mpnn_lstm_bwd<<<lgrid, kRowsThreads, smem, st>>>(l);
  STMP_LAUNCH_OK("k_mpnn_lstm_bwd");
  MpBnBwd bn = {R, lgrid, training, b.part_l, r2, b.g2, bn2_weight, b.st.stats + 2 * kH, b.dY, kH, dbn + 2 * kH, dbn + 3 * kH};
  k_mpnn_bn_bwd<<<grid, kRowsThreads, 0, st>>>(bn);
  STMP_LAUNCH_OK("k_mpnn_bn_bwd");
  MpGatherBwd g = {};
  g.rowptr = plan->bwd[0].rowptr; g.cv = plan->bwd[0].cv; g.n = R; g.cin = (int)cin; g.nodes = (int)num_nodes; g.window = T;
  g.scale = scale; g.w = w2; g.dY = b.dY; g.stats = b.st.stats; g.b = b; g.gout = gout;
  k_mpnn_conv2_bwd<<<grid, kRowsThreads, 0, st>>>(g);
  STMP_LAUNCH_OK("k_mpnn_conv2_bwd");
  bn = {R, grid, training, b.part_c, r1, b.g1, bn1_weight, b.st.stats, b.dY, 0, dbn, dbn + kH};
  k_mpnn_bn_bwd<<<grid, kRowsThreads, 0, st>>>(bn);
  STMP_LAUNCH_OK("k_mpnn_bn_bwd");
  if (dx) {
    g.w = w1; g.dx = dx;
    k_mpnn_dx<<<grid, kRowsThreads, 0, st>>>(g);
    STMP_LAUNCH_OK("k_mpnn_dx");
  }
  return STMP_OK;
}

extern "C" int stmp_mpnn_rows_wgrad(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window, void* stash, void* workspace,
                                    float* dw, float* db, void* stream) {
  const char* fn = "stmp_mpnn_rows_wgrad";
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: plan is NULL", fn);
  STMP_REQUIRE(mpnn_supported(plan, cin, hidden, window), STMP_EUNSUPPORTED, "%s: outside the envelope of stmp_mpnn_rows_supported", fn);
  STMP_REQUIRE(stash && workspace && dw && db, STMP_EINVAL, "%s: NULL tensor", fn);
  const void* ps[] = {stash, workspace, dw, db};
  for (const void* q : ps) STMP_REQUIRE(((uintptr_t)q & 15u) == 0, STMP_ESHAPE, "%s: tensor not 16-byte aligned", fn);
  const int R = plan->n, M = R / (int)window;
  float* wpart;
  const MpBwdBuf b = bwd_buf(workspace, R, lstm_bwd_grid(M), rows_grid(R), &wpart);
  const MpStash sh = stash_of(stash, R);
  WideWgradOps<5> op = {{b.basis1, b.basis1, b.basis2, b.basis2, sh.a}, {b.dpre1, b.dpre1 + 64, b.dpre2, b.dpre2 + 64, b.dY},
                        {128, 128, 128, 128, 64}};
  const int parts = wide_wgrad_parts(R);
  cudaStream_t st = (cudaStream_t)stream;
  k_wide_rows_wgrad<5><<<dim3(parts, 5), kWideWgThreads, 0, st>>>(R, kLd, op, wpart);
  STMP_LAUNCH_OK("k_mpnn_wgrad");
  const int total = 5 * 64 * kLd + 5 * 64;
  k_wide_rows_wgrad_reduce<5><<<(total + 31) / 32, 256, 0, st>>>(parts, kLd, kLd, wpart, 0, 0, nullptr, dw, db, nullptr);
  STMP_LAUNCH_OK("k_mpnn_wgrad_reduce");
  return STMP_OK;
}
