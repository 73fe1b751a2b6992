// agcrn.cu -- AGCRN, the adaptive graph convolutional recurrent cell (DESIGN §4u), in exact fp32.  One call of the reference's
// AGCRN.forward (nn/recurrent/agcrn.py) with its two AVWGCNs, gate (z = 0: Co = 2 out) and update (z = 1: Co = out), Ci = in + out:
//
//   S = softmax(relu(E E^T)), T_1 = S, T_2 = 2 S S - I          AVWGCN_z(Y)[b, n] = sum_k (T_k Y)[b, n] W_z,n[k] + E[n] bias_pool_z
//   W_z,n = E[n] weights_pool_z                                Y1 = [X | H], Z | R = sigmoid(AVWGCN_0(Y1)), Y2 = [X | Z H]
//   H' = R H + (1 - R) tanh(AVWGCN_1(Y2))                      (T_0 = I; at K = 1 the single weight block multiplies Y + S Y)
//
//   forward   k_agcrn_support        one warp per row: logits relu(e_n . e_m), row max, sum of exp in a fixed order, S
//             k_agcrn_gemm<T2>       K = 3: T_2 = 2 S S - I
//             k_agcrn_gemm<NodeW>    both AVWGCNs' node weights [W_n | b_n] = E [weights_pool | bias_pool], one product
//             k_agcrn_gemm<Sup<0>>   P1 = T_t [X | H] for every batch: the stacked supports times each batch's Y1
//             k_agcrn_gemm<Con<0>>   per node: [Y1 | P1 | 1] [W_n ; b_n] for all its batch rows -> Z, R, Z H
//             k_agcrn_gemm<Sup<1>>   P2 = T_t (Z H); the X columns of T_t Y2 are P1's
//             k_agcrn_gemm<Con<1>>   per node: [Y2 | P2 | 1] [W_n ; b_n] -> tanh -> H'
//   backward  k_agcrn_pw_update, then per AVWGCN (update, then gate, with k_agcrn_pw_gate between): dF = dOut W_n^T and
//             [dW_n ; db_n] = F^T dOut per node, summed over b in order; dY = dF_0 + sum_t T_t^T dF_t.  Then the pools' gradients
//             E^T [dW | db] (summed over n in order) and, for dE, dT_t = sum_b dF_t Y^T, dS (K = 3 through T_2), the softmax and ReLU
//             backward (k_agcrn_softmax_bwd) and dE = [dW | db] [pools]^T + (dA + dA^T) E as one product.
//
// Every product is one FFMA tile kernel (k_agcrn_gemm) instantiated per operand layout: 64 x 64 output tiles, a 16-deep k loop, 4 x 4
// outputs per thread, each sum running over k in one fixed order.  No atomics, no tensor cores: repeated calls are bit-identical and the
// training forward is the inference forward.
#include "rows.cuh"

namespace stmp {
namespace {

constexpr int kThreads = 256;
constexpr int kTm = 64, kTn = 64, kTk = 16;
constexpr int kMaxN = 4096, kMaxOut = 64, kMaxCi = 128, kMaxD = 64, kMaxK = 3;
constexpr int kSupRows = kThreads / 32;      // k_agcrn_support / _softmax_bwd: one row per warp
constexpr int kZMax = 65535;                 // gridDim.z; larger batches loop

struct Ag {
  int B, N, in, out, Ci, K, Kt, d;           // Kt = max(K - 1, 1): the supports kept (T_1, T_2)
  int kci;                                   // K Ci feature columns per node; row kci of W is the bias
  const float *x, *h, *e;                    // X (B, N, in), H (B, N, out) or NULL (zeros), E (N, d)
  const float* wp[2];                        // weights_pool (d, K, Ci, Co)
  const float* bp[2];                        // bias_pool (d, Co)
  float* S;                                  // (Kt, N, N)
  float* W[2];                               // (N, kci + 1, Co)
  float* P1;                                 // (B, N, Kt, Ci): T_t Y1
  float* P2;                                 // (B, N, Kt, out): T_t (Z H)
  float* ZR;                                 // (B, N, 2 out)
  float* ZH;                                 // (B, N, out)
  float* HC;                                 // (B, N, out): tanh of the update, the training stash (NULL in inference)
  float* hout;                               // (B, N, out)
  const float* gh;                           // dL/dH'
  float *dU, *dG;                            // (B, N, out), (B, N, 2 out): gradients of the pre-activations
  float* dF[2];                              // (B, N, kci)
  float* dY2;                                // (B, N, Ci)
  float* dW[2];                              // (N, kci + 1, Co)
  float *dT, *dS, *dA;                       // (Kt, N, N), (N, N) at K = 3, (N, N)
  float* part;                               // split-k partial sums (split_of), (problem, split, M, N)
  int splits;                                // k splits of the launch (1: no split, the epilogue stores directly)
  float *dx, *dh, *de, *dwp[2], *dbp[2];
};

__device__ __forceinline__ int co_of(const Ag& g, int z) { return z == 0 ? 2 * g.out : g.out; }
// the dF slot that support t (0-based) multiplies: slot 0 is the identity's, and at K = 1 also S's
__device__ __forceinline__ int slot_of(const Ag& g, int t) { return g.K == 1 ? 0 : t + 1; }
__device__ __forceinline__ float hval(const Ag& g, size_t bn, int c) { return g.h ? g.h[bn * g.out + c] : 0.f; }

// channel i of Y_z at (b, n) = bn: [X | H] for the gate, [X | Z H] for the update
template <int Z>
__device__ __forceinline__ float yval(const Ag& g, size_t bn, int i) {
  if (i < g.in) return g.x[bn * g.in + i];
  return Z == 0 ? hval(g, bn, i - g.in) : g.ZH[bn * g.out + i - g.in];
}

// column j of node n's feature row for AVWGCN z: slot s = j / Ci (0: Y, s > 0: T_s Y; K = 1: Y + S Y), channel i; column kci is the
// bias's 1
template <int Z>
__device__ __forceinline__ float feat(const Ag& g, int b, int n, int j) {
  if (j >= g.kci) return 1.f;
  const int s = j / g.Ci, i = j - s * g.Ci;
  const size_t bn = (size_t)b * g.N + n;
  float p = 0.f;
  if (s > 0 || g.K == 1) {
    const size_t bt = bn * g.Kt + (s > 0 ? s - 1 : 0);
    p = (Z == 0 || i < g.in) ? g.P1[bt * g.Ci + i] : g.P2[bt * g.out + i - g.in];
    if (s > 0) return p;
  }
  const float y = yval<Z>(g, bn, i);
  return g.K == 1 ? __fadd_rn(y, p) : y;
}

// ---- the FFMA tile product: C_z[r][c] = sum_k A_z[r][k] B_z[k][c], one 64 x 64 tile of one problem z per CTA pass.  Op supplies the
// problem count, each problem's M / N / K, element reads and the epilogue (store), and which index runs along memory in each operand, so
// that the tile loads are coalesced (kAm: A's m index, else its k index; kBn: B's n index, else its k index).
template <class Op>
__global__ void __launch_bounds__(kThreads, 2) k_agcrn_gemm(const Ag g) {
  __shared__ __align__(16) float As[kTk][kTm + 4];
  __shared__ __align__(16) float Bs[kTk][kTn + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int n0 = blockIdx.x * kTn;
  const int S = g.splits, nzs = Op::nz(g) * S;
  for (int zs = blockIdx.z; zs < nzs; zs += gridDim.z) {
    const int z = zs / S, sp = zs - z * S;
    const int M = Op::m(g, z), Nc = Op::n(g, z);
    const int Kall = Op::k(g, z);
    const int chunk = ((Kall + S - 1) / S + kTk - 1) / kTk * kTk;   // split sp sums k in [k_lo, Kd)
    const int k_lo = sp * chunk, Kd = k_lo + chunk < Kall ? k_lo + chunk : Kall;
    if (n0 >= Nc) continue;                  // block-uniform
    for (int m0 = blockIdx.y * kTm; m0 < M; m0 += gridDim.y * kTm) {
      float acc[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
      for (int k0 = k_lo; k0 < Kd; k0 += kTk) {
        float ra[4], rb[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int idx = tid + kThreads * q;
          const int am = Op::kAm ? (idx & 63) : (idx >> 4), ak = Op::kAm ? (idx >> 6) : (idx & 15);
          const int bn = Op::kBn ? (idx & 63) : (idx >> 4), bk = Op::kBn ? (idx >> 6) : (idx & 15);
          ra[q] = (m0 + am < M && k0 + ak < Kd) ? Op::a(g, z, m0 + am, k0 + ak) : 0.f;
          rb[q] = (n0 + bn < Nc && k0 + bk < Kd) ? Op::b(g, z, k0 + bk, n0 + bn) : 0.f;
        }
        __syncthreads();                     // the previous tile's reads are done
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int idx = tid + kThreads * q;
          As[Op::kAm ? (idx >> 6) : (idx & 15)][Op::kAm ? (idx & 63) : (idx >> 4)] = ra[q];
          Bs[Op::kBn ? (idx >> 6) : (idx & 15)][Op::kBn ? (idx & 63) : (idx >> 4)] = rb[q];
        }
        __syncthreads();
        float part[4][4];                    // this k tile's sums, added to acc once: two-level summation keeps long sums (dE: up to
#pragma unroll                               // (K Ci + 1) 3 out + N terms) as accurate as a blocked BLAS sum
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) part[i][j] = 0.f;
#pragma unroll
        for (int kk = 0; kk < kTk; ++kk) {
          const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
          const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
          const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) part[i][j] = fmaf(av[i], bv[j], part[i][j]);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] += part[i][j];
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int r = m0 + ty * 4 + i, c = n0 + tx * 4 + j;
          if (r < M && c < Nc) {
            if (S == 1) Op::store(g, z, r, c, acc[i][j]);
            else g.part[((size_t)zs * M + r) * Nc + c] = acc[i][j];
          }
        }
    }
  }
}

// T_2 = 2 S S - I
struct OpT2 {
  static constexpr bool kAm = false, kBn = true;
  static constexpr const char* kName = "k_agcrn_gemm_t2";
  __device__ static int nz(const Ag&) { return 1; }
  __device__ static int m(const Ag& g, int) { return g.N; }
  __device__ static int n(const Ag& g, int) { return g.N; }
  __device__ static int k(const Ag& g, int) { return g.N; }
  __device__ static float a(const Ag& g, int, int r, int k) { return g.S[(size_t)r * g.N + k]; }
  __device__ static float b(const Ag& g, int, int k, int c) { return g.S[(size_t)k * g.N + c]; }
  __device__ static void store(const Ag& g, int, int r, int c, float v) {
    g.S[(size_t)g.N * g.N + (size_t)r * g.N + c] = __fsub_rn(2.f * v, r == c ? 1.f : 0.f);
  }
};

// [W_z,n | b_z,n] = E[n] [weights_pool_z | bias_pool_z], z = 0, 1
struct OpNodeW {
  static constexpr bool kAm = false, kBn = true;
  static constexpr const char* kName = "k_agcrn_gemm_nodew";
  __device__ static int nz(const Ag&) { return 2; }
  __device__ static int m(const Ag& g, int) { return g.N; }
  __device__ static int n(const Ag& g, int z) { return (g.kci + 1) * co_of(g, z); }
  __device__ static int k(const Ag& g, int) { return g.d; }
  __device__ static float a(const Ag& g, int, int r, int k) { return g.e[(size_t)r * g.d + k]; }
  __device__ static float b(const Ag& g, int z, int k, int c) {
    const int Co = co_of(g, z), w = g.kci * Co;
    return c < w ? g.wp[z][(size_t)k * w + c] : g.bp[z][k * Co + c - w];
  }
  __device__ static void store(const Ag& g, int z, int r, int c, float v) { g.W[z][(size_t)r * (g.kci + 1) * co_of(g, z) + c] = v; }
};

// batch b = z: rows (t, n) of the stacked supports times Y1 (Z = 0: all Ci columns) or Z H (Z = 1)
template <int Z>
struct OpSup {
  static constexpr bool kAm = false, kBn = true;
  static constexpr const char* kName = Z == 0 ? "k_agcrn_gemm_sup_gate" : "k_agcrn_gemm_sup_update";
  __device__ static int nz(const Ag& g) { return g.B; }
  __device__ static int m(const Ag& g, int) { return g.Kt * g.N; }
  __device__ static int n(const Ag& g, int) { return Z == 0 ? g.Ci : g.out; }
  __device__ static int k(const Ag& g, int) { return g.N; }
  __device__ static float a(const Ag& g, int, int r, int k) { return g.S[(size_t)r * g.N + k]; }
  __device__ static float b(const Ag& g, int z, int k, int c) {
    const size_t bn = (size_t)z * g.N + k;
    return Z == 0 ? yval<0>(g, bn, c) : g.ZH[bn * g.out + c];
  }
  __device__ static void store(const Ag& g, int z, int r, int c, float v) {
    const int t = r / g.N, nn = r - t * g.N;
    const size_t bt = ((size_t)z * g.N + nn) * g.Kt + t;
    if (Z == 0) g.P1[bt * g.Ci + c] = v;
    else g.P2[bt * g.out + c] = v;
  }
};

// node n = z: its feature rows for every batch times [W_n ; b_n]; epilogue: the gate (Z = 0) or the update and the GRU combination
template <int Z>
struct OpCon {
  static constexpr bool kAm = false, kBn = true;
  static constexpr const char* kName = Z == 0 ? "k_agcrn_gemm_con_gate" : "k_agcrn_gemm_con_update";
  __device__ static int nz(const Ag& g) { return g.N; }
  __device__ static int m(const Ag& g, int) { return g.B; }
  __device__ static int n(const Ag& g, int) { return co_of(g, Z); }
  __device__ static int k(const Ag& g, int) { return g.kci + 1; }
  __device__ static float a(const Ag& g, int z, int r, int k) { return feat<Z>(g, r, z, k); }
  __device__ static float b(const Ag& g, int z, int k, int c) { return g.W[Z][((size_t)z * (g.kci + 1) + k) * co_of(g, Z) + c]; }
  __device__ static void store(const Ag& g, int z, int r, int c, float v) {
    const size_t bn = (size_t)r * g.N + z;
    if (Z == 0) {
      const float s = sigmoidf_acc(v);
      g.ZR[bn * 2 * g.out + c] = s;
      if (c < g.out) g.ZH[bn * g.out + c] = __fmul_rn(s, hval(g, bn, c));
    } else {
      const float hc = tanhf(v), rr = g.ZR[bn * 2 * g.out + g.out + c], h = hval(g, bn, c);
      g.hout[bn * g.out + c] = __fadd_rn(__fmul_rn(rr, h), __fmul_rn(__fsub_rn(1.f, rr), hc));
      if (g.HC) g.HC[bn * g.out + c] = hc;
    }
  }
};

// node n = z: dF_z = dOut W_n^T (the bias row has no feature gradient)
template <int Z>
struct OpDF {
  static constexpr bool kAm = false, kBn = false;
  static constexpr const char* kName = Z == 0 ? "k_agcrn_gemm_df_gate" : "k_agcrn_gemm_df_update";
  __device__ static int nz(const Ag& g) { return g.N; }
  __device__ static int m(const Ag& g, int) { return g.B; }
  __device__ static int n(const Ag& g, int) { return g.kci; }
  __device__ static int k(const Ag& g, int) { return co_of(g, Z); }
  __device__ static float a(const Ag& g, int z, int r, int k) {
    const size_t bn = (size_t)r * g.N + z;
    return Z == 0 ? g.dG[bn * 2 * g.out + k] : g.dU[bn * g.out + k];
  }
  __device__ static float b(const Ag& g, int z, int k, int c) { return g.W[Z][((size_t)z * (g.kci + 1) + c) * co_of(g, Z) + k]; }
  __device__ static void store(const Ag& g, int z, int r, int c, float v) { g.dF[Z][((size_t)r * g.N + z) * g.kci + c] = v; }
};

// node n = z: [dW_n ; db_n] = [F ; 1]^T dOut, summed over the batch rows in order
template <int Z>
struct OpDW {
  static constexpr bool kAm = true, kBn = true;
  static constexpr const char* kName = Z == 0 ? "k_agcrn_gemm_dw_gate" : "k_agcrn_gemm_dw_update";
  __device__ static int nz(const Ag& g) { return g.N; }
  __device__ static int m(const Ag& g, int) { return g.kci + 1; }
  __device__ static int n(const Ag& g, int) { return co_of(g, Z); }
  __device__ static int k(const Ag& g, int) { return g.B; }
  __device__ static float a(const Ag& g, int z, int r, int k) { return feat<Z>(g, k, z, r); }
  __device__ static float b(const Ag& g, int z, int k, int c) {
    const size_t bn = (size_t)k * g.N + z;
    return Z == 0 ? g.dG[bn * 2 * g.out + c] : g.dU[bn * g.out + c];
  }
  __device__ static void store(const Ag& g, int z, int r, int c, float v) {
    g.dW[Z][((size_t)z * (g.kci + 1) + r) * co_of(g, Z) + c] = v;
  }
};

// batch b = z: dY_z = dF_z,0 + sum_t T_t^T dF_z,slot(t).  Update: -> dY2.  Gate: the X columns plus dY2's -> dX, the H columns added
// to dH (which k_agcrn_pw_gate wrote)
template <int Z>
struct OpSupT {
  static constexpr bool kAm = true, kBn = true;
  static constexpr const char* kName = Z == 0 ? "k_agcrn_gemm_supt_gate" : "k_agcrn_gemm_supt_update";
  __device__ static int nz(const Ag& g) { return g.B; }
  __device__ static int m(const Ag& g, int) { return g.N; }
  __device__ static int n(const Ag& g, int) { return g.Ci; }
  __device__ static int k(const Ag& g, int) { return g.Kt * g.N; }
  __device__ static float a(const Ag& g, int, int r, int k) { return g.S[(size_t)k * g.N + r]; }
  __device__ static float b(const Ag& g, int z, int k, int c) {
    const int t = k / g.N, mm = k - t * g.N;
    return g.dF[Z][((size_t)z * g.N + mm) * g.kci + slot_of(g, t) * g.Ci + c];
  }
  __device__ static void store(const Ag& g, int z, int r, int c, float v) {
    const size_t bn = (size_t)z * g.N + r;
    v = __fadd_rn(v, g.dF[Z][bn * g.kci + c]);
    if (Z == 1) {
      g.dY2[bn * g.Ci + c] = v;
    } else if (c < g.in) {
      if (g.dx) g.dx[bn * g.in + c] = __fadd_rn(v, g.dY2[bn * g.Ci + c]);
    } else if (g.dh) {
      float* p = g.dh + bn * g.out + c - g.in;
      *p = __fadd_rn(*p, v);
    }
  }
};

// z = AVWGCN: [d weights_pool | d bias_pool] = E^T [dW | db], summed over the nodes in order
struct OpDPool {
  static constexpr bool kAm = true, kBn = true;
  static constexpr const char* kName = "k_agcrn_gemm_dpool";
  __device__ static int nz(const Ag&) { return 2; }
  __device__ static int m(const Ag& g, int) { return g.d; }
  __device__ static int n(const Ag& g, int z) { return (g.kci + 1) * co_of(g, z); }
  __device__ static int k(const Ag& g, int) { return g.N; }
  __device__ static float a(const Ag& g, int, int r, int k) { return g.e[(size_t)k * g.d + r]; }
  __device__ static float b(const Ag& g, int z, int k, int c) { return g.dW[z][(size_t)k * (g.kci + 1) * co_of(g, z) + c]; }
  __device__ static void store(const Ag& g, int z, int r, int c, float v) {
    const int Co = co_of(g, z), w = g.kci * Co;
    if (c < w) {
      if (g.dwp[z]) g.dwp[z][(size_t)r * w + c] = v;
    } else if (g.dbp[z]) {
      g.dbp[z][r * Co + c - w] = v;
    }
  }
};

// support t = z: dT_t = sum_b (dF_0,slot(t) Y1^T + dF_1,slot(t) Y2^T), the k index running over (b, channel of [Y1 | Y2])
struct OpDT {
  static constexpr bool kAm = false, kBn = false;
  static constexpr const char* kName = "k_agcrn_gemm_dt";
  static constexpr const char* kReduceName = "k_agcrn_split_reduce_dt";
  __device__ static int nz(const Ag& g) { return g.Kt; }
  __device__ static int m(const Ag& g, int) { return g.N; }
  __device__ static int n(const Ag& g, int) { return g.N; }
  __device__ static int k(const Ag& g, int) { return g.B * 2 * g.Ci; }   // < 2^31: agcrn_supported caps B
  __device__ static float a(const Ag& g, int z, int r, int k) {
    const int b = k / (2 * g.Ci), q = k - b * 2 * g.Ci, zz = q >= g.Ci;
    return g.dF[zz][((size_t)b * g.N + r) * g.kci + slot_of(g, z) * g.Ci + q - zz * g.Ci];
  }
  __device__ static float b(const Ag& g, int, int k, int c) {
    const int b = k / (2 * g.Ci), q = k - b * 2 * g.Ci;
    const size_t bn = (size_t)b * g.N + c;
    return q < g.Ci ? yval<0>(g, bn, q) : yval<1>(g, bn, q - g.Ci);
  }
  __device__ static void store(const Ag& g, int z, int r, int c, float v) { g.dT[((size_t)z * g.N + r) * g.N + c] = v; }
};

// K = 3: dS = dT_1 + 2 (dT_2 S^T + S^T dT_2)
struct OpDS {
  static constexpr bool kAm = false, kBn = true;
  static constexpr const char* kName = "k_agcrn_gemm_ds";
  __device__ static int nz(const Ag&) { return 1; }
  __device__ static int m(const Ag& g, int) { return g.N; }
  __device__ static int n(const Ag& g, int) { return g.N; }
  __device__ static int k(const Ag& g, int) { return 2 * g.N; }
  __device__ static float a(const Ag& g, int, int r, int k) {
    const size_t NN = (size_t)g.N * g.N;
    return k < g.N ? g.dT[NN + (size_t)r * g.N + k] : g.S[(size_t)(k - g.N) * g.N + r];
  }
  __device__ static float b(const Ag& g, int, int k, int c) {
    const size_t NN = (size_t)g.N * g.N;
    return k < g.N ? g.S[(size_t)c * g.N + k] : g.dT[NN + (size_t)(k - g.N) * g.N + c];
  }
  __device__ static void store(const Ag& g, int, int r, int c, float v) {
    const size_t i = (size_t)r * g.N + c;
    g.dS[i] = __fadd_rn(g.dT[i], 2.f * v);
  }
};

// dE = [dW_0 | db_0 | dW_1 | db_1] [pools_0 | pools_1]^T + (dA + dA^T) E, the k index running over the three segments
struct OpDE {
  static constexpr bool kAm = false, kBn = false;
  static constexpr const char* kName = "k_agcrn_gemm_de";
  static constexpr const char* kReduceName = "k_agcrn_split_reduce_de";
  __device__ static int nz(const Ag&) { return 1; }
  __device__ static int m(const Ag& g, int) { return g.N; }
  __device__ static int n(const Ag& g, int) { return g.d; }
  __device__ static int k(const Ag& g, int) { return (g.kci + 1) * 3 * g.out + g.N; }
  __device__ static float a(const Ag& g, int, int r, int k) {
    const int L0 = (g.kci + 1) * 2 * g.out, L1 = (g.kci + 1) * g.out;
    if (k < L0) return g.dW[0][(size_t)r * L0 + k];
    if (k < L0 + L1) return g.dW[1][(size_t)r * L1 + k - L0];
    const int m = k - L0 - L1;
    return __fadd_rn(g.dA[(size_t)r * g.N + m], g.dA[(size_t)m * g.N + r]);
  }
  __device__ static float b(const Ag& g, int, int k, int c) {
    const int L0 = (g.kci + 1) * 2 * g.out, L1 = (g.kci + 1) * g.out;
    if (k >= L0 + L1) return g.e[(size_t)(k - L0 - L1) * g.d + c];
    const int z = k >= L0, Co = co_of(g, z), w = g.kci * Co, j = k - z * L0;
    return j < w ? g.wp[z][(size_t)c * w + j] : g.bp[z][c * Co + j - w];
  }
  __device__ static void store(const Ag& g, int, int r, int c, float v) { g.de[(size_t)r * g.d + c] = v; }
};

// f(m, relu(e_n . e_m)) for every column m of row n (one warp per row; all threads of the block call it): E staged 32 rows at a time,
// each dot product in the order of the embedding dimensions
template <class F>
__device__ __forceinline__ void for_logits(const Ag& g, int n, float (&es)[32][kMaxD + 1], const float* en, F f) {
  const int lane = threadIdx.x & 31;
  for (int m0 = 0; m0 < g.N; m0 += 32) {
    __syncthreads();
    for (int i = threadIdx.x; i < 32 * g.d; i += kThreads) {
      const int r = i / g.d, dd = i - r * g.d;
      es[r][dd] = m0 + r < g.N ? g.e[(size_t)(m0 + r) * g.d + dd] : 0.f;
    }
    __syncthreads();
    if (n < g.N && m0 + lane < g.N) {
      float s = 0.f;
      for (int dd = 0; dd < g.d; ++dd) s = fmaf(en[dd], es[lane][dd], s);
      f(m0 + lane, s < 0.f ? 0.f : s);
    }
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// S = softmax(relu(E E^T), dim=1): the logits go to S's row, then exp(l - max) and the row sum (per lane in column order, then a
// butterfly: every lane holds the same sum), then the division
__global__ void __launch_bounds__(kThreads) k_agcrn_support(const Ag g) {
  __shared__ float es[32][kMaxD + 1];
  __shared__ float en[kSupRows][kMaxD];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, n = blockIdx.x * kSupRows + w;
  for (int dd = lane; dd < g.d; dd += 32) en[w][dd] = n < g.N ? g.e[(size_t)n * g.d + dd] : 0.f;
  float* row = g.S + (size_t)n * g.N;
  float mx = 0.f;
  for_logits(g, n, es, en[w], [&](int m, float l) {
    row[m] = l;
    mx = fmaxf(mx, l);
  });
  if (n >= g.N) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float s = 0.f;
  for (int m = lane; m < g.N; m += 32) {
    const float v = expf(__fsub_rn(row[m], mx));
    row[m] = v;
    s += v;
  }
  s = warp_sum(s);
  for (int m = lane; m < g.N; m += 32) row[m] = __fdiv_rn(row[m], s);
}

// dA = relu'(logits) * S * (dS - rowsum(dS * S)), one warp per row; relu' is 0 where the logit is 0, as torch's
__global__ void __launch_bounds__(kThreads) k_agcrn_softmax_bwd(const Ag g) {
  __shared__ float es[32][kMaxD + 1];
  __shared__ float en[kSupRows][kMaxD];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, n = blockIdx.x * kSupRows + w;
  for (int dd = lane; dd < g.d; dd += 32) en[w][dd] = n < g.N ? g.e[(size_t)n * g.d + dd] : 0.f;
  const float* ds = (g.K == 3 ? g.dS : g.dT) + (size_t)n * g.N;
  const float* sr = g.S + (size_t)n * g.N;
  float dot = 0.f;
  if (n < g.N)
    for (int m = lane; m < g.N; m += 32) dot = fmaf(ds[m], sr[m], dot);
  dot = warp_sum(dot);
  float* da = g.dA + (size_t)n * g.N;
  for_logits(g, n, es, en[w], [&](int m, float l) { da[m] = l > 0.f ? __fmul_rn(sr[m], __fsub_rn(ds[m], dot)) : 0.f; });
}

// dU = dH' (1 - R) (1 - HC^2)
__global__ void __launch_bounds__(kThreads) k_agcrn_pw_update(const Ag g) {
  const size_t total = (size_t)g.B * g.N * g.out;
  for (size_t i = blockIdx.x * (size_t)kThreads + threadIdx.x; i < total; i += (size_t)gridDim.x * kThreads) {
    const size_t bn = i / g.out;
    const int c = (int)(i - bn * g.out);
    const float r = g.ZR[bn * 2 * g.out + g.out + c], hc = g.HC[i];
    g.dU[i] = __fmul_rn(__fmul_rn(g.gh[i], __fsub_rn(1.f, r)), __fsub_rn(1.f, __fmul_rn(hc, hc)));
  }
}

// dZ = dY2[Z H] H, dR = dH' (H - HC), dG = [dZ | dR] sigmoid'; dH = dH' R + dY2[Z H] Z (the gate's own H columns follow)
__global__ void __launch_bounds__(kThreads) k_agcrn_pw_gate(const Ag g) {
  const size_t total = (size_t)g.B * g.N * g.out;
  for (size_t i = blockIdx.x * (size_t)kThreads + threadIdx.x; i < total; i += (size_t)gridDim.x * kThreads) {
    const size_t bn = i / g.out;
    const int c = (int)(i - bn * g.out);
    const float z = g.ZR[bn * 2 * g.out + c], r = g.ZR[bn * 2 * g.out + g.out + c];
    const float h = hval(g, bn, c), go = g.gh[i], dzh = g.dY2[bn * g.Ci + g.in + c];
    const float dz = __fmul_rn(dzh, h), dr = __fmul_rn(go, __fsub_rn(h, g.HC[i]));
    g.dG[bn * 2 * g.out + c] = __fmul_rn(__fmul_rn(dz, __fsub_rn(1.f, z)), z);
    g.dG[bn * 2 * g.out + g.out + c] = __fmul_rn(__fmul_rn(dr, __fsub_rn(1.f, r)), r);
    if (g.dh) g.dh[i] = __fadd_rn(__fmul_rn(go, r), __fmul_rn(dzh, z));
  }
}

// The split-k partials of a launch added in split order, then Op's epilogue (problems of one Op share M and N)
template <class Op>
__global__ void __launch_bounds__(kThreads) k_agcrn_split_reduce(const Ag g) {
  const int S = g.splits, M = Op::m(g, 0), Nc = Op::n(g, 0);
  const size_t per = (size_t)M * Nc, total = (size_t)Op::nz(g) * per;
  for (size_t i = blockIdx.x * (size_t)kThreads + threadIdx.x; i < total; i += (size_t)gridDim.x * kThreads) {
    const int z = (int)(i / per);
    const size_t rc = i - (size_t)z * per;
    const float* p = g.part + (size_t)z * S * per + rc;
    float v = p[0];
    for (int sp = 1; sp < S; ++sp) v += p[(size_t)sp * per];
    Op::store(g, z, (int)(rc / Nc), (int)(rc % Nc), v);
  }
}

// k splits of a long-k product with `tiles` output tiles: enough CTAs to fill two per SM of a 132-SM part, at least 512 k per split,
// at most 32 splits.  A function of the shapes alone, so the summation order (and every bit of the result) does not depend on the GPU.
inline int split_of(long long tiles, long long Kd) {
  const long long want = (264 + tiles - 1) / tiles, cap = Kd / 512;
  long long sp = want < cap ? want : cap;
  if (sp > 32) sp = 32;
  return sp > 1 ? (int)sp : 1;
}
inline long long tiles_of(long long M, long long Nc, long long nz) { return ((M + kTm - 1) / kTm) * ((Nc + kTn - 1) / kTn) * nz; }

inline int pw_grid(size_t total) {
  const size_t blocks = (total + kThreads - 1) / kThreads;
  return blocks < 4096 ? (blocks > 0 ? (int)blocks : 1) : 4096;
}

template <class Op>
int gemm(const Ag& g, long long M, long long Nc, long long nz, cudaStream_t st) {
  if (M <= 0 || Nc <= 0 || nz <= 0) return STMP_OK;
  const long long mt = (M + kTm - 1) / kTm;
  const dim3 grid((unsigned)((Nc + kTn - 1) / kTn), (unsigned)(mt < kZMax ? mt : kZMax), (unsigned)(nz < kZMax ? nz : kZMax));
  Ag g1 = g;
  g1.splits = 1;
  k_agcrn_gemm<Op><<<grid, kThreads, 0, st>>>(g1);
  STMP_LAUNCH_OK(Op::kName);                 // one call site per instantiation, so one path counter per Op
  return STMP_OK;
}

// A long-k product (dT, dE): split over k when its tiles alone leave the GPU mostly idle, the partials summed in order by
// k_agcrn_split_reduce, which applies the epilogue
template <class Op>
int gemm_split(const Ag& g, long long M, long long Nc, long long nz, long long Kd, cudaStream_t st) {
  if (M <= 0 || Nc <= 0 || nz <= 0) return STMP_OK;
  const int S = split_of(tiles_of(M, Nc, nz), Kd);
  if (S == 1) return gemm<Op>(g, M, Nc, nz, st);
  Ag gs = g;
  gs.splits = S;
  const dim3 grid((unsigned)((Nc + kTn - 1) / kTn), (unsigned)((M + kTm - 1) / kTm), (unsigned)(nz * S));
  k_agcrn_gemm<Op><<<grid, kThreads, 0, st>>>(gs);
  STMP_LAUNCH_OK(Op::kName);
  k_agcrn_split_reduce<Op><<<pw_grid((size_t)(nz * M * Nc)), kThreads, 0, st>>>(gs);
  STMP_LAUNCH_OK(Op::kReduceName);
  return STMP_OK;
}

// B (2 (in + out)) < 2^31: dT's reduction over (batch, channel) is counted in 32 bits
bool agcrn_supported(int64_t b, int64_t n, int64_t in, int64_t out, int64_t K, int64_t d) {
  return b >= 0 && b <= INT32_MAX / kMaxCi / 2 && n >= 1 && n <= kMaxN && in >= 1 && out >= 1 && out <= kMaxOut && in + out <= kMaxCi && K >= 1 && K <= kMaxK && d >= 1 &&
         d <= kMaxD;
}

// The float counts of each buffer, every one rounded up to 4 floats so each starts 16-byte aligned
struct Sizes {
  int64_t S, W0, W1, P1, P2, ZR, ZH;                   // scratch
  int64_t HC;                                          // stash
  int64_t dU, dG, dF0, dF1, dY2, dW0, dW1, dT, dS, dA, part; // workspace
};
inline int64_t r4(int64_t v) { return (v + 3) / 4 * 4; }
Sizes sizes(int64_t B, int64_t N, int64_t in, int64_t out, int64_t K) {
  const int64_t Ci = in + out, Kt = K > 1 ? K - 1 : 1, kci = K * Ci, BN = B * N;
  Sizes s;
  s.S = r4(Kt * N * N);
  s.W0 = r4(N * (kci + 1) * 2 * out);
  s.W1 = r4(N * (kci + 1) * out);
  s.P1 = r4(BN * Kt * Ci);
  s.P2 = r4(BN * Kt * out);
  s.ZR = r4(BN * 2 * out);
  s.ZH = r4(BN * out);
  s.HC = r4(BN * out);
  s.dU = r4(BN * out);
  s.dG = r4(BN * 2 * out);
  s.dF0 = s.dF1 = r4(BN * kci);
  s.dY2 = r4(BN * Ci);
  s.dW0 = s.W0;
  s.dW1 = s.W1;
  s.dT = s.S;
  s.dS = K == 3 ? r4(N * N) : 0;
  s.dA = r4(N * N);
  // the split-k partials of dT and of dE (d <= 64: one column tile), used one after the other
  const long long sdt = split_of(tiles_of(N, N, Kt), B * 2 * Ci), sde = split_of(tiles_of(N, kMaxD, 1), (kci + 1) * 3 * out + N);
  const long long pdt = sdt > 1 ? sdt * Kt * N * N : 0, pde = sde > 1 ? sde * N * kMaxD : 0;
  s.part = r4(pdt > pde ? pdt : pde);
  return s;
}

Ag make_ag(int64_t B, int64_t N, int64_t in, int64_t out, int64_t K, int64_t d, const float* x, const float* e, const float* h,
           const float* wp0, const float* bp0, const float* wp1, const float* bp1, void* scratch) {
  Ag g = {};
  g.B = (int)B; g.N = (int)N; g.in = (int)in; g.out = (int)out; g.Ci = (int)(in + out); g.K = (int)K;
  g.Kt = K > 1 ? (int)K - 1 : 1; g.d = (int)d; g.kci = g.K * g.Ci;
  g.x = x; g.e = e; g.h = h; g.wp[0] = wp0; g.bp[0] = bp0; g.wp[1] = wp1; g.bp[1] = bp1;
  const Sizes s = sizes(B, N, in, out, K);
  float* p = reinterpret_cast<float*>(scratch);
  g.S = p; p += s.S;
  g.W[0] = p; p += s.W0;
  g.W[1] = p; p += s.W1;
  g.P1 = p; p += s.P1;
  g.P2 = p; p += s.P2;
  g.ZR = p; p += s.ZR;
  g.ZH = p;
  return g;
}

int check_args(const char* fn, int64_t B, int64_t N, int64_t in, int64_t out, int64_t K, int64_t d) {
  STMP_REQUIRE(B >= 0, STMP_EINVAL, "%s: negative batch %lld", fn, (long long)B);
  STMP_REQUIRE(agcrn_supported(B, N, in, out, K, d), STMP_EUNSUPPORTED,
               "%s: B=%lld N=%lld in=%lld out=%lld K=%lld d=%lld outside the envelope (B <= 8388607, N <= 4096, out <= 64, in + out <= "
               "128, K <= 3, d <= 64)", fn, (long long)B, (long long)N, (long long)in, (long long)out, (long long)K, (long long)d);
  return STMP_OK;
}

}  // namespace
}  // namespace stmp

using namespace stmp;

extern "C" int stmp_agcrn_supported(int64_t b, int64_t n, int64_t in, int64_t out, int64_t K, int64_t d) {
  return agcrn_supported(b, n, in, out, K, d) ? 1 : 0;
}

extern "C" int64_t stmp_agcrn_scratch_bytes(int64_t b, int64_t n, int64_t in, int64_t out, int64_t K) {
  if (!agcrn_supported(b, n, in, out, K, 1)) return 0;
  const Sizes s = sizes(b, n, in, out, K);
  return 4 * (s.S + s.W0 + s.W1 + s.P1 + s.P2 + s.ZR + s.ZH);
}

extern "C" int64_t stmp_agcrn_stash_bytes(int64_t b, int64_t n, int64_t in, int64_t out, int64_t K) {
  if (!agcrn_supported(b, n, in, out, K, 1)) return 0;
  return 4 * sizes(b, n, in, out, K).HC;
}

extern "C" int64_t stmp_agcrn_workspace_bytes(int64_t b, int64_t n, int64_t in, int64_t out, int64_t K) {
  if (!agcrn_supported(b, n, in, out, K, 1)) return 0;
  const Sizes s = sizes(b, n, in, out, K);
  return 4 * (s.dU + s.dG + s.dF0 + s.dF1 + s.dY2 + s.dW0 + s.dW1 + s.dT + s.dS + s.dA + s.part);
}

extern "C" int stmp_agcrn_fwd(int64_t b, int64_t n, int64_t in, int64_t out, int64_t K, int64_t d, const float* x, const float* e,
                              const float* h, const float* wp_gate, const float* bp_gate, const float* wp_update, const float* bp_update,
                              void* scratch, void* stash, float* hout, void* stream) {
  const char* fn = "stmp_agcrn_fwd";
  if (int rc = check_args(fn, b, n, in, out, K, d)) return rc;
  STMP_REQUIRE(e && wp_gate && bp_gate && wp_update && bp_update && (b == 0 || (x && scratch && hout)), STMP_EINVAL, "%s: NULL tensor",
               fn);
  const void* ps[] = {x, e, h, wp_gate, bp_gate, wp_update, bp_update, scratch, stash, hout};
  for (const void* q : ps) STMP_REQUIRE(rows::al4(q), STMP_ESHAPE, "%s: misaligned tensor", fn);
  if (b == 0) return STMP_OK;
  Ag g = make_ag(b, n, in, out, K, d, x, e, h, wp_gate, bp_gate, wp_update, bp_update, scratch);
  g.HC = reinterpret_cast<float*>(stash);
  g.hout = hout;
  cudaStream_t st = (cudaStream_t)stream;
  k_agcrn_support<<<ceil_div((int)n, kSupRows), kThreads, 0, st>>>(g);
  STMP_LAUNCH_OK("k_agcrn_support");
  int rc;
  if (K == 3 && (rc = gemm<OpT2>(g, n, n, 1, st))) return rc;
  const int64_t kci = K * (in + out);
  if ((rc = gemm<OpNodeW>(g, n, (kci + 1) * 2 * out, 2, st))) return rc;
  if ((rc = gemm<OpSup<0>>(g, g.Kt * n, in + out, b, st))) return rc;
  if ((rc = gemm<OpCon<0>>(g, b, 2 * out, n, st))) return rc;
  if ((rc = gemm<OpSup<1>>(g, g.Kt * n, out, b, st))) return rc;
  return gemm<OpCon<1>>(g, b, out, n, st);
}

extern "C" int stmp_agcrn_bwd(int64_t b, int64_t n, int64_t in, int64_t out, int64_t K, int64_t d, const float* x, const float* e,
                              const float* h, const float* wp_gate, const float* bp_gate, const float* wp_update, const float* bp_update,
                              void* scratch, void* stash, const float* gh, void* workspace, float* dx, float* dh, float* de,
                              float* dwp_gate, float* dbp_gate, float* dwp_update, float* dbp_update, void* stream) {
  const char* fn = "stmp_agcrn_bwd";
  if (int rc = check_args(fn, b, n, in, out, K, d)) return rc;
  STMP_REQUIRE(e && wp_gate && bp_gate && wp_update && bp_update && (b == 0 || (x && scratch && stash && gh && workspace)), STMP_EINVAL,
               "%s: NULL tensor", fn);
  const void* ps[] = {x, e, h, wp_gate, bp_gate, wp_update, bp_update, scratch, stash, gh, workspace, dx, dh, de, dwp_gate, dbp_gate,
                      dwp_update, dbp_update};
  for (const void* q : ps) STMP_REQUIRE(rows::al4(q), STMP_ESHAPE, "%s: misaligned tensor", fn);
  const bool pools = dwp_gate || dbp_gate || dwp_update || dbp_update;
  if (b == 0) {                              // no rows: every gradient is a zero sum (cudaMemsetAsync is not a kernel launch)
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t kci = K * (in + out);
    float* zs[] = {de, dwp_gate, dbp_gate, dwp_update, dbp_update};
    const int64_t ns[] = {n * d, d * kci * 2 * out, d * 2 * out, d * kci * out, d * out};
    for (int i = 0; i < 5; ++i)
      if (zs[i]) STMP_CUDA_OK(cudaMemsetAsync(zs[i], 0, 4 * ns[i], st));
    return STMP_OK;
  }
  Ag g = make_ag(b, n, in, out, K, d, x, e, h, wp_gate, bp_gate, wp_update, bp_update, scratch);
  g.HC = reinterpret_cast<float*>(stash);
  g.gh = gh;
  const Sizes s = sizes(b, n, in, out, K);
  float* p = reinterpret_cast<float*>(workspace);
  g.dU = p; p += s.dU;
  g.dG = p; p += s.dG;
  g.dF[0] = p; p += s.dF0;
  g.dF[1] = p; p += s.dF1;
  g.dY2 = p; p += s.dY2;
  g.dW[0] = p; p += s.dW0;
  g.dW[1] = p; p += s.dW1;
  g.dT = p; p += s.dT;
  g.dS = p; p += s.dS;
  g.dA = p; p += s.dA;
  g.part = p;
  g.dx = dx; g.dh = dh; g.de = de;
  g.dwp[0] = dwp_gate; g.dbp[0] = dbp_gate; g.dwp[1] = dwp_update; g.dbp[1] = dbp_update;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t Ci = in + out, kci = K * Ci, BNo = b * n * out;
  int rc;
  k_agcrn_pw_update<<<pw_grid(BNo), kThreads, 0, st>>>(g);
  STMP_LAUNCH_OK("k_agcrn_pw_update");
  if ((rc = gemm<OpDF<1>>(g, b, kci, n, st))) return rc;
  if ((pools || de) && (rc = gemm<OpDW<1>>(g, kci + 1, out, n, st))) return rc;
  if ((rc = gemm<OpSupT<1>>(g, n, Ci, b, st))) return rc;
  k_agcrn_pw_gate<<<pw_grid(BNo), kThreads, 0, st>>>(g);
  STMP_LAUNCH_OK("k_agcrn_pw_gate");
  if ((pools || de) && (rc = gemm<OpDW<0>>(g, kci + 1, 2 * out, n, st))) return rc;
  if (dx || dh || de) {
    if ((rc = gemm<OpDF<0>>(g, b, kci, n, st))) return rc;
    if ((dx || dh) && (rc = gemm<OpSupT<0>>(g, n, Ci, b, st))) return rc;
  }
  if (pools && (rc = gemm<OpDPool>(g, d, (kci + 1) * 2 * out, 2, st))) return rc;
  if (!de) return STMP_OK;
  if ((rc = gemm_split<OpDT>(g, n, n, g.Kt, b * 2 * Ci, st))) return rc;
  if (K == 3 && (rc = gemm<OpDS>(g, n, n, 1, st))) return rc;
  k_agcrn_softmax_bwd<<<ceil_div((int)n, kSupRows), kThreads, 0, st>>>(g);
  STMP_LAUNCH_OK("k_agcrn_softmax_bwd");
  return gemm_split<OpDE>(g, n, d, 1, (kci + 1) * 3 * out + n, st);
}
