// dcrnn_narrow.cu -- the DCRNN recurrence for narrow states (cout <= 4, cin <= 4, K <= 4): forward and backward, each one
// persistent launch.  This is the model every index-batching script of the reference trains, BatchedDCRNN(F, F, K=3) with F = 1 or 2
// (examples/indexBatching/DCRNN/pems_ddp.py:81); the hidden-32 kernels (dcrnn_seq.cu, dcrnn_seq_tc.cu) cannot be narrowed to it.
//
// Layout (both kernels):
//  * a CTA serves P windows at once ("packing"): row n of every shared-memory state buffer holds the P windows' C = cin + cout
//    channels side by side, each padded to CP = 4 or 8 floats, so one gather of a source row serves all P windows (the diffusion is
//    linear and shares one operator).  Row pitch PW = P * CP.  P is chosen at launch (choose_pack); the grid is persistent over the
//    ceil(B / P) window groups.
//  * a thread owns whole (node, window) tasks -- task = n * P + p -- for all T steps, and does every multiply-add of its task in the
//    same order whatever P is, so the results do not depend on the launch shape.  Pad channels are never folded into a result.
//  * both operators live in shared memory as stage_graph builds them (dcrnn_common.cuh): padded (src * PW, val) entries per task.
//
// Forward, per step: U = [X_t | H]; the pre-activations of z | r start from block 0 (U @ (W[0,0] + W[1,0])) and every diffusion hop
// T_k,o (k = 1: P_o U; k >= 2: 2 P_o T_{k-1},o - U, dcrnn.py:80,106) is folded into them as soon as it is produced: only T_{k-1} of
// both operators is kept (two ping-pong pairs of [N][PW] buffers), never the (2K-1)-block basis.  The candidate repeats this on
// [X_t | H * R].  Contraction and gates in fp32 FFMA; the stash (Z, R, H~) of every step feeds the backward.
//
// Backward, per step in reverse (the algebra of the per-step branch of _DcrnnSeqFn.backward: gru_bwd_carry, adjoint_inplace,
// gru_bwd_zr): dph -> dS2 = dph Whs^T block by block, the adjoint of the K-hop basis through the transposed operators (again only the
// running block of each operator in shared memory), z/r derivatives, dS1 = dpzr Wzr^T and its adjoint, dL/dH_{t-1} and dX_t.
// dL/dH stays in registers of the owning thread; the d pre-activations are written out for the weight-gradient contraction.
#include "common.cuh"
#include "dcrnn_common.cuh"

namespace stmp {
namespace {

constexpr int kNarrowThreads = 256;
constexpr int kMaxSmemNarrow = 232448;  // 227 KB opt-in limit per CTA on sm_90
constexpr int kMaxPack = 8;

inline long long align_up_n(long long v, long long a) { return (v + a - 1) / a * a; }

struct NarrowLayout {
  int N, CIN, COUT, K, CP, P, PW, NB;
  int nbuf;                 // [N][PW] state buffers
  int off_buf, off_W, off_bias, off_gstart, off_order, off_ce;
  int smem_bytes;
  int tpt;                  // tasks per thread: 1, 2, 4 (forward) / 1, 2 (backward)
};

// Shared-memory carve-up for P packed windows; false if it does not fit or the tasks exceed the thread capacity (N * P <= 1024 in the
// forward, <= 512 in the backward).  Sizes are summed in 64 bits: an edge count is not bounded by N (duplicate edges are legal).
bool narrow_layout(const stmp_plan* plan, const Csr* ops, int cin, int cout, int K, int P, bool bwd, NarrowLayout* L) {
  L->N = plan->n; L->CIN = cin; L->COUT = cout; L->K = K; L->P = P;
  L->CP = (cin + cout) <= 4 ? 4 : 8;
  L->PW = P * L->CP;
  L->NB = 2 * K - 1;
  L->nbuf = bwd ? 4 : 5;
  const long long C = cin + cout, N = L->N;
  long long off = 0, o[6];
  o[0] = off; off += align_up_n(L->nbuf * N * L->PW * 4, 128);
  // forward: W[(blk*C + c)][z | r | h] (3 cout columns); backward: Whs^T (cout rows) | Wzr^T (2 cout rows) of (2K-1) C columns
  o[1] = off; off += align_up_n(L->NB * C * 3 * cout * 4, 16);
  o[2] = off; off += align_up_n(3LL * cout * 4, 16);
  o[3] = off; off += align_up_n((2 * N + 1) * 4, 16);
  o[4] = off; off += align_up_n(2 * N * 4, 16);
  o[5] = off; off += align_up_n(((long long)ops[0].nnz + ops[1].nnz + 6 * N + 4) * 8, 16);
  const long long tasks = N * P;
  const int max_tpt = bwd ? 2 : 4;         // the backward's registers hold two tasks without spilling
  L->tpt = tasks <= kNarrowThreads ? 1 : (tasks <= 2 * kNarrowThreads ? 2 : 4);
  if (off > kMaxSmemNarrow || tasks > (long long)max_tpt * kNarrowThreads) return false;
  L->off_buf = (int)o[0]; L->off_W = (int)o[1]; L->off_bias = (int)o[2];
  L->off_gstart = (int)o[3]; L->off_order = (int)o[4]; L->off_ce = (int)o[5];
  L->smem_bytes = (int)off;
  return true;
}

// Per-pack launch counters ("k_dcrnn_narrow_seq[pack P]"), so callers and tests can see the launch shape that served a call.
void count_pack(bool bwd, int P) {
  static const char* const kFwd[kMaxPack] = {"k_dcrnn_narrow_seq[pack 1]", "k_dcrnn_narrow_seq[pack 2]", "k_dcrnn_narrow_seq[pack 3]",
                                             "k_dcrnn_narrow_seq[pack 4]", "k_dcrnn_narrow_seq[pack 5]", "k_dcrnn_narrow_seq[pack 6]",
                                             "k_dcrnn_narrow_seq[pack 7]", "k_dcrnn_narrow_seq[pack 8]"};
  static const char* const kBwd[kMaxPack] = {"k_dcrnn_narrow_bwd[pack 1]", "k_dcrnn_narrow_bwd[pack 2]", "k_dcrnn_narrow_bwd[pack 3]",
                                             "k_dcrnn_narrow_bwd[pack 4]", "k_dcrnn_narrow_bwd[pack 5]", "k_dcrnn_narrow_bwd[pack 6]",
                                             "k_dcrnn_narrow_bwd[pack 7]", "k_dcrnn_narrow_bwd[pack 8]"};
  struct Slots { int s[2][kMaxPack]; };
  static const Slots slots = [] {     // registered once (thread-safe static initialisation)
    Slots r;
    for (int i = 0; i < kMaxPack; ++i) { r.s[0][i] = path_slot(kFwd[i]); r.s[1][i] = path_slot(kBwd[i]); }
    return r;
  }();
  count_path(slots.s[bwd ? 1 : 0][P - 1]);
}

bool narrow_shape_ok(const stmp_plan* plan, long long cin, long long cout, long long K) {
  if (!plan || plan->flavor != STMP_FLAVOR_DCONV || plan->n_ops != 2) return false;
  return cout >= 1 && cout <= 4 && cin >= 1 && cin <= 4 && K >= 1 && K <= 4;
}

// Windows per CTA: the option "dcrnn_narrow_pack" (> 0) or, automatically, the largest P <= 8 that still gives every SM a CTA
// (P = 1 at the reference's batch of 64); then lowered until the layout fits, which includes the thread capacity N * P <= 1024
// (forward) / 512 (backward): at 1056 windows on 132 SMs METR-LA runs P = 4 forward and 2 backward, PEMS-BAY P = 3 and 1.
// 0 = not even P = 1 fits.
int choose_pack(const stmp_plan* plan, const Csr* ops, long long B, int cin, int cout, int K, bool bwd, int sms, NarrowLayout* L) {
  int P = g_narrow_pack > 0 ? g_narrow_pack : (int)(B / (sms > 0 ? sms : 1));
  if (P > kMaxPack) P = kMaxPack;
  if (P < 1) P = 1;
  for (; P >= 1; --P)
    if (narrow_layout(plan, ops, cin, cout, K, P, bwd, L)) return P;
  return 0;
}

// Per-CTA graph staging shared by both kernels.
struct GraphArgs {
  const int* rp[2];
  const int2* cv[2];
};

// ============================================================================================================================
// forward
// ============================================================================================================================
struct NarrowFwdParams {
  NarrowLayout L;
  int T;
  long long B, G;           // windows, window groups (ceil(B / P))
  GraphArgs g;
  const float* x;
  const long long* win_start;
  long long x_bstride, x_tstride;
  const float* w[3];
  const float* bias[3];
  const float* h0;
  float* out;
  float* stash;
};

// v[c] (c < CP) of the task's row in block `src` gathered through operator `op`: one gather_row per float4
template <int CP>
__device__ __forceinline__ void gather_task(const float* src, const GraphSmem& g, int N, int op, int n, int coff, float (&v)[CP]) {
  const int task = op * N + n;
  const int beg = g.gstart[task], end = g.gstart[task + 1];
#pragma unroll
  for (int q = 0; q < CP / 4; ++q) {
    const float4 a = gather_row(src + coff + 4 * q, g.ce, beg, end);
    v[4 * q] = a.x; v[4 * q + 1] = a.y; v[4 * q + 2] = a.z; v[4 * q + 3] = a.w;
  }
}

// acc[q] += sum_{c < C} v[c] * W[(row0 + c) * WLD + col0 + q]   (c ascending: the fold order of every block)
template <int CP, int NQ>
__device__ __forceinline__ void fold(const float (&v)[CP], int C, const float* W, int row0, int WLD, int col0, float (&acc)[NQ]) {
#pragma unroll
  for (int c = 0; c < CP; ++c) {
    if (c < C) {
      const float* w = W + (row0 + c) * WLD + col0;
#pragma unroll
      for (int q = 0; q < NQ; ++q) acc[q] = fmaf(v[c], w[q], acc[q]);
    }
  }
}

template <int CP>
__device__ __forceinline__ void ld_row(const float* p, float (&v)[CP]) {
#pragma unroll
  for (int q = 0; q < CP / 4; ++q) {
    const float4 a = ld4(p + 4 * q);
    v[4 * q] = a.x; v[4 * q + 1] = a.y; v[4 * q + 2] = a.z; v[4 * q + 3] = a.w;
  }
}
template <int CP>
__device__ __forceinline__ void st_row(float* p, const float (&v)[CP]) {
#pragma unroll
  for (int q = 0; q < CP / 4; ++q) st4(p + 4 * q, make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]));
}

// One diffusion round of the forward: acc (NQ columns of W starting at col0) += U @ W_blk0 + sum_k (T_k,o @ W_blk(k,o)), folded hop by
// hop.  U is already in place; ends behind a block barrier once the last hop's gathers are done (or with no barrier when K = 1: nothing
// crossed rows).  `pp` is the ping-pong index, carried across rounds.
template <int CP, int TPT, int NQ>
__device__ __forceinline__ void fwd_round(const NarrowLayout& L, const GraphSmem& gs, float* U, const float* W, int col0,
                                          float (&acc)[TPT][NQ], int tid) {
  const int N = L.N, P = L.P, PW = L.PW, C = L.CIN + L.COUT, K = L.K, WLD = 3 * L.COUT, NPW = N * PW;
  // T buffers follow U: [1 + 2 * set + op] * NPW, set = ping-pong index
#pragma unroll
  for (int j = 0; j < TPT; ++j) {
    const int task = tid + j * kNarrowThreads;
    if (task < N * P) {
      const int n = task / P, pw = task - n * P;
      float u[CP];
      ld_row<CP>(U + n * PW + pw * CP, u);
      fold<CP, NQ>(u, C, W, 0, WLD, col0, acc[j]);
    }
  }
  int cur = 0;
  for (int hop = 1; hop < K; ++hop) {
#pragma unroll
    for (int j = 0; j < TPT; ++j) {
      const int task = tid + j * kNarrowThreads;
      if (task < N * P) {
        const int n = task / P, pw = task - n * P, coff = pw * CP;
        float u[CP];
        if (hop >= 2) ld_row<CP>(U + n * PW + coff, u);
#pragma unroll
        for (int op = 0; op < 2; ++op) {
          float v[CP];
          gather_task<CP>(hop == 1 ? U : U + (1 + 2 * (cur ^ 1) + op) * NPW, gs, N, op, n, coff, v);
          if (hop >= 2) {
#pragma unroll
            for (int c = 0; c < CP; ++c) v[c] = 2.0f * v[c] - u[c];
          }
          st_row<CP>(U + (1 + 2 * cur + op) * NPW + n * PW + coff, v);
          fold<CP, NQ>(v, C, W, (1 + 2 * (hop - 1) + op) * C, WLD, col0, acc[j]);
        }
      }
    }
    __syncthreads();
    cur ^= 1;
  }
}

template <int COUT, int CP, int TPT>
__global__ void __launch_bounds__(kNarrowThreads, 1) k_dcrnn_narrow_seq(const NarrowFwdParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr int NT = kNarrowThreads;
  const NarrowLayout& L = p.L;
  const int tid = threadIdx.x;
  const int N = L.N, CIN = L.CIN, C = CIN + COUT, K = L.K, T = p.T, P = L.P, PW = L.PW, NB = L.NB;
  constexpr int WLD = 3 * COUT;
  float* U = reinterpret_cast<float*>(smem + L.off_buf);
  float* W = reinterpret_cast<float*>(smem + L.off_W);
  float* Bs = reinterpret_cast<float*>(smem + L.off_bias);
  int2* s_ce = reinterpret_cast<int2*>(smem + L.off_ce);
  int* s_gstart = reinterpret_cast<int*>(smem + L.off_gstart);
  int* s_order = reinterpret_cast<int*>(smem + L.off_order);
  if (blockIdx.x >= p.G) return;

  stage_graph<NT>(p.g.rp[0], p.g.rp[1], p.g.cv[0], p.g.cv[1], N, PW, s_ce, s_gstart, s_order, tid);
  const GraphSmem gs{s_ce, s_gstart, s_order};
  // stacked weights, reference channel order [X | H]: block 0 = W[0,0] + W[1,0], block 1 + 2(k-1) + o = W[o,k]
  for (int idx = tid; idx < NB * C * WLD; idx += NT) {
    const int row = idx / WLD, col = idx - row * WLD;
    const int blk = row / C, ch = row - blk * C;
    const int gt = col / COUT, o = col - gt * COUT;
    const float* wg = p.w[gt];
    float v;
    if (blk == 0) v = wg[((0 * K + 0) * C + ch) * COUT + o] + wg[((1 * K + 0) * C + ch) * COUT + o];
    else v = wg[(((blk - 1) & 1) * K + 1 + (blk - 1) / 2) * C * COUT + ch * COUT + o];
    W[idx] = v;
  }
  for (int idx = tid; idx < WLD; idx += NT) {
    const int gt = idx / COUT;
    Bs[idx] = p.bias[gt] ? p.bias[gt][idx - gt * COUT] : 0.f;
  }
  for (int idx = tid; idx < L.nbuf * N * PW; idx += NT) U[idx] = 0.f;    // pad channels stay zero
  __syncthreads();

  for (long long grp = blockIdx.x; grp < p.G; grp += gridDim.x) {
    float h[TPT][COUT], xn[TPT][4];
    long long bw[TPT];
#pragma unroll
    for (int j = 0; j < TPT; ++j) {
      const int task = tid + j * NT;
      const int n = task / P, pw = task - n * P;
      const long long b = grp * P + pw;
      bw[j] = (task < N * P && b < p.B) ? b : -1;
      const float* xb = bw[j] >= 0 ? p.x + (p.win_start ? p.win_start[b] * p.x_tstride : b * p.x_bstride) + (long long)n * CIN : nullptr;
#pragma unroll
      for (int o = 0; o < COUT; ++o) h[j][o] = (bw[j] >= 0 && p.h0) ? __ldg(p.h0 + (b * N + n) * COUT + o) : 0.f;
#pragma unroll
      for (int c = 0; c < 4; ++c) xn[j][c] = (xb && c < CIN) ? __ldg(xb + c) : 0.f;
    }
    for (int t = 0; t < T; ++t) {
      // U = [X_t | H] (own rows; every cross-row read of U ended behind the previous round's barriers)
#pragma unroll
      for (int j = 0; j < TPT; ++j) {
        const int task = tid + j * NT;
        if (task < N * P) {
          const int n = task / P, pw = task - n * P;
          float* u = U + n * PW + pw * CP;
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (c < CIN) u[c] = xn[j][c];
#pragma unroll
          for (int o = 0; o < COUT; ++o) u[CIN + o] = h[j][o];
        }
      }
      // prefetch X_{t+1} while this step computes
#pragma unroll
      for (int j = 0; j < TPT; ++j) {
        if (bw[j] >= 0 && t + 1 < T) {
          const int n = (tid + j * NT) / P;
          const long long b = bw[j];
          const float* xb = p.x + (p.win_start ? p.win_start[b] * p.x_tstride : b * p.x_bstride) + (t + 1) * p.x_tstride + (long long)n * CIN;
#pragma unroll
          for (int c = 0; c < 4; ++c) xn[j][c] = c < CIN ? __ldg(xb + c) : 0.f;
        }
      }
      __syncthreads();
      // ---- z | r: diffusion of [X | H] folded hop by hop
      float acc[TPT][2 * COUT];
#pragma unroll
      for (int j = 0; j < TPT; ++j)
#pragma unroll
        for (int q = 0; q < 2 * COUT; ++q) acc[j][q] = 0.f;
      fwd_round<CP, TPT, 2 * COUT>(L, gs, U, W, 0, acc, tid);
      float z[TPT][COUT];
#pragma unroll
      for (int j = 0; j < TPT; ++j) {
        const int task = tid + j * NT;
        if (task < N * P) {
          const int n = task / P, pw = task - n * P;
          float r[COUT];
#pragma unroll
          for (int o = 0; o < COUT; ++o) {
            z[j][o] = sigmoidf_acc(acc[j][o] + Bs[o]);
            r[o] = sigmoidf_acc(acc[j][COUT + o] + Bs[COUT + o]);
          }
          float* u = U + n * PW + pw * CP;           // own row only: the gathers of U ended behind the last hop's barrier
#pragma unroll
          for (int o = 0; o < COUT; ++o) u[CIN + o] = h[j][o] * r[o];
          if (bw[j] >= 0 && p.stash) {
            float* sp = p.stash + ((bw[j] * T + t) * 3 * N + n) * COUT;
#pragma unroll
            for (int o = 0; o < COUT; ++o) { sp[o] = z[j][o]; sp[(long long)N * COUT + o] = r[o]; }
          }
        }
      }
      __syncthreads();
      // ---- candidate: diffusion of [X | H * R]
      float acch[TPT][COUT];
#pragma unroll
      for (int j = 0; j < TPT; ++j)
#pragma unroll
        for (int q = 0; q < COUT; ++q) acch[j][q] = 0.f;
      fwd_round<CP, TPT, COUT>(L, gs, U, W, 2 * COUT, acch, tid);
#pragma unroll
      for (int j = 0; j < TPT; ++j) {
        if ((tid + j * NT) < N * P) {
          const int n = (tid + j * NT) / P;
          float ht[COUT];
#pragma unroll
          for (int o = 0; o < COUT; ++o) {
            ht[o] = tanhf(acch[j][o] + Bs[2 * COUT + o]);
            h[j][o] = z[j][o] * h[j][o] + (1.0f - z[j][o]) * ht[o];   // dcrnn.py:190-192
          }
          if (bw[j] >= 0) {
            const long long row = (bw[j] * T + t) * N + n;
#pragma unroll
            for (int o = 0; o < COUT; ++o) p.out[row * COUT + o] = h[j][o];
            if (p.stash) {
              float* sp = p.stash + ((bw[j] * T + t) * 3 * N + 2 * (long long)N + n) * COUT;
#pragma unroll
              for (int o = 0; o < COUT; ++o) sp[o] = ht[o];
            }
          }
        }
      }
    }
  }
}

// ============================================================================================================================
// backward
// ============================================================================================================================
struct NarrowBwdParams {
  NarrowLayout L;
  int T;
  long long B, G;
  GraphArgs g;              // transposed operators (by source)
  const float* gout; const float* out; const float* h0; const float* stash;
  const float* whsT; const float* wzrT;     // (cout, (2K-1)C), (2cout, (2K-1)C)
  float* dph_all; float* dpzr_all;          // (T,B,N,cout), (T,B,N,2cout)
  float* dx;                                // (B,T,N,cin) or null
  float* dh0;                               // (B,N,cout)
};

// v[i] for a run-time i < CP, without indexing the register array dynamically (which would put it in local memory)
template <int CP>
__device__ __forceinline__ float pick(const float (&v)[CP], int i) {
  float r = v[0];
#pragma unroll
  for (int c = 1; c < CP; ++c) r = i == c ? v[c] : r;
  return r;
}

// dS[c] of basis block `blk` for d pre-activations dp (NQ of them): sum_q dp[q] * WT[q][blk*C + c]  (q ascending)
template <int CP, int NQ>
__device__ __forceinline__ void dS_block(const float (&dp)[NQ], const float* WT, int nbC, int C, int blk, float (&v)[CP]) {
#pragma unroll
  for (int c = 0; c < CP; ++c) {
    float a = 0.f;
    if (c < C) {
#pragma unroll
      for (int q = 0; q < NQ; ++q) a = fmaf(dp[q], WT[q * nbC + blk * C + c], a);
    }
    v[c] = a;
  }
}

// dU = adjoint of U -> [U | P_o U | P_i U | 2 P_o T_1o - U | ...] applied to dS = dp @ W^T, for every task of the thread (the order of
// adjoint_inplace in nn/recurrent/dcrnn.py: hops K-1 .. 2, operator 0 then 1, then the first hop).  Starts with no cross-row reads pending
// on D; ends behind a block barrier.
template <int CP, int TPT, int NQ>
__device__ __forceinline__ void bwd_adjoint(const NarrowLayout& L, const GraphSmem& gs, float* D, const float (&dp)[TPT][NQ],
                                            const float* WT, float (&dU)[TPT][CP], int tid) {
  const int N = L.N, P = L.P, PW = L.PW, C = L.CIN + L.COUT, K = L.K, nbC = L.NB * C, NPW = N * PW;
  // running block of operator op in ping-pong set s: D + (2 * s + op) * NPW
#pragma unroll
  for (int j = 0; j < TPT; ++j) {
    const int task = tid + j * kNarrowThreads;
    if (task < N * P) {
      const int n = task / P, pw = task - n * P, coff = pw * CP;
      dS_block<CP, NQ>(dp[j], WT, nbC, C, 0, dU[j]);
      if (K > 1) {
#pragma unroll
        for (int op = 0; op < 2; ++op) {
          float v[CP];
          dS_block<CP, NQ>(dp[j], WT, nbC, C, 1 + 2 * (K - 2) + op, v);
          st_row<CP>(D + op * NPW + n * PW + coff, v);
        }
      }
    }
  }
  if (K == 1) return;
  __syncthreads();
  int cur = 0;
  for (int k = K - 1; k >= 2; --k) {                  // d[k-1,o] += 2 P_o^T d[k,o];  d0 -= d[k,o]
#pragma unroll
    for (int j = 0; j < TPT; ++j) {
      const int task = tid + j * kNarrowThreads;
      if (task < N * P) {
        const int n = task / P, pw = task - n * P, coff = pw * CP;
#pragma unroll
        for (int op = 0; op < 2; ++op) {
          float v[CP], s[CP], dk[CP];
          const float* Dc = D + (2 * cur + op) * NPW;
          gather_task<CP>(Dc, gs, N, op, n, coff, v);
          dS_block<CP, NQ>(dp[j], WT, nbC, C, 1 + 2 * (k - 2) + op, s);
          ld_row<CP>(Dc + n * PW + coff, dk);
#pragma unroll
          for (int c = 0; c < CP; ++c) {
            v[c] = fmaf(2.0f, v[c], s[c]);
            dU[j][c] = dU[j][c] - dk[c];
          }
          st_row<CP>(D + (2 * (cur ^ 1) + op) * NPW + n * PW + coff, v);
        }
      }
    }
    __syncthreads();
    cur ^= 1;
  }
#pragma unroll
  for (int j = 0; j < TPT; ++j) {                     // d0 += P_0^T d[1,0];  d0 += P_1^T d[1,1]
    const int task = tid + j * kNarrowThreads;
    if (task < N * P) {
      const int n = task / P, pw = task - n * P, coff = pw * CP;
#pragma unroll
      for (int op = 0; op < 2; ++op) {
        float v[CP];
        gather_task<CP>(D + (2 * cur + op) * NPW, gs, N, op, n, coff, v);
#pragma unroll
        for (int c = 0; c < CP; ++c) dU[j][c] = v[c] + dU[j][c];
      }
    }
  }
  __syncthreads();   // no gather of D is pending when the next adjoint writes its first blocks
}

template <int COUT, int CP, int TPT>
__global__ void __launch_bounds__(kNarrowThreads, 1) k_dcrnn_narrow_bwd(const NarrowBwdParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr int NT = kNarrowThreads;
  const NarrowLayout& L = p.L;
  const int tid = threadIdx.x;
  const int N = L.N, CIN = L.CIN, C = CIN + COUT, T = p.T, P = L.P, PW = L.PW, nbC = L.NB * C;
  const long long NH = (long long)N * COUT;
  float* buf = reinterpret_cast<float*>(smem + L.off_buf);
  float* Whs = reinterpret_cast<float*>(smem + L.off_W);
  float* Wzr = Whs + COUT * nbC;
  int2* s_ce = reinterpret_cast<int2*>(smem + L.off_ce);
  int* s_gstart = reinterpret_cast<int*>(smem + L.off_gstart);
  int* s_order = reinterpret_cast<int*>(smem + L.off_order);
  if (blockIdx.x >= p.G) return;

  stage_graph<NT>(p.g.rp[0], p.g.rp[1], p.g.cv[0], p.g.cv[1], N, PW, s_ce, s_gstart, s_order, tid);
  const GraphSmem gs{s_ce, s_gstart, s_order};
  for (int i = tid; i < COUT * nbC; i += NT) Whs[i] = __ldg(p.whsT + i);
  for (int i = tid; i < 2 * COUT * nbC; i += NT) Wzr[i] = __ldg(p.wzrT + i);
  for (int i = tid; i < L.nbuf * N * PW; i += NT) buf[i] = 0.f;
  __syncthreads();

  for (long long grp = blockIdx.x; grp < p.G; grp += gridDim.x) {
    float dh[TPT][COUT];                              // dL/dH_t carried from step t+1 (zero at the last step)
    long long bw[TPT];
#pragma unroll
    for (int j = 0; j < TPT; ++j) {
      const int task = tid + j * NT;
      const int n = task / P, pw = task - n * P;
      const long long b = grp * P + pw;
      bw[j] = (task < N * P && b < p.B) ? b : -1;
      (void)n;
#pragma unroll
      for (int o = 0; o < COUT; ++o) dh[j][o] = 0.f;
    }
    for (int t = T - 1; t >= 0; --t) {
      // ---- open step t: g = gout_t + dH,  dph = g (1-Z)(1-Ht^2)
      float g[TPT][COUT], z[TPT][COUT], dph[TPT][COUT];
#pragma unroll
      for (int j = 0; j < TPT; ++j) {
        const int n = (tid + j * NT) / P;
        const long long b = bw[j];
#pragma unroll
        for (int o = 0; o < COUT; ++o) {
          float go = 0.f, zz = 0.f, hh = 0.f;
          if (b >= 0) {
            const long long bt = b * T + t;
            go = __ldg(p.gout + bt * NH + n * COUT + o);
            zz = __ldg(p.stash + bt * 3 * NH + n * COUT + o);
            hh = __ldg(p.stash + bt * 3 * NH + 2 * NH + n * COUT + o);
          }
          g[j][o] = go + dh[j][o];
          z[j][o] = zz;
          dph[j][o] = g[j][o] * (1.f - zz) * (1.f - hh * hh);
        }
        if (b >= 0) {
          float* d = p.dph_all + ((long long)t * p.B + b) * NH + n * COUT;
#pragma unroll
          for (int o = 0; o < COUT; ++o) d[o] = dph[j][o];
        }
      }
      // ---- dU2 = adjoint(dph Whs^T)
      float dU2[TPT][CP];
      bwd_adjoint<CP, TPT, COUT>(L, gs, buf, dph, Whs, dU2, tid);
      // ---- z / r: dpz = g (H_{t-1} - Ht) Z (1-Z),  dpr = dHR H_{t-1} R (1-R)
      float dpzr[TPT][2 * COUT], r[TPT][COUT];
#pragma unroll
      for (int j = 0; j < TPT; ++j) {
        const int n = (tid + j * NT) / P;
        const long long b = bw[j];
#pragma unroll
        for (int o = 0; o < COUT; ++o) {
          float hp = 0.f, rr = 0.f, hh = 0.f;
          if (b >= 0) {
            const long long bt = b * T + t;
            const float* hsrc = t > 0 ? p.out + (bt - 1) * NH : (p.h0 ? p.h0 + b * NH : nullptr);
            if (hsrc) hp = __ldg(hsrc + n * COUT + o);
            rr = __ldg(p.stash + bt * 3 * NH + NH + n * COUT + o);
            hh = __ldg(p.stash + bt * 3 * NH + 2 * NH + n * COUT + o);
          }
          r[j][o] = rr;
          dpzr[j][o] = g[j][o] * (hp - hh) * z[j][o] * (1.f - z[j][o]);
          dpzr[j][COUT + o] = pick<CP>(dU2[j], CIN + o) * hp * rr * (1.f - rr);
        }
        if (b >= 0) {
          float* d = p.dpzr_all + ((long long)t * p.B + b) * 2 * NH + n * 2 * COUT;
#pragma unroll
          for (int q = 0; q < 2 * COUT; ++q) d[q] = dpzr[j][q];
        }
      }
      // ---- dU1 = adjoint(dpzr Wzr^T)
      float dU1[TPT][CP];
      bwd_adjoint<CP, TPT, 2 * COUT>(L, gs, buf, dpzr, Wzr, dU1, tid);
      // ---- close step t: dH_{t-1} = g Z + dHR R + dU1[cin:],  dX_t = dU2[:cin] + dU1[:cin]
#pragma unroll
      for (int j = 0; j < TPT; ++j) {
        const int n = (tid + j * NT) / P;
        const long long b = bw[j];
#pragma unroll
        for (int o = 0; o < COUT; ++o) dh[j][o] = g[j][o] * z[j][o] + pick<CP>(dU2[j], CIN + o) * r[j][o] + pick<CP>(dU1[j], CIN + o);
        if (b >= 0 && p.dx) {
          float* d = p.dx + ((b * T + t) * N + n) * (long long)CIN;
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (c < CIN) d[c] = dU2[j][c] + dU1[j][c];
        }
      }
    }
#pragma unroll
    for (int j = 0; j < TPT; ++j) {
      if (bw[j] >= 0) {
        const int n = (tid + j * NT) / P;
#pragma unroll
        for (int o = 0; o < COUT; ++o) p.dh0[bw[j] * NH + n * COUT + o] = dh[j][o];
      }
    }
  }
}

// ---- launch helpers ---------------------------------------------------------------------------------------------------------
template <typename KernelT, typename ParamsT>
int launch_kernel(KernelT kern, const ParamsT& p, int grid, int smem, cudaStream_t st) {
  STMP_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  kern<<<grid, kNarrowThreads, smem, st>>>(p);
  return STMP_OK;
}

template <int COUT, int CP>
int fwd_tpt(const NarrowFwdParams& p, int grid, cudaStream_t st) {
  switch (p.L.tpt) {
    case 1: return launch_kernel(k_dcrnn_narrow_seq<COUT, CP, 1>, p, grid, p.L.smem_bytes, st);
    case 2: return launch_kernel(k_dcrnn_narrow_seq<COUT, CP, 2>, p, grid, p.L.smem_bytes, st);
    default: return launch_kernel(k_dcrnn_narrow_seq<COUT, CP, 4>, p, grid, p.L.smem_bytes, st);
  }
}
template <int COUT>
int fwd_cp(const NarrowFwdParams& p, int grid, cudaStream_t st) {
  return p.L.CP == 4 ? fwd_tpt<COUT, 4>(p, grid, st) : fwd_tpt<COUT, 8>(p, grid, st);
}
template <int COUT, int CP>
int bwd_tpt(const NarrowBwdParams& p, int grid, cudaStream_t st) {
  if (p.L.tpt == 1) return launch_kernel(k_dcrnn_narrow_bwd<COUT, CP, 1>, p, grid, p.L.smem_bytes, st);
  return launch_kernel(k_dcrnn_narrow_bwd<COUT, CP, 2>, p, grid, p.L.smem_bytes, st);
}
template <int COUT>
int bwd_cp(const NarrowBwdParams& p, int grid, cudaStream_t st) {
  return p.L.CP == 4 ? bwd_tpt<COUT, 4>(p, grid, st) : bwd_tpt<COUT, 8>(p, grid, st);
}

int sm_count(int* sms) {
  int dev = 0;
  STMP_CUDA_OK(cudaGetDevice(&dev));
  STMP_CUDA_OK(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
  return STMP_OK;
}

}  // namespace

// ---- entry points used by dcrnn_seq.cu (forward) --------------------------------------------------------------------------------
bool dcrnn_narrow_supported(const stmp_plan* plan, long long cin, long long cout, long long K) {
  if (!narrow_shape_ok(plan, cin, cout, K)) return false;
  NarrowLayout L;
  return narrow_layout(plan, plan->fwd, (int)cin, (int)cout, (int)K, 1, false, &L);
}

int dcrnn_narrow_launch(const stmp_plan* plan, long long B, long long T, long long cin, long long cout, long long K, const float* x,
                        const long long* win_start, long long x_bstride, long long x_tstride, const float* w_z, const float* w_r,
                        const float* w_h, const float* b_z, const float* b_r, const float* b_h, const float* h0, float* out, float* stash,
                        cudaStream_t st) {
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc != STMP_OK) return rc;
  NarrowFwdParams p;
  if (choose_pack(plan, plan->fwd, B, (int)cin, (int)cout, (int)K, false, sms, &p.L) == 0)
    return set_error(STMP_EUNSUPPORTED, "narrow DCRNN kernel: the graph (N=%d) does not fit shared memory", plan->n);
  p.T = (int)T; p.B = B; p.G = (B + p.L.P - 1) / p.L.P;
  for (int o = 0; o < 2; ++o) { p.g.rp[o] = plan->fwd[o].rowptr; p.g.cv[o] = plan->fwd[o].cv; }
  p.x = x; p.win_start = win_start; p.x_bstride = x_bstride; p.x_tstride = x_tstride;
  p.w[0] = w_z; p.w[1] = w_r; p.w[2] = w_h;
  p.bias[0] = b_z; p.bias[1] = b_r; p.bias[2] = b_h;
  p.h0 = h0; p.out = out; p.stash = stash;
  const int grid = (int)(p.G < sms ? p.G : sms);
  int r = STMP_OK;
  switch (cout) {
    case 1: r = fwd_cp<1>(p, grid, st); break;
    case 2: r = fwd_cp<2>(p, grid, st); break;
    case 3: r = fwd_cp<3>(p, grid, st); break;
    default: r = fwd_cp<4>(p, grid, st); break;
  }
  if (r != STMP_OK) return r;
  STMP_LAUNCH_OK("k_dcrnn_narrow_seq");
  count_pack(false, p.L.P);
  return STMP_OK;
}

}  // namespace stmp

using namespace stmp;

extern "C" int stmp_dcrnn_narrow_bwd_supported(const stmp_plan* plan, int64_t cin, int64_t cout, int64_t K) {
  if (!narrow_shape_ok(plan, cin, cout, K)) return 0;
  NarrowLayout L;
  return narrow_layout(plan, plan->bwd, (int)cin, (int)cout, (int)K, 1, true, &L) ? 1 : 0;
}

extern "C" int stmp_dcrnn_narrow_bwd_seq(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K,
                                         const float* gout, const float* out, const float* h0, const float* stash, const float* whsT,
                                         const float* wzrT, float* dph_all, float* dpzr_all, float* dx, float* dh0, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_dcrnn_narrow_bwd_seq: plan is NULL");
  STMP_REQUIRE(B >= 0 && T >= 0, STMP_EINVAL, "stmp_dcrnn_narrow_bwd_seq: negative B/T");
  if (!narrow_shape_ok(plan, cin, cout, K))
    return set_error(STMP_EUNSUPPORTED, "narrow DCRNN backward supports cin, cout in 1..4 and K in 1..4 on a DConv plan (got cin=%lld cout=%lld K=%lld)",
                     (long long)cin, (long long)cout, (long long)K);
  STMP_REQUIRE(gout && out && stash && whsT && wzrT && dph_all && dpzr_all && dh0, STMP_EINVAL, "stmp_dcrnn_narrow_bwd_seq: NULL tensor");
  if (B == 0 || T == 0) return STMP_OK;
  int sms = 0;
  const int rc = sm_count(&sms);
  if (rc != STMP_OK) return rc;
  NarrowBwdParams p;
  if (choose_pack(plan, plan->bwd, B, (int)cin, (int)cout, (int)K, true, sms, &p.L) == 0)
    return set_error(STMP_EUNSUPPORTED, "narrow DCRNN backward: the graph (N=%d) does not fit shared memory", plan->n);
  p.T = (int)T; p.B = B; p.G = (B + p.L.P - 1) / p.L.P;
  for (int o = 0; o < 2; ++o) { p.g.rp[o] = plan->bwd[o].rowptr; p.g.cv[o] = plan->bwd[o].cv; }
  p.gout = gout; p.out = out; p.h0 = h0; p.stash = stash; p.whsT = whsT; p.wzrT = wzrT;
  p.dph_all = dph_all; p.dpzr_all = dpzr_all; p.dx = dx; p.dh0 = dh0;
  const int grid = (int)(p.G < sms ? p.G : sms);
  cudaStream_t st = (cudaStream_t)stream;
  int r = STMP_OK;
  switch (cout) {
    case 1: r = bwd_cp<1>(p, grid, st); break;
    case 2: r = bwd_cp<2>(p, grid, st); break;
    case 3: r = bwd_cp<3>(p, grid, st); break;
    default: r = bwd_cp<4>(p, grid, st); break;
  }
  if (r != STMP_OK) return r;
  STMP_LAUNCH_OK("k_dcrnn_narrow_bwd");
  count_pack(true, p.L.P);
  return STMP_OK;
}
