// dcrnn_bwd.cu -- backward of the fused DCRNN sequence for graphs that fit one SM's shared memory (K = 2, 32 hidden).
//
// What autograd would replay for BatchedDCRNN.forward (torch_geometric_temporal/nn/recurrent/dcrnn.py:429-475, cell
// :172-219) is a reverse-time recurrence on dL/dH.  Two kernels:
//
//   k_dcrnn_bwd_basis  one CTA per (t, window): rebuilds S1 = [U | P_o U | P_i U] for U = [X_t | H_{t-1}] and
//                      S2 for U = [X_t | H_{t-1} * R_t] from the forward outputs and the gate stash -- the
//                      operands of the weight-gradient contractions, which do NOT depend on the recurrence
//                      and are therefore done for all steps at once (two GEMMs over all (t,b,n) rows).
//   k_dcrnn_bwd_seq    one CTA per window, persistent over the T steps in reverse: per step
//                        dS2 = dpre_h @ Wh^T            (FFMA, operands in shared memory)
//                        dU2 = adjoint of the basis     (transposed-CSR gather out of shared memory)
//                        gate derivatives (z, r)        (pointwise, stash read from global)
//                        dS1 = dpre_zr @ Wzr^T ; dU1 = adjoint ; dH_{t-1}, dX_t
//                      dL/dH never leaves shared memory; d pre-activations are streamed out for the weight GEMMs.
//
// Everything here is fp32 FFMA: the per-window GEMMs are 207x32x102 / 207x64x102, the problem is latency-bound on
// the serial recurrence with 64 windows per step (the reference's batch size), not throughput-bound.
#include "dcrnn_common.cuh"

namespace stmp {
namespace {

constexpr int kCo = 32;          // hidden size served by these kernels
constexpr int kBwdThreads = 512;
constexpr int kBatch = 4;        // vector slots per thread whose global operands are fetched together (latency paid once)
// dynamic shared memory a k_dcrnn_bwd_seq block may request: the 227 KB opt-in limit covers static shared memory too, and the
// cluster-pair variant's static mbarrier (dbar) takes 16 bytes (8, padded to the dynamic block's alignment; cuobjdump -res-usage)
constexpr size_t kBwdSmemMax = 227 * 1024 - 16;

// basis width [U | Op_0 U | .. | Op_{nops-1} U], U = [X | H], rounded up to whole 8-column groups
__host__ __device__ constexpr int ncol_of(int cin, int nops = 2) { return ((nops + 1) * (cin + kCo) + 7) / 8 * 8; }

// ---- 1- or 2-float vector access (rows have C = cin + 32 channels; C even -> float2 slots halve the instruction count)
template <int V> __device__ __forceinline__ void ldv(const float* p, float (&v)[V]);
template <> __device__ __forceinline__ void ldv<1>(const float* p, float (&v)[1]) { v[0] = *p; }
template <> __device__ __forceinline__ void ldv<2>(const float* p, float (&v)[2]) { const float2 t = *reinterpret_cast<const float2*>(p); v[0] = t.x; v[1] = t.y; }
template <int V> __device__ __forceinline__ void ldgv(const float* p, float (&v)[V]);
template <> __device__ __forceinline__ void ldgv<1>(const float* p, float (&v)[1]) { v[0] = __ldg(p); }
template <> __device__ __forceinline__ void ldgv<2>(const float* p, float (&v)[2]) { const float2 t = __ldg(reinterpret_cast<const float2*>(p)); v[0] = t.x; v[1] = t.y; }
template <int V> __device__ __forceinline__ void stv(float* p, const float (&v)[V]);
template <> __device__ __forceinline__ void stv<1>(float* p, const float (&v)[1]) { *p = v[0]; }
template <> __device__ __forceinline__ void stv<2>(float* p, const float (&v)[2]) { *reinterpret_cast<float2*>(p) = make_float2(v[0], v[1]); }

// ---- one sparse operator, read from global memory (L1-cached) or from a compressed shared-memory copy
template <bool SG> struct Gr;
template <> struct Gr<false> {
  const int* rp; const int2* cv;
  __device__ __forceinline__ int begin(int n) const { return __ldg(rp + n); }
  __device__ __forceinline__ int end(int n) const { return __ldg(rp + n + 1); }
  __device__ __forceinline__ void edge(int k, int& col, float& w) const { const int2 e = __ldg(cv + k); col = e.x; w = __int_as_float(e.y); }
};
template <> struct Gr<true> {          // N <= 256: column in one byte; row pointers in 16 bits
  const unsigned short* rp; const float* val; const unsigned char* col;
  __device__ __forceinline__ int begin(int n) const { return rp[n]; }
  __device__ __forceinline__ int end(int n) const { return rp[n + 1]; }
  __device__ __forceinline__ void edge(int k, int& c, float& w) const { c = col[k]; w = val[k]; }
};

// ------------------------------------------------------------------------------------------------------------------
struct BasisParams {
  const int* rp[2]; const int2* cv[2];      // forward CSRs (by destination): y[i] = sum_k val_k x[col_k]
  int N, B, T, ld;
  const float* x; long long x_bs, x_ts;     // X[b,t] = x + b*x_bs + t*x_ts, (N, cin) dense
  const float* out; const float* h0; const float* stash;
  float* S1; float* S2;                     // (T*B, N, ld), ld >= 3*(cin+Co)
};

template <int CIN, int NOPS>
__global__ void __launch_bounds__(256) k_dcrnn_bwd_basis(BasisParams p) {
  constexpr int C = CIN + kCo, V = (C % 2 == 0) ? 2 : 1, CP = C / V;
  extern __shared__ __align__(16) float sm[];
  const int N = p.N, NP = N * CP;
  float* U1 = sm;
  float* U2 = sm + N * C;
  const int q = blockIdx.x, t = q / p.B, b = q - t * p.B;
  const long long bt = (long long)b * p.T + t;
  float* s1 = p.S1 + (long long)q * N * p.ld;
  float* s2 = p.S2 + (long long)q * N * p.ld;
  const float* hsrc = t > 0 ? p.out + (bt - 1) * N * kCo : (p.h0 ? p.h0 + (long long)b * N * kCo : nullptr);
  const float* rsrc = p.stash + (bt * 3 + 1) * N * kCo;
  const float* xsrc = p.x + b * p.x_bs + t * p.x_ts;
#pragma unroll 1
  for (int base = threadIdx.x; base < NP; base += kBatch * 256) {
    float h[kBatch][V], r[kBatch][V];
#pragma unroll
    for (int j = 0; j < kBatch; ++j) {
      const int s = base + j * 256, n = s / CP, c0 = (s - n * CP) * V;
#pragma unroll
      for (int e = 0; e < V; ++e) { h[j][e] = 0.f; r[j][e] = 1.f; }
      if (s < NP) {
        if (c0 < CIN) ldgv<V>(xsrc + n * CIN + c0, h[j]);
        else {
          if (hsrc) ldgv<V>(hsrc + n * kCo + c0 - CIN, h[j]);
          ldgv<V>(rsrc + n * kCo + c0 - CIN, r[j]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < kBatch; ++j) {
      const int s = base + j * 256;
      if (s < NP) {
        const int n = s / CP, c0 = (s - n * CP) * V;
        float v2[V];
#pragma unroll
        for (int e = 0; e < V; ++e) v2[e] = c0 < CIN ? h[j][e] : h[j][e] * r[j][e];
        stv<V>(U1 + n * C + c0, h[j]); stv<V>(U2 + n * C + c0, v2);
        stv<V>(s1 + (long long)n * p.ld + c0, h[j]); stv<V>(s2 + (long long)n * p.ld + c0, v2);
      }
    }
  }
  __syncthreads();
#pragma unroll
  for (int op = 0; op < NOPS; ++op) {
    const Gr<false> g{p.rp[op], p.cv[op]};
    for (int s = threadIdx.x; s < NP; s += 256) {
      const int n = s / CP, c0 = (s - n * CP) * V;
      float a1[V], a2[V];
#pragma unroll
      for (int e = 0; e < V; ++e) a1[e] = a2[e] = 0.f;
      const int k1 = g.end(n);
#pragma unroll 4
      for (int k = g.begin(n); k < k1; ++k) {        // same multiply / add order as k_spmm (bit-identical basis)
        int col; float w;
        g.edge(k, col, w);
        float u1[V], u2[V];
        ldv<V>(U1 + col * C + c0, u1); ldv<V>(U2 + col * C + c0, u2);
#pragma unroll
        for (int e = 0; e < V; ++e) { a1[e] = __fadd_rn(a1[e], __fmul_rn(w, u1[e])); a2[e] = __fadd_rn(a2[e], __fmul_rn(w, u2[e])); }
      }
      stv<V>(s1 + (long long)n * p.ld + (1 + op) * C + c0, a1);
      stv<V>(s2 + (long long)n * p.ld + (1 + op) * C + c0, a2);
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
struct BwdParams {
  const int* rp[2]; const int2* cv[2];      // transposed CSRs (by source): (A^T y)[j] = sum over edges leaving j
  int nnz[2];
  int N, B, T;
  const float* gout; const float* out; const float* h0; const float* stash;
  const float* whsT; const float* wzrT;     // (Co, 3C) and (2Co, 3C), row-major
  float* dph_all; float* dpzr_all;          // (T,B,N,Co), (T,B,N,2Co)
  float* dx;                                // (B,T,N,cin) or null
  float* dh0;                               // (B,N,Co)
};

// buf[r0 + RT rg ..+RT)[8cg..8cg+8) = sum_k dpT[k][r0 + RT rg ..] (x) W[k][8cg..]: one thread per RT x 8 output tile, RG row groups starting at
// row r0.  Per k a thread issues RT/4 + 2 LDS.128 (the rows -- dp is kept TRANSPOSED, k-major, so they are contiguous -- and the 8 weight
// columns) for 8 RT FFMA: with RT = 8 the shared-memory pipe and the FMA pipe are balanced (a 1 x 52 tile was 4x LSU-bound).  Adjacent
// lanes take adjacent column groups, so the tile stores of a warp spread over the banks.  PEER: the tile is also pushed into the partner
// CTA's buf (distributed shared memory), whose adjoint gathers read rows of both halves.
template <int NCOL, int KD, int RT, bool PEER>
__device__ __forceinline__ void gemm_tiles(const float* __restrict__ dpT, int dpp, const float* __restrict__ W, float* __restrict__ buf,
                                           int r0, int RG, uint32_t peer_buf, uint32_t peer_bar) {
  constexpr int CGN = NCOL / 8;
  const int tid = threadIdx.x;
  const bool active = tid < RG * CGN;
  const int rg = active ? tid / CGN : 0, cg = active ? tid - rg * CGN : 0;
  float acc[RT][8];
#pragma unroll
  for (int i = 0; i < RT; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  const float* ap = dpT + r0 + RT * rg;
  const float* wp = W + 8 * cg;
  if (active) {
  // 4-row tiles (the cluster-pair variant) have half the FMAs per operand load: their k loop is unrolled 4 deep to keep the LDS latency covered
  // (the profile of the first version showed 77 % of the FMA line's stalls on the short scoreboard); packed FFMA2 halves the issue slots
  // (bit-identical: two independent IEEE fmas per instruction)
#pragma unroll (RT == 4 ? 4 : 2)
  for (int k = 0; k < KD; ++k) {
    float a[RT];
#pragma unroll
    for (int q = 0; q < RT / 4; ++q) {
      const float4 t = *reinterpret_cast<const float4*>(ap + k * dpp + 4 * q);
      a[4 * q] = t.x; a[4 * q + 1] = t.y; a[4 * q + 2] = t.z; a[4 * q + 3] = t.w;
    }
    const float4 w0 = *reinterpret_cast<const float4*>(wp + k * NCOL), w1 = *reinterpret_cast<const float4*>(wp + k * NCOL + 4);
    const float w[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
    for (int i = 0; i < RT; ++i)
#pragma unroll
      for (int j = 0; j < 8; j += 2) {
        const float2 r = ffma2(make_float2(a[i], a[i]), make_float2(w[j], w[j + 1]), make_float2(acc[i][j], acc[i][j + 1]));
        acc[i][j] = r.x; acc[i][j + 1] = r.y;
      }
  }
  }
  if constexpr (PEER) cluster_wait();          // the pair has finished gathering from buf (signalled at the end of the previous phase)
  if (!active) return;
#pragma unroll
  for (int i = 0; i < RT; ++i) {
    const int off = (r0 + RT * rg + i) * NCOL + 8 * cg;
    const float4 v0 = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]), v1 = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
    float4* o = reinterpret_cast<float4*>(buf + off);
    o[0] = v0; o[1] = v1;
    if constexpr (PEER) { st4_async_cluster(peer_buf + off * 4, v0, peer_bar); st4_async_cluster(peer_buf + off * 4 + 16, v1, peer_bar); }
  }
}

// dU[n][c..c+V) = dS[n][c..] + sum_op sum_{edges of row n of A_op^T} val * dS[col][(1+op)*C + c..]   (adjoint of U -> [U|Op_0 U|..])
template <int NOPS, int NCOL, int C, int V, bool SG, int NG>
__device__ __forceinline__ void adjoint_at(const Gr<SG> (&g)[NG], const float* __restrict__ buf, int n, int c, float (&v)[V]) {
  ldv<V>(buf + n * NCOL + c, v);
#pragma unroll
  for (int op = 0; op < NOPS; ++op) {
    const int k1 = g[op].end(n);
    const float* src = buf + (1 + op) * C + c;
#pragma unroll 4
    for (int k = g[op].begin(n); k < k1; ++k) {
      int col; float w;
      g[op].edge(k, col, w);
      float s[V];
      ldv<V>(src + col * NCOL, s);
#pragma unroll
      for (int e = 0; e < V; ++e) v[e] = fmaf(w, s[e], v[e]);
    }
  }
}

// SPLIT = 2: a thread-block cluster of two CTAs per window (launched when 2 B CTAs still fit the machine, i.e. at the reference's batch of 64
// on 132 SMs): each CTA owns half of the node rows (a multiple of 8), runs the GEMMs / adjoints / gate derivatives of its rows only, and
// pushes its rows of dS into the partner's buf so that the adjoint gathers stay local.  Behind a GEMM the pair meets at a release / acquire
// cluster barrier (dS visible); behind a gather phase each CTA only signals "done reading buf" (relaxed arrival) and the matching wait sits
// in the next GEMM between its FFMA loop and its stores.
// NOPS: operators of the basis (2: DCRNN's P_o, P_i; 1: a Chebyshev K = 2 / GCN operator; 0: none).
template <int CIN, bool SG, int SPLIT, int NOPS>
__global__ void __launch_bounds__(kBwdThreads, 1) k_dcrnn_bwd_seq(BwdParams p) {
  constexpr int C = CIN + kCo, NB = NOPS + 1, NCOL = ncol_of(CIN, NOPS), V = (C % 2 == 0) ? 2 : 1, CP = C / V, RT = SPLIT == 2 ? 4 : 8;
  extern __shared__ __align__(16) float sm[];
  const int N = p.N, T = p.T, b = blockIdx.x / SPLIT, tid = threadIdx.x;
  const int RG = (N + 7) / 8, dpp = RG * 8 + 4, NH = N * kCo;
  // rows [r_lo, r_hi) are this CTA's; the GEMM covers whole groups of RT rows (pad rows of dpT are zero)
  const int half_rows = ((RG + 1) / 2) * 8;
  const int hrank = SPLIT == 2 ? (int)cluster_rank() : 0;
  const int r_lo = SPLIT == 2 ? hrank * half_rows : 0;
  const int r_hi = SPLIT == 2 ? (r_lo + half_rows < N ? r_lo + half_rows : N) : N;
  const int g_r0 = r_lo, g_RG = SPLIT == 2 ? ((hrank == 0 ? half_rows : RG * 8 - half_rows) / RT) : RG;
  const int s_lo = r_lo * CP, NP = r_hi * CP;                     // slot range of the pointwise loops
  float* Wh = sm;                            // [Co][NCOL]
  float* Wzr = Wh + kCo * NCOL;              // [2Co][NCOL]
  float* buf = Wzr + 2 * kCo * NCOL;         // [8RG][NCOL]
  float* dpT = buf + RG * 8 * NCOL;          // [2Co][dpp]  d pre-activations, k-major (transposed)
  float* G = dpT + 2 * kCo * dpp;            // [N][Co]     dL/dH_t (open) -> partial dL/dH_{t-1}
  float* dXp = G + N * kCo;                  // [N][4]      dU2[:, :cin] waiting for dU1
  Gr<SG> g[NOPS > 0 ? NOPS : 1];
  if constexpr (SG) {                        // compressed copy of the transposed operators: val f32 | col u8 | rowptr u16 (nnz of absent ones = 0)
    float* gval = dXp + N * 4;
    unsigned char* gcol = reinterpret_cast<unsigned char*>(gval + p.nnz[0] + p.nnz[1]);
    unsigned short* grp = reinterpret_cast<unsigned short*>(gcol + ((p.nnz[0] + p.nnz[1] + 3) & ~3));
#pragma unroll
    for (int op = 0; op < NOPS; ++op) {
      float* val = gval + (op ? p.nnz[0] : 0);
      unsigned char* col = gcol + (op ? p.nnz[0] : 0);
      unsigned short* rp = grp + op * (N + 1);
      for (int k = tid; k < p.nnz[op]; k += kBwdThreads) { const int2 e = __ldg(p.cv[op] + k); val[k] = __int_as_float(e.y); col[k] = (unsigned char)e.x; }
      for (int n = tid; n <= N; n += kBwdThreads) rp[n] = (unsigned short)__ldg(p.rp[op] + n);
      g[op].rp = rp; g[op].val = val; g[op].col = col;
    }
  } else {
#pragma unroll
    for (int op = 0; op < NOPS; ++op) { g[op].rp = p.rp[op]; g[op].cv = p.cv[op]; }
  }
  // ---- weights, zero padded to NCOL columns; padded rows of dpT stay zero for the whole kernel
  for (int i = tid; i < 3 * kCo * NCOL; i += kBwdThreads) {
    const int r = i / NCOL, c = i - r * NCOL;
    float v = 0.f;
    if (c < NB * C) v = r < kCo ? __ldg(p.whsT + r * NB * C + c) : __ldg(p.wzrT + (r - kCo) * NB * C + c);
    sm[i] = v;
  }
  for (int i = tid; i < 2 * kCo * dpp; i += kBwdThreads) dpT[i] = 0.f;
  // The partner's rows of dS arrive by st.async: every 16-byte store completes 16 transaction bytes on MY mbarrier `dbar`, which thread 0 arms
  // with the byte count of the partner's half before each phase -- no release / acquire cluster barrier on the data path (that barrier and
  // its memory fence were 47 % + 12 % of the warp time of the first cluster version).
  __shared__ __align__(8) uint64_t dbar;
  uint32_t peer_buf = 0, peer_bar = 0, dpar = 0;
  const uint32_t expect_bytes = (uint32_t)((hrank == 0 ? RG * 8 - half_rows : half_rows) * NCOL * 4);   // what the partner sends per GEMM
  if constexpr (SPLIT == 2) {
    peer_buf = map_to_peer(buf, (uint32_t)(hrank ^ 1));
    peer_bar = map_to_peer(&dbar, (uint32_t)(hrank ^ 1));
    if (tid == 0) {
      mbar_init(&dbar, 1);
      fence_mbar_init();
      mbar_arrive_expect_tx(&dbar, expect_bytes);
    }
  }
  // data_sync: behind a GEMM (dS of both halves complete and visible); free_sync: behind a gather phase (block barrier for dpT / G, plus the
  // relaxed "done reading buf" arrival that the next GEMM waits for just before it stores)
  auto data_sync = [&]() {
    __syncthreads();                                           // my own rows of dS (and dpT / G) are visible inside the CTA
    if constexpr (SPLIT == 2) {
      mbar_wait(&dbar, dpar);                                  // the partner's rows have landed
      dpar ^= 1u;
      if (tid == 0) mbar_arrive_expect_tx(&dbar, expect_bytes);   // armed for the next GEMM (the partner cannot send before my next arrival)
    }
  };
  auto free_sync = [&]() { if constexpr (SPLIT == 2) cluster_arrive_relaxed(); __syncthreads(); };
  if constexpr (SPLIT == 2) cluster_sync_all(); else __syncthreads();     // barriers initialised, weights / graph staged
  // ---- open step T-1
  const long long bT = (long long)b * T;
  for (int i = r_lo * kCo + tid; i < r_hi * kCo; i += kBwdThreads) {
    const int n = i / kCo, cc = i - n * kCo;
    const long long bt = bT + (T - 1);
    const float gg = __ldg(p.gout + bt * NH + i);
    const float z = __ldg(p.stash + (bt * 3 + 0) * NH + i), ht = __ldg(p.stash + (bt * 3 + 2) * NH + i);
    const float d = gg * (1.f - z) * (1.f - ht * ht);
    G[i] = gg;
    dpT[cc * dpp + n] = d;
    p.dph_all[(((long long)(T - 1) * p.B + b) * N) * kCo + i] = d;
  }
  free_sync();
#pragma unroll 1
  for (int t = T - 1; t >= 0; --t) {
    const long long bt = bT + t;
    const float* st = p.stash + bt * 3 * NH;
    const float* hprev = t > 0 ? p.out + (bt - 1) * NH : (p.h0 ? p.h0 + (long long)b * NH : nullptr);
    // dS2 = dpre_h @ Wh^T
    gemm_tiles<NCOL, kCo, RT, SPLIT == 2>(dpT, dpp, Wh, buf, g_r0, g_RG, peer_buf, peer_bar);
    data_sync();
    // dU2 = adjoint; d pre-activations of z and r; partial carry  g*Z + dHR*R
    float* dpzr = p.dpzr_all + (((long long)t * p.B + b) * N) * 2 * kCo;
#pragma unroll 1
    for (int base = s_lo + tid; base < NP; base += kBatch * kBwdThreads) {
      float hp[kBatch][V], zz[kBatch][V], rr[kBatch][V], hh[kBatch][V];
#pragma unroll
      for (int j = 0; j < kBatch; ++j) {                       // all global operands of the batch in flight together
        const int s = base + j * kBwdThreads, n = s / CP, c0 = (s - n * CP) * V, i = n * kCo + c0 - CIN;
#pragma unroll
        for (int e = 0; e < V; ++e) hp[j][e] = zz[j][e] = rr[j][e] = hh[j][e] = 0.f;
        if (s < NP && c0 >= CIN) {
          if (hprev) ldgv<V>(hprev + i, hp[j]);
          ldgv<V>(st + i, zz[j]); ldgv<V>(st + NH + i, rr[j]); ldgv<V>(st + 2 * NH + i, hh[j]);
        }
      }
#pragma unroll
      for (int j = 0; j < kBatch; ++j) {
        const int s = base + j * kBwdThreads;
        if (s < NP) {
          const int n = s / CP, c0 = (s - n * CP) * V;
          float v[V];
          adjoint_at<NOPS, NCOL, C, V, SG>(g, buf, n, c0, v);
          if (c0 < CIN) {
#pragma unroll
            for (int e = 0; e < V; ++e) dXp[n * 4 + c0 + e] = v[e];
          } else {
            const int cc = c0 - CIN, i = n * kCo + cc;
            float gg[V], dz[V], dr[V], gn[V];
            ldv<V>(G + i, gg);
#pragma unroll
            for (int e = 0; e < V; ++e) {
              dz[e] = gg[e] * (hp[j][e] - hh[j][e]) * zz[j][e] * (1.f - zz[j][e]);
              dr[e] = v[e] * hp[j][e] * rr[j][e] * (1.f - rr[j][e]);
              gn[e] = gg[e] * zz[j][e] + v[e] * rr[j][e];
              dpT[(cc + e) * dpp + n] = dz[e];
              dpT[(kCo + cc + e) * dpp + n] = dr[e];
            }
            stv<V>(dpzr + n * 2 * kCo + cc, dz);
            stv<V>(dpzr + n * 2 * kCo + kCo + cc, dr);
            stv<V>(G + i, gn);
          }
        }
      }
    }
    free_sync();
    // dS1 = dpre_zr @ Wzr^T
    gemm_tiles<NCOL, 2 * kCo, RT, SPLIT == 2>(dpT, dpp, Wzr, buf, g_r0, g_RG, peer_buf, peer_bar);
    data_sync();
    // dU1 = adjoint; dX_t; dL/dH_{t-1}; open step t-1
    const float* stn = st - 3 * NH;          // stash of step t-1 (only dereferenced when t > 0)
    float* dphn = p.dph_all + (((long long)(t - 1) * p.B + b) * N) * kCo;
#pragma unroll 1
    for (int base = s_lo + tid; base < NP; base += kBatch * kBwdThreads) {
      float go[kBatch][V], zz[kBatch][V], hh[kBatch][V];
#pragma unroll
      for (int j = 0; j < kBatch; ++j) {
        const int s = base + j * kBwdThreads, n = s / CP, c0 = (s - n * CP) * V, i = n * kCo + c0 - CIN;
#pragma unroll
        for (int e = 0; e < V; ++e) go[j][e] = zz[j][e] = hh[j][e] = 0.f;
        if (s < NP && c0 >= CIN && t > 0) {
          ldgv<V>(p.gout + (bt - 1) * NH + i, go[j]); ldgv<V>(stn + i, zz[j]); ldgv<V>(stn + 2 * NH + i, hh[j]);
        }
      }
#pragma unroll
      for (int j = 0; j < kBatch; ++j) {
        const int s = base + j * kBwdThreads;
        if (s < NP) {
          const int n = s / CP, c0 = (s - n * CP) * V;
          float v[V];
          adjoint_at<NOPS, NCOL, C, V, SG>(g, buf, n, c0, v);
          if (c0 < CIN) {
            if (p.dx) {
#pragma unroll
              for (int e = 0; e < V; ++e) p.dx[(bt * N + n) * CIN + c0 + e] = dXp[n * 4 + c0 + e] + v[e];
            }
          } else {
            const int cc = c0 - CIN, i = n * kCo + cc;
            float gg[V], d[V];
            ldv<V>(G + i, gg);
#pragma unroll
            for (int e = 0; e < V; ++e) gg[e] += v[e];                       // dL/dH_{t-1}
            if (t > 0) {
#pragma unroll
              for (int e = 0; e < V; ++e) {
                gg[e] += go[j][e];
                d[e] = gg[e] * (1.f - zz[j][e]) * (1.f - hh[j][e] * hh[j][e]);
                dpT[(cc + e) * dpp + n] = d[e];
              }
              stv<V>(G + i, gg);
              stv<V>(dphn + i, d);
            } else {
              stv<V>(p.dh0 + (long long)b * NH + i, gg);
            }
          }
        }
      }
    }
    free_sync();
  }
  if constexpr (SPLIT == 2) cluster_wait();      // pairs with the last arrival; nobody leaves while the partner may still be in its phase
}

inline size_t seq_smem_base(int N, int cin, int nops = 2) {
  const int ncol = ncol_of(cin, nops), rg = (N + 7) / 8;
  return sizeof(float) * ((size_t)3 * kCo * ncol + (size_t)rg * 8 * ncol + (size_t)2 * kCo * (rg * 8 + 4) + (size_t)N * (kCo + 4));
}
inline size_t seq_smem_graph(const stmp_plan* plan, int nops = 2) {
  size_t nnz = 0;
  for (int op = 0; op < nops; ++op) nnz += (size_t)plan->bwd[op].nnz;
  return 4 * nnz + ((nnz + 3) & ~(size_t)3) + 2 * (size_t)nops * ((size_t)plan->n + 1) + 8;
}
inline bool graph_in_smem(const stmp_plan* plan, int cin, int nops = 2) {
  if (nops == 0) return false;                   // nothing to stage
  for (int op = 0; op < nops; ++op)
    if (plan->bwd[op].nnz >= 65536) return false;
  return plan->n <= 256 && seq_smem_base(plan->n, cin, nops) + seq_smem_graph(plan, nops) <= kBwdSmemMax;
}
// the graph fits one SM: the GEMM tiles fit the block, the per-window buffers its shared memory, the basis kernel's [X|H] copies 100 KB
inline bool fits_one_sm(const stmp_plan* plan, long long cin, int nops) {
  return ((plan->n + 7) / 8) * (ncol_of((int)cin, nops) / 8) <= kBwdThreads && seq_smem_base(plan->n, (int)cin, nops) <= kBwdSmemMax &&
         2 * sizeof(float) * (size_t)plan->n * (cin + kCo) <= 100 * 1024;
}
inline bool bwd_supported(const stmp_plan* plan, long long cin, long long cout, long long K) {
  if (!plan || plan->flavor != STMP_FLAVOR_DCONV || plan->n_ops != 2) return false;
  if (K != 2 || cout != kCo || cin < 1 || cin > 4) return false;
  // cin == 2 (float2 slots, 104 columns) is the benchmark configuration; cin 1, 3, 4 (scalar slots / 112 columns) are served too
  // (tests/test_gpu_dcrnn.py::test_training_persistent_backward_other_channel_counts).
  return fits_one_sm(plan, cin, 2);
}
inline bool gru_bwd_supported(const stmp_plan* plan, long long n_ops, long long cin, long long cout) {
  if (!plan || n_ops < 0 || n_ops > 2 || n_ops > plan->n_ops) return false;
  if (cout != kCo || cin < 1 || cin > 4) return false;
  return fits_one_sm(plan, cin, (int)n_ops);
}

template <int CIN, int NOPS>
int launch_basis(const BasisParams& p, size_t smem, cudaStream_t st) {
  STMP_CUDA_OK(cudaFuncSetAttribute(k_dcrnn_bwd_basis<CIN, NOPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_dcrnn_bwd_basis<CIN, NOPS><<<(unsigned)(p.B * p.T), 256, smem, st>>>(p);
  return STMP_OK;
}
template <int NOPS>
int dispatch_basis(const BasisParams& p, int cin, size_t smem, cudaStream_t st) {
  switch (cin) {
    case 1: return launch_basis<1, NOPS>(p, smem, st);
    case 2: return launch_basis<2, NOPS>(p, smem, st);
    case 3: return launch_basis<3, NOPS>(p, smem, st);
    default: return launch_basis<4, NOPS>(p, smem, st);
  }
}
template <int CIN, bool SG, int NOPS>
int launch_seq(const BwdParams& p, size_t smem, int split, cudaStream_t st) {
  if (split == 2) {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_dcrnn_bwd_seq<CIN, SG, 2, NOPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)p.B * 2); cfg.blockDim = dim3(kBwdThreads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    STMP_CUDA_OK(cudaLaunchKernelEx(&cfg, k_dcrnn_bwd_seq<CIN, SG, 2, NOPS>, p));
    return STMP_OK;
  }
  STMP_CUDA_OK(cudaFuncSetAttribute(k_dcrnn_bwd_seq<CIN, SG, 1, NOPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_dcrnn_bwd_seq<CIN, SG, 1, NOPS><<<(unsigned)p.B, kBwdThreads, smem, st>>>(p);
  return STMP_OK;
}
template <int CIN, int NOPS>
int launch_seq_sg(const BwdParams& p, bool sg, size_t smem, int split, cudaStream_t st) {
  if constexpr (NOPS > 0) {
    if (sg) return launch_seq<CIN, true, NOPS>(p, smem, split, st);
  }
  return launch_seq<CIN, false, NOPS>(p, smem, split, st);
}
template <int NOPS>
int dispatch_seq(const BwdParams& p, int cin, bool sg, size_t smem, int split, cudaStream_t st) {
  switch (cin) {
    case 1: return launch_seq_sg<1, NOPS>(p, sg, smem, split, st);
    case 2: return launch_seq_sg<2, NOPS>(p, sg, smem, split, st);
    case 3: return launch_seq_sg<3, NOPS>(p, sg, smem, split, st);
    default: return launch_seq_sg<4, NOPS>(p, sg, smem, split, st);
  }
}

// Splits the prepacked forward weights wcat [96][112] (columns H | Op0 H | Op1 H | X | Op0 X | Op1 X | pad) into the transposed stacked weights
// of the backward GEMMs in basis order [X | H] per block: whsT (32, NB C) from the candidate rows, wzrT (64, NB C) from the z | r rows.
__global__ void k_gru_pack_bwd_weights(int cin, int nb, const float* __restrict__ wcat, float* __restrict__ whsT, float* __restrict__ wzrT) {
  const int C = cin + kCo, W = nb * C;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 3 * kCo * W) return;
  const int r = i / W, m = i - r * W, blk = m / C, c = m - blk * C;
  const int col = c < cin ? 96 + 4 * blk + c : 32 * blk + (c - cin);
  if (r < kCo) whsT[r * W + m] = wcat[(2 * kCo + r) * 112 + col];
  else wzrT[(r - kCo) * W + m] = wcat[(r - kCo) * 112 + col];
}

int basis_impl(const stmp_plan* plan, int nops, int64_t B, int64_t T, int64_t cin, const float* x, int64_t x_bstride, int64_t x_tstride,
               const float* out, const float* h0, const float* stash, float* S1, float* S2, int64_t ld, cudaStream_t st) {
  BasisParams p;
  for (int o = 0; o < 2; ++o) { p.rp[o] = o < nops ? plan->fwd[o].rowptr : nullptr; p.cv[o] = o < nops ? plan->fwd[o].cv : nullptr; }
  p.N = plan->n; p.B = (int)B; p.T = (int)T; p.ld = (int)ld;
  p.x = x; p.x_bs = x_bstride; p.x_ts = x_tstride; p.out = out; p.h0 = h0; p.stash = stash; p.S1 = S1; p.S2 = S2;
  const size_t smem = sizeof(float) * 2 * (size_t)plan->n * (cin + kCo);
  switch (nops) {
    case 0: return dispatch_basis<0>(p, (int)cin, smem, st);
    case 1: return dispatch_basis<1>(p, (int)cin, smem, st);
    default: return dispatch_basis<2>(p, (int)cin, smem, st);
  }
}

int seq_impl(const stmp_plan* plan, int nops, int64_t B, int64_t T, int64_t cin, const float* gout, const float* out, const float* h0,
             const float* stash, const float* whsT, const float* wzrT, float* dph_all, float* dpzr_all, float* dx, float* dh0, cudaStream_t st,
             int* split_out, bool* global_out) {
  BwdParams p;
  for (int o = 0; o < 2; ++o) {
    const bool on = o < nops;
    p.rp[o] = on ? plan->bwd[o].rowptr : nullptr; p.cv[o] = on ? plan->bwd[o].cv : nullptr; p.nnz[o] = on ? plan->bwd[o].nnz : 0;
  }
  p.N = plan->n; p.B = (int)B; p.T = (int)T;
  p.gout = gout; p.out = out; p.h0 = h0; p.stash = stash; p.whsT = whsT; p.wzrT = wzrT;
  p.dph_all = dph_all; p.dpzr_all = dpzr_all; p.dx = dx; p.dh0 = dh0;
  const bool sg = graph_in_smem(plan, (int)cin, nops);
  const size_t smem = seq_smem_base(plan->n, (int)cin, nops) + (sg ? seq_smem_graph(plan, nops) : 0);
  int dev = 0, sms = 0;
  STMP_CUDA_OK(cudaGetDevice(&dev));
  STMP_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int split = (g_bwd_split && 2 * B <= sms && plan->n >= 16) ? 2 : 1;      // small batches: two CTAs per window (cluster), rows halved
  *split_out = split;
  *global_out = nops > 0 && !sg;          // the transposed operators are read from the global CSR, not a staged copy
  switch (nops) {
    case 0: return dispatch_seq<0>(p, (int)cin, sg, smem, split, st);
    case 1: return dispatch_seq<1>(p, (int)cin, sg, smem, split, st);
    default: return dispatch_seq<2>(p, (int)cin, sg, smem, split, st);
  }
}

}  // namespace
}  // namespace stmp

using namespace stmp;

extern "C" int stmp_dcrnn_bwd_supported(const stmp_plan* plan, int64_t cin, int64_t cout, int64_t K) {
  return bwd_supported(plan, cin, cout, K) ? 1 : 0;
}

extern "C" int stmp_dcrnn_bwd_basis(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, const float* x,
                                    int64_t x_bstride, int64_t x_tstride, const float* out, const float* h0, const float* stash,
                                    float* S1, float* S2, int64_t ld, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_dcrnn_bwd_basis: plan is NULL");
  STMP_REQUIRE(bwd_supported(plan, cin, cout, 2), STMP_EUNSUPPORTED, "stmp_dcrnn_bwd_basis: configuration not served (K=2, cout=32, cin<=4, small graph)");
  STMP_REQUIRE(x && out && stash && S1 && S2, STMP_EINVAL, "stmp_dcrnn_bwd_basis: NULL tensor");
  STMP_REQUIRE(B >= 0 && T > 0 && ld >= 3 * (cin + cout), STMP_ESHAPE, "stmp_dcrnn_bwd_basis: bad sizes");
  const bool vec2 = (cin + cout) % 2 == 0;
  STMP_REQUIRE(!vec2 || (ld % 2 == 0 && x_bstride % 2 == 0 && x_tstride % 2 == 0 && ((uintptr_t)x % 8) == 0 && ((uintptr_t)S1 % 8) == 0 &&
                         ((uintptr_t)S2 % 8) == 0), STMP_ESHAPE, "stmp_dcrnn_bwd_basis: operands must be 8-byte aligned with even strides");
  if (B == 0) return STMP_OK;
  const int rc = basis_impl(plan, 2, B, T, cin, x, x_bstride, x_tstride, out, h0, stash, S1, S2, ld, (cudaStream_t)stream);
  if (rc != STMP_OK) return rc;
  STMP_LAUNCH_OK("k_dcrnn_bwd_basis");
  return STMP_OK;
}

extern "C" int stmp_dcrnn_bwd_seq(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, const float* gout,
                                  const float* out, const float* h0, const float* stash, const float* whsT, const float* wzrT,
                                  float* dph_all, float* dpzr_all, float* dx, float* dh0, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_dcrnn_bwd_seq: plan is NULL");
  STMP_REQUIRE(bwd_supported(plan, cin, cout, 2), STMP_EUNSUPPORTED, "stmp_dcrnn_bwd_seq: configuration not served (K=2, cout=32, cin<=4, small graph)");
  STMP_REQUIRE(gout && out && stash && whsT && wzrT && dph_all && dpzr_all && dh0, STMP_EINVAL, "stmp_dcrnn_bwd_seq: NULL tensor");
  STMP_REQUIRE(B >= 0 && T > 0, STMP_ESHAPE, "stmp_dcrnn_bwd_seq: bad sizes");
  auto al8 = [](const void* q) { return ((uintptr_t)q % 8) == 0; };
  STMP_REQUIRE(al8(gout) && al8(out) && al8(stash) && al8(dph_all) && al8(dpzr_all) && al8(dh0) && (!h0 || al8(h0)), STMP_ESHAPE,
               "stmp_dcrnn_bwd_seq: operands must be 8-byte aligned");
  if (B == 0) return STMP_OK;
  int split = 1;
  bool global = false;
  const int rc = seq_impl(plan, 2, B, T, cin, gout, out, h0, stash, whsT, wzrT, dph_all, dpzr_all, dx, dh0, (cudaStream_t)stream, &split,
                          &global);
  if (rc != STMP_OK) return rc;
  STMP_LAUNCH_OK("k_dcrnn_bwd_seq");
  if (split == 2) { static const int slot2 = path_slot("k_dcrnn_bwd_seq[cluster2]"); count_path(slot2); }
  if (global) { static const int slotg = path_slot("k_dcrnn_bwd_seq[graph-global]"); count_path(slotg); }
  return STMP_OK;
}

// ---- generic graph-GRU backward (the twin of stmp_gru_seq_fwd): the same kernels with n_ops operators of any plan flavor --------------
extern "C" int stmp_gru_bwd_supported(const stmp_plan* plan, int n_ops, int64_t cin, int64_t cout) {
  return gru_bwd_supported(plan, n_ops, cin, cout) ? 1 : 0;
}

extern "C" int stmp_gru_bwd_basis(const stmp_plan* plan, int n_ops, int64_t B, int64_t T, int64_t cin, const float* x, int64_t x_bstride,
                                  int64_t x_tstride, const float* out, const float* h0, int64_t h0_bstride, const float* stash, float* S1,
                                  float* S2, int64_t ld, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_gru_bwd_basis: plan is NULL");
  STMP_REQUIRE(gru_bwd_supported(plan, n_ops, cin, kCo), STMP_EUNSUPPORTED,
               "stmp_gru_bwd_basis: configuration not served (n_ops <= plan's, cout = 32, cin <= 4, graph fits one SM)");
  STMP_REQUIRE(!h0 || h0_bstride != 0, STMP_EUNSUPPORTED, "stmp_gru_bwd_basis: a shared h0 (batch stride 0) is not served");
  STMP_REQUIRE(x && out && stash && S1 && S2, STMP_EINVAL, "stmp_gru_bwd_basis: NULL tensor");
  const int64_t C = cin + kCo;
  STMP_REQUIRE(B >= 0 && T > 0 && ld == ncol_of((int)cin, n_ops) && (!h0 || h0_bstride == (int64_t)plan->n * kCo), STMP_ESHAPE,
               "stmp_gru_bwd_basis: bad sizes (ld must be (n_ops+1)(cin+32) rounded up to 8, h0 (B, N, 32) dense)");
  STMP_REQUIRE(C % 2 != 0 || (x_bstride % 2 == 0 && x_tstride % 2 == 0 && ((uintptr_t)x % 8) == 0 && ((uintptr_t)S1 % 8) == 0 &&
                              ((uintptr_t)S2 % 8) == 0), STMP_ESHAPE, "stmp_gru_bwd_basis: operands must be 8-byte aligned with even strides");
  if (B == 0) return STMP_OK;
  const int rc = basis_impl(plan, n_ops, B, T, cin, x, x_bstride, x_tstride, out, h0, stash, S1, S2, ld, (cudaStream_t)stream);
  if (rc != STMP_OK) return rc;
  STMP_LAUNCH_OK("k_gru_bwd_basis");
  return STMP_OK;
}

extern "C" int stmp_gru_bwd_seq(const stmp_plan* plan, int n_ops, int64_t B, int64_t T, int64_t cin, const float* gout, const float* out,
                                const float* h0, int64_t h0_bstride, const float* stash, const float* whsT, const float* wzrT, float* dph_all,
                                float* dpzr_all, float* dx, float* dh0, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_gru_bwd_seq: plan is NULL");
  STMP_REQUIRE(gru_bwd_supported(plan, n_ops, cin, kCo), STMP_EUNSUPPORTED,
               "stmp_gru_bwd_seq: configuration not served (n_ops <= plan's, cout = 32, cin <= 4, graph fits one SM)");
  STMP_REQUIRE(!h0 || h0_bstride != 0, STMP_EUNSUPPORTED, "stmp_gru_bwd_seq: a shared h0 (batch stride 0) is not served");
  STMP_REQUIRE(gout && out && stash && whsT && wzrT && dph_all && dpzr_all && dh0, STMP_EINVAL, "stmp_gru_bwd_seq: NULL tensor");
  STMP_REQUIRE(B >= 0 && T > 0 && (!h0 || h0_bstride == (int64_t)plan->n * kCo), STMP_ESHAPE,
               "stmp_gru_bwd_seq: bad sizes (h0 must be (B, N, 32) dense)");
  auto al8 = [](const void* q) { return ((uintptr_t)q % 8) == 0; };
  STMP_REQUIRE(al8(gout) && al8(out) && al8(stash) && al8(dph_all) && al8(dpzr_all) && al8(dh0) && (!h0 || al8(h0)), STMP_ESHAPE,
               "stmp_gru_bwd_seq: operands must be 8-byte aligned");
  if (B == 0) return STMP_OK;
  int split = 1;
  bool global = false;
  const int rc = seq_impl(plan, n_ops, B, T, cin, gout, out, h0, stash, whsT, wzrT, dph_all, dpzr_all, dx, dh0, (cudaStream_t)stream, &split,
                          &global);
  if (rc != STMP_OK) return rc;
  STMP_LAUNCH_OK("k_gru_bwd_seq");
  if (split == 2) { static const int slot2 = path_slot("k_gru_bwd_seq[cluster2]"); count_path(slot2); }
  if (global) { static const int slotg = path_slot("k_gru_bwd_seq[graph-global]"); count_path(slotg); }
  return STMP_OK;
}

extern "C" int stmp_gru_pack_bwd_weights(int n_ops, int64_t cin, const float* wcat, float* whsT, float* wzrT, void* stream) {
  STMP_REQUIRE(wcat && whsT && wzrT, STMP_EINVAL, "stmp_gru_pack_bwd_weights: NULL tensor");
  STMP_REQUIRE(n_ops >= 0 && n_ops <= 2 && cin >= 1 && cin <= 4, STMP_EUNSUPPORTED, "stmp_gru_pack_bwd_weights: n_ops <= 2, cin <= 4 only");
  const int total = 3 * kCo * (n_ops + 1) * (int)(cin + kCo);
  k_gru_pack_bwd_weights<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>((int)cin, n_ops + 1, wcat, whsT, wzrT);
  STMP_LAUNCH_OK("k_gru_pack_bwd_weights");
  return STMP_OK;
}
