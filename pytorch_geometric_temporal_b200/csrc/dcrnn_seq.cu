// dcrnn_seq.cu -- K1..K5 fused: the whole DCRNN recurrence of one window in one persistent CTA.
//
// Reference path replaced: BatchedDCRNN.forward (nn/recurrent/dcrnn.py:429-475) = Python loop over T of
// 3 x BatchedDConv (:258-325) + gates (:398-427); with B=T=1 it is DCRNN.forward (:194-219).
//
// Design (sm_90a):
//  * grid = min(B, #SM) persistent CTAs; CTA b owns window b, b+grid, ...  Everything a window needs
//    lives in shared memory for all T steps: both diffusion operators (CSR, (col,val) packed 8 B/edge),
//    the three gates' weights, and the basis matrix S[N][NB*CP] = [U | P_o U | P_i U | ...] whose block 0
//    is U = [H | X_t].  HBM traffic per window is the compulsory minimum: read X window once, write H_t.
//  * X windows arrive by TMA 1-D bulk copies (cp.async.bulk -> mbarrier), double buffered: the next
//    window's X streams in while the current one computes.
//  * gather/scatter: a half-warp owns one (destination row, operator); lanes are float4-vectorised along
//    the feature axis; per-destination accumulation is in registers in CSR order (no atomics).
//  * z and r share the diffusion of [X|H] (the reference recomputes it per gate); only the H*R columns
//    are re-diffused for the candidate.
//  * contraction S @ [Wz|Wr] and S @ Wh in exact fp32 FFMA (strict-parity mode): warp w owns output
//    channels 4w..4w+3 of every gate, lane l owns rows l, l+32, ...; A rows are read as float4 along K
//    with LD/4 odd => conflict-free LDS.128; B is a warp-uniform broadcast.  The gate epilogue
//    (sigmoid/tanh/Hadamard/convex combine) runs on the accumulators in registers.
#include "common.cuh"
#include "dcrnn_common.cuh"

namespace stmp {
// wgmma variant (dcrnn_seq_tc.cu)
bool dcrnn_tc_supported(const stmp_plan* plan, long long cin, long long cout, long long K);
int dcrnn_tc_launch(const stmp_plan* plan, long long B, long long T, long long cin, const float* x, const long long* win_start,
                    long long x_bstride, long long x_tstride, const float* w_z, const float* w_r, const float* w_h, const float* b_z,
                    const float* b_r, const float* b_h, const float* h0, float* out, float* stash, const void* wimage,
                    void* workspace, cudaStream_t st);
int tc_pack_weight_image(const float* wcat, const float* bcat, const float* w0, const float* w1, const float* w2, const float* b0,
                         const float* b1, const float* b2, int cin, void* image, cudaStream_t st);
int tc_weight_image_bytes();

bool gru_tc_supported(const stmp_plan* plan, long long cin, int n_ops);
int gru_tc_launch(const stmp_plan* plan, int n_ops, long long B, long long T, long long cin, const float* x, const long long* win_start,
                  long long x_bstride, long long x_tstride, const float* wcat, const float* bcat, const float* h0, long long h0_bstride,
                  float* out, float* stash, const void* wimage, void* workspace, cudaStream_t st);
long long tc_workspace_bytes(const stmp_plan* plan, long long T, long long cin);

// narrow-state variant, cout <= 4 (dcrnn_narrow.cu)
bool dcrnn_narrow_supported(const stmp_plan* plan, long long cin, long long cout, long long K);
int dcrnn_narrow_launch(const stmp_plan* plan, long long B, long long T, long long cin, long long cout, long long K, const float* x,
                        const long long* win_start, long long x_bstride, long long x_tstride, const float* w_z, const float* w_r,
                        const float* w_h, const float* b_z, const float* b_r, const float* b_h, const float* h0, float* out, float* stash,
                        cudaStream_t st);

namespace {

constexpr int kMaxSmem = 232448;  // 227 KB opt-in limit per CTA on sm_90

struct DcrnnParams {
  int N, CIN, K, T;
  long long B;
  int CP, NB, LD;
  const int* rowptr[2];
  const int2* cv[2];
  int nnz[2];
  const float* x;
  const long long* win_start;
  long long x_bstride, x_tstride;
  const float* w[3];
  const float* bias[3];
  const float* h0;
  float* out;
  float* stash;
  int off_S, off_W, off_bias, off_rowptr[2], off_cv[2], off_x[2], off_bar;
  int x_floats;  // T*N*CIN
  int use_tma;
};

// One diffusion hop.  H columns: LPR = OUT/4 lanes per task, lane j owns float4 j, so a warp covers
// 32/LPR destination rows per pass and every gather is one full 128-byte shared-memory wavefront.
// X columns (one float4 at column OUT): one thread per task, only when `with_x`.
// dst block = P_op * src (hop 1) or 2 * P_op * src - U (hop >= 2; the reference never advances Tx_0 past
// X, dcrnn.py:80,106).
template <int OUT, int NT>
__device__ __forceinline__ void diffuse(float* S, const GraphSmem g, int N, int LD, int CP, int hop, bool with_x, int tid) {
  constexpr int LPR = OUT / 4;
  const int j = tid & (LPR - 1);
  for (int slot = tid / LPR; slot < 2 * N; slot += NT / LPR) {
    const int task = g.order[slot];
    const int op = task >= N ? 1 : 0;
    const int i = task - op * N;
    const int sb = (hop == 1) ? 0 : (1 + 2 * (hop - 2) + op);
    const int db = 1 + 2 * (hop - 1) + op;
    float4 acc = gather_row(S + sb * CP + 4 * j, g.ce, g.gstart[task], g.gstart[task + 1]);
    if (hop >= 2) {
      const float4 u = ld4(S + i * LD + 4 * j);
      acc.x = 2.0f * acc.x - u.x; acc.y = 2.0f * acc.y - u.y; acc.z = 2.0f * acc.z - u.z; acc.w = 2.0f * acc.w - u.w;
    }
    st4(S + i * LD + db * CP + 4 * j, acc);
  }
  if (with_x) {
    for (int slot = tid; slot < 2 * N; slot += NT) {
      const int task = g.order[slot];
      const int op = task >= N ? 1 : 0;
      const int i = task - op * N;
      const int sb = (hop == 1) ? 0 : (1 + 2 * (hop - 2) + op);
      const int db = 1 + 2 * (hop - 1) + op;
      float4 acc = gather_row(S + sb * CP + OUT, g.ce, g.gstart[task], g.gstart[task + 1]);
      if (hop >= 2) {
        const float4 u = ld4(S + i * LD + OUT);
        acc.x = 2.0f * acc.x - u.x; acc.y = 2.0f * acc.y - u.y; acc.z = 2.0f * acc.z - u.z; acc.w = 2.0f * acc.w - u.w;
      }
      st4(S + i * LD + db * CP + OUT, acc);
    }
  }
}

// Thread mapping of the contraction: warp w owns rows [w*RQ*RT, (w+1)*RQ*RT); inside the warp lane =
// (cg, rq) with cg = lane % CG the group of 4 output channels and rq = lane / CG the row phase; the
// thread owns rows w*RQ*RT + rq + RQ*i (i < RT) x channels 4cg..4cg+3 of EVERY gate, so Z, H and H~ of an
// element meet in one thread's registers.  A (rows of S, float4 along K): RQ distinct rows per LDS.128,
// consecutive rows are LD words apart with LD/4 odd => distinct bank groups, one wavefront.  B (weights):
// CG distinct consecutive float4 = <= 128 B, one wavefront.
template <int OUT, int RT, int NW>
__global__ void __launch_bounds__(NW * 32, 1) k_dcrnn_seq(const DcrnnParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  constexpr int NT = NW * 32;
  constexpr int WLD = 3 * OUT;
  constexpr int CG = OUT / 4;
  constexpr int RQ = 32 / CG;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int N = p.N, CIN = p.CIN, K = p.K, T = p.T, CP = p.CP, LD = p.LD;
  const int C = OUT + CIN;

  float* S = reinterpret_cast<float*>(smem + p.off_S);
  float* W = reinterpret_cast<float*>(smem + p.off_W);
  float* Bs = reinterpret_cast<float*>(smem + p.off_bias);
  int2* s_ce = reinterpret_cast<int2*>(smem + p.off_cv[0]);
  int* s_gstart = reinterpret_cast<int*>(smem + p.off_rowptr[0]);
  int* s_order = reinterpret_cast<int*>(smem + p.off_rowptr[1]);
  float* xbuf0 = reinterpret_cast<float*>(smem + p.off_x[0]);
  float* xbuf1 = reinterpret_cast<float*>(smem + p.off_x[1]);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + p.off_bar);

  const long long b_first = blockIdx.x;
  if (b_first >= p.B) return;
  const uint32_t x_bytes = (uint32_t)p.x_floats * 4u;
  auto x_base = [&](long long b) -> const float* {
    return p.x + (p.win_start ? p.win_start[b] * p.x_tstride : b * p.x_bstride);
  };

  // ---- one-time per CTA: barriers, first TMA, graph, weights, zero S --------------------------------
  if (p.use_tma && tid == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    fence_mbar_init();
    mbar_arrive_expect_tx(&bars[0], x_bytes);
    tma_bulk_g2s(xbuf0, x_base(b_first), x_bytes, &bars[0]);
  }
  stage_graph<NT>(p.rowptr[0], p.rowptr[1], p.cv[0], p.cv[1], N, LD, s_ce, s_gstart, s_order, tid);
  const GraphSmem gs{s_ce, s_gstart, s_order};
  // weights -> Wcat[kidx][z|r|h], internal channel order [H(OUT) | X(CIN) | pad], block 0 = W[0,0]+W[1,0]
  for (int idx = tid; idx < LD * WLD; idx += NT) {
    const int kidx = idx / WLD, col = idx - kidx * WLD;
    const int g = col / OUT, o = col - g * OUT;
    const int blk = kidx / CP, ci = kidx - blk * CP;
    float v = 0.f;
    if (ci < C) {
      const int ch = ci < OUT ? CIN + ci : ci - OUT;
      const float* wg = g == 0 ? p.w[0] : (g == 1 ? p.w[1] : p.w[2]);
      if (blk == 0) {
        v = wg[((0 * K + 0) * C + ch) * OUT + o] + wg[((1 * K + 0) * C + ch) * OUT + o];
      } else {
        const int hop = (blk - 1) / 2 + 1, d = (blk - 1) & 1;
        v = wg[((d * K + hop) * C + ch) * OUT + o];
      }
    }
    W[idx] = v;
  }
  for (int idx = tid; idx < WLD; idx += NT) {
    const int g = idx / OUT;
    const float* bg = g == 0 ? p.bias[0] : (g == 1 ? p.bias[1] : p.bias[2]);
    Bs[idx] = bg ? bg[idx - g * OUT] : 0.f;
  }
  for (int idx = tid; idx < N * LD; idx += NT) S[idx] = 0.f;
  __syncthreads();

  const int cg = lane % CG, rq = lane / CG;
  const int c0 = cg * 4;
  const int row0 = warp * (RQ * RT) + rq;
  int soff[RT];  // clamped row offsets (rows >= N read row N-1, their results are discarded)
#pragma unroll
  for (int i = 0; i < RT; ++i) {
    const int r = row0 + RQ * i;
    soff[i] = (r < N ? r : N - 1) * LD;
  }
  const int KG = LD / 4;
  uint32_t phase0 = 0u, phase1 = 0u;
  int it = 0;

  for (long long b = b_first; b < p.B; b += gridDim.x, ++it) {
    const int buf = it & 1;
    const float* xw;
    if (p.use_tma) {
      if (buf == 0) { mbar_wait(&bars[0], phase0); phase0 ^= 1u; } else { mbar_wait(&bars[1], phase1); phase1 ^= 1u; }
      const long long bn = b + gridDim.x;
      if (tid == 0 && bn < p.B) {  // stream the next window in while this one computes
        fence_proxy_async();
        mbar_arrive_expect_tx(&bars[buf ^ 1], x_bytes);
        tma_bulk_g2s(buf ? xbuf0 : xbuf1, x_base(bn), x_bytes, &bars[buf ^ 1]);
      }
      xw = buf ? xbuf1 : xbuf0;
    } else {
      const float* xb = x_base(b);
      for (int t = 0; t < T; ++t)
        for (int idx = tid; idx < N * CIN; idx += NT) xbuf0[t * N * CIN + idx] = __ldg(xb + t * p.x_tstride + idx);
      xw = xbuf0;
    }
    // H_0 and X_0 into block 0
    for (int idx = tid; idx < N * OUT; idx += NT) {
      const int n = idx / OUT, c = idx - n * OUT;
      S[n * LD + c] = p.h0 ? __ldg(p.h0 + (b * N + n) * OUT + c) : 0.f;
    }
    __syncthreads();  // (non-TMA path: xbuf visible)
    for (int idx = tid; idx < N * CIN; idx += NT) {
      const int n = idx / CIN, c = idx - n * CIN;
      S[n * LD + OUT + c] = xw[idx];
    }
    __syncthreads();

    for (int t = 0; t < T; ++t) {
      // ---- round 1: diffuse U = [H | X_t] ------------------------------------------------------------
      for (int hop = 1; hop < K; ++hop) {
        diffuse<OUT, NT>(S, gs, N, LD, CP, hop, true, tid);
        __syncthreads();
      }
      // ---- GEMM 1: [z|r] pre-activations -------------------------------------------------------------
      float2 accz[RT][2], accr[RT][2];
#pragma unroll
      for (int i = 0; i < RT; ++i)
#pragma unroll
        for (int c = 0; c < 2; ++c) { accz[i][c] = make_float2(0.f, 0.f); accr[i][c] = make_float2(0.f, 0.f); }
#pragma unroll 1
      for (int kg = 0; kg < KG; ++kg) {
        float4 a[RT];
#pragma unroll
        for (int i = 0; i < RT; ++i) a[i] = ld4(S + soff[i] + 4 * kg);
        const float* wrow = W + (4 * kg) * WLD + c0;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const float4 bz = ld4(wrow + kk * WLD);
          const float4 br = ld4(wrow + kk * WLD + OUT);
#pragma unroll
          for (int i = 0; i < RT; ++i) {
            const float av = kk == 0 ? a[i].x : (kk == 1 ? a[i].y : (kk == 2 ? a[i].z : a[i].w));
            const float2 aa = make_float2(av, av);
            accz[i][0] = ffma2(aa, make_float2(bz.x, bz.y), accz[i][0]);
            accz[i][1] = ffma2(aa, make_float2(bz.z, bz.w), accz[i][1]);
            accr[i][0] = ffma2(aa, make_float2(br.x, br.y), accr[i][0]);
            accr[i][1] = ffma2(aa, make_float2(br.z, br.w), accr[i][1]);
          }
        }
      }
      // gates; keep Z and H in registers, R only lives long enough to form H*R
      float hreg[RT][4], zreg[RT][4], rreg[RT][4];
      {
        const float4 bz = ld4(Bs + c0), br = ld4(Bs + OUT + c0);
        const float bzv[4] = {bz.x, bz.y, bz.z, bz.w}, brv[4] = {br.x, br.y, br.z, br.w};
#pragma unroll
        for (int i = 0; i < RT; ++i) {
          const float4 h = ld4(S + soff[i] + c0);
          hreg[i][0] = h.x; hreg[i][1] = h.y; hreg[i][2] = h.z; hreg[i][3] = h.w;
          const float pz[4] = {accz[i][0].x, accz[i][0].y, accz[i][1].x, accz[i][1].y};
          const float pr[4] = {accr[i][0].x, accr[i][0].y, accr[i][1].x, accr[i][1].y};
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            zreg[i][c] = sigmoidf_acc(pz[c] + bzv[c]);
            rreg[i][c] = sigmoidf_acc(pr[c] + brv[c]);
          }
        }
      }
      __syncthreads();  // every warp is done reading block 0 as the GEMM A operand
      const long long obase = (b * T + t) * (long long)N;
#pragma unroll
      for (int i = 0; i < RT; ++i) {
        const int r = row0 + RQ * i;
        if (r < N) {
          st4(S + r * LD + c0, make_float4(hreg[i][0] * rreg[i][0], hreg[i][1] * rreg[i][1],
                                           hreg[i][2] * rreg[i][2], hreg[i][3] * rreg[i][3]));
          if (p.stash) {
            float* sp = p.stash + ((obase * 3) + r) * OUT + c0;
            st4(sp, make_float4(zreg[i][0], zreg[i][1], zreg[i][2], zreg[i][3]));
            st4(sp + (long long)N * OUT, make_float4(rreg[i][0], rreg[i][1], rreg[i][2], rreg[i][3]));
          }
        }
      }
      __syncthreads();
      // ---- round 2: re-diffuse only the H*R columns ---------------------------------------------------
      for (int hop = 1; hop < K; ++hop) {
        diffuse<OUT, NT>(S, gs, N, LD, CP, hop, false, tid);
        __syncthreads();
      }
      // ---- GEMM 2: candidate --------------------------------------------------------------------------
      float2 acch[RT][2];
#pragma unroll
      for (int i = 0; i < RT; ++i) { acch[i][0] = make_float2(0.f, 0.f); acch[i][1] = make_float2(0.f, 0.f); }
#pragma unroll 1
      for (int kg = 0; kg < KG; ++kg) {
        float4 a[RT];
#pragma unroll
        for (int i = 0; i < RT; ++i) a[i] = ld4(S + soff[i] + 4 * kg);
        const float* wrow = W + (4 * kg) * WLD + 2 * OUT + c0;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          const float4 bh = ld4(wrow + kk * WLD);
#pragma unroll
          for (int i = 0; i < RT; ++i) {
            const float av = kk == 0 ? a[i].x : (kk == 1 ? a[i].y : (kk == 2 ? a[i].z : a[i].w));
            const float2 aa = make_float2(av, av);
            acch[i][0] = ffma2(aa, make_float2(bh.x, bh.y), acch[i][0]);
            acch[i][1] = ffma2(aa, make_float2(bh.z, bh.w), acch[i][1]);
          }
        }
      }
      __syncthreads();  // all reads of S for this step are done
      {
        const float4 bh = ld4(Bs + 2 * OUT + c0);
        const float bhv[4] = {bh.x, bh.y, bh.z, bh.w};
#pragma unroll
        for (int i = 0; i < RT; ++i) {
          const int r = row0 + RQ * i;
          if (r < N) {
            float hn[4], ht[4];
            const float ph[4] = {acch[i][0].x, acch[i][0].y, acch[i][1].x, acch[i][1].y};
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              ht[c] = tanhf(ph[c] + bhv[c]);
              hn[c] = zreg[i][c] * hreg[i][c] + (1.0f - zreg[i][c]) * ht[c];  // dcrnn.py:190-192
            }
            const float4 hv = make_float4(hn[0], hn[1], hn[2], hn[3]);
            st4(S + r * LD + c0, hv);
            st4(p.out + (obase + r) * OUT + c0, hv);
            if (p.stash) st4(p.stash + ((obase * 3) + 2 * (long long)N + r) * OUT + c0, make_float4(ht[0], ht[1], ht[2], ht[3]));
          }
        }
      }
      if (t + 1 < T) {
        const float* xt = xw + (t + 1) * N * CIN;
        for (int idx = tid; idx < N * CIN; idx += NT) {
          const int n = idx / CIN, c = idx - n * CIN;
          S[n * LD + OUT + c] = xt[idx];
        }
      }
      __syncthreads();
    }
  }
}

struct Layout {
  DcrnnParams p;
  int smem_bytes;
};

inline int align_up(int v, int a) { return (v + a - 1) / a * a; }

// Fills the shape-derived fields and the shared-memory carve-up; returns false if it cannot fit.
bool make_layout(const stmp_plan* plan, int cin, int cout, int K, int T, Layout* L) {
  DcrnnParams& p = L->p;
  p.N = plan->n; p.CIN = cin; p.K = K; p.T = T;
  p.CP = align_up(cout + cin, 4);
  p.NB = 2 * K - 1;
  p.LD = p.NB * p.CP;
  int off = 0;
  p.off_S = off; off += align_up(p.N * p.LD * 4, 128);
  p.off_W = off; off += align_up(p.LD * 3 * cout * 4, 128);
  p.off_bias = off; off += align_up(3 * cout * 4, 128);
  // off_rowptr[0] = gstart[2N+1], off_rowptr[1] = order[2N]; off_cv[0] = padded edge entries (<= nnz + 3 per task)
  p.off_rowptr[0] = off; off += align_up((2 * p.N + 1) * 4, 16);
  p.off_rowptr[1] = off; off += align_up(2 * p.N * 4, 16);
  p.off_cv[0] = off; off += align_up((plan->fwd[0].nnz + plan->fwd[1].nnz + 6 * p.N + 4) * 8, 16);
  p.off_cv[1] = off;
  off = align_up(off, 128);
  p.x_floats = T * p.N * cin;
  for (int i = 0; i < 2; ++i) { p.off_x[i] = off; off += align_up(p.x_floats * 4, 128); }
  p.off_bar = off; off += 16;
  L->smem_bytes = off;
  return off <= kMaxSmem;
}

template <int OUT, int RT, int NW>
int launch(const Layout& L, int grid, cudaStream_t st) {
  auto kern = k_dcrnn_seq<OUT, RT, NW>;
  STMP_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L.smem_bytes));
  kern<<<grid, NW * 32, L.smem_bytes, st>>>(L.p);
  STMP_LAUNCH_OK("k_dcrnn_seq");
  // per-instance launch counter ("k_dcrnn_seq[<OUT,RT,NW>]"), so callers and tests can see which row mapping served a call
  static const int slot = [] {
    static char name[40];
    snprintf(name, sizeof(name), "k_dcrnn_seq[<%d,%d,%d>]", OUT, RT, NW);
    return path_slot(name);
  }();
  count_path(slot);
  return STMP_OK;
}

// rows covered = NW * (128/OUT) * RT
template <int OUT>
int launch_rt(const Layout& L, int grid, cudaStream_t st) {
  constexpr int RQ = 128 / OUT;
  const int n = L.p.N;
  if (n <= 8 * RQ * 1) return launch<OUT, 1, 8>(L, grid, st);
  if (n <= 8 * RQ * 2) return launch<OUT, 2, 8>(L, grid, st);
  if (n <= 8 * RQ * 4) return launch<OUT, 4, 8>(L, grid, st);
  if (n <= 8 * RQ * 7) return launch<OUT, 7, 8>(L, grid, st);
  if (n <= 16 * RQ * 4) return launch<OUT, 4, 16>(L, grid, st);
  return set_error(STMP_EUNSUPPORTED, "fused DCRNN kernel: N=%d exceeds the row capacity", n);
}

bool shape_ok(const stmp_plan* plan, int64_t cin, int64_t cout, int64_t K) {
  if (!plan || plan->flavor != STMP_FLAVOR_DCONV || plan->n_ops != 2) return false;
  if (!(cout == 16 || cout == 32)) return false;
  if (cin < 1 || cin > 4 || K < 1 || K > 4) return false;
  if (plan->n > 16 * (128 / (int)cout) * 4) return false;
  return true;
}

}  // namespace
}  // namespace stmp

using namespace stmp;

extern "C" int stmp_dcrnn_seq_supported(const stmp_plan* plan, int64_t cin, int64_t cout, int64_t K) {
  if (cout >= 1 && cout <= 4) return dcrnn_narrow_supported(plan, cin, cout, K) ? 1 : 0;   // narrow states: dcrnn_narrow.cu
  if (!shape_ok(plan, cin, cout, K)) return 0;
  if (g_dcrnn_tc && dcrnn_tc_supported(plan, cin, cout, K)) return 1;   // the wgmma kernel's envelope is wider in cin than the FFMA kernel's
  Layout L;
  return make_layout(plan, (int)cin, (int)cout, (int)K, 12, &L) ? 1 : 0;
}

extern "C" int stmp_dcrnn_seq_fwd(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K,
                                  const float* x, const int64_t* win_start, int64_t x_bstride, int64_t x_tstride,
                                  const float* w_z, const float* w_r, const float* w_h, const float* b_z,
                                  const float* b_r, const float* b_h, const float* h0, float* out, float* stash,
                                  const void* wimage, void* workspace, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_dcrnn_seq_fwd: plan is NULL");
  STMP_REQUIRE(plan->flavor == STMP_FLAVOR_DCONV, STMP_EINVAL, "stmp_dcrnn_seq_fwd: plan is not a DConv plan");
  STMP_REQUIRE(B >= 0 && T >= 0, STMP_EINVAL, "stmp_dcrnn_seq_fwd: negative B/T");
  STMP_REQUIRE(K > 0, STMP_EINVAL, "K must be > 0");  // assert K > 0, dcrnn.py:23
  STMP_REQUIRE(x && w_z && w_r && w_h && out, STMP_EINVAL, "stmp_dcrnn_seq_fwd: NULL tensor");
  if (cout >= 1 && cout <= 4) {   // narrow states (the reference's BatchedDCRNN(F, F, K) training model): dcrnn_narrow.cu
    if (!dcrnn_narrow_supported(plan, cin, cout, K))
      return set_error(STMP_EUNSUPPORTED, "narrow DCRNN kernel supports cin in 1..4, K in 1..4 and graphs whose layout fits shared memory "
                       "(got N=%d cin=%lld cout=%lld K=%lld)", plan->n, (long long)cin, (long long)cout, (long long)K);
    if (B == 0 || T == 0) return STMP_OK;
    return dcrnn_narrow_launch(plan, B, T, cin, cout, K, x, reinterpret_cast<const long long*>(win_start), x_bstride, x_tstride, w_z, w_r,
                               w_h, b_z, b_r, b_h, h0, out, stash, (cudaStream_t)stream);
  }
  if (!shape_ok(plan, cin, cout, K))
    return set_error(STMP_EUNSUPPORTED, "fused DCRNN kernel supports N<=256 (cout 32), cin<=4, cout in {16,32}, K<=4 (got N=%d cin=%lld cout=%lld K=%lld)",
                     plan->n, (long long)cin, (long long)cout, (long long)K);
  if (B == 0 || T == 0) return STMP_OK;
  // tensor-core variant unless disabled (stmp_set_option("dcrnn_tc", 0)) or outside its envelope
  if (g_dcrnn_tc && dcrnn_tc_supported(plan, cin, cout, K))
    return dcrnn_tc_launch(plan, B, T, cin, x, reinterpret_cast<const long long*>(win_start), x_bstride, x_tstride, w_z, w_r, w_h,
                           b_z, b_r, b_h, h0, out, stash, wimage, workspace, (cudaStream_t)stream);
  STMP_REQUIRE(T * (long long)plan->n * cin < (1ll << 24), STMP_ESHAPE, "window too long for the shared-memory X buffer");
  Layout L;
  if (!make_layout(plan, (int)cin, (int)cout, (int)K, (int)T, &L))
    return set_error(STMP_EUNSUPPORTED, "fused DCRNN kernel needs %d B of shared memory (> %d)", L.smem_bytes, kMaxSmem);
  DcrnnParams& p = L.p;
  p.B = B;
  for (int op = 0; op < 2; ++op) {
    p.rowptr[op] = plan->fwd[op].rowptr;
    p.cv[op] = plan->fwd[op].cv;
    p.nnz[op] = plan->fwd[op].nnz;
  }
  p.x = x; p.win_start = reinterpret_cast<const long long*>(win_start); p.x_bstride = x_bstride; p.x_tstride = x_tstride;
  p.w[0] = w_z; p.w[1] = w_r; p.w[2] = w_h;
  p.bias[0] = b_z; p.bias[1] = b_r; p.bias[2] = b_h;
  p.h0 = h0; p.out = out; p.stash = stash;
  // TMA bulk copies need a contiguous window, 16-byte aligned start and size
  const long long row_elems = (long long)plan->n * cin;
  bool tma = (x_tstride == row_elems) && ((p.x_floats * 4) % 16 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
  if (win_start) tma = tma && ((row_elems * 4) % 16 == 0);
  else tma = tma && ((x_bstride * 4) % 16 == 0);
  p.use_tma = tma ? 1 : 0;
  int dev = 0, sms = 0;
  STMP_CUDA_OK(cudaGetDevice(&dev));
  STMP_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  int grid = (int)(B < sms ? B : sms);
  cudaStream_t st = (cudaStream_t)stream;
  const int rc = cout == 16 ? launch_rt<16>(L, grid, st) : launch_rt<32>(L, grid, st);
  if (rc == STMP_OK && !p.use_tma) { static const int slotp = path_slot("k_dcrnn_seq[x-plain]"); count_path(slotp); }
  return rc;
}

extern "C" int stmp_gru_seq_supported(const stmp_plan* plan, int n_ops, int64_t cin, int64_t cout) {
  if (!plan || n_ops < 0 || n_ops > 2 || n_ops > plan->n_ops || cout != 32) return 0;
  return gru_tc_supported(plan, cin, n_ops) ? 1 : 0;
}

extern "C" int stmp_gru_seq_fwd(const stmp_plan* plan, int n_ops, int64_t B, int64_t T, int64_t cin, const float* x,
                                const int64_t* win_start, int64_t x_bstride, int64_t x_tstride, const float* wcat,
                                const float* bcat, const float* h0, int64_t h0_bstride, float* out, float* stash,
                                const void* wimage, void* workspace, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_gru_seq_fwd: plan is NULL");
  STMP_REQUIRE(n_ops >= 0 && n_ops <= 2 && n_ops <= plan->n_ops, STMP_EINVAL, "stmp_gru_seq_fwd: n_ops=%d not available in this plan", n_ops);
  STMP_REQUIRE(B >= 0 && T >= 0, STMP_EINVAL, "stmp_gru_seq_fwd: negative B/T");
  STMP_REQUIRE(x && wcat && bcat && out, STMP_EINVAL, "stmp_gru_seq_fwd: NULL tensor");
  if (!gru_tc_supported(plan, cin, n_ops))
    return set_error(STMP_EUNSUPPORTED, "fused graph-GRU kernel supports N<=207, cin<=4, cout=32 (got N=%d cin=%lld)", plan->n, (long long)cin);
  if (B == 0 || T == 0) return STMP_OK;
  return gru_tc_launch(plan, n_ops, B, T, cin, x, reinterpret_cast<const long long*>(win_start), x_bstride, x_tstride, wcat, bcat, h0,
                       h0_bstride, out, stash, wimage, workspace, (cudaStream_t)stream);
}

extern "C" int64_t stmp_gru_weight_image_bytes(void) { return tc_weight_image_bytes(); }
extern "C" int64_t stmp_seq_workspace_bytes(const stmp_plan* plan, int64_t T, int64_t cin) {
  return (plan && T > 0 && cin > 0) ? tc_workspace_bytes(plan, T, cin) : 0;
}

extern "C" int stmp_dcrnn_pack_weights(int64_t cin, int64_t cout, int64_t K, const float* w_z, const float* w_r, const float* w_h,
                                       const float* b_z, const float* b_r, const float* b_h, void* image, void* stream) {
  STMP_REQUIRE(w_z && w_r && w_h && image, STMP_EINVAL, "stmp_dcrnn_pack_weights: NULL pointer");
  if (cout != 32 || K != 2 || cin < 1 || cin > 4)
    return set_error(STMP_EUNSUPPORTED, "weight images exist for the wgmma kernel only (cout=32, K=2, cin<=4)");
  return tc_pack_weight_image(nullptr, nullptr, w_z, w_r, w_h, b_z, b_r, b_h, (int)cin, image, (cudaStream_t)stream);
}

extern "C" int stmp_gru_pack_weights(const float* wcat, const float* bcat, void* image, void* stream) {
  STMP_REQUIRE(wcat && bcat && image, STMP_EINVAL, "stmp_gru_pack_weights: NULL pointer");
  return tc_pack_weight_image(wcat, bcat, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 4, image, (cudaStream_t)stream);
}
