// cells.cu -- K5 gate epilogues for the tiled (large-graph) path and K8 window gather.
// All HBM-bound elementwise kernels: float4-vectorised when the element count allows, grid-stride.
#include "common.cuh"

namespace stmp {
namespace {

constexpr int kT = 256;
inline unsigned grid_for(long long n) {
  long long b = (n + kT - 1) / kT;
  if (b < 1) b = 1;
  if (b > 132ll * 32) b = 132ll * 32;
  return (unsigned)b;
}

__global__ void __launch_bounds__(kT) k_gru_zr(long long n, const float* __restrict__ pz, const float* __restrict__ pr,
                                               const float* __restrict__ h, float* __restrict__ z, float* __restrict__ r,
                                               float* __restrict__ hr) {
  for (long long i = blockIdx.x * (long long)kT + threadIdx.x; i < n; i += (long long)gridDim.x * kT) {
    float zv = sigmoidf_acc(pz[i]), rv = sigmoidf_acc(pr[i]);
    z[i] = zv;
    r[i] = rv;
    hr[i] = h[i] * rv;
  }
}
__global__ void __launch_bounds__(kT) k_gru_out(long long n, const float* __restrict__ ph, const float* __restrict__ z,
                                                const float* __restrict__ h, float* __restrict__ ht, float* __restrict__ hnew) {
  for (long long i = blockIdx.x * (long long)kT + threadIdx.x; i < n; i += (long long)gridDim.x * kT) {
    float t = tanhf(ph[i]);
    float zv = z[i];
    if (ht) ht[i] = t;
    hnew[i] = zv * h[i] + (1.0f - zv) * t;
  }
}
__global__ void __launch_bounds__(kT) k_lstm_ifc(long long n, int cout, const float* __restrict__ pi, const float* __restrict__ pf,
                                                 const float* __restrict__ pc, const float* __restrict__ c,
                                                 const float* __restrict__ wci, const float* __restrict__ wcf,
                                                 const float* __restrict__ bi, const float* __restrict__ bf,
                                                 const float* __restrict__ bc, float* __restrict__ ig, float* __restrict__ fg,
                                                 float* __restrict__ tg, float* __restrict__ cnew) {
  for (long long i = blockIdx.x * (long long)kT + threadIdx.x; i < n; i += (long long)gridDim.x * kT) {
    const int ch = (int)(i % cout);
    const float cv = c[i];
    // ((conv + w_c*C) + b): the reference adds the peephole then the bias (gconv_lstm.py:171-173)
    const float iv = sigmoidf_acc(__fadd_rn(__fadd_rn(pi[i], __fmul_rn(wci[ch], cv)), bi[ch]));
    const float fv = sigmoidf_acc(__fadd_rn(__fadd_rn(pf[i], __fmul_rn(wcf[ch], cv)), bf[ch]));
    const float tv = tanhf(__fadd_rn(pc[i], bc[ch]));
    if (ig) ig[i] = iv;
    if (fg) fg[i] = fv;
    if (tg) tg[i] = tv;
    cnew[i] = __fadd_rn(__fmul_rn(fv, cv), __fmul_rn(iv, tv));
  }
}
__global__ void __launch_bounds__(kT) k_lstm_oh(long long n, int cout, const float* __restrict__ po, const float* __restrict__ cnew,
                                                const float* __restrict__ wco, const float* __restrict__ bo,
                                                float* __restrict__ og, float* __restrict__ hnew) {
  for (long long i = blockIdx.x * (long long)kT + threadIdx.x; i < n; i += (long long)gridDim.x * kT) {
    const int ch = (int)(i % cout);
    const float cv = cnew[i];
    const float ov = sigmoidf_acc(__fadd_rn(__fadd_rn(po[i], __fmul_rn(wco[ch], cv)), bo[ch]));
    if (og) og[i] = ov;
    hnew[i] = ov * tanhf(cv);
  }
}

// Gate derivatives of the peephole LSTM cell (hand-written backward of gconv_lstm.py:168-202), one thread per (row, channel).
//   pre [rows][4*Co] = pre-activations i|f|c|o of the contraction INCLUDING the ChebConv biases (recomputed by the backward GEMM),
//   c_old / c_new [rows][Co], gh = dL/dH' , gc = dL/dC' arriving from later steps (nullable);
//   dpre [rows][4*Co] = dL/d pre, dc_old [rows][Co] = dL/dC_{t-1}.
__global__ void __launch_bounds__(kT) k_lstm_gate_bwd(long long n, int cout, const float* __restrict__ pre, const float* __restrict__ c_old,
                                                      const float* __restrict__ c_new, const float* __restrict__ gh,
                                                      const float* __restrict__ gc, const float* __restrict__ wci,
                                                      const float* __restrict__ wcf, const float* __restrict__ wco,
                                                      const float* __restrict__ bi, const float* __restrict__ bf,
                                                      const float* __restrict__ bc, const float* __restrict__ bo,
                                                      float* __restrict__ dpre, float* __restrict__ dc_old) {
  for (long long i = blockIdx.x * (long long)kT + threadIdx.x; i < n; i += (long long)gridDim.x * kT) {
    const long long row = i / cout;
    const int ch = (int)(i - row * cout);
    const float* pr = pre + row * 4 * cout;
    const float co = c_old[i], cn = c_new[i];
    const float iv = sigmoidf_acc(__fadd_rn(__fadd_rn(pr[ch], __fmul_rn(wci[ch], co)), bi[ch]));
    const float fv = sigmoidf_acc(__fadd_rn(__fadd_rn(pr[cout + ch], __fmul_rn(wcf[ch], co)), bf[ch]));
    const float tv = tanhf(__fadd_rn(pr[2 * cout + ch], bc[ch]));
    const float ov = sigmoidf_acc(__fadd_rn(__fadd_rn(pr[3 * cout + ch], __fmul_rn(wco[ch], cn)), bo[ch]));
    const float tc = tanhf(cn);
    const float g = gh ? gh[i] : 0.f;
    const float dpo = g * tc * ov * (1.0f - ov);
    const float dcn = (gc ? gc[i] : 0.f) + g * ov * (1.0f - tc * tc) + dpo * wco[ch];
    const float dpi = dcn * tv * iv * (1.0f - iv);
    const float dpf = dcn * co * fv * (1.0f - fv);
    const float dpc = dcn * iv * (1.0f - tv * tv);
    float* dp = dpre + row * 4 * cout;
    dp[ch] = dpi;
    dp[cout + ch] = dpf;
    dp[2 * cout + ch] = dpc;
    dp[3 * cout + ch] = dpo;
    dc_old[i] = dcn * fv + dpi * wci[ch] + dpf * wcf[ch];
  }
}

// x[b, t, :] = series[start[b] + t, :]  for t in [0,h);  y[b, t, :] = series[start[b] + h + t, :]
template <typename V>
__global__ void __launch_bounds__(kT) k_window_gather(const V* __restrict__ series, long long row_v, const long long* __restrict__ start,
                                                      long long B, int h, V* __restrict__ x, V* __restrict__ y) {
  const long long per = (long long)h * row_v;
  const long long total = B * per * (y ? 2 : 1);
  for (long long i = blockIdx.x * (long long)kT + threadIdx.x; i < total; i += (long long)gridDim.x * kT) {
    const long long half = i / (B * per);
    const long long j = i - half * B * per;
    const long long b = j / per, o = j - b * per;
    const V v = series[(start[b] + half * h) * row_v + o];
    (half ? y : x)[j] = v;
  }
}


// ---- reverse-time GRU gate derivatives (hand-written backward of the DCRNN sequence, dcrnn.py:172-192) -------------
// One thread per (b, n, c), c < Co.  `close` finishes step t+1 (dH_t+1 -> dH_t, dX_{t+1}), `open` starts step t
// (g_t = dL/dH_t, d pre-activation of the candidate); both halves are optional so one kernel serves the first step,
// the steady state and the final flush.
struct GruBwdCarry {
  long long total; int N, Ci, Co; long long du_ld;
  const float* g_prev; const float* z_prev; const float* r_prev; const float* du2; const float* du1;
  float* dx; long long dx_bs;
  const float* gout; long long gout_bs; const float* z; const float* ht; long long stash_bs;
  float* g; float* dph; float* dh_out;
};
__global__ void __launch_bounds__(kT) k_gru_bwd_carry(GruBwdCarry p) {
  const int Co = p.Co, Ci = p.Ci;
  const long long per = (long long)p.N * Co;
  for (long long i = blockIdx.x * (long long)kT + threadIdx.x; i < p.total; i += (long long)gridDim.x * kT) {
    const long long b = i / per, rem = i - b * per;
    const int n = (int)(rem / Co), c = (int)(rem - (long long)n * Co);
    float dh = 0.f;
    if (p.g_prev) {
      const long long row = (b * p.N + n) * p.du_ld;
      const float dhr = p.du2[row + Ci + c];
      dh = p.g_prev[i] * p.z_prev[b * p.stash_bs + rem] + dhr * p.r_prev[b * p.stash_bs + rem] + p.du1[row + Ci + c];
      if (p.dx)
        for (int ci = c; ci < Ci; ci += Co) p.dx[b * p.dx_bs + (long long)n * Ci + ci] = p.du2[row + ci] + p.du1[row + ci];
    }
    if (p.dh_out) p.dh_out[i] = dh;
    if (p.gout) {
      const float g = p.gout[b * p.gout_bs + rem] + dh;
      const float z = p.z[b * p.stash_bs + rem], ht = p.ht[b * p.stash_bs + rem];
      p.g[i] = g;
      p.dph[i] = g * (1.f - z) * (1.f - ht * ht);
    }
  }
}
// d pre-activations of the update and reset gates at step t:  dpz = g (H_{t-1} - Ht) Z (1-Z),  dpr = dHR H_{t-1} R (1-R)
__global__ void __launch_bounds__(kT) k_gru_bwd_zr(long long total, int N, int Ci, int Co, long long du_ld, const float* __restrict__ g,
                                                   const float* __restrict__ hprev, long long hprev_bs, const float* __restrict__ z,
                                                   const float* __restrict__ r, const float* __restrict__ ht, long long stash_bs,
                                                   const float* __restrict__ du2, float* __restrict__ dpzr) {
  const long long per = (long long)N * Co;
  for (long long i = blockIdx.x * (long long)kT + threadIdx.x; i < total; i += (long long)gridDim.x * kT) {
    const long long b = i / per, rem = i - b * per;
    const int n = (int)(rem / Co), c = (int)(rem - (long long)n * Co);
    const float hp = hprev ? hprev[b * hprev_bs + rem] : 0.f;
    const float zv = z[b * stash_bs + rem], rv = r[b * stash_bs + rem], hv = ht[b * stash_bs + rem];
    const float dhr = du2[(b * N + n) * du_ld + Ci + c];
    float* o = dpzr + (b * N + n) * 2 * Co;
    o[c] = g[i] * (hp - hv) * zv * (1.f - zv);
    o[Co + c] = dhr * hp * rv * (1.f - rv);
  }
}


// ---- masked MAE of the index-batching examples (examples/indexBatching/DCRNN/utils.py:10-18) -----------------------
//   mask = (y != 0); mask /= mean(mask); loss = mean(nan_to_zero(|p - y| * mask))   ==   sum_i nz(|p_i-y_i| m_i) / sum_i m_i
// Deterministic two-stage reduction (per-block partials, then one block in fixed order).
constexpr int kMaeBlocks = 512;
__global__ void __launch_bounds__(kT) k_masked_mae_partial(long long n, const float* __restrict__ p, const float* __restrict__ y,
                                                           float* __restrict__ part) {
  float s = 0.f, m = 0.f;
  for (long long i = blockIdx.x * (long long)kT + threadIdx.x; i < n; i += (long long)gridDim.x * kT) {
    const float yy = y[i], t = fabsf(p[i] - yy);
    if (yy != 0.f) { m += 1.f; if (t == t) s += t; }         // NaN terms are zeroed (utils.py:16), masked-out terms are 0
  }
  __shared__ float ss[kT / 32], sm[kT / 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); m += __shfl_xor_sync(0xffffffffu, m, o); }
  if ((threadIdx.x & 31) == 0) { ss[threadIdx.x >> 5] = s; sm[threadIdx.x >> 5] = m; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < kT / 32; ++w) { a += ss[w]; b += sm[w]; }
    part[2 * blockIdx.x] = a; part[2 * blockIdx.x + 1] = b;
  }
}
__global__ void k_masked_mae_final(int blocks, const float* __restrict__ part, float* __restrict__ loss, float* __restrict__ s0) {
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int i = 0; i < blocks; ++i) { a += part[2 * i]; b += part[2 * i + 1]; }
    *s0 = b;
    *loss = b > 0.f ? a / b : 0.f;                            // mean(mask) == 0 -> every term is NaN -> zeroed -> loss 0
  }
}
__global__ void __launch_bounds__(kT) k_masked_mae_bwd(long long n, const float* __restrict__ p, const float* __restrict__ y,
                                                       const float* __restrict__ s0, const float* __restrict__ gout,
                                                       float* __restrict__ gp) {
  const float b = *s0, scale = b > 0.f ? *gout / b : 0.f;
  for (long long i = blockIdx.x * (long long)kT + threadIdx.x; i < n; i += (long long)gridDim.x * kT) {
    const float yy = y[i], d = p[i] - yy;
    float g = 0.f;
    if (yy != 0.f && d == d) g = d > 0.f ? scale : (d < 0.f ? -scale : 0.f);
    gp[i] = g;
  }
}

// ---- transposed stacked DConv weights for the backward kernels: W (2,K,C,Co) -> rows of W_stacked^T ------------------
// stacked block 0 = W[0,0] + W[1,0]; block 1+2(k-1)+o = W[o,k]  (nn/recurrent/dcrnn.py::_stack_weight)
__global__ void __launch_bounds__(kT) k_pack_bwd_weights(int C, int Co, int K, const float* __restrict__ wz, const float* __restrict__ wr,
                                                         const float* __restrict__ wh, float* __restrict__ whsT, float* __restrict__ wzrT) {
  const int nbC = (2 * K - 1) * C, total = 3 * Co * nbC;
  for (int i = blockIdx.x * kT + threadIdx.x; i < total; i += gridDim.x * kT) {
    const int gate = i / (Co * nbC), r = i - gate * Co * nbC, o = r / nbC, col = r - o * nbC, blk = col / C, c = col - blk * C;
    const float* w = gate == 0 ? wh : (gate == 1 ? wz : wr);
    float v;
    if (blk == 0) v = w[((0 * K + 0) * C + c) * Co + o] + w[((1 * K + 0) * C + c) * Co + o];
    else { const int dir = (blk - 1) & 1, k = 1 + ((blk - 1) >> 1); v = w[((dir * K + k) * C + c) * Co + o]; }
    if (gate == 0) whsT[o * nbC + col] = v;
    else wzrT[((gate - 1) * Co + o) * nbC + col] = v;
  }
}

}  // namespace
}  // namespace stmp

using namespace stmp;

extern "C" int stmp_gru_zr(int64_t n, const float* pz, const float* pr, const float* h, float* z, float* r, float* hr,
                           void* stream) {
  STMP_REQUIRE(n >= 0 && pz && pr && h && z && r && hr, STMP_EINVAL, "stmp_gru_zr: bad argument");
  if (n == 0) return STMP_OK;
  k_gru_zr<<<grid_for(n), kT, 0, (cudaStream_t)stream>>>(n, pz, pr, h, z, r, hr);
  STMP_LAUNCH_OK("k_gru_zr");
  return STMP_OK;
}
extern "C" int stmp_gru_out(int64_t n, const float* ph, const float* z, const float* h, float* ht, float* hnew,
                            void* stream) {
  STMP_REQUIRE(n >= 0 && ph && z && h && hnew, STMP_EINVAL, "stmp_gru_out: bad argument");
  if (n == 0) return STMP_OK;
  k_gru_out<<<grid_for(n), kT, 0, (cudaStream_t)stream>>>(n, ph, z, h, ht, hnew);
  STMP_LAUNCH_OK("k_gru_out");
  return STMP_OK;
}
extern "C" int stmp_lstm_ifc(int64_t rows, int64_t cout, const float* pi, const float* pf, const float* pc, const float* c,
                             const float* wci, const float* wcf, const float* bi, const float* bf, const float* bc,
                             float* i, float* f, float* t, float* cnew, void* stream) {
  STMP_REQUIRE(rows >= 0 && cout > 0 && pi && pf && pc && c && wci && wcf && bi && bf && bc && cnew, STMP_EINVAL,
               "stmp_lstm_ifc: bad argument");
  if (rows == 0) return STMP_OK;
  k_lstm_ifc<<<grid_for(rows * cout), kT, 0, (cudaStream_t)stream>>>(rows * cout, (int)cout, pi, pf, pc, c, wci, wcf, bi,
                                                                      bf, bc, i, f, t, cnew);
  STMP_LAUNCH_OK("k_lstm_ifc");
  return STMP_OK;
}
extern "C" int stmp_lstm_oh(int64_t rows, int64_t cout, const float* po, const float* cnew, const float* wco,
                            const float* bo, float* o, float* hnew, void* stream) {
  STMP_REQUIRE(rows >= 0 && cout > 0 && po && cnew && wco && bo && hnew, STMP_EINVAL, "stmp_lstm_oh: bad argument");
  if (rows == 0) return STMP_OK;
  k_lstm_oh<<<grid_for(rows * cout), kT, 0, (cudaStream_t)stream>>>(rows * cout, (int)cout, po, cnew, wco, bo, o, hnew);
  STMP_LAUNCH_OK("k_lstm_oh");
  return STMP_OK;
}
extern "C" int stmp_lstm_gate_bwd(int64_t rows, int64_t cout, const float* pre, const float* c_old, const float* c_new, const float* gh,
                                  const float* gc, const float* wci, const float* wcf, const float* wco, const float* bi, const float* bf,
                                  const float* bc, const float* bo, float* dpre, float* dc_old, void* stream) {
  STMP_REQUIRE(rows >= 0 && cout > 0, STMP_EINVAL, "stmp_lstm_gate_bwd: bad size");
  STMP_REQUIRE(pre && c_old && c_new && wci && wcf && wco && bi && bf && bc && bo && dpre && dc_old, STMP_EINVAL, "stmp_lstm_gate_bwd: NULL tensor");
  if (rows == 0) return STMP_OK;
  k_lstm_gate_bwd<<<grid_for(rows * cout), kT, 0, (cudaStream_t)stream>>>(rows * cout, (int)cout, pre, c_old, c_new, gh, gc, wci, wcf, wco, bi,
                                                                        bf, bc, bo, dpre, dc_old);
  STMP_LAUNCH_OK("k_lstm_gate_bwd");
  return STMP_OK;
}

extern "C" int stmp_window_gather(const float* series, int64_t t_total, int64_t row_elems, const int64_t* start, int64_t B,
                                  int64_t horizon, float* x, float* y, void* stream) {
  STMP_REQUIRE(series && start && x, STMP_EINVAL, "stmp_window_gather: NULL pointer");
  STMP_REQUIRE(B >= 0 && horizon > 0 && row_elems > 0 && t_total >= (y ? 2 : 1) * horizon, STMP_EINVAL,
               "stmp_window_gather: bad sizes");
  if (B == 0) return STMP_OK;
  const long long total = B * horizon * row_elems * (y ? 2 : 1);
  auto al = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (row_elems % 4 == 0 && al(series) && al(x) && (!y || al(y))) {
    k_window_gather<float4><<<grid_for(total / 4), kT, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const float4*>(series), row_elems / 4, (const long long*)start, B, (int)horizon,
        reinterpret_cast<float4*>(x), reinterpret_cast<float4*>(y));
  } else {
    k_window_gather<float><<<grid_for(total), kT, 0, (cudaStream_t)stream>>>(series, row_elems, (const long long*)start, B,
                                                                              (int)horizon, x, y);
  }
  STMP_LAUNCH_OK("k_window_gather");
  return STMP_OK;
}

extern "C" int stmp_gru_bwd_carry(int64_t B, int64_t N, int64_t cin, int64_t cout, int64_t du_ld, const float* g_prev,
                                  const float* z_prev, const float* r_prev, const float* du2, const float* du1, float* dx,
                                  int64_t dx_bstride, const float* gout, int64_t gout_bstride, const float* z, const float* ht,
                                  int64_t stash_bstride, float* g, float* dph, float* dh_out, void* stream) {
  STMP_REQUIRE(B >= 0 && N > 0 && cin >= 0 && cout > 0 && du_ld >= cin + cout, STMP_EINVAL, "stmp_gru_bwd_carry: bad sizes");
  STMP_REQUIRE(!g_prev || (z_prev && r_prev && du2 && du1), STMP_EINVAL, "stmp_gru_bwd_carry: incomplete `close` operands");
  STMP_REQUIRE(!gout || (z && ht && g && dph), STMP_EINVAL, "stmp_gru_bwd_carry: incomplete `open` operands");
  STMP_REQUIRE(g_prev || gout, STMP_EINVAL, "stmp_gru_bwd_carry: nothing to do");
  if (B == 0) return STMP_OK;
  GruBwdCarry p;
  p.total = B * N * cout; p.N = (int)N; p.Ci = (int)cin; p.Co = (int)cout; p.du_ld = du_ld;
  p.g_prev = g_prev; p.z_prev = z_prev; p.r_prev = r_prev; p.du2 = du2; p.du1 = du1; p.dx = dx; p.dx_bs = dx_bstride;
  p.gout = gout; p.gout_bs = gout_bstride; p.z = z; p.ht = ht; p.stash_bs = stash_bstride; p.g = g; p.dph = dph; p.dh_out = dh_out;
  k_gru_bwd_carry<<<grid_for(p.total), kT, 0, (cudaStream_t)stream>>>(p);
  STMP_LAUNCH_OK("k_gru_bwd_carry");
  return STMP_OK;
}
extern "C" int stmp_gru_bwd_zr(int64_t B, int64_t N, int64_t cin, int64_t cout, int64_t du_ld, const float* g, const float* hprev,
                               int64_t hprev_bstride, const float* z, const float* r, const float* ht, int64_t stash_bstride,
                               const float* du2, float* dpzr, void* stream) {
  STMP_REQUIRE(B >= 0 && N > 0 && cin >= 0 && cout > 0 && du_ld >= cin + cout && g && z && r && ht && du2 && dpzr, STMP_EINVAL,
               "stmp_gru_bwd_zr: bad argument");
  if (B == 0) return STMP_OK;
  k_gru_bwd_zr<<<grid_for(B * N * cout), kT, 0, (cudaStream_t)stream>>>(B * N * cout, (int)N, (int)cin, (int)cout, du_ld, g, hprev,
                                                                         hprev_bstride, z, r, ht, stash_bstride, du2, dpzr);
  STMP_LAUNCH_OK("k_gru_bwd_zr");
  return STMP_OK;
}

extern "C" int64_t stmp_masked_mae_workspace_floats(void) { return 2 * kMaeBlocks; }
extern "C" int stmp_masked_mae_fwd(int64_t n, const float* pred, const float* target, float* workspace, float* loss, float* s0,
                                   void* stream) {
  STMP_REQUIRE(n >= 0 && pred && target && workspace && loss && s0, STMP_EINVAL, "stmp_masked_mae_fwd: bad argument");
  int blocks = (int)((n + kT - 1) / kT);
  if (blocks < 1) blocks = 1;
  if (blocks > kMaeBlocks) blocks = kMaeBlocks;
  k_masked_mae_partial<<<blocks, kT, 0, (cudaStream_t)stream>>>(n, pred, target, workspace);
  STMP_LAUNCH_OK("k_masked_mae_partial");
  k_masked_mae_final<<<1, 32, 0, (cudaStream_t)stream>>>(blocks, workspace, loss, s0);
  STMP_LAUNCH_OK("k_masked_mae_final");
  return STMP_OK;
}
extern "C" int stmp_masked_mae_bwd(int64_t n, const float* pred, const float* target, const float* s0, const float* gout,
                                   float* gpred, void* stream) {
  STMP_REQUIRE(n >= 0 && pred && target && s0 && gout && gpred, STMP_EINVAL, "stmp_masked_mae_bwd: bad argument");
  if (n == 0) return STMP_OK;
  k_masked_mae_bwd<<<grid_for(n), kT, 0, (cudaStream_t)stream>>>(n, pred, target, s0, gout, gpred);
  STMP_LAUNCH_OK("k_masked_mae_bwd");
  return STMP_OK;
}
extern "C" int stmp_dcrnn_pack_bwd_weights(int64_t cin, int64_t cout, int64_t K, const float* wz, const float* wr, const float* wh,
                                           float* whsT, float* wzrT, void* stream) {
  STMP_REQUIRE(cin >= 0 && cout > 0 && K > 0 && wz && wr && wh && whsT && wzrT, STMP_EINVAL, "stmp_dcrnn_pack_bwd_weights: bad argument");
  const long long total = 3 * cout * (2 * K - 1) * (cin + cout);
  k_pack_bwd_weights<<<grid_for(total), kT, 0, (cudaStream_t)stream>>>((int)(cin + cout), (int)cout, (int)K, wz, wr, wh, whsT, wzrT);
  STMP_LAUNCH_OK("k_pack_bwd_weights");
  return STMP_OK;
}
