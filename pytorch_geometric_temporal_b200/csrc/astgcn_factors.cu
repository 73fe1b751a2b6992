// astgcn_factors.cu -- the small-matrix front of an ASTGCN block in ONE launch (nn/attention/astgcn.py): temporal attention
// (TemporalAttention.forward :311-328), X~ = X E (:427-430) and the two (B,N,T) factors of the spatial attention (:245-256)
//     E      = softmax_dim1( Ve @ sigmoid( ((X^T U1) U2) @ (U3 X) + be ) )                       (B, T, T)
//     lhs_s  = ((X~ W1) W2)          (B, N, T)            rhs_s = (W3 X~)^T                        (B, T, N)
// which the reference (and round 1 of this engine) runs as ~25 matmul / permute / pointwise launches per block.  X~ is never
// materialised: by linearity  (X~ W1)[n,f] = sum_t X[n,t,f] (E W1)[t]   and   (W3 X~)[n,u] = sum_t (W3 . X[n,t,:]) E[t,u].
// One CTA per batch row; X[b] (channels-last (N, T, F)) is streamed twice (the second pass hits L2), everything else lives in shared
// memory.  Bytes: 2 x 4*N*T*F read, 8*N*T written; the N x N products downstream are stmp_spatial_attention_fwd's job.
#include "common.cuh"

namespace stmp {
namespace {

struct FactorArgs {
  int N, T, F;
  const float* x;       // [B][N][T][F]
  const float* U1;      // [N]
  const float* U2;      // [F][N]
  const float* U3;      // [F]
  const float* be;      // [T][T]
  const float* Ve;      // [T][T]
  const float* W1;      // [T]
  const float* W2;      // [F][T]
  const float* W3;      // [F]
  float* lhs_s;         // [B][N][T]
  float* rhs_s;         // [B][T][N]
  float* E_out;         // [B][T][T] or null
};

constexpr int FA_NT = 512;
constexpr int FA_TMAX = 12;

__device__ __forceinline__ float sigmoid_a(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }

// LPR lanes share a node's rows; each lane owns VEC consecutive features: F == LPR * VEC
template <int LPR, int VEC>
__global__ void __launch_bounds__(FA_NT) k_astgcn_factors(const FactorArgs a) {
  extern __shared__ __align__(16) float sm[];
  const int N = a.N, T = a.T, F = a.F;
  float* Rt = sm;                    // [N][T]  U3 . X[n,t,:]
  float* Xw3 = Rt + N * T;           // [N][T]  W3 . X[n,t,:]
  float* LHS = Xw3 + N * T;          // [T][N]
  float* lhs1 = LHS + N * T;         // [T][F]
  float* Em = lhs1 + T * F;          // [T][T] prod -> sigmoid -> E
  float* E0 = Em + T * T;            // [T][T] Ve @ sigmoid
  float* e1 = E0 + T * T;            // [T]
  const int tid = threadIdx.x;
  const long long b = blockIdx.x;
  const float* xb = a.x + b * (long long)N * T * F;
  constexpr int SLOTS = FA_NT / LPR;
  const int slot = tid / LPR, li = tid % LPR;

  for (int i = tid; i < T * F; i += FA_NT) lhs1[i] = 0.f;
  __syncthreads();

  // ---- pass 1: Rt, Xw3 (dot over F), lhs1 += U1[n] X[n,t,:] ------------------------------------------------------------
  {
    float u3[VEC], w3[VEC], acc[FA_TMAX][VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v) { u3[v] = __ldg(a.U3 + li * VEC + v); w3[v] = __ldg(a.W3 + li * VEC + v); }
#pragma unroll
    for (int t = 0; t < FA_TMAX; ++t)
#pragma unroll
      for (int v = 0; v < VEC; ++v) acc[t][v] = 0.f;
    for (int n0 = 0; n0 < N; n0 += SLOTS) {          // uniform trip count: the shuffles below need every lane of the warp
      const int n = n0 + slot;
      const bool nv = n < N;
      const float u1 = nv ? __ldg(a.U1 + n) : 0.f;
      // all T rows of the node are requested before the first one is used (the shuffles below would otherwise serialise the loads:
      // one HBM round trip per (node, t) -- measured 120 us of a 158 us kernel)
      float xa[FA_TMAX][VEC];
#pragma unroll
      for (int t = 0; t < FA_TMAX; ++t) {
        if (t < T) {
          const float* src = xb + ((long long)(nv ? n : 0) * T + t) * F + li * VEC;
          if (VEC == 4) {
            const float4 q = __ldg(reinterpret_cast<const float4*>(src));
            xa[t][0] = q.x; xa[t][1 % VEC] = q.y; xa[t][2 % VEC] = q.z; xa[t][3 % VEC] = q.w;
          } else {
#pragma unroll
            for (int v = 0; v < VEC; ++v) xa[t][v] = __ldg(src + v);
          }
        }
      }
#pragma unroll
      for (int t = 0; t < FA_TMAX; ++t) {
        if (t < T) {
          float xv[VEC];
#pragma unroll
          for (int v = 0; v < VEC; ++v) xv[v] = xa[t][v];
          float d3 = 0.f, dw = 0.f;
#pragma unroll
          for (int v = 0; v < VEC; ++v) {
            d3 = fmaf(u3[v], xv[v], d3);
            dw = fmaf(w3[v], xv[v], dw);
            acc[t][v] = fmaf(u1, xv[v], acc[t][v]);
          }
#pragma unroll
          for (int o = LPR / 2; o > 0; o >>= 1) {
            d3 += __shfl_xor_sync(0xffffffffu, d3, o);
            dw += __shfl_xor_sync(0xffffffffu, dw, o);
          }
          if (li == 0 && nv) { Rt[n * T + t] = d3; Xw3[n * T + t] = dw; }
        }
      }
    }
#pragma unroll
    for (int t = 0; t < FA_TMAX; ++t)
      if (t < T)
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          float part = acc[t][v];
#pragma unroll
          for (int o = 16; o >= LPR; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);   // the slots of a warp own the same (t, f)
          if ((threadIdx.x & 31) < LPR) atomicAdd(&lhs1[t * F + li * VEC + v], part);
        }
  }
  __syncthreads();
  // ---- LHS[t][n] = sum_f lhs1[t][f] U2[f][n] ----------------------------------------------------------------------------
  // thread = node n: U2[f][n] is read once (coalesced over n, 8 loads in flight) and feeds all T rows; lhs1 is a shared-memory broadcast
  for (int n = tid; n < N; n += FA_NT) {
    float s[FA_TMAX];
#pragma unroll
    for (int t = 0; t < FA_TMAX; ++t) s[t] = 0.f;
    for (int f0 = 0; f0 < F; f0 += 8) {
      float u[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) u[j] = (f0 + j < F) ? __ldg(a.U2 + (long long)(f0 + j) * N + n) : 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (f0 + j < F) {
#pragma unroll
          for (int t = 0; t < FA_TMAX; ++t)
            if (t < T) s[t] = fmaf(lhs1[t * F + f0 + j], u[j], s[t]);
        }
    }
#pragma unroll
    for (int t = 0; t < FA_TMAX; ++t)
      if (t < T) LHS[t * N + n] = s[t];
  }
  __syncthreads();
  // ---- prod = LHS @ Rt ; sigmoid(prod + be) ; E0 = Ve @ .. ; softmax over dim 1 (rows) ------------------------------------
  for (int idx = tid; idx < T * T; idx += FA_NT) {
    const int t = idx / T, u = idx - t * T;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    int n = 0;
    for (; n + 4 <= N; n += 4) {
      s0 = fmaf(LHS[t * N + n], Rt[n * T + u], s0);
      s1 = fmaf(LHS[t * N + n + 1], Rt[(n + 1) * T + u], s1);
      s2 = fmaf(LHS[t * N + n + 2], Rt[(n + 2) * T + u], s2);
      s3 = fmaf(LHS[t * N + n + 3], Rt[(n + 3) * T + u], s3);
    }
    for (; n < N; ++n) s0 = fmaf(LHS[t * N + n], Rt[n * T + u], s0);
    Em[idx] = sigmoid_a((s0 + s1) + (s2 + s3) + __ldg(a.be + idx));
  }
  __syncthreads();
  for (int idx = tid; idx < T * T; idx += FA_NT) {
    const int t = idx / T, u = idx - t * T;
    float s = 0.f;
    for (int k = 0; k < T; ++k) s = fmaf(__ldg(a.Ve + t * T + k), Em[k * T + u], s);
    E0[idx] = s;
  }
  __syncthreads();
  if (tid < T) {                        // column u = tid: softmax over the rows t
    const int u = tid;
    float mx = -INFINITY;
    for (int t = 0; t < T; ++t) mx = fmaxf(mx, E0[t * T + u]);
    float sum = 0.f;
    for (int t = 0; t < T; ++t) sum += __expf(E0[t * T + u] - mx);
    const float inv = 1.0f / sum;
    for (int t = 0; t < T; ++t) Em[t * T + u] = __expf(E0[t * T + u] - mx) * inv;
  }
  __syncthreads();
  if (tid < T) {                        // e1 = E @ W1
    float s = 0.f;
    for (int u = 0; u < T; ++u) s = fmaf(Em[tid * T + u], __ldg(a.W1 + u), s);
    e1[tid] = s;
  }
  if (a.E_out)
    for (int idx = tid; idx < T * T; idx += FA_NT) a.E_out[b * T * T + idx] = Em[idx];
  // ---- rhs_s[u][n] = sum_t Xw3[n][t] E[t][u] -----------------------------------------------------------------------------
  for (int idx = tid; idx < T * N; idx += FA_NT) {
    const int u = idx / N, n = idx - u * N;
    float s = 0.f;
    for (int t = 0; t < T; ++t) s = fmaf(Xw3[n * T + t], Em[t * T + u], s);
    a.rhs_s[b * (long long)T * N + idx] = s;
  }
  __syncthreads();
  // ---- pass 2: a[n][f] = sum_t X[n,t,f] e1[t] ; lhs_s[n][u] = sum_f a[n][f] W2[f][u] ---------------------------------------
  {
    float w2[VEC][FA_TMAX];
#pragma unroll
    for (int v = 0; v < VEC; ++v)
#pragma unroll
      for (int u = 0; u < FA_TMAX; ++u) w2[v][u] = u < T ? __ldg(a.W2 + (long long)(li * VEC + v) * T + u) : 0.f;
    for (int n0 = 0; n0 < N; n0 += SLOTS) {
      const int n = n0 + slot;
      const bool nv = n < N;
      float av[VEC];
#pragma unroll
      for (int v = 0; v < VEC; ++v) av[v] = 0.f;
      float xa[FA_TMAX][VEC];
#pragma unroll
      for (int t = 0; t < FA_TMAX; ++t) {
        if (t < T) {
          const float* src = xb + ((long long)(nv ? n : 0) * T + t) * F + li * VEC;
          if (VEC == 4) {
            const float4 q = __ldg(reinterpret_cast<const float4*>(src));
            xa[t][0] = q.x; xa[t][1 % VEC] = q.y; xa[t][2 % VEC] = q.z; xa[t][3 % VEC] = q.w;
          } else {
#pragma unroll
            for (int v = 0; v < VEC; ++v) xa[t][v] = __ldg(src + v);
          }
        }
      }
#pragma unroll
      for (int t = 0; t < FA_TMAX; ++t) {
        if (t < T) {
          const float et = e1[t];
#pragma unroll
          for (int v = 0; v < VEC; ++v) av[v] = fmaf(et, xa[t][v], av[v]);
        }
      }
#pragma unroll
      for (int u = 0; u < FA_TMAX; ++u) {
        if (u < T) {
          float s = 0.f;
#pragma unroll
          for (int v = 0; v < VEC; ++v) s = fmaf(av[v], w2[v][u], s);
#pragma unroll
          for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
          if (li == 0 && nv) a.lhs_s[(b * N + n) * T + u] = s;
        }
      }
    }
  }
}

template <int LPR, int VEC>
int fa_launch(const FactorArgs& a, long long B, size_t smem, cudaStream_t st) {
  STMP_CUDA_OK(cudaFuncSetAttribute(k_astgcn_factors<LPR, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  k_astgcn_factors<LPR, VEC><<<(unsigned)B, FA_NT, smem, st>>>(a);
  STMP_LAUNCH_OK("k_astgcn_factors");
  return STMP_OK;
}

}  // namespace
}  // namespace stmp

using namespace stmp;

extern "C" int stmp_astgcn_factors_fwd(int64_t B, int64_t n_nodes, int64_t n_steps, int64_t f_in, const float* x, const float* U1,
                                       const float* U2, const float* U3, const float* be, const float* Ve, const float* W1, const float* W2,
                                       const float* W3, float* lhs_s, float* rhs_s, float* E_out, void* stream) {
  STMP_REQUIRE(B >= 0 && n_nodes >= 1 && n_steps >= 1 && f_in >= 1, STMP_EINVAL, "stmp_astgcn_factors_fwd: bad sizes");
  const bool vec4 = f_in % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
  const int lpr = (int)(vec4 ? f_in / 4 : f_in);
  const size_t smem = ((size_t)3 * n_nodes * n_steps + n_steps * f_in + 2 * n_steps * n_steps + n_steps + 16) * sizeof(float);
  if (n_steps > FA_TMAX || (lpr != 1 && lpr != 2 && lpr != 4 && lpr != 8 && lpr != 16) || smem > 200 * 1024 || B > 65535)
    return set_error(STMP_EUNSUPPORTED, "fused ASTGCN factors: T <= 12, F in {1,2,4,8,16,32,64} (got T=%lld F=%lld N=%lld)", (long long)n_steps,
                     (long long)f_in, (long long)n_nodes);
  if (B == 0) return STMP_OK;
  STMP_REQUIRE(x && U1 && U2 && U3 && be && Ve && W1 && W2 && W3 && lhs_s && rhs_s, STMP_EINVAL, "stmp_astgcn_factors_fwd: NULL pointer");
  FactorArgs a;
  a.N = (int)n_nodes; a.T = (int)n_steps; a.F = (int)f_in; a.x = x; a.U1 = U1; a.U2 = U2; a.U3 = U3; a.be = be; a.Ve = Ve;
  a.W1 = W1; a.W2 = W2; a.W3 = W3; a.lhs_s = lhs_s; a.rhs_s = rhs_s; a.E_out = E_out;
  cudaStream_t st = (cudaStream_t)stream;
  if (vec4) {
    switch (lpr) {
      case 1: return fa_launch<1, 4>(a, B, smem, st);
      case 2: return fa_launch<2, 4>(a, B, smem, st);
      case 4: return fa_launch<4, 4>(a, B, smem, st);
      case 8: return fa_launch<8, 4>(a, B, smem, st);
      default: return fa_launch<16, 4>(a, B, smem, st);
    }
  }
  switch (lpr) {
    case 1: return fa_launch<1, 1>(a, B, smem, st);
    case 2: return fa_launch<2, 1>(a, B, smem, st);
    case 4: return fa_launch<4, 1>(a, B, smem, st);
    case 8: return fa_launch<8, 1>(a, B, smem, st);
    default: return fa_launch<16, 1>(a, B, smem, st);
  }
}
