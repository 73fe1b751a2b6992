// train.cu -- the two pieces of a DCRNN training step that sit between the recurrence kernels and the collective:
//
//   k_dcrnn_wgrad (+ _reduce)   weight / bias gradients of the three gates over ALL (t, b, n) rows: dW = S^T dpre, db = 1^T dpre, for
//                               the stacked bases S1 / S2 written by k_dcrnn_bwd_basis and the d pre-activations streamed out by
//                               k_dcrnn_bwd_seq.  What autograd records for the `torch.matmul(basis, W)` / `+ bias` of
//                               torch_geometric_temporal/nn/recurrent/dcrnn.py:86-111 once per step, per gate, per diffusion hop.
//                               The contraction axis is the long one (T*B*N rows = 159 k at the reference's batch size), the output is
//                               102 x 96: every CTA takes a strided set of 16-row tiles (TMA bulk copies, four stages), keeps an 8 x 8
//                               register tile per thread (4 LDS.128 per 64 FFMA) and writes ONE partial; a second launch sums the
//                               partials in a fixed order (deterministic) and scatters them straight into the (2, K, C, Co) weight
//                               gradients (block 0 of the stack feeds W[0,0] and W[1,0]).
//   k_adam_flat                 torch.optim.Adam's update (examples/indexBatching/DCRNN/pems_ddp.py:90,104-121) over the ONE flat
//                               parameter / gradient buffer of distributed.FlatGradSync: one launch instead of the ~35 of the
//                               capturable foreach implementation; the step counter lives on the device (CUDA-graph replay), the
//                               gradient average over ranks and the zeroing of the gradient buffer are folded in.
#include "rows.cuh"

namespace stmp {
int wgrad_tc_launch(int c3, long long rows, int ld, const float* S1, const float* S2, const float* dpzr, const float* dph, float* partial,
                    int max_parts, cudaStream_t st, int* parts);
namespace {

constexpr int kWgTK = 16;            // rows per staged tile
constexpr int kWgStages = 4;         // tiles in flight per CTA: 3 x 19 KB x 2 CTAs per SM keeps ~115 KB per SM on the wire (2 stages of 32 rows were load-latency bound)
constexpr int kWgThreads = 192;      // >= 12 * ceil(3C/8) for cin <= 4
constexpr int kCo = 32;

struct WgradParams {
  const float* S1; const float* S2; const float* dpzr; const float* dph;
  long long rows;
  int ld, n_tiles, MG;
  float* partial;                    // [grid][MG*8*(64+N2) + 64+N2]
};

__device__ __forceinline__ float4 ld4s(const float* p) { return *reinterpret_cast<const float4*>(p); }

// N2 = the column count of the second operand: 32 for the GRU cells (S2^T dph), 64 for the LSTM cell (S^T [dpc | dpo]).
template <int N2>
__global__ void __launch_bounds__(kWgThreads, 2) k_dcrnn_wgrad(WgradParams p) {
  extern __shared__ __align__(128) unsigned char smraw[];
  const int ld = p.ld, tid = threadIdx.x, MG = p.MG;
  const int stage_floats = kWgTK * (2 * ld + 2 * kCo + N2);
  float* stages = reinterpret_cast<float*>(smraw);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smraw + (size_t)kWgStages * stage_floats * 4);
  if (tid == 0) {
    for (int i = 0; i < kWgStages; ++i) mbar_init(&bars[i], 1);
    fence_mbar_init();
  }
  __syncthreads();

  auto issue = [&](int tile, int s) {
    const long long r0 = (long long)tile * kWgTK;
    const int nr = (int)((p.rows - r0) < kWgTK ? (p.rows - r0) : kWgTK);
    float* st = stages + (size_t)s * stage_floats;
    const uint32_t bs = (uint32_t)nr * ld * 4u, bzr = (uint32_t)nr * 2 * kCo * 4u, bh = (uint32_t)nr * N2 * 4u;
    mbar_arrive_expect_tx(&bars[s], 2 * bs + bzr + bh);
    tma_bulk_g2s(st, p.S1 + r0 * ld, bs, &bars[s]);
    tma_bulk_g2s(st + kWgTK * ld, p.S2 + r0 * ld, bs, &bars[s]);
    tma_bulk_g2s(st + 2 * kWgTK * ld, p.dpzr + r0 * 2 * kCo, bzr, &bars[s]);
    tma_bulk_g2s(st + 2 * kWgTK * ld + kWgTK * 2 * kCo, p.dph + r0 * N2, bh, &bars[s]);
  };

  // roles: threads [0, 8 MG) own the 8x8 tiles of S1^T dpzr (MG x 8 tiles), threads [8 MG, (8 + N2/8) MG) those of S2^T dph (MG x N2/8)
  constexpr int NG2 = N2 / 8;
  const int n1 = 8 * MG, n2 = NG2 * MG;
  const bool prod = tid >= n1;
  const bool active = tid < n1 + n2;
  const int u = prod ? tid - n1 : tid;
  constexpr int LG2 = N2 == 64 ? 3 : 2;
  const int mg = prod ? (u >> LG2) : (u >> 3), ng = prod ? (u & (NG2 - 1)) : (u & 7);
  const int a_off = (prod ? kWgTK * ld : 0) + 8 * mg;
  const int b_off = 2 * kWgTK * ld + (prod ? kWgTK * 2 * kCo : 0) + 8 * ng;
  const int b_pitch = prod ? N2 : 2 * kCo;

  float acc[8][8], bsum[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    bsum[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  }
  if (tid == 0) {
    for (int q = 0; q < kWgStages - 1; ++q)
      if ((int)blockIdx.x + q * (int)gridDim.x < p.n_tiles) issue(blockIdx.x + q * gridDim.x, q);
  }
  int it = 0;
  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x, ++it) {
    const int s = it % kWgStages;
    // the stage refilled here was consumed in iteration it - 1 and released by the barrier at its end
    if (tid == 0 && tile + (kWgStages - 1) * (int)gridDim.x < p.n_tiles) issue(tile + (kWgStages - 1) * gridDim.x, (it + kWgStages - 1) % kWgStages);
    mbar_wait(&bars[s], (it / kWgStages) & 1);
    if (active) {
      const long long r0 = (long long)tile * kWgTK;
      const int nr = (int)((p.rows - r0) < kWgTK ? (p.rows - r0) : kWgTK);
      const float* A = stages + (size_t)s * stage_floats + a_off;
      const float* Bp = stages + (size_t)s * stage_floats + b_off;
#pragma unroll 4
      for (int k = 0; k < nr; ++k) {
        const float4 a0 = ld4s(A + k * ld), a1 = ld4s(A + k * ld + 4);
        const float4 b0 = ld4s(Bp + k * b_pitch), b1 = ld4s(Bp + k * b_pitch + 4);
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        if (mg == 0) {
#pragma unroll
          for (int j = 0; j < 8; ++j) bsum[j] += b[j];
        }
      }
    }
    __syncthreads();
  }
  if (active) {
    float* out = p.partial + (size_t)blockIdx.x * ((size_t)MG * 8 * (2 * kCo + N2) + 2 * kCo + N2);
    float* o = prod ? out + (size_t)MG * 8 * 2 * kCo : out;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float4* q = reinterpret_cast<float4*>(o + (size_t)(8 * mg + i) * b_pitch + 8 * ng);
      q[0] = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      q[1] = make_float4(acc[i][4], acc[i][5], acc[i][6], acc[i][7]);
    }
    if (mg == 0) {
      float4* q = reinterpret_cast<float4*>(out + (size_t)MG * 8 * (2 * kCo + N2) + (prod ? 2 * kCo : 0) + 8 * ng);
      q[0] = make_float4(bsum[0], bsum[1], bsum[2], bsum[3]);
      q[1] = make_float4(bsum[4], bsum[5], bsum[6], bsum[7]);
    }
  }
}

// Sum the partials in a fixed order (fixed_order_sum, rows.cuh; a block covers 32 consecutive outputs) and scatter: gate weights
// W (2, 2, C, Co) <- stacked rows (block 0 -> W[0,0] and W[1,0]; block 1 + o -> W[o,1]).
__global__ void __launch_bounds__(256) k_dcrnn_wgrad_reduce(int parts, int MG, int C, const float* __restrict__ partial, float* __restrict__ gz,
                                                            float* __restrict__ gr, float* __restrict__ gh, float* __restrict__ gbz,
                                                            float* __restrict__ gbr, float* __restrict__ gbh) {
  __shared__ float sub[8][32];
  const int per_w = 4 * C * kCo, total = 3 * per_w + 3 * kCo;
  const int x = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + x;
  const size_t stride = (size_t)MG * 8 * 3 * kCo + 3 * kCo;
  size_t src = 0;
  float* dst = nullptr;
  if (i < 3 * per_w) {
    const int gate = i / per_w, r = i - gate * per_w;            // 0 = z, 1 = r, 2 = h
    const int o = r / (2 * C * kCo), r2 = r - o * 2 * C * kCo, k = r2 / (C * kCo), r3 = r2 - k * C * kCo, c = r3 / kCo, j = r3 - c * kCo;
    const int m = (k == 0 ? 0 : 1 + o) * C + c;
    src = gate == 2 ? (size_t)MG * 8 * 2 * kCo + (size_t)m * kCo + j : (size_t)m * 2 * kCo + gate * kCo + j;
    dst = (gate == 0 ? gz : gate == 1 ? gr : gh) + r;
  } else if (i < total) {
    const int b = i - 3 * per_w;                                 // bias sums are stored z | r | h
    src = (size_t)MG * 8 * 3 * kCo + b;
    float* base = b < kCo ? gbz : (b < 2 * kCo ? gbr : gbh);
    dst = base ? base + (b & (kCo - 1)) : nullptr;
  }
  const float t = fixed_order_sum(partial + src, stride, parts, dst != nullptr, sub);
  if (w == 0 && dst) *dst = t;
}

// The same fixed-order sum for the generic graph-GRU (bases [U | Op_0 U | ..] of nb = n_ops + 1 blocks), scattered straight into the layout
// of the forward's prepacked weights: dwcat [96][112] (row gate*32 + o; columns H | Op0 H | Op1 H | X | Op0 X | Op1 X | pad -- zero for absent
// operators, absent X channels and the padding) and dbcat [96] (nullable).
__global__ void __launch_bounds__(256) k_gru_wgrad_reduce(int parts, int MG, int cin, int nb, const float* __restrict__ partial,
                                                          float* __restrict__ dwcat, float* __restrict__ dbcat) {
  __shared__ float sub[8][32];
  const int C = cin + kCo;
  const int x = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + x;
  const size_t stride = (size_t)MG * 8 * 3 * kCo + 3 * kCo;
  size_t src = 0;
  float* dst = nullptr;
  bool zero = false;
  if (i < 96 * 112) {
    const int row = i / 112, col = i - row * 112, gate = row >> 5, o = row & 31;
    const int blk = col < 96 ? col >> 5 : (col - 96) >> 2, c = col < 96 ? cin + (col & 31) : (col - 96) & 3;
    dst = dwcat + i;
    zero = blk >= nb || (col >= 96 && c >= cin);
    const int m = blk * C + c;                                   // column of the basis
    src = gate == 2 ? (size_t)MG * 8 * 2 * kCo + (size_t)m * kCo + o : (size_t)m * 2 * kCo + gate * kCo + o;
  } else if (i < 96 * 112 + 3 * kCo) {
    const int b = i - 96 * 112;                                  // bias sums are stored z | r | h
    src = (size_t)MG * 8 * 3 * kCo + b;
    dst = dbcat ? dbcat + b : nullptr;
  }
  const float t = fixed_order_sum(partial + src, stride, parts, dst && !zero, sub);
  if (w == 0 && dst) *dst = zero ? 0.f : t;
}

// ---- Adam over one flat buffer -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_adam_flat(long long n, float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                                                   float* __restrict__ v, float* step, unsigned* ticket, float lr, float b1, float b2,
                                                   float eps, float wd, float gscale, int zero_grad) {
  __shared__ float s_c[2];
  if (threadIdx.x == 0) {
    const double t = (double)*step + 1.0;                        // every block reads the counter before the last one to finish bumps it
    s_c[0] = (float)((double)lr / (1.0 - pow((double)b1, t)));
    s_c[1] = (float)sqrt(1.0 - pow((double)b2, t));
  }
  __syncthreads();
  const float step_size = s_c[0], bc2 = s_c[1], w1 = 1.f - b1, w2 = 1.f - b2;
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    float gi = g[i] * gscale;
    const float pi = p[i];
    if (wd != 0.f) gi = fmaf(wd, pi, gi);
    const float mi = fmaf(w1, gi - m[i], m[i]);                  // exp_avg.lerp_(grad, 1 - beta1)
    const float vi = fmaf(w2 * gi, gi, v[i] * b2);               // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value = 1 - beta2)
    const float denom = sqrtf(vi) / bc2 + eps;
    m[i] = mi; v[i] = vi;
    p[i] = pi - step_size * (mi / denom);
    if (zero_grad) g[i] = 0.f;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(ticket, 1u) == gridDim.x - 1) { *step += 1.f; *ticket = 0u; __threadfence(); }
  }
}

}  // namespace
}  // namespace stmp

using namespace stmp;

extern "C" int64_t stmp_dcrnn_bwd_wgrad_workspace_bytes(int64_t cin) {
  const int64_t MG = (3 * (cin + kCo) + 7) / 8;
  return (int64_t)wgrad_ffma_max_parts() * (MG * 8 * 3 * kCo + 3 * kCo) * 4;
}

extern "C" int stmp_dcrnn_bwd_wgrad(int64_t cin, int64_t cout, int64_t K, int64_t rows, int64_t ld, const float* S1, const float* S2,
                                    const float* dpzr, const float* dph, void* workspace, float* gz, float* gr, float* gh, float* gbz,
                                    float* gbr, float* gbh, void* stream) {
  STMP_REQUIRE(S1 && S2 && dpzr && dph && workspace && gz && gr && gh && rows >= 0, STMP_EINVAL, "stmp_dcrnn_bwd_wgrad: bad argument");
  STMP_REQUIRE(K == 2 && cout == kCo && cin >= 1 && cin <= 4, STMP_EUNSUPPORTED, "stmp_dcrnn_bwd_wgrad: K = 2, cout = 32, cin <= 4 only");
  const int C = (int)(cin + cout), MG = (3 * C + 7) / 8;
  STMP_REQUIRE(ld == 8 * MG, STMP_EINVAL, "stmp_dcrnn_bwd_wgrad: the basis row pitch must be 3(cin+cout) rounded up to 8");
  cudaStream_t st = (cudaStream_t)stream;
  if (rows == 0) {                                   // nothing to contract: the gradients are zero
    const size_t wbytes = (size_t)4 * C * kCo * 4;
    STMP_CUDA_OK(cudaMemsetAsync(gz, 0, wbytes, st));
    STMP_CUDA_OK(cudaMemsetAsync(gr, 0, wbytes, st));
    STMP_CUDA_OK(cudaMemsetAsync(gh, 0, wbytes, st));
    if (gbz) STMP_CUDA_OK(cudaMemsetAsync(gbz, 0, kCo * 4, st));
    if (gbr) STMP_CUDA_OK(cudaMemsetAsync(gbr, 0, kCo * 4, st));
    if (gbh) STMP_CUDA_OK(cudaMemsetAsync(gbh, 0, kCo * 4, st));
    return STMP_OK;
  }
  float* partial = reinterpret_cast<float*>(workspace);
  int parts = 0;
  const int rc = g_wgrad_tc ? wgrad_tc_launch(3 * C, rows, (int)ld, S1, S2, dpzr, dph, partial, wgrad_ffma_max_parts(), st, &parts)
                            : wgrad_ffma_launch(kCo, rows, (int)ld, S1, S2, dpzr, dph, partial, st, &parts);
  if (rc != STMP_OK) return rc;
  const int total = 3 * 4 * C * kCo + 3 * kCo;
  k_dcrnn_wgrad_reduce<<<(total + 31) / 32, 256, 0, st>>>(parts, MG, C, partial, gz, gr, gh, gbz, gbr, gbh);
  STMP_LAUNCH_OK("k_dcrnn_wgrad_reduce");
  return STMP_OK;
}

extern "C" int64_t stmp_gru_bwd_wgrad_workspace_bytes(int n_ops, int64_t cin) {
  const int64_t MG = ((n_ops + 1) * (cin + kCo) + 7) / 8;
  return (int64_t)wgrad_ffma_max_parts() * (MG * 8 * 3 * kCo + 3 * kCo) * 4;
}

extern "C" int stmp_gru_bwd_wgrad(int n_ops, int64_t cin, int64_t rows, int64_t ld, const float* S1, const float* S2, const float* dpzr,
                                  const float* dph, void* workspace, float* dwcat, float* dbcat, void* stream) {
  STMP_REQUIRE(S1 && S2 && dpzr && dph && workspace && dwcat && rows >= 0, STMP_EINVAL, "stmp_gru_bwd_wgrad: bad argument");
  STMP_REQUIRE(n_ops >= 0 && n_ops <= 2 && cin >= 1 && cin <= 4, STMP_EUNSUPPORTED, "stmp_gru_bwd_wgrad: n_ops <= 2, cin <= 4 only");
  const int C = (int)cin + kCo, C3 = (n_ops + 1) * C, MG = (C3 + 7) / 8;
  STMP_REQUIRE(ld == 8 * MG, STMP_ESHAPE, "stmp_gru_bwd_wgrad: the basis row pitch must be (n_ops+1)(cin+32) rounded up to 8");
  cudaStream_t st = (cudaStream_t)stream;
  if (rows == 0) {                                   // nothing to contract: the gradients are zero
    STMP_CUDA_OK(cudaMemsetAsync(dwcat, 0, (size_t)96 * 112 * 4, st));
    if (dbcat) STMP_CUDA_OK(cudaMemsetAsync(dbcat, 0, (size_t)96 * 4, st));
    return STMP_OK;
  }
  float* partial = reinterpret_cast<float*>(workspace);
  int parts = 0;
  const int rc = wgrad_tc_launch(C3, rows, (int)ld, S1, S2, dpzr, dph, partial, wgrad_ffma_max_parts(), st, &parts);
  if (rc != STMP_OK) return rc;
  const int total = 96 * 112 + 3 * kCo;
  k_gru_wgrad_reduce<<<(total + 31) / 32, 256, 0, st>>>(parts, MG, (int)cin, n_ops + 1, partial, dwcat, dbcat);
  STMP_LAUNCH_OK("k_gru_wgrad_reduce");
  return STMP_OK;
}

namespace stmp {
int wgrad_ffma_max_parts() {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return 2 * sms;
}

int wgrad_ffma_launch(int n2, long long rows, int ld, const float* S1, const float* S2, const float* A, const float* B, float* partial,
                      cudaStream_t st, int* parts) {
  WgradParams p;
  p.S1 = S1; p.S2 = S2; p.dpzr = A; p.dph = B; p.rows = rows; p.ld = ld; p.MG = ld / 8;
  p.n_tiles = (int)((rows + kWgTK - 1) / kWgTK);
  p.partial = partial;
  int grid = wgrad_ffma_max_parts();
  if (p.n_tiles < grid) grid = p.n_tiles > 0 ? p.n_tiles : 1;
  const int smem = kWgStages * kWgTK * (2 * ld + 2 * kCo + n2) * 4 + 64;
  if (n2 == 64) {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_dcrnn_wgrad<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k_dcrnn_wgrad<64><<<grid, kWgThreads, smem, st>>>(p);
  } else {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_dcrnn_wgrad<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k_dcrnn_wgrad<32><<<grid, kWgThreads, smem, st>>>(p);
  }
  STMP_LAUNCH_OK("k_dcrnn_wgrad");
  *parts = grid;
  return STMP_OK;
}
}  // namespace stmp

extern "C" int stmp_adam_flat(int64_t n, float* param, float* grad, float* exp_avg, float* exp_avg_sq, float* step, void* ticket, float lr,
                              float beta1, float beta2, float eps, float weight_decay, float grad_scale, int zero_grad, void* stream) {
  STMP_REQUIRE(n >= 0 && param && grad && exp_avg && exp_avg_sq && step && ticket, STMP_EINVAL, "stmp_adam_flat: bad argument");
  if (n == 0) return STMP_OK;
  long long blocks = (n + 255) / 256;
  if (blocks > 1184) blocks = 1184;
  k_adam_flat<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(n, param, grad, exp_avg, exp_avg_sq, step, reinterpret_cast<unsigned*>(ticket),
                                                                  lr, beta1, beta2, eps, weight_decay, grad_scale, zero_grad);
  STMP_LAUNCH_OK("k_adam_flat");
  return STMP_OK;
}
