// gru_rows.cu -- the generic graph-GRU cell (out = 32, n_ops <= 1: GConvGRU K <= 2) on graphs of ANY size, split over CTAs by destination
// rows (DESIGN §4i).  One graph, one step per call; the two all-to-all dependencies of a step -- Op(H*R) in the forward and Op^T(.) in the
// backward -- split a cell into a short chain of launches, each a gather + contraction + gate math fused per row:
//
//   forward, H given   k_gru_rows_fwd_a<1>  gather Op[X | H]; Z, R, H*R and the X half of the candidate pre-activation -> scratch
//                      k_gru_rows_fwd_b     gather Op(H*R); pre_h, Ht = tanh(pre_h), H' = Z*H + (1-Z)*Ht
//   forward, H = None  k_gru_rows_fwd_a<0>  gather Op X; Z and H' = (1-Z)*tanh(pre_h) (R is dead: H*R = 0)
//   backward           k_gru_rows_bwd_a     dph, dpz and dS2 = dph W_h^T (rowwise)
//                      k_gru_rows_bwd_b     gather Op^T of dS2's H*R block: d(H*R), dpr, dS1 = [dpz | dpr] W_zr^T, the own-row dH / dX
//                      k_gru_rows_bwd_c     gather Op^T of the operator blocks of dS1 (+ dS2's X columns): dH, dX complete
//
// Mapping: one warp per destination row, lane = output channel (and X channel for lane < cin); a CTA owns tiles of kRowTile consecutive
// rows (grid-strided) and stages the weights it needs in shared memory once.  The contraction is exact fp32 FFMA: every basis value is
// broadcast with a shuffle and multiplied into the lane's column of the staged weights (pitch 97: the lane-indexed rows and the
// lane-indexed columns are both free of bank conflicts).  Gathers walk the plan's CSR rows in entry order with separate multiply and
// add, as stmp_spmm does.  No atomics anywhere; every result depends on its row alone, so repeated calls are bit-identical.
#include "rows.cuh"

namespace stmp {
namespace {

using namespace rows;
constexpr int kScrPitch = 192;               // backward scratch row: dS2 (96) | Op^T operand Q (96)
constexpr int kFwdScrPitch = 96;             // forward scratch row: H*R | X half of pre_h | Z

struct RowsFwd {
  const int* rowptr; const int2* cv;         // operator 0 by destination (n_ops = 1)
  int n, cin, nops, nb;                      // nb = (nops + 1)(cin + 32) basis columns
  const float* x; const float* h;            // (N, cin), (N, 32) or NULL (H = None)
  const float* w; const float* b;            // packed [96][nb], [96]
  float* out;                                // (N, 32)
  float* scr;                                // (N, 96)  H given
  float* stash;                              // (3, N, 32) Z | R | Ht, nullable
  float* S1; float* S2; int ld;              // (N, ld) weight-gradient bases, nullable
};

// HAS_H = 1: launch A of the two-launch forward.  HAS_H = 0: the whole H = None cell.
template <bool HAS_H>
__global__ void __launch_bounds__(kRowsThreads, 2) k_gru_rows_fwd_a(RowsFwd a) {
  extern __shared__ float ws[];              // [96][kWPitch]
  stage_w(ws, a.w, a.nb, 0, 96);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + kCo;
  const float bz = __ldg(a.b + lane), br = __ldg(a.b + kCo + lane), bh = __ldg(a.b + 2 * kCo + lane);
  const size_t NC = (size_t)a.n * kCo;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const float xv = lane < cin ? __ldg(a.x + (size_t)i * cin + lane) : 0.f;
      const float hv = HAS_H ? __ldg(a.h + (size_t)i * kCo + lane) : 0.f;
      float lh = 0.f, lx = 0.f;
      if (a.nops) gather_row<HAS_H>(a.rowptr, a.cv, i, a.h, kCo, a.x, cin, cin, lane, lh, lx);
      float pz = bz, pr = br, ph = bh;       // pre = b + [U | Op U] W^T in basis order; ph takes the X columns only here
      for (int blk = 0; blk <= a.nops; ++blk) {
        const float sx = blk ? lx : xv, sh = blk ? lh : hv;
        const float* wb = ws + blk * C;
        for (int c = 0; c < cin; ++c) {
          const float s = __shfl_sync(0xffffffffu, sx, c);
          pz = fmaf(s, wb[lane * kWPitch + c], pz);
          if (HAS_H) pr = fmaf(s, wb[(kCo + lane) * kWPitch + c], pr);
          ph = fmaf(s, wb[(2 * kCo + lane) * kWPitch + c], ph);
        }
        if (HAS_H) {
#pragma unroll 8
          for (int o = 0; o < kCo; ++o) {
            const float s = __shfl_sync(0xffffffffu, sh, o);
            pz = fmaf(s, wb[lane * kWPitch + cin + o], pz);
            pr = fmaf(s, wb[(kCo + lane) * kWPitch + cin + o], pr);
          }
        }
      }
      const float Z = sigmoidf_acc(pz);
      if (HAS_H) {
        const float R = sigmoidf_acc(pr), hr = hv * R;
        float* s = a.scr + (size_t)i * kFwdScrPitch;
        s[lane] = hr;
        s[kCo + lane] = ph;
        s[2 * kCo + lane] = Z;
        if (a.stash) {
          a.stash[(size_t)i * kCo + lane] = Z;
          a.stash[NC + (size_t)i * kCo + lane] = R;
        }
        if (a.S2) a.S2[(size_t)i * a.ld + cin + lane] = hr;
      } else {
        const float Ht = tanhf(ph), hn = (1.f - Z) * Ht;
        a.out[(size_t)i * kCo + lane] = hn;
        if (a.stash) {
          a.stash[(size_t)i * kCo + lane] = Z;
          a.stash[2 * NC + (size_t)i * kCo + lane] = Ht;
        }
      }
      if (a.S1) {                            // [X | H | Op X | Op H] (+ zero padding); H = None: H columns zero
        float* r1 = a.S1 + (size_t)i * a.ld;
        if (lane < cin) r1[lane] = xv;
        r1[cin + lane] = hv;
        if (a.nops) {
          if (lane < cin) r1[C + lane] = lx;
          r1[C + cin + lane] = lh;
        }
        if (a.nb + lane < a.ld) r1[a.nb + lane] = 0.f;
        if (HAS_H && a.S2) {                 // S2's X columns and padding; H*R above, Op(H*R) in launch B
          float* r2 = a.S2 + (size_t)i * a.ld;
          if (lane < cin) r2[lane] = xv;
          if (a.nops && lane < cin) r2[C + lane] = lx;
          if (a.nb + lane < a.ld) r2[a.nb + lane] = 0.f;
        }
      }
    }
  }
}

__global__ void __launch_bounds__(kRowsThreads, 2) k_gru_rows_fwd_b(RowsFwd a) {
  extern __shared__ float ws[];              // candidate rows of the weights: [32][kWPitch]
  stage_w(ws, a.w, a.nb, 2 * kCo, kCo);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + kCo;
  const size_t NC = (size_t)a.n * kCo;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const float* s = a.scr + (size_t)i * kFwdScrPitch;
      const float hr = s[lane];
      float ph = s[kCo + lane], lhr = 0.f, unused;
      if (a.nops) gather_row<true>(a.rowptr, a.cv, i, a.scr, kFwdScrPitch, a.scr, kFwdScrPitch, 0, lane, lhr, unused);
      for (int blk = 0; blk <= a.nops; ++blk) {
        const float sh = blk ? lhr : hr;
        const float* wr = ws + lane * kWPitch + blk * C + cin;
#pragma unroll 8
        for (int o = 0; o < kCo; ++o) ph = fmaf(__shfl_sync(0xffffffffu, sh, o), wr[o], ph);
      }
      const float Z = s[2 * kCo + lane], hv = __ldg(a.h + (size_t)i * kCo + lane);
      const float Ht = tanhf(ph);
      a.out[(size_t)i * kCo + lane] = Z * hv + (1.f - Z) * Ht;
      if (a.stash) a.stash[2 * NC + (size_t)i * kCo + lane] = Ht;
      if (a.S2 && a.nops) a.S2[(size_t)i * a.ld + C + cin + lane] = lhr;
    }
  }
}

struct RowsBwd {
  const int* rowptr; const int2* cv;         // operator 0 by SOURCE (the transposed product)
  int n, cin, nops, nb;
  const float* gout; const float* h;         // (N, 32); h NULL for H = None
  const float* stash; const float* w;        // (3, N, 32), packed [96][nb]
  float* dph; float* dpzr;                   // (N, 32), (N, 64)
  float* scr;                                // (N, 192): dS2 | Q
  float* dx; float* dh;                      // (N, cin), (N, 32), nullable
};

// rowwise: dph, dpz (dpr = 0 when H = None), dS2 = dph W_h^T -> scratch; H = None: also dS1 = [dpz | 0] W_zr^T and the X gradient's own row
// and its Op^T operand (the X columns of both bases).
template <bool HAS_H>
__global__ void __launch_bounds__(kRowsThreads, 2) k_gru_rows_bwd_a(RowsBwd a) {
  extern __shared__ float ws[];              // [96][kWPitch]
  stage_w(ws, a.w, a.nb, 0, 96);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + kCo;
  const size_t NC = (size_t)a.n * kCo;
  const bool need_ds = HAS_H || a.dx != nullptr;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const size_t io = (size_t)i * kCo + lane;
      const float g = a.gout[io], Z = a.stash[io], Ht = a.stash[2 * NC + io];
      const float hp = HAS_H ? a.h[io] : 0.f;
      const float dph = g * (1.f - Z) * (1.f - Ht * Ht);
      const float dpz = g * (hp - Ht) * Z * (1.f - Z);
      a.dph[io] = dph;
      a.dpzr[(size_t)i * 2 * kCo + lane] = dpz;
      if (!HAS_H) a.dpzr[(size_t)i * 2 * kCo + kCo + lane] = 0.f;
      if (!need_ds) continue;
      float d2[3] = {0.f, 0.f, 0.f}, d1[3] = {0.f, 0.f, 0.f};      // basis columns m = lane + 32 q
#pragma unroll 4
      for (int o = 0; o < kCo; ++o) {
        const float s2 = __shfl_sync(0xffffffffu, dph, o);
        const float s1 = HAS_H ? 0.f : __shfl_sync(0xffffffffu, dpz, o);
#pragma unroll
        for (int q = 0; q < 3; ++q) {
          d2[q] = fmaf(s2, ws[(2 * kCo + o) * kWPitch + lane + 32 * q], d2[q]);
          if (!HAS_H) d1[q] = fmaf(s1, ws[o * kWPitch + lane + 32 * q], d1[q]);
        }
      }
      float* sr = a.scr + (size_t)i * kScrPitch;
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int m = lane + 32 * q;
        if (m >= a.nb) continue;
        if (HAS_H) {
          sr[m] = d2[q];
        } else {                             // only the X columns carry a gradient
          const float v = d2[q] + d1[q];
          if (m < cin) a.dx[(size_t)i * cin + m] = v;
          else if (m >= C && m < C + cin) sr[kScrPitch / 2 + m - C] = v;
        }
      }
    }
  }
}

// H given: gather Op^T of dS2's H*R block -> d(H*R), dpr, dS1 = [dpz | dpr] W_zr^T; the own-row parts of dH and dX; Q = the Op^T operand of
// the final gather (dS1's operator block, plus dS2's operator-block X columns).
__global__ void __launch_bounds__(kRowsThreads, 2) k_gru_rows_bwd_b(RowsBwd a) {
  extern __shared__ float ws[];              // z | r rows: [64][kWPitch], then one 96-float row buffer per warp
  stage_w(ws, a.w, a.nb, 0, 2 * kCo);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin, C = cin + kCo;
  float* sb = ws + 2 * kCo * kWPitch + warp * 96;
  const size_t NC = (size_t)a.n * kCo;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int j = t0 + warp; j < t1; j += kRowsWarps) {
      const size_t io = (size_t)j * kCo + lane;
      const float* sr = a.scr + (size_t)j * kScrPitch;
      float dhr = sr[cin + lane];
      if (a.nops) {
        float t, unused;
        gather_row<true>(a.rowptr, a.cv, j, a.scr + C + cin, kScrPitch, a.scr, kScrPitch, 0, lane, t, unused);
        dhr += t;
      }
      const float g = a.gout[io], Z = a.stash[io], R = a.stash[NC + io], hp = a.h[io];
      const float dpr = dhr * hp * R * (1.f - R);
      const float dpz = a.dpzr[(size_t)j * 2 * kCo + lane];
      a.dpzr[(size_t)j * 2 * kCo + kCo + lane] = dpr;
      float d1[3] = {0.f, 0.f, 0.f};
#pragma unroll 4
      for (int o = 0; o < kCo; ++o) {
        const float sz = __shfl_sync(0xffffffffu, dpz, o), sp = __shfl_sync(0xffffffffu, dpr, o);
#pragma unroll
        for (int q = 0; q < 3; ++q)
          d1[q] = fmaf(sp, ws[(kCo + o) * kWPitch + lane + 32 * q], fmaf(sz, ws[o * kWPitch + lane + 32 * q], d1[q]));
      }
#pragma unroll
      for (int q = 0; q < 3; ++q) sb[lane + 32 * q] = d1[q];
      __syncwarp();
      if (a.dh) a.dh[io] = g * Z + dhr * R + sb[cin + lane];
      if (a.dx && lane < cin) a.dx[(size_t)j * cin + lane] = sr[lane] + sb[lane];
      if (a.nops)
        for (int c = lane; c < C; c += 32) a.scr[(size_t)j * kScrPitch + kScrPitch / 2 + c] = sb[C + c] + (c < cin ? sr[C + c] : 0.f);
      __syncwarp();
    }
  }
}

// dH += Op^T Q[:, cin:], dX += Op^T Q[:, :cin]  (either nullable)
__global__ void __launch_bounds__(kRowsThreads) k_gru_rows_bwd_c(RowsBwd a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, cin = a.cin;
  const float* q = a.scr + kScrPitch / 2;
  for (int t0 = blockIdx.x * kRowTile; t0 < a.n; t0 += gridDim.x * kRowTile) {
    const int t1 = min(t0 + kRowTile, a.n);
    for (int j = t0 + warp; j < t1; j += kRowsWarps) {
      float th, tx;
      if (a.dh) gather_row<true>(a.rowptr, a.cv, j, q + cin, kScrPitch, q, kScrPitch, a.dx ? cin : 0, lane, th, tx);
      else gather_row<false>(a.rowptr, a.cv, j, q + cin, kScrPitch, q, kScrPitch, cin, lane, th, tx);
      if (a.dh) a.dh[(size_t)j * kCo + lane] += th;
      if (a.dx && lane < cin) a.dx[(size_t)j * cin + lane] += tx;
    }
  }
}

// w [96][nb]: row gate*32 + o, column m = blk*(cin+32) + c of the basis [X | H | Op X | Op H]; b [96] = bx + bh (zeros without biases)
__global__ void k_gru_rows_pack(int nops, int cin, const float* __restrict__ wx, const float* __restrict__ wh, const float* __restrict__ bx,
                                const float* __restrict__ bh, float* __restrict__ w, float* __restrict__ b) {
  const int C = cin + kCo, nbk = nops + 1, nb = nbk * C;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 96 * nb) {
    const int row = i / nb, m = i - row * nb, gate = row >> 5, o = row & 31, blk = m / C, c = m - blk * C;
    w[i] = c < cin ? wx[(((size_t)gate * nbk + blk) * kCo + o) * cin + c] : wh[(((size_t)gate * nbk + blk) * kCo + o) * kCo + c - cin];
  } else if (i < 96 * nb + 96) {
    const int r = i - 96 * nb;
    b[r] = bx ? bx[r] + bh[r] : 0.f;
  }
}

}  // namespace
}  // namespace stmp

using namespace stmp;

static bool rows_supported(const stmp_plan* plan, int n_ops, int64_t cin, int64_t cout) {
  return plan && n_ops >= 0 && n_ops <= 1 && n_ops <= plan->n_ops && cout == kCo && cin >= 1 && cin <= kMaxCin;
}

extern "C" int stmp_gru_rows_supported(const stmp_plan* plan, int n_ops, int64_t cin, int64_t cout) {
  return rows_supported(plan, n_ops, cin, cout) ? 1 : 0;
}

extern "C" int stmp_gru_rows_pack_weights(int n_ops, int64_t cin, const float* wx, const float* wh, const float* bx, const float* bh,
                                          float* w, float* b, void* stream) {
  STMP_REQUIRE(wx && wh && w && b, STMP_EINVAL, "stmp_gru_rows_pack_weights: NULL tensor");
  STMP_REQUIRE(!bx == !bh, STMP_EINVAL, "stmp_gru_rows_pack_weights: give both bias stacks or neither");
  STMP_REQUIRE(n_ops >= 0 && n_ops <= 1 && cin >= 1 && cin <= kMaxCin, STMP_EUNSUPPORTED, "stmp_gru_rows_pack_weights: n_ops <= 1, cin 1..16 only");
  const int total = 96 * (n_ops + 1) * ((int)cin + kCo) + 96;
  k_gru_rows_pack<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n_ops, (int)cin, wx, wh, bx, bh, w, b);
  STMP_LAUNCH_OK("k_gru_rows_pack");
  return STMP_OK;
}

extern "C" int stmp_gru_rows_fwd(const stmp_plan* plan, int n_ops, int64_t cin, const float* x, const float* h, const float* w, const float* b,
                                 float* scratch, float* out, float* stash, float* S1, float* S2, int64_t ld, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_gru_rows_fwd: plan is NULL");
  STMP_REQUIRE(rows_supported(plan, n_ops, cin, kCo), STMP_EUNSUPPORTED,
               "stmp_gru_rows_fwd: n_ops <= min(1, plan's operators), cin 1..16 only (n_ops=%d, cin=%lld)", n_ops, (long long)cin);
  STMP_REQUIRE(x && w && b && out && (!h || scratch), STMP_EINVAL, "stmp_gru_rows_fwd: NULL tensor");
  STMP_REQUIRE(!S2 || (S1 && h), STMP_EINVAL, "stmp_gru_rows_fwd: S2 needs S1 and h (H = None: S2 = S1)");
  const int nb = (n_ops + 1) * ((int)cin + kCo);
  STMP_REQUIRE(!S1 || ld == (nb + 7) / 8 * 8, STMP_ESHAPE, "stmp_gru_rows_fwd: the basis row pitch must be (n_ops+1)(cin+32) rounded up to 8");
  const void* ps[] = {x, h, w, b, scratch, out, stash, S1, S2};
  for (const void* p : ps) STMP_REQUIRE(al4(p), STMP_ESHAPE, "stmp_gru_rows_fwd: misaligned tensor");
  STMP_REQUIRE(!S1 || (((uintptr_t)S1 | (uintptr_t)S2) & 15u) == 0, STMP_ESHAPE, "stmp_gru_rows_fwd: S1 / S2 must be 16-byte aligned");
  if (plan->n == 0) return STMP_OK;
  RowsFwd a;
  a.rowptr = plan->fwd[0].rowptr; a.cv = plan->fwd[0].cv;
  a.n = plan->n; a.cin = (int)cin; a.nops = n_ops; a.nb = nb;
  a.x = x; a.h = h; a.w = w; a.b = b; a.out = out; a.scr = scratch; a.stash = stash; a.S1 = S1; a.S2 = S2; a.ld = (int)ld;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = rows_grid(plan->n), smem = 96 * kWPitch * 4;
  if (h) {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_gru_rows_fwd_a<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k_gru_rows_fwd_a<true><<<grid, kRowsThreads, smem, st>>>(a);
    STMP_LAUNCH_OK("k_gru_rows_fwd_a");
    k_gru_rows_fwd_b<<<grid, kRowsThreads, kCo * kWPitch * 4, st>>>(a);
    STMP_LAUNCH_OK("k_gru_rows_fwd_b");
  } else {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_gru_rows_fwd_a<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k_gru_rows_fwd_a<false><<<grid, kRowsThreads, smem, st>>>(a);
    STMP_LAUNCH_OK("k_gru_rows_fwd_a");
  }
  return STMP_OK;
}

extern "C" int64_t stmp_gru_rows_scratch_bytes(const stmp_plan* plan) {
  return plan ? (int64_t)plan->n * kScrPitch * 4 : 0;
}

extern "C" int stmp_gru_rows_bwd(const stmp_plan* plan, int n_ops, int64_t cin, const float* gout, const float* h, const float* stash,
                                 const float* w, float* scratch, float* dph, float* dpzr, float* dx, float* dh, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_gru_rows_bwd: plan is NULL");
  STMP_REQUIRE(rows_supported(plan, n_ops, cin, kCo), STMP_EUNSUPPORTED,
               "stmp_gru_rows_bwd: n_ops <= min(1, plan's operators), cin 1..16 only (n_ops=%d, cin=%lld)", n_ops, (long long)cin);
  STMP_REQUIRE(gout && stash && w && scratch && dph && dpzr, STMP_EINVAL, "stmp_gru_rows_bwd: NULL tensor");
  STMP_REQUIRE(h || !dh, STMP_EINVAL, "stmp_gru_rows_bwd: dh needs h (H = None has no state gradient)");
  const void* ps[] = {gout, h, stash, w, scratch, dph, dpzr, dx, dh};
  for (const void* p : ps) STMP_REQUIRE(al4(p), STMP_ESHAPE, "stmp_gru_rows_bwd: misaligned tensor");
  if (plan->n == 0) return STMP_OK;
  RowsBwd a;
  a.rowptr = plan->bwd[0].rowptr; a.cv = plan->bwd[0].cv;
  a.n = plan->n; a.cin = (int)cin; a.nops = n_ops; a.nb = (n_ops + 1) * ((int)cin + kCo);
  a.gout = gout; a.h = h; a.stash = stash; a.w = w; a.dph = dph; a.dpzr = dpzr; a.scr = scratch; a.dx = dx; a.dh = dh;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = rows_grid(plan->n), smem = 96 * kWPitch * 4, smem_b = (2 * kCo * kWPitch + kRowsWarps * 96) * 4;
  if (h) {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_gru_rows_bwd_a<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k_gru_rows_bwd_a<true><<<grid, kRowsThreads, smem, st>>>(a);
    STMP_LAUNCH_OK("k_gru_rows_bwd_a");
    k_gru_rows_bwd_b<<<grid, kRowsThreads, smem_b, st>>>(a);
    STMP_LAUNCH_OK("k_gru_rows_bwd_b");
  } else {
    STMP_CUDA_OK(cudaFuncSetAttribute(k_gru_rows_bwd_a<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k_gru_rows_bwd_a<false><<<grid, kRowsThreads, smem, st>>>(a);
    STMP_LAUNCH_OK("k_gru_rows_bwd_a");
  }
  if (n_ops && (dh || dx)) {
    k_gru_rows_bwd_c<<<grid, kRowsThreads, 0, st>>>(a);
    STMP_LAUNCH_OK("k_gru_rows_bwd_c");
  }
  return STMP_OK;
}
