// spatial_attention_tiled.cu -- ASTGCN spatial attention (nn/attention/astgcn.py SpatialAttention) for graphs too wide for one CTA row
// tile: up to 1024 nodes, the PeMS03 / PeMS07 networks.  Computes the quantity of stmp_spatial_attention_fwd (gemm_blocks.cu, MODE_SPATT):
//
//   ST[b, j, i] = softmax_dim1( Vs @ sigmoid(LHS @ RHS + bs) )[b, i, j]        rows (b, j), softmax over the columns i
//
// gemm_blocks.cu holds a 128-row tile x ALL columns in one CTA so that the softmax is thread-local in its epilogue; that stops at 320
// columns (the accumulators of 320 columns already spill).  Here the columns are tiled as well, in two launches, deterministic, no atomics:
//   k_spatt_tiles  grid (128-row tiles of (b, j)) x (column tiles of <= 256 i).  A CTA generates its A operand
//                  sigmoid(sum_t LHS[b,k,t] RHS[b,t,j] + bs[k][j]) k-block by k-block exactly as MODE_SPATT does (so A is regenerated once
//                  per column tile), splits it into fp16 hi / lo and runs the three wgmma passes lo*hi + hi*lo + hi*hi against its rows of
//                  the packed Vs^T (stmp_gemm_prepack layout, [P][P], P = nodes rounded up to 64).  It writes the unnormalised logits
//                  into ST and one (max, sum exp(l - max)) pair per (row, column tile) into the workspace.
//   k_spatt_norm   one warp per row: combines the row's tile pairs in tile order and rewrites the row as exp(l - m) / s, zero in the
//                  padding columns -- the same __expf and IEEE division as the one-CTA softmax epilogue.
#include "common.cuh"
#include "tc_common.cuh"

namespace stmp {
namespace {

constexpr int SA_NT = 256;
constexpr int SA_BM = 128;
constexpr int SA_A_BYTES = SA_BM * 128;   // one K-block of A (hi or lo): 128 rows x 64 fp16
constexpr int SA_MAXCT = 256;             // columns per CTA: 4 accumulators of m64n64 per warpgroup
constexpr int SA_NCH = SA_MAXCT / 64;
constexpr int SA_MAXN = 1024;
constexpr int SA_MAXT = 12;

struct SaParams {
  int Nn, Tn;                 // nodes, timesteps
  int Npad;                   // nodes rounded up to 64: the K extent and the column extent of the product
  int ct, ntiles;             // column tile width (% 64 == 0); tile c covers columns [c ct, min((c + 1) ct, Npad))
  const float* lhs;           // [B][Nn][Tn]
  const float* rhs;           // [B][Tn][Nn]
  const float* bsT;           // [Nn][Nn]  bsT[j][k] = bs[k][j]
  const __half* w_hi;         // [Npad][Npad]  Vs^T, row = output column i, column = k
  const __half* w_lo;
  float* st; long long ld;    // [B][Nn][ld]
  float2* part;               // [B Nn][ntiles]  (max, sum exp(l - max)) of a row's columns in one tile
};

__device__ __forceinline__ float sigmoid_g(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }

__global__ void __launch_bounds__(SA_NT, 1) k_spatt_tiles(const SaParams p) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  // every row tile lies inside one batch element (ceil(Nn/128) tiles each), so LHS addresses are warp-uniform
  const int rtiles = (p.Nn + SA_BM - 1) / SA_BM;
  const int bt = (int)(blockIdx.x / rtiles), j0 = (int)(blockIdx.x % rtiles) * SA_BM;
  const int tile = blockIdx.y, c0 = tile * p.ct, w = min(p.ct, p.Npad - c0);
  const int rows_here = min(SA_BM, p.Nn - j0);
  const int b_bytes = p.ct * 128;                    // one K-block of B (hi or lo) at the widest tile
  const int stage_bytes = 2 * SA_A_BYTES + 2 * b_bytes;
  float* red = reinterpret_cast<float*>(smem + 2 * stage_bytes);   // [2][128] epilogue exchange
  const int wg = warp >> 2, wt = tid & 127;
  const int nkb = p.Npad / 64;
  float acc[SA_NCH][32];

  // A generator: thread = 4 consecutive rows (b, j..j+3) x 8 k of every k-block; the RHS columns of my rows stay in registers
  float rj[4][SA_MAXT];
  int sj[4];
  const int r0 = lane * 4, k8 = warp * 8;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int jr = j0 + r0 + r;
    sj[r] = jr < p.Nn ? jr : p.Nn - 1;
#pragma unroll
    for (int t = 0; t < SA_MAXT; ++t) rj[r][t] = t < p.Tn ? __ldg(p.rhs + ((long long)bt * p.Tn + t) * p.Nn + sj[r]) : 0.f;
  }

  for (int kb = 0; kb < nkb; ++kb) {
    const int s = kb & 1;
    unsigned char* a_hi = smem + s * stage_bytes;
    unsigned char* a_lo = a_hi + SA_A_BYTES;
    unsigned char* b_hi = a_lo + SA_A_BYTES;
    unsigned char* b_lo = b_hi + b_bytes;
    if (kb >= 2) {  // the MMAs of k-block kb-2 must have drained this stage; those of kb-1 keep running
      wgmma_wait<1>();
      __syncthreads();
    }
    const int k0 = kb * 64;
    // B: rows c0 .. c0 + w of the packed Vs^T, k-block kb (L2-resident: every row tile reads it) -> SWIZZLE_128B by hand
    for (int base = 0; base < w * 8; base += 4 * SA_NT) {
      uint4 h[4], l[4];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int idx = base + tid + jj * SA_NT;
        if (idx < w * 8) {
          const long long g = (long long)(c0 + (idx >> 3)) * p.Npad + k0 + 8 * (idx & 7);
          h[jj] = __ldg(reinterpret_cast<const uint4*>(p.w_hi + g));
          l[jj] = __ldg(reinterpret_cast<const uint4*>(p.w_lo + g));
        }
      }
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int idx = base + tid + jj * SA_NT;
        if (idx < w * 8) {
          const int n = idx >> 3, c = idx & 7;
          const int off = n * 128 + ((c ^ (n & 7)) << 4);
          *reinterpret_cast<uint4*>(b_hi + off) = h[jj];
          *reinterpret_cast<uint4*>(b_lo + off) = l[jj];
        }
      }
    }
    // A generated: A[(b,j)][k] = sigmoid(sum_t LHS[b,k,t] RHS[b,t,j] + bsT[j][k]), zero for k >= Nn
    {
      const int Tn = p.Tn;
      float o[4][8];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const float* bsr = p.bsT + (long long)sj[r] * p.Nn + k0 + k8;
#pragma unroll
        for (int e = 0; e < 8; ++e) o[r][e] = (k0 + k8 + e < p.Nn) ? __ldg(bsr + e) : 0.f;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int k = k0 + k8 + e;
        float l[SA_MAXT];
#pragma unroll
        for (int t = 0; t < SA_MAXT; ++t) l[t] = 0.f;
        if (k < p.Nn) {
          const float* lk = p.lhs + ((long long)bt * p.Nn + k) * Tn;
          if (Tn == 12) {                              // 48-byte rows: three 16-byte broadcast loads
#pragma unroll
            for (int q4 = 0; q4 < 3; ++q4) {
              const float4 v4 = __ldg(reinterpret_cast<const float4*>(lk) + q4);
              l[4 * q4] = v4.x; l[4 * q4 + 1] = v4.y; l[4 * q4 + 2] = v4.z; l[4 * q4 + 3] = v4.w;
            }
          } else {
#pragma unroll
            for (int t = 0; t < SA_MAXT; ++t)
              if (t < Tn) l[t] = __ldg(lk + t);
          }
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          float a = o[r][e];
#pragma unroll
          for (int t = 0; t < SA_MAXT; ++t) a = fmaf(l[t], rj[r][t], a);
          o[r][e] = a;
        }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
#pragma unroll
        for (int e = 0; e < 8; ++e) o[r][e] = (k0 + k8 + e < p.Nn) ? sigmoid_g(o[r][e]) : 0.f;
        store_split4(a_hi, a_lo, r0 + r, k8, make_float4(o[r][0], o[r][1], o[r][2], o[r][3]));
        store_split4(a_hi, a_lo, r0 + r, k8 + 4, make_float4(o[r][4], o[r][5], o[r][6], o[r][7]));
      }
    }
    fence_proxy_async();        // generic-proxy operand stores -> visible to the tensor core (async proxy)
    __syncthreads();
    const uint32_t ah = smem_u32(a_hi) + wg * 64 * 128, al = smem_u32(a_lo) + wg * 64 * 128, bh = smem_u32(b_hi), bl = smem_u32(b_lo);
    wgmma_fence();
#pragma unroll
    for (int pass = 0; pass < 3; ++pass) {          // lo*hi, hi*lo, hi*hi
      const uint32_t ab = pass == 0 ? al : ah, bb = pass == 1 ? bl : bh;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int c = 0; c < SA_NCH; ++c)
          if (64 * c < w)
            wgmma_f16_n64(acc[c], gmma_desc_sw128(ab + ks * 32), gmma_desc_sw128(bb + c * 64 * 128 + ks * 32), (kb | pass | ks) ? 1u : 0u);
      }
    }
    wgmma_commit();
  }
  wgmma_wait<0>();
#pragma unroll
  for (int c = 0; c < SA_NCH; ++c) acc_fence(acc[c]);
  // the accumulators go to a row-major fp32 tile over the (now idle) operand stages, so that the epilogue walks rows
  __syncthreads();
  float* ctile = reinterpret_cast<float*>(smem);
  const int cp = p.ct + 8;      // row pitch (floats)
#pragma unroll
  for (int c = 0; c < SA_NCH; ++c)
    if (64 * c < w) acc_store(ctile, cp, 64 * wg, 64 * c, wt, acc[c]);
  __syncthreads();

  // ---- epilogue: thread == row; the two warp halves take alternate 16-column chunks and exchange their partial max / sum --------
  const int q = warp & 3, half = warp >> 2;
  const int trow = q * 32 + lane;
  const long long row = (long long)bt * p.Nn + j0 + trow;
  const bool live = trow < rows_here;
  const int nvalid = min(w, p.Nn - c0);            // columns i < Nn of this tile (>= 1: a tile starts below Npad - 63 < Nn)
  const int nchunk = w / 16;
  float mx = -INFINITY;
  for (int ch = half; ch < nchunk; ch += 2) {
    uint32_t v[16];
    acc_ld<16>(ctile, cp, trow, 16 * ch, v);
#pragma unroll
    for (int jj = 0; jj < 16; ++jj)
      if (16 * ch + jj < nvalid) mx = fmaxf(mx, __uint_as_float(v[jj]));
    if (live) {                                      // the raw logits; k_spatt_norm rewrites them in place
      float* dst = p.st + row * p.ld + c0 + 16 * ch; // ld % 4 == 0, st 16-byte aligned (checked on the host)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj)
        *reinterpret_cast<float4*>(dst + 4 * jj) = make_float4(__uint_as_float(v[4 * jj]), __uint_as_float(v[4 * jj + 1]),
                                                               __uint_as_float(v[4 * jj + 2]), __uint_as_float(v[4 * jj + 3]));
    }
  }
  red[half * 128 + trow] = mx;
  __syncthreads();
  mx = fmaxf(red[trow], red[128 + trow]);
  __syncthreads();
  float sum = 0.f;
  for (int ch = half; ch < nchunk; ch += 2) {
    uint32_t v[16];
    acc_ld<16>(ctile, cp, trow, 16 * ch, v);
#pragma unroll
    for (int jj = 0; jj < 16; ++jj)
      if (16 * ch + jj < nvalid) sum += __expf(__uint_as_float(v[jj]) - mx);
  }
  red[half * 128 + trow] = sum;
  __syncthreads();
  if (half == 0 && live) p.part[row * p.ntiles + tile] = make_float2(mx, red[trow] + red[128 + trow]);
}

// one warp per row (b, j): m = max over the tiles, s = sum_t s_t exp(m_t - m) in tile order, then exp(l - m) / s for i < Nn, 0 beyond
__global__ void __launch_bounds__(256) k_spatt_norm(float* __restrict__ st, long long ld, const float2* __restrict__ part, long long rows,
                                                    int Nn, int Npad, int ntiles) {
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float2* pr = part + row * ntiles;
  float m = -INFINITY;
  for (int t = 0; t < ntiles; ++t) m = fmaxf(m, pr[t].x);
  float s = 0.f;
  for (int t = 0; t < ntiles; ++t) {
    const float2 q = pr[t];
    s += q.y * __expf(q.x - m);
  }
  const float inv = 1.0f / s;
  float* r = st + row * ld;
  for (int c = 4 * lane; c < Npad; c += 128) {
    float4 v = *reinterpret_cast<const float4*>(r + c);
    v.x = c < Nn ? __expf(v.x - m) * inv : 0.f;
    v.y = c + 1 < Nn ? __expf(v.y - m) * inv : 0.f;
    v.z = c + 2 < Nn ? __expf(v.z - m) * inv : 0.f;
    v.w = c + 3 < Nn ? __expf(v.w - m) * inv : 0.f;
    *reinterpret_cast<float4*>(r + c) = v;
  }
}

// column tiling of a padded width: as few tiles of <= 256 columns as possible, as even as multiples of 64 allow (896 -> 256 x 3 + 128)
void sa_tiling(int Npad, int* ct, int* ntiles) {
  const int n64 = Npad / 64, nt = (Npad + SA_MAXCT - 1) / SA_MAXCT;
  *ct = 64 * ((n64 + nt - 1) / nt);
  *ntiles = (Npad + *ct - 1) / *ct;
}

}  // namespace
}  // namespace stmp

using namespace stmp;

extern "C" int64_t stmp_spatial_attention_tiled_workspace_bytes(int64_t B, int64_t n_nodes) {
  if (B < 0 || n_nodes < 1 || n_nodes > SA_MAXN) return -1;
  int ct, nt;
  sa_tiling((int)((n_nodes + 63) / 64 * 64), &ct, &nt);
  return B * n_nodes * nt * (int64_t)sizeof(float2);
}

extern "C" int stmp_spatial_attention_tiled_fwd(int64_t B, int64_t n_nodes, int64_t n_steps, const float* lhs, const float* rhs,
                                                const float* bsT, const void* vsT_packed, float* st_out, int64_t ld_out, void* workspace,
                                                int64_t workspace_bytes, void* stream) {
  STMP_REQUIRE(B >= 0 && n_nodes >= 1 && n_steps >= 1, STMP_EINVAL, "stmp_spatial_attention_tiled_fwd: bad sizes");
  if (n_nodes > SA_MAXN || n_steps > SA_MAXT)
    return set_error(STMP_EUNSUPPORTED, "tiled spatial attention takes <= %d nodes and <= %d timesteps (nodes=%lld steps=%lld)", SA_MAXN,
                     SA_MAXT, (long long)n_nodes, (long long)n_steps);
  const int Npad = (int)((n_nodes + 63) / 64 * 64);
  STMP_REQUIRE(ld_out >= Npad && ld_out % 4 == 0, STMP_ESHAPE,
               "stmp_spatial_attention_tiled_fwd: ld_out=%lld must be >= %d (nodes rounded up to 64) and a multiple of 4", (long long)ld_out, Npad);
  const int rtiles = (int)((n_nodes + SA_BM - 1) / SA_BM);
  if (B * rtiles >= (1ll << 31) || B * n_nodes >= (1ll << 33))
    return set_error(STMP_EUNSUPPORTED, "tiled spatial attention: B=%lld too large", (long long)B);
  if (B == 0) return STMP_OK;
  STMP_REQUIRE(lhs && rhs && bsT && vsT_packed && st_out && workspace, STMP_EINVAL, "stmp_spatial_attention_tiled_fwd: NULL pointer");
  STMP_REQUIRE((reinterpret_cast<uintptr_t>(st_out) & 15) == 0, STMP_ESHAPE, "stmp_spatial_attention_tiled_fwd: st_out must be 16-byte aligned");
  STMP_REQUIRE((reinterpret_cast<uintptr_t>(vsT_packed) & 15) == 0, STMP_EINVAL, "stmp_spatial_attention_tiled_fwd: vsT_packed must be 16-byte aligned");
  const int64_t need = stmp_spatial_attention_tiled_workspace_bytes(B, n_nodes);
  STMP_REQUIRE(workspace_bytes >= need && (reinterpret_cast<uintptr_t>(workspace) & 7) == 0, STMP_EINVAL,
               "stmp_spatial_attention_tiled_fwd: workspace of %lld bytes (8-byte aligned) needed, %lld given", (long long)need,
               (long long)workspace_bytes);
  STMP_REQUIRE(n_steps != 12 || (reinterpret_cast<uintptr_t>(lhs) & 15) == 0, STMP_EINVAL,
               "stmp_spatial_attention_tiled_fwd: lhs must be 16-byte aligned");
  SaParams p = {};
  p.Nn = (int)n_nodes; p.Tn = (int)n_steps; p.Npad = Npad;
  sa_tiling(Npad, &p.ct, &p.ntiles);
  p.lhs = lhs; p.rhs = rhs; p.bsT = bsT;
  p.w_hi = reinterpret_cast<const __half*>(vsT_packed); p.w_lo = p.w_hi + (int64_t)Npad * Npad;
  p.st = st_out; p.ld = ld_out; p.part = reinterpret_cast<float2*>(workspace);
  cudaStream_t st = (cudaStream_t)stream;
  const int smem = 2 * (2 * SA_A_BYTES + 2 * p.ct * 128) + 2 * SA_BM * (int)sizeof(float);
  STMP_CUDA_OK(cudaFuncSetAttribute(k_spatt_tiles, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_spatt_tiles<<<dim3((unsigned)(B * rtiles), (unsigned)p.ntiles), SA_NT, smem, st>>>(p);
  STMP_LAUNCH_OK("k_spatt_tiles");
  const long long rows = B * n_nodes;
  k_spatt_norm<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(st_out, ld_out, p.part, rows, p.Nn, Npad, p.ntiles);
  STMP_LAUNCH_OK("k_spatt_norm");
  return STMP_OK;
}
