// spmm.cu -- K1/K3: gather of source-node rows -> edge-weighted accumulate per destination, with the
// Chebyshev/diffusion axpby fused into the epilogue.  One group of G lanes owns one (batch, destination) row, lanes are
// vectorised along the feature axis (float4/float2/float), edge metadata is one 64-bit load per edge, 4 gathers in flight.
// A CTA owns 8 x (256 / G) consecutive destination rows of one batch element.
// Bound (cfg5 probe, random 10^4-node graph): L2 throughput -- 4*nnz*F*B = 1.8 GB of gathered rows per launch on top of the 0.33 GB of
// compulsory HBM traffic.  Variants kept selectable for A/B runs (tests/perf/spmm_variants.py, spmm_blocked.py): entries preloaded once
// + shuffles, predicated batches without a scalar tail, TMA-staged source rows (k_spmm_tma below), 1024-thread CTAs.
// Deterministic: per destination the sum runs in the reference's scatter order with separate
// multiply and add, which makes the result bit-identical to CPU index_select -> mul -> scatter_add_.
#include <cstdlib>

#include "common.cuh"

namespace stmp {
int g_spmm_rows_per_group = 8;   // consecutive destination rows walked by one lane group (stmp_set_option("spmm_rows_per_group")): cfg5 probe
                                 // 1: 1451 GB/s, 4: 1810, 8: 1855, 16: 1700 on the random graph; 1533 / 1920 / 1986 / 1879 on a banded one
int g_spmm_block = 256;          // threads per CTA (stmp_set_option("spmm_block"): 256 or 1024)
int g_spmm_variant = -1;   // 0 (default): k_spmm register gather; 1 / 2: k_spmm_tma with 8 / 16 staged rows per warp
namespace {

template <int VEC> struct VecT;
template <> struct VecT<1> { using T = float; };
template <> struct VecT<2> { using T = float2; };
template <> struct VecT<4> { using T = float4; };

template <int VEC>
__device__ __forceinline__ void ld_vec(const float* p, float (&v)[VEC]) {
  using T = typename VecT<VEC>::T;
  T t = __ldg(reinterpret_cast<const T*>(p));
  const float* f = reinterpret_cast<const float*>(&t);
#pragma unroll
  for (int i = 0; i < VEC; ++i) v[i] = f[i];
}
template <int VEC>
__device__ __forceinline__ void st_vec(float* p, const float (&v)[VEC]) {
  using T = typename VecT<VEC>::T;
  T t;
  float* f = reinterpret_cast<float*>(&t);
#pragma unroll
  for (int i = 0; i < VEC; ++i) f[i] = v[i];
  *reinterpret_cast<T*>(p) = t;
}

struct SpmmArgs {
  const int* rowptr;
  const int2* cv;
  int n;
  long long batch;
  int f;
  const float* x; long long ldx, bsx;
  float* y; long long ldy, bsy;
  const float* z; long long ldz, bsz;
  float alpha, beta;
  const float* att;  // [batch, n, att_ld] or null
  long long att_ld;  // row stride of att (n unless the attention is handed in padded)
  int att_transposed; // entry (dst=i, src=c): forward uses att[b,i,c]; transposed product / transposed attention uses att[b,c,i]
};

// G lanes per row (power of two, <=32).  blockDim.x = 256.
// A CTA owns `rpg` * (256 / G) CONSECUTIVE destination rows of one batch element and walks them 256 / G rows at a time: with a node
// numbering that has locality (sensor networks numbered along the roads) the source rows of neighbouring destinations overlap and are
// re-used out of L1 instead of crossing the L2 -> SM crossbar once per edge.
template <int VEC, int BLOCK>
__global__ void __launch_bounds__(BLOCK) k_spmm(SpmmArgs a, int G, int log2G, int rpg, int blocks_per_b) {
  const int lane_in_group = threadIdx.x & (G - 1);
  const int gpc = BLOCK >> log2G;
  const long long b = blockIdx.x / blocks_per_b;
  const int blk = blockIdx.x - (int)(b * blocks_per_b);
  const float* xb = a.x + b * a.bsx;
  const float* attb = a.att ? a.att + b * (long long)a.n * a.att_ld : nullptr;
  for (int r = 0; r < rpg; ++r) {
  const int i = (blk * rpg + r) * gpc + (threadIdx.x >> log2G);
  if (i >= a.n) return;
  const int beg = a.rowptr[i], end = a.rowptr[i + 1];

  for (int f0 = lane_in_group * VEC; f0 < a.f; f0 += G * VEC) {
    float acc[VEC];
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[v] = 0.f;
    int k = beg;
    for (; k + 4 <= end; k += 4) {
      int2 e[4];
      float xv[4][VEC];
      float w[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) e[u] = __ldg(&a.cv[k + u]);
#pragma unroll
      for (int u = 0; u < 4; ++u) ld_vec<VEC>(xb + (long long)e[u].x * a.ldx + f0, xv[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        w[u] = __int_as_float(e[u].y);
        if (attb) {
          float s = a.att_transposed ? __ldg(&attb[(long long)e[u].x * a.att_ld + i]) : __ldg(&attb[(long long)i * a.att_ld + e[u].x]);
          w[u] = __fmul_rn(w[u], s);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < VEC; ++v) acc[v] = __fadd_rn(acc[v], __fmul_rn(w[u], xv[u][v]));
    }
    for (; k < end; ++k) {
      int2 e = __ldg(&a.cv[k]);
      float xv[VEC];
      ld_vec<VEC>(xb + (long long)e.x * a.ldx + f0, xv);
      float w = __int_as_float(e.y);
      if (attb) {
        float s = a.att_transposed ? __ldg(&attb[(long long)e.x * a.att_ld + i]) : __ldg(&attb[(long long)i * a.att_ld + e.x]);
        w = __fmul_rn(w, s);
      }
#pragma unroll
      for (int v = 0; v < VEC; ++v) acc[v] = __fadd_rn(acc[v], __fmul_rn(w, xv[v]));
    }
    float o[VEC];
    if (a.z) {
      float zv[VEC];
      ld_vec<VEC>(a.z + b * a.bsz + (long long)i * a.ldz + f0, zv);
#pragma unroll
      for (int v = 0; v < VEC; ++v) o[v] = __fadd_rn(__fmul_rn(a.alpha, acc[v]), __fmul_rn(a.beta, zv[v]));
    } else {
#pragma unroll
      for (int v = 0; v < VEC; ++v) o[v] = (a.alpha == 1.0f) ? acc[v] : __fmul_rn(a.alpha, acc[v]);
    }
    st_vec<VEC>(a.y + b * a.bsy + (long long)i * a.ldy + f0, o);
  }
  }
}

// ---- TMA-staged gather ---------------------------------------------------------------------------------------------------------
// One warp per (batch, destination) row, persistent over rows.  The source rows of the destination's CSR row are fetched by TMA bulk
// copies (cp.async.bulk global -> shared, one per edge, 4*f bytes each, completion on the warp's mbarrier) into the warp's slots in
// shared memory, up to SLOTS rows per batch -- the loads in flight are bounded by shared memory (SLOTS x 4f bytes per warp), not by
// the L1's outstanding-load tracking that caps the register gather (k_spmm: ~64 KB per SM in flight whatever the unroll depth:
// tests/perf/spmm_variants.py).  Lanes then read their float4 of every staged row (conflict-free) and accumulate in CSR order with
// separate multiply and add -- bit-identical to k_spmm.  Needs f % 4 == 0, 16-byte aligned rows, f <= 32 * 4 * JMAX, no attention.
template <int SLOTS, int JMAX>
__global__ void __launch_bounds__(256) k_spmm_tma(SpmmArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rowbytes = a.f * 4;
  float* slots = reinterpret_cast<float*>(smem_raw) + (size_t)warp * SLOTS * a.f;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw + (size_t)8 * SLOTS * rowbytes) + warp;
  if (lane == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncwarp();
  const long long total = a.batch * (long long)a.n;
  uint32_t parity = 0;
  for (long long group = (long long)blockIdx.x * 8 + warp; group < total; group += (long long)gridDim.x * 8) {
    const int i = (int)(group % a.n);
    const long long b = group / a.n;
    const float* xb = a.x + b * a.bsx;
    const int beg = __ldg(a.rowptr + i), end = __ldg(a.rowptr + i + 1);
    float acc[JMAX][4];
#pragma unroll
    for (int j = 0; j < JMAX; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    for (int c0 = beg; c0 < end; c0 += SLOTS) {
      const int nh = min(SLOTS, end - c0);
      const int2 mine = lane < nh ? __ldg(a.cv + c0 + lane) : make_int2(0, 0);
      if (lane == 0) mbar_arrive_expect_tx(bar, (uint32_t)(nh * rowbytes));
      __syncwarp();
      if (lane < nh) tma_bulk_g2s(slots + (size_t)lane * a.f, xb + (long long)mine.x * a.ldx, (uint32_t)rowbytes, bar);
      mbar_wait(bar, parity);
      parity ^= 1u;
      for (int u = 0; u < nh; ++u) {
        const float w = __int_as_float(__shfl_sync(0xffffffffu, mine.y, u));
#pragma unroll
        for (int j = 0; j < JMAX; ++j) {
          const int f0 = (j * 32 + lane) * 4;
          if (f0 < a.f) {
            const float4 xv = *reinterpret_cast<const float4*>(slots + (size_t)u * a.f + f0);
            acc[j][0] = __fadd_rn(acc[j][0], __fmul_rn(w, xv.x));
            acc[j][1] = __fadd_rn(acc[j][1], __fmul_rn(w, xv.y));
            acc[j][2] = __fadd_rn(acc[j][2], __fmul_rn(w, xv.z));
            acc[j][3] = __fadd_rn(acc[j][3], __fmul_rn(w, xv.w));
          }
        }
      }
      __syncwarp();          // every lane is done with the slots before the next batch of copies overwrites them
    }
#pragma unroll
    for (int j = 0; j < JMAX; ++j) {
      const int f0 = (j * 32 + lane) * 4;
      if (f0 < a.f) {
        float o[4];
        if (a.z) {
          const float4 zv = __ldg(reinterpret_cast<const float4*>(a.z + b * a.bsz + (long long)i * a.ldz + f0));
          o[0] = __fadd_rn(__fmul_rn(a.alpha, acc[j][0]), __fmul_rn(a.beta, zv.x));
          o[1] = __fadd_rn(__fmul_rn(a.alpha, acc[j][1]), __fmul_rn(a.beta, zv.y));
          o[2] = __fadd_rn(__fmul_rn(a.alpha, acc[j][2]), __fmul_rn(a.beta, zv.z));
          o[3] = __fadd_rn(__fmul_rn(a.alpha, acc[j][3]), __fmul_rn(a.beta, zv.w));
        } else {
#pragma unroll
          for (int v = 0; v < 4; ++v) o[v] = (a.alpha == 1.0f) ? acc[j][v] : __fmul_rn(a.alpha, acc[j][v]);
        }
        *reinterpret_cast<float4*>(a.y + b * a.bsy + (long long)i * a.ldy + f0) = make_float4(o[0], o[1], o[2], o[3]);
      }
    }
  }
}

// d(att)[b,i,c] += val * <gy[b,i,:], x[b,c,:]> : one warp per (b, entry); entries are unique (dst,src)
// pairs except the doubled self loops of CHEB_ATT, hence atomicAdd.
__global__ void __launch_bounds__(256) k_att_grad(const int* __restrict__ rowptr, const int2* __restrict__ cv, int n,
                                                  long long batch, int f, const float* __restrict__ gy, long long ldg,
                                                  long long bsg, const float* __restrict__ x, long long ldx, long long bsx,
                                                  float* __restrict__ datt) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long total = batch * (long long)n;
  if (warp >= total) return;
  const int i = (int)(warp % n);
  const long long b = warp / n;
  const float* g = gy + b * bsg + (long long)i * ldg;
  for (int k = rowptr[i]; k < rowptr[i + 1]; ++k) {
    int2 e = __ldg(&cv[k]);
    const float* xr = x + b * bsx + (long long)e.x * ldx;
    float s = 0.f;
    for (int c = lane; c < f; c += 32) s = fmaf(g[c], xr[c], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) atomicAdd(&datt[(b * n + i) * (long long)n + e.x], __int_as_float(e.y) * s);
  }
}

inline bool aligned(const void* p, int bytes) { return (reinterpret_cast<uintptr_t>(p) % bytes) == 0; }

}  // namespace
}  // namespace stmp

using namespace stmp;

static int spmm_impl(const stmp_plan* plan, int op, int transposed, int64_t batch, int64_t f, const float* x,
                     int64_t ldx, int64_t bsx, float* y, int64_t ldy, int64_t bsy, float alpha, const float* z,
                     int64_t ldz, int64_t bsz, float beta, const float* att, int64_t att_ld, int att_is_transposed, void* stream);

extern "C" int stmp_spmm(const stmp_plan* plan, int op, int transposed, int64_t batch, int64_t f, const float* x,
                         int64_t ldx, int64_t bsx, float* y, int64_t ldy, int64_t bsy, float alpha, const float* z,
                         int64_t ldz, int64_t bsz, float beta, const float* att, void* stream) {
  return spmm_impl(plan, op, transposed, batch, f, x, ldx, bsx, y, ldy, bsy, alpha, z, ldz, bsz, beta, att, plan ? plan->n : 0, 0, stream);
}

extern "C" int stmp_spmm_att_t(const stmp_plan* plan, int op, int64_t batch, int64_t f, const float* x, int64_t ldx, int64_t bsx,
                              float* y, int64_t ldy, int64_t bsy, float alpha, const float* z, int64_t ldz, int64_t bsz, float beta,
                              const float* attT, int64_t att_ld, void* stream) {
  STMP_REQUIRE(attT != nullptr, STMP_EINVAL, "stmp_spmm_att_t: attT is NULL");
  STMP_REQUIRE(plan == nullptr || att_ld >= plan->n, STMP_ESHAPE, "stmp_spmm_att_t: att_ld smaller than the node count");
  return spmm_impl(plan, op, 0, batch, f, x, ldx, bsx, y, ldy, bsy, alpha, z, ldz, bsz, beta, attT, att_ld, 1, stream);
}

static int spmm_impl(const stmp_plan* plan, int op, int transposed, int64_t batch, int64_t f, const float* x,
                     int64_t ldx, int64_t bsx, float* y, int64_t ldy, int64_t bsy, float alpha, const float* z,
                     int64_t ldz, int64_t bsz, float beta, const float* att, int64_t att_ld, int att_is_transposed, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_spmm: plan is NULL");
  STMP_REQUIRE(op >= 0 && op < plan->n_ops, STMP_EINVAL, "stmp_spmm: op %d out of range", op);
  STMP_REQUIRE(x && y, STMP_EINVAL, "stmp_spmm: x/y is NULL");
  STMP_REQUIRE(batch >= 0 && f >= 0, STMP_EINVAL, "stmp_spmm: negative size");
  STMP_REQUIRE(ldx >= f && ldy >= f && (!z || ldz >= f), STMP_ESHAPE, "stmp_spmm: row stride smaller than f");
  STMP_REQUIRE(x != y, STMP_EINVAL, "stmp_spmm: in-place product is not supported");
  if (batch == 0 || f == 0) return STMP_OK;
  const Csr& c = transposed ? plan->bwd[op] : plan->fwd[op];
  SpmmArgs a;
  a.rowptr = c.rowptr; a.cv = c.cv; a.n = c.n; a.batch = batch; a.f = (int)f;
  a.x = x; a.ldx = ldx; a.bsx = bsx; a.y = y; a.ldy = ldy; a.bsy = bsy;
  a.z = z; a.ldz = z ? ldz : 0; a.bsz = z ? bsz : 0; a.alpha = alpha; a.beta = beta;
  a.att = att; a.att_ld = att_ld; a.att_transposed = (transposed ? 1 : 0) ^ (att_is_transposed ? 1 : 0);
  // widest vector the shapes/alignments allow
  auto ok = [&](int v) {
    int bytes = 4 * v;
    bool r = (f % v == 0) && (ldx % v == 0) && (ldy % v == 0) && (bsx % v == 0) && (bsy % v == 0) &&
             aligned(x, bytes) && aligned(y, bytes);
    if (z) r = r && (ldz % v == 0) && (bsz % v == 0) && aligned(z, bytes);
    return r;
  };
  int vec = ok(4) ? 4 : (ok(2) ? 2 : 1);
  int lanes = (int)((f + vec - 1) / vec);
  int G = 1, lg = 0;
  while (G < lanes && G < 32) { G <<= 1; ++lg; }
  long long groups = batch * (long long)c.n;
  const int blk = g_spmm_block == 1024 ? 1024 : 256;
  const int gpc = blk / G;
  int rpg = g_spmm_rows_per_group;
  if (rpg < 1) rpg = 1;
  // small problems keep one row per group: the row blocks must still fill the machine (>= 8 CTAs of 256 threads per SM's worth of blocks)
  while (rpg > 1 && batch * ((c.n + (long long)gpc * rpg - 1) / ((long long)gpc * rpg)) < 1184) rpg >>= 1;
  const int blocks_per_b = (int)((c.n + (long long)gpc * rpg - 1) / ((long long)gpc * rpg));
  long long blocks = batch * (long long)blocks_per_b;
  STMP_REQUIRE(blocks < (1ll << 31), STMP_ESHAPE, "stmp_spmm: problem too large for one launch");
  cudaStream_t st = (cudaStream_t)stream;
  if (g_spmm_variant < 0) {
    const char* v = getenv("STMP_SPMM_VARIANT");
    g_spmm_variant = v ? atoi(v) : 0;
  }
  if ((g_spmm_variant == 1 || g_spmm_variant == 2) && !att && vec == 4 && f <= 512 && (long long)groups >= 8) {
    // TMA-staged gather: SLOTS x 4f bytes of shared memory per warp
    const int slots = g_spmm_variant == 1 ? 8 : 16;
    const size_t smem = (size_t)8 * slots * f * 4 + 8 * 8;
    if (smem <= 200 * 1024) {
      int dev = 0, sms = 0;
      STMP_CUDA_OK(cudaGetDevice(&dev));
      STMP_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
      int per_sm = (int)((220 * 1024) / (smem + 1024));
      if (per_sm > 8) per_sm = 8;
      if (per_sm < 1) per_sm = 1;
      long long want = (groups + 7) / 8;
      unsigned grid = (unsigned)(want < (long long)sms * per_sm ? want : (long long)sms * per_sm);
      const int jm = (int)((f + 127) / 128);
#define STMP_TMA_LAUNCH(S, J)                                                                                          \
  do {                                                                                                                 \
    STMP_CUDA_OK(cudaFuncSetAttribute(k_spmm_tma<S, J>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));      \
    k_spmm_tma<S, J><<<grid, 256, smem, st>>>(a);                                                                      \
  } while (0)
      if (slots == 8) {
        if (jm == 1) STMP_TMA_LAUNCH(8, 1); else if (jm == 2) STMP_TMA_LAUNCH(8, 2); else STMP_TMA_LAUNCH(8, 4);
      } else {
        if (jm == 1) STMP_TMA_LAUNCH(16, 1); else if (jm == 2) STMP_TMA_LAUNCH(16, 2); else STMP_TMA_LAUNCH(16, 4);
      }
#undef STMP_TMA_LAUNCH
      STMP_LAUNCH_OK("k_spmm_tma");
      return STMP_OK;
    }
  }
  if (blk == 1024) {
    if (vec == 4) k_spmm<4, 1024><<<(unsigned)blocks, 1024, 0, st>>>(a, G, lg, rpg, blocks_per_b);
    else if (vec == 2) k_spmm<2, 1024><<<(unsigned)blocks, 1024, 0, st>>>(a, G, lg, rpg, blocks_per_b);
    else k_spmm<1, 1024><<<(unsigned)blocks, 1024, 0, st>>>(a, G, lg, rpg, blocks_per_b);
  } else {
    if (vec == 4) k_spmm<4, 256><<<(unsigned)blocks, 256, 0, st>>>(a, G, lg, rpg, blocks_per_b);
    else if (vec == 2) k_spmm<2, 256><<<(unsigned)blocks, 256, 0, st>>>(a, G, lg, rpg, blocks_per_b);
    else k_spmm<1, 256><<<(unsigned)blocks, 256, 0, st>>>(a, G, lg, rpg, blocks_per_b);
  }
  STMP_LAUNCH_OK("k_spmm");
  return STMP_OK;
}

extern "C" int stmp_spmm_att_grad(const stmp_plan* plan, int op, int64_t batch, int64_t f, const float* gy, int64_t ldg,
                                  int64_t bsg, const float* x, int64_t ldx, int64_t bsx, float* datt, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_spmm_att_grad: plan is NULL");
  STMP_REQUIRE(op >= 0 && op < plan->n_ops, STMP_EINVAL, "stmp_spmm_att_grad: op %d out of range", op);
  STMP_REQUIRE(gy && x && datt, STMP_EINVAL, "stmp_spmm_att_grad: NULL pointer");
  if (batch == 0 || f == 0) return STMP_OK;
  const Csr& c = plan->fwd[op];
  long long warps = batch * (long long)c.n;
  long long blocks = (warps * 32 + 255) / 256;
  k_att_grad<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(c.rowptr, c.cv, c.n, batch, (int)f, gy, ldg, bsg, x, ldx,
                                                                  bsx, datt);
  STMP_LAUNCH_OK("k_att_grad");
  return STMP_OK;
}
