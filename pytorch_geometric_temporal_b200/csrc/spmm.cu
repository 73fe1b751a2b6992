// spmm.cu -- K1/K3: gather of source-node rows -> edge-weighted accumulate per destination, with the
// Chebyshev/diffusion axpby fused into the epilogue.  One group of G lanes owns one (batch, destination) row, lanes are
// vectorised along the feature axis (float4/float2/float), edge metadata is one 64-bit load per edge, 4 gathers in flight.
// A CTA of 256 threads owns 8 x (256 / G) consecutive destination rows of one batch element.
// Bound (cfg5 probe, random 10^4-node graph): L2 throughput -- 4*nnz*F*B = 1.8 GB of gathered rows per launch on top of the 0.33 GB of
// compulsory HBM traffic.  Measured dead ends (B200): TMA-staged source rows 0.90x / 0.95x, 1024-thread CTAs 0.94x.
// Deterministic: per destination the sum runs in the reference's scatter order with separate
// multiply and add, which makes the result bit-identical to CPU index_select -> mul -> scatter_add_.
#include "common.cuh"

namespace stmp {
namespace {

constexpr int kSpmmThreads = 256;
constexpr int kSpmmRowsPerGroup = 8;   // consecutive destination rows walked by one lane group: cfg5 probe (B200) 1: 1451 GB/s, 4: 1810,
                                       // 8: 1855, 16: 1700 on the random graph; 1533 / 1920 / 1986 / 1879 on a banded one

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
template <int VEC>
__global__ void __launch_bounds__(kSpmmThreads) k_spmm(SpmmArgs a, int G, int log2G, int rpg, int blocks_per_b) {
  const int lane_in_group = threadIdx.x & (G - 1);
  const int gpc = kSpmmThreads >> log2G;
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
  STMP_REQUIRE(attT != nullptr || batch == 0 || f == 0, STMP_EINVAL, "stmp_spmm_att_t: attT is NULL");
  STMP_REQUIRE(plan == nullptr || att_ld >= plan->n, STMP_ESHAPE, "stmp_spmm_att_t: att_ld smaller than the node count");
  return spmm_impl(plan, op, 0, batch, f, x, ldx, bsx, y, ldy, bsy, alpha, z, ldz, bsz, beta, attT, att_ld, 1, stream);
}

static int spmm_impl(const stmp_plan* plan, int op, int transposed, int64_t batch, int64_t f, const float* x,
                     int64_t ldx, int64_t bsx, float* y, int64_t ldy, int64_t bsy, float alpha, const float* z,
                     int64_t ldz, int64_t bsz, float beta, const float* att, int64_t att_ld, int att_is_transposed, void* stream) {
  STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "stmp_spmm: plan is NULL");
  STMP_REQUIRE(op >= 0 && op < plan->n_ops, STMP_EINVAL, "stmp_spmm: op %d out of range", op);
  STMP_REQUIRE(batch >= 0 && f >= 0, STMP_EINVAL, "stmp_spmm: negative size");
  STMP_REQUIRE(ldx >= f && ldy >= f && (!z || ldz >= f), STMP_ESHAPE, "stmp_spmm: row stride smaller than f");
  if (batch == 0 || f == 0) return STMP_OK;     // empty tensors may come with NULL data pointers
  STMP_REQUIRE(x && y, STMP_EINVAL, "stmp_spmm: x/y is NULL");
  STMP_REQUIRE(x != y, STMP_EINVAL, "stmp_spmm: in-place product is not supported");
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
  const int gpc = kSpmmThreads / G;
  int rpg = kSpmmRowsPerGroup;
  // small problems keep one row per group: the row blocks must still fill the machine (>= 8 CTAs of 256 threads per SM's worth of blocks)
  while (rpg > 1 && batch * ((c.n + (long long)gpc * rpg - 1) / ((long long)gpc * rpg)) < 1184) rpg >>= 1;
  const int blocks_per_b = (int)((c.n + (long long)gpc * rpg - 1) / ((long long)gpc * rpg));
  long long blocks = batch * (long long)blocks_per_b;
  STMP_REQUIRE(blocks < (1ll << 31), STMP_ESHAPE, "stmp_spmm: problem too large for one launch");
  cudaStream_t st = (cudaStream_t)stream;
  if (vec == 4) k_spmm<4><<<(unsigned)blocks, kSpmmThreads, 0, st>>>(a, G, lg, rpg, blocks_per_b);
  else if (vec == 2) k_spmm<2><<<(unsigned)blocks, kSpmmThreads, 0, st>>>(a, G, lg, rpg, blocks_per_b);
  else k_spmm<1><<<(unsigned)blocks, kSpmmThreads, 0, st>>>(a, G, lg, rpg, blocks_per_b);
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
