// hetero_rows.cu -- HeteroGCLSTM (DESIGN §4v), the heterogeneous graph LSTM, for every node type in ONE row-split launch.
//
// For a destination node type t with incoming edge types e_1 .. e_R (src(e_r) = s_r), each gate's pre-activation is
//   pre_g = X_t W_g + b_g + sum_r ( mean_{e_r}(H_{s_r}) lin_l^{g,e_r}^T + lin_l^{g,e_r}.bias + H_t lin_r^{g,e_r}^T )
// i.e. S w^T + b on the basis S = [X_t | H_t | mean_{e_1}(H_{s_1}) | ... | mean_{e_R}(H_{s_R})] with, per gate, the packed row block
// [W_g^T | sum_r lin_r^{g,e_r} | lin_l^{g,e_1} | ... ] and b = b_g + sum_r lin_l^{g,e_r}.bias (packed by the module, in edge-type order).
// mean_e is the bipartite SAGE mean operator of edge type e: an STMP_FLAVOR_RGCN plan of one relation built on max(N_src, N_dst) nodes,
// whose rows < N_dst are read and whose columns are < N_src (checked when the plan is made).
//
//   k_hetero_lstm_fwd<NC, HAS_H>   CTAs take grid-strided 16-row tiles of the concatenated destination types from the type table (a
//                                  kernel parameter); a CTA stages its type's packed weight [4 CO][nb] once per type change, one warp per
//                                  row gathers the means in CSR entry order (rows::gather_rows), lane = channel (lane + 32 j, j < NC)
//
// The contraction runs over the basis columns in order with fmaf, the gathers with separate multiply and add, no atomics: repeated calls
// are bit-identical.  Node-type state stays in the caller's per-type tensors: the table carries each type's pointers, so the launch
// count is one whatever the number of types and no concatenation copies are made.
#include "rows.cuh"

namespace stmp {
namespace {

using namespace rows;

constexpr int kHgMaxTypes = STMP_HETERO_MAX_TYPES;
constexpr int kHgMaxRel = STMP_HETERO_MAX_REL;
constexpr int kHgMaxCin = 32;                 // the lane carries the X channel

// staged pitch (odd: lane-indexed weight rows are conflict-free) and the widest basis of each width: out 32 with four incoming edge
// types (32 + 32 * 5 = 192 columns, 98 816 B, two CTAs per SM), out 64 with one (32 + 64 * 2 = 160 columns, 164 864 B, one CTA per SM)
template <int NC> struct HgWd;
template <> struct HgWd<1> { static constexpr int CO = 32, MAXREL = 4, P = 193, CTAS = 2; };
template <> struct HgWd<2> { static constexpr int CO = 64, MAXREL = 1, P = 161, CTAS = 1; };

struct HgType {
  const float* x; const float* h; const float* c; const float* w; const float* b;
  float* hout; float* cout;
  const int* rowptr[kHgMaxRel]; const int2* cv[kHgMaxRel]; const float* hs[kHgMaxRel];
  float* stash; float* S;                      // training: I, F, T, O (4 planes of N x CO) and the basis rows (N x nb); NULL for inference
  int n, cin, nrel, tile0;
};

struct HgArgs {
  HgType t[kHgMaxTypes];
  int ntypes, tiles;
};

template <int NC, bool HAS_H, bool TRAIN>
__global__ void __launch_bounds__(kRowsThreads, 1) k_hetero_lstm_fwd(const __grid_constant__ HgArgs a) {
  extern __shared__ float ws[];
  constexpr int CO = HgWd<NC>::CO, P = HgWd<NC>::P, MR = HgWd<NC>::MAXREL;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int staged = -1;
  for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
    int ti = 0;
    while (ti + 1 < a.ntypes && tile >= a.t[ti + 1].tile0) ++ti;
    const HgType& T = a.t[ti];
    const int cin = T.cin, nrel = T.nrel;
    if (ti != staged) {
      __syncthreads();                         // every warp is done with the previous type's weights
      stage_w<P>(ws, T.w, cin + CO * (1 + nrel), 0, 4 * CO);
      staged = ti;
    }
    const int t0 = (tile - T.tile0) * kRowTile, t1 = min(t0 + kRowTile, T.n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      const float xv = lane < cin ? __ldg(T.x + (size_t)i * cin + lane) : 0.f;
      float hv[NC], m[MR][NC];
#pragma unroll
      for (int j = 0; j < NC; ++j) {
        hv[j] = HAS_H ? __ldg(T.h + (size_t)i * CO + lane + 32 * j) : 0.f;
#pragma unroll
        for (int r = 0; r < MR; ++r) m[r][j] = 0.f;
      }
      if (HAS_H) {
        float unused;
#pragma unroll
        for (int r = 0; r < MR; ++r)
          if (r < nrel) gather_rows<NC, true>(T.rowptr[r], T.cv[r], i, T.hs[r], CO, nullptr, 0, 0, lane, m[r], unused);
      }
      float p[4][NC];                          // pre = b + S w^T, S's columns in basis order
#pragma unroll
      for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int j = 0; j < NC; ++j) p[g][j] = __ldg(T.b + g * CO + lane + 32 * j);
      auto col = [&](float s, int k) {
#pragma unroll
        for (int g = 0; g < 4; ++g)
#pragma unroll
          for (int j = 0; j < NC; ++j) p[g][j] = fmaf(s, ws[(g * CO + lane + 32 * j) * P + k], p[g][j]);
      };
      for (int k = 0; k < cin; ++k) col(__shfl_sync(0xffffffffu, xv, k), k);
      if (HAS_H) {                             // H = None: the H and mean columns are zero and skipped
#pragma unroll
        for (int jo = 0; jo < NC; ++jo) {
#pragma unroll 8
          for (int o = 0; o < 32; ++o) col(__shfl_sync(0xffffffffu, hv[jo], o), cin + 32 * jo + o);
        }
#pragma unroll
        for (int r = 0; r < MR; ++r) {
          if (r < nrel) {
#pragma unroll
            for (int jo = 0; jo < NC; ++jo) {
#pragma unroll 8
              for (int o = 0; o < 32; ++o) col(__shfl_sync(0xffffffffu, m[r][jo], o), cin + CO * (1 + r) + 32 * jo + o);
            }
          }
        }
      }
#pragma unroll
      for (int j = 0; j < NC; ++j) {
        const size_t io = (size_t)i * CO + lane + 32 * j;
        const float cp = T.c ? __ldg(T.c + io) : 0.f;
        const float I = sigmoidf_acc(p[0][j]), F = sigmoidf_acc(p[1][j]), Tc = tanhf(p[2][j]);
        const float cn = F * cp + I * Tc;
        const float O = sigmoidf_acc(p[3][j]);   // no peephole: O does not read the new cell state
        T.hout[io] = O * tanhf(cn);
        T.cout[io] = cn;
        if (TRAIN) {
          const size_t NCn = (size_t)T.n * CO;
          T.stash[io] = I;
          T.stash[NCn + io] = F;
          T.stash[2 * NCn + io] = Tc;
          T.stash[3 * NCn + io] = O;
        }
      }
      if (TRAIN) {                             // the weight-gradient basis row; H = None: its H and mean columns are zero
        const int nb = cin + CO * (1 + nrel);
        float* Sr = T.S + (size_t)i * nb;
        if (lane < cin) Sr[lane] = xv;
#pragma unroll
        for (int j = 0; j < NC; ++j) {
          Sr[cin + lane + 32 * j] = hv[j];
#pragma unroll
          for (int r = 0; r < MR; ++r)
            if (r < nrel) Sr[cin + CO * (1 + r) + lane + 32 * j] = m[r][j];
        }
      }
    }
  }
}

bool hg_envelope(int64_t out, int64_t cin, int64_t nrel) {
  if (cin < 1 || cin > kHgMaxCin || nrel < 1) return false;
  return (out == 32 && nrel <= HgWd<1>::MAXREL) || (out == 64 && nrel <= HgWd<2>::MAXREL);
}

int hg_cap(int ctas) {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return ctas * sms;
}

template <int NC, bool HAS_H, bool TRAIN>
int hg_launch(const HgArgs& a, cudaStream_t st) {
  constexpr int smem = 4 * HgWd<NC>::CO * HgWd<NC>::P * 4;
  const int cap = hg_cap(HgWd<NC>::CTAS);
  STMP_CUDA_OK(cudaFuncSetAttribute(k_hetero_lstm_fwd<NC, HAS_H, TRAIN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_hetero_lstm_fwd<NC, HAS_H, TRAIN><<<a.tiles < cap ? a.tiles : cap, kRowsThreads, smem, st>>>(a);
  STMP_LAUNCH_OK("k_hetero_lstm_fwd");
  return STMP_OK;
}

// ---- backward ---------------------------------------------------------------------------------------------------------------------
//   k_hetero_lstm_bwd_rows<NC>   per row of every type: dpre from the stash, dC, then dS = dpre w (lane = basis column, the 4 CO packed
//                                rows summed in order): dX, the own-row dH and Q_r = dpre lin_l^{e_r} per incoming edge type
//   k_hetero_lstm_bwd_gather<NC> per row of every source type: dH_s = own + sum over its outgoing edge types (metadata order) of
//                                Op_e^T Q_e (the plan's CSR by source, entry order)
//   k_hetero_wgrad               partials of [dW | db] = dpre^T [S | 1] over fixed row chunks, 64 x 64 output tiles
//   k_hetero_wgrad_reduce        the chunk partials summed in chunk order
constexpr int kHgMaxOut = 8;                   // outgoing edge types per source type of the fused backward
constexpr int kWgChunk = 2048, kWgTile = 64, kWgSlab = 16;

struct HgBwdType {
  const float* w; const float* stash; const float* c; const float* cn; const float* gh; const float* gc;
  float* dpre; float* dx; float* dh; float* dc; float* q[kHgMaxRel];
  int n, cin, nrel, tile0;
};
struct HgBwdArgs { HgBwdType t[kHgMaxTypes]; int ntypes, tiles; };

template <int NC>
__global__ void __launch_bounds__(kRowsThreads, 1) k_hetero_lstm_bwd_rows(const __grid_constant__ HgBwdArgs a) {
  extern __shared__ float ws[];
  constexpr int CO = HgWd<NC>::CO, P = HgWd<NC>::P, NQ = (P - 1) / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int staged = -1;
  for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
    int ti = 0;
    while (ti + 1 < a.ntypes && tile >= a.t[ti + 1].tile0) ++ti;
    const HgBwdType& T = a.t[ti];
    const int cin = T.cin, nb = cin + CO * (1 + T.nrel);
    const bool want_s = T.dx || T.dh;
    if (ti != staged && want_s) {
      __syncthreads();
      stage_w<P>(ws, T.w, nb, 0, 4 * CO);
      staged = ti;
    }
    const int t0 = (tile - T.tile0) * kRowTile, t1 = min(t0 + kRowTile, T.n);
    const size_t NCn = (size_t)T.n * CO;
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      float dp[4][NC];
#pragma unroll
      for (int j = 0; j < NC; ++j) {
        const size_t io = (size_t)i * CO + lane + 32 * j;
        const float I = T.stash[io], F = T.stash[NCn + io], Tc = T.stash[2 * NCn + io], O = T.stash[3 * NCn + io];
        const float cp = T.c ? T.c[io] : 0.f, cn = T.cn[io];
        const float ghv = T.gh ? T.gh[io] : 0.f, gcv = T.gc ? T.gc[io] : 0.f;
        const float tc = tanhf(cn);
        const float dcn = gcv + ghv * O * (1.f - tc * tc);
        dp[0][j] = dcn * Tc * I * (1.f - I);
        dp[1][j] = dcn * cp * F * (1.f - F);
        dp[2][j] = dcn * I * (1.f - Tc * Tc);
        dp[3][j] = ghv * tc * O * (1.f - O);
        if (T.dc) T.dc[io] = dcn * F;
#pragma unroll
        for (int g = 0; g < 4; ++g) T.dpre[(size_t)i * 4 * CO + g * CO + lane + 32 * j] = dp[g][j];
      }
      if (!want_s) continue;
      float acc[NQ];
#pragma unroll
      for (int q = 0; q < NQ; ++q) acc[q] = 0.f;
#pragma unroll
      for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int j = 0; j < NC; ++j) {
#pragma unroll 4
          for (int c = 0; c < 32; ++c) {
            const float v = __shfl_sync(0xffffffffu, dp[g][j], c);
            const float* wr = ws + (g * CO + 32 * j + c) * P + lane;
#pragma unroll
            for (int q = 0; q < NQ; ++q) acc[q] = fmaf(v, wr[32 * q], acc[q]);
          }
        }
#pragma unroll
      for (int q = 0; q < NQ; ++q) {
        const int k = lane + 32 * q;
        if (k < cin) {
          if (T.dx) T.dx[(size_t)i * cin + k] = acc[q];
        } else if (k < cin + CO) {
          if (T.dh) T.dh[(size_t)i * CO + k - cin] = acc[q];
        } else if (k < nb) {
          const int r = (k - cin - CO) / CO;
          if (T.dh) T.q[r][(size_t)i * CO + (k - cin - CO) - r * CO] = acc[q];
        }
      }
    }
  }
}

struct HgGatherType {
  float* dh; const int* rowptr[kHgMaxOut]; const int2* cv[kHgMaxOut]; const float* q[kHgMaxOut];
  int n, nout, tile0;
};
struct HgGatherArgs { HgGatherType t[kHgMaxTypes]; int ntypes, tiles; };

template <int NC>
__global__ void __launch_bounds__(kRowsThreads) k_hetero_lstm_bwd_gather(const __grid_constant__ HgGatherArgs a) {
  constexpr int CO = 32 * NC;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int tile = blockIdx.x; tile < a.tiles; tile += gridDim.x) {
    int ti = 0;
    while (ti + 1 < a.ntypes && tile >= a.t[ti + 1].tile0) ++ti;
    const HgGatherType& T = a.t[ti];
    const int t0 = (tile - T.tile0) * kRowTile, t1 = min(t0 + kRowTile, T.n);
    for (int i = t0 + warp; i < t1; i += kRowsWarps) {
      float acc[NC];
#pragma unroll
      for (int j = 0; j < NC; ++j) acc[j] = T.dh[(size_t)i * CO + lane + 32 * j];     // the own-row term first
      for (int o = 0; o < T.nout; ++o) {
        float g[NC], unused;
        gather_rows<NC, true>(T.rowptr[o], T.cv[o], i, T.q[o], CO, nullptr, 0, 0, lane, g, unused);
#pragma unroll
        for (int j = 0; j < NC; ++j) acc[j] = __fadd_rn(acc[j], g[j]);
      }
#pragma unroll
      for (int j = 0; j < NC; ++j) T.dh[(size_t)i * CO + lane + 32 * j] = acc[j];
    }
  }
}

struct HgWgType {
  const float* dpre; const float* S; float* part; float* dw;
  int n, nb, item0, tk, chunks;               // output tiles: (4 CO / 64) x tk per chunk
};
struct HgWgArgs { HgWgType t[kHgMaxTypes]; int ntypes, items, M; };

// one 64 x 64 tile of [dW | db] (M x (nb + 1)) over one chunk of rows, rows summed in order; column nb of the basis is the constant 1
__global__ void __launch_bounds__(256) k_hetero_wgrad(const __grid_constant__ HgWgArgs a) {
  __shared__ float sp[kWgSlab][kWgTile], ss[kWgSlab][kWgTile];
  int ti = 0;
  while (ti + 1 < a.ntypes && (int)blockIdx.x >= a.t[ti + 1].item0) ++ti;
  const HgWgType& T = a.t[ti];
  const int item = blockIdx.x - T.item0, tm = a.M / kWgTile;
  const int chunk = item / (tm * T.tk), rest = item - chunk * tm * T.tk;
  const int m0 = (rest / T.tk) * kWgTile, k0 = (rest % T.tk) * kWgTile, ld = T.nb + 1;
  const int r0 = chunk * kWgChunk, r1 = min(r0 + kWgChunk, T.n);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4] = {};
  for (int s0 = r0; s0 < r1; s0 += kWgSlab) {
    __syncthreads();
    for (int e = threadIdx.x; e < kWgSlab * kWgTile; e += 256) {
      const int r = e / kWgTile, cc = e - r * kWgTile, row = s0 + r, k = k0 + cc;
      const bool live = row < r1;
      sp[r][cc] = live ? T.dpre[(size_t)row * a.M + m0 + cc] : 0.f;
      ss[r][cc] = !live || k > T.nb ? 0.f : (k == T.nb ? 1.f : T.S[(size_t)row * T.nb + k]);
    }
    __syncthreads();
#pragma unroll 4
    for (int r = 0; r < kWgSlab; ++r) {
      float pv[4], sv[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) { pv[u] = sp[r][ty * 4 + u]; sv[u] = ss[r][tx * 4 + u]; }
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = fmaf(pv[u], sv[v], acc[u][v]);
    }
  }
  float* part = T.part + (size_t)chunk * a.M * ld;
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int m = m0 + ty * 4 + u, k = k0 + tx * 4 + v;
      if (k < ld) part[(size_t)m * ld + k] = acc[u][v];
    }
}

__global__ void k_hetero_wgrad_reduce(const __grid_constant__ HgWgArgs a, int total) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
    int ti = 0, base = 0;
    while (ti + 1 < a.ntypes && e >= base + a.M * (a.t[ti].nb + 1)) { base += a.M * (a.t[ti].nb + 1); ++ti; }
    const HgWgType& T = a.t[ti];
    const size_t sz = (size_t)a.M * (T.nb + 1);
    const int o = e - base;
    float s = 0.f;
    for (int c = 0; c < T.chunks; ++c) s = __fadd_rn(s, T.part[c * sz + o]);
    T.dw[o] = s;
  }
}

}  // namespace
}  // namespace stmp

using namespace stmp;

extern "C" int stmp_hetero_lstm_supported(int64_t out_channels, int64_t in_channels, int64_t num_rel) {
  return hg_envelope(out_channels, in_channels, num_rel) ? 1 : 0;
}

static int hg_common(const char* fn, int64_t out_channels, int64_t num_types, const int64_t* desc) {
  STMP_REQUIRE(desc != nullptr, STMP_EINVAL, "%s: desc is NULL", fn);
  STMP_REQUIRE(num_types >= 1 && num_types <= kHgMaxTypes, STMP_EUNSUPPORTED, "%s: %lld node types, 1..%d supported", fn,
               (long long)num_types, kHgMaxTypes);
  STMP_REQUIRE(out_channels == 32 || out_channels == 64, STMP_EUNSUPPORTED, "%s: out_channels %lld, 32 or 64 supported", fn,
               (long long)out_channels);
  for (int t = 0; t < num_types; ++t) {
    const int64_t* d = desc + (size_t)t * STMP_HETERO_DESC;
    STMP_REQUIRE(hg_envelope(out_channels, d[1], d[2]), STMP_EUNSUPPORTED,
                 "%s: type %d has in_channels %lld and %lld incoming edge types, outside the envelope at out_channels %lld", fn, t,
                 (long long)d[1], (long long)d[2], (long long)out_channels);
    STMP_REQUIRE(d[0] >= 1 && d[0] < (1ll << 31) / 256, STMP_EUNSUPPORTED, "%s: type %d has %lld nodes", fn, t, (long long)d[0]);
  }
  return STMP_OK;
}

static float* fp(int64_t v) { return reinterpret_cast<float*>(static_cast<intptr_t>(v)); }
static const stmp_plan* pp(int64_t v) { return reinterpret_cast<const stmp_plan*>(static_cast<intptr_t>(v)); }
static int hg_nb(int64_t out, const int64_t* d) { return (int)(d[1] + out * (1 + d[2])); }
static int hg_chunks(const int64_t* d) { return (int)((d[0] + kWgChunk - 1) / kWgChunk); }

extern "C" int stmp_hetero_lstm_fwd(int64_t out_channels, int64_t num_types, const int64_t* desc, int has_h, void* stream) {
  const char* fn = "stmp_hetero_lstm_fwd";
  if (int rc = hg_common(fn, out_channels, num_types, desc)) return rc;
  HgArgs a = {};
  a.ntypes = (int)num_types;
  long long tiles = 0;
  bool train = false;
  for (int t = 0; t < num_types; ++t) {
    const int64_t* d = desc + (size_t)t * STMP_HETERO_DESC;
    const int64_t n = d[0], cin = d[1], nrel = d[2];
    HgType& T = a.t[t];
    T.n = (int)n; T.cin = (int)cin; T.nrel = (int)nrel; T.tile0 = (int)tiles;
    T.x = fp(d[3]); T.h = fp(d[4]); T.c = fp(d[5]); T.w = fp(d[6]); T.b = fp(d[7]); T.hout = fp(d[8]); T.cout = fp(d[9]);
    T.stash = fp(d[18]); T.S = fp(d[19]);
    if (t == 0) train = T.stash != nullptr;
    STMP_REQUIRE(T.x && T.w && T.b && T.hout && T.cout && (!has_h || T.h), STMP_EINVAL, "%s: type %d: NULL tensor", fn, t);
    STMP_REQUIRE((T.stash != nullptr) == train && (T.S != nullptr) == train, STMP_EINVAL,
                 "%s: type %d: stash and basis must be given for every type or none", fn, t);
    const void* ps[] = {T.x, T.h, T.c, T.w, T.b, T.hout, T.cout, T.stash, T.S};
    for (const void* q : ps) STMP_REQUIRE(al4(q), STMP_ESHAPE, "%s: type %d: misaligned tensor", fn, t);
    for (int r = 0; r < nrel; ++r) {
      const stmp_plan* plan = pp(d[10 + r]);
      STMP_REQUIRE(plan != nullptr, STMP_EINVAL, "%s: type %d: plan %d is NULL", fn, t, r);
      STMP_REQUIRE(plan->flavor == STMP_FLAVOR_RGCN && plan->n_ops >= 1 && plan->n >= n, STMP_EINVAL,
                   "%s: type %d: plan %d is not a mean plan over at least %lld rows", fn, t, r, (long long)n);
      T.rowptr[r] = plan->fwd[0].rowptr;
      T.cv[r] = plan->fwd[0].cv;
      T.hs[r] = fp(d[10 + kHgMaxRel + r]);
      STMP_REQUIRE(!has_h || (T.hs[r] && al4(T.hs[r])), STMP_EINVAL, "%s: type %d: source state %d is NULL or misaligned", fn, t, r);
    }
    tiles += (n + kRowTile - 1) / kRowTile;
  }
  a.tiles = (int)tiles;
  cudaStream_t st = (cudaStream_t)stream;
  if (out_channels == 32) {
    if (train) return has_h ? hg_launch<1, true, true>(a, st) : hg_launch<1, false, true>(a, st);
    return has_h ? hg_launch<1, true, false>(a, st) : hg_launch<1, false, false>(a, st);
  }
  if (train) return has_h ? hg_launch<2, true, true>(a, st) : hg_launch<2, false, true>(a, st);
  return has_h ? hg_launch<2, true, false>(a, st) : hg_launch<2, false, false>(a, st);
}

extern "C" int64_t stmp_hetero_lstm_workspace_bytes(int64_t out_channels, int64_t num_types, const int64_t* desc) {
  if (hg_common("stmp_hetero_lstm_workspace_bytes", out_channels, num_types, desc)) return 0;
  int64_t total = 0;
  for (int t = 0; t < num_types; ++t) {
    const int64_t* d = desc + (size_t)t * STMP_HETERO_DESC;
    total += (int64_t)hg_chunks(d) * 4 * out_channels * (hg_nb(out_channels, d) + 1);
  }
  return 4 * total;
}

template <int NC>
static int hg_bwd(const int64_t* desc, int num_types, int want_dh, void* workspace, cudaStream_t st) {
  constexpr int CO = 32 * NC;
  HgBwdArgs a = {};
  HgGatherArgs g = {};
  HgWgArgs wg = {};
  a.ntypes = g.ntypes = wg.ntypes = num_types;
  wg.M = 4 * CO;
  int tiles = 0, items = 0, total = 0;
  size_t off = 0;
  bool wgrad = false;
  int order[kHgMaxTypes * kHgMaxRel][2], nedge = 0;   // (type, relation) of every edge, by metadata rank
  for (int t = 0; t < num_types; ++t) {
    const int64_t* d = desc + (size_t)t * STMP_HETERO_DESC;
    HgBwdType& T = a.t[t];
    T.n = (int)d[0]; T.cin = (int)d[1]; T.nrel = (int)d[2]; T.tile0 = tiles;
    T.w = fp(d[6]); T.c = fp(d[5]); T.cn = fp(d[9]); T.stash = fp(d[18]);
    T.gh = fp(d[20]); T.gc = fp(d[21]); T.dpre = fp(d[22]); T.dx = fp(d[23]); T.dh = want_dh ? fp(d[24]) : nullptr; T.dc = fp(d[25]);
    STMP_REQUIRE(T.w && T.cn && T.stash && T.dpre && fp(d[19]), STMP_EINVAL, "stmp_hetero_lstm_bwd: type %d: NULL tensor", t);
    STMP_REQUIRE(!want_dh || T.dh, STMP_EINVAL, "stmp_hetero_lstm_bwd: type %d: dh is NULL", t);
    for (int r = 0; r < T.nrel; ++r) {
      T.q[r] = want_dh ? fp(d[26 + r]) : nullptr;
      STMP_REQUIRE(!want_dh || T.q[r], STMP_EINVAL, "stmp_hetero_lstm_bwd: type %d: Q %d is NULL", t, r);
      const int64_t src = d[30 + r], rank = d[34 + r];
      STMP_REQUIRE(src >= 0 && src < num_types && rank >= 0 && rank < kHgMaxTypes * kHgMaxRel, STMP_EINVAL,
                   "stmp_hetero_lstm_bwd: type %d: source %lld or rank %lld out of range", t, (long long)src, (long long)rank);
      order[nedge][0] = t; order[nedge][1] = r; ++nedge;
    }
    tiles += (T.n + kRowTile - 1) / kRowTile;
    HgWgType& W = wg.t[t];
    W.dpre = T.dpre; W.S = fp(d[19]); W.dw = fp(d[38]); W.n = T.n; W.nb = hg_nb(CO, d);
    W.tk = (W.nb + 1 + kWgTile - 1) / kWgTile; W.chunks = hg_chunks(d); W.item0 = items;
    W.part = reinterpret_cast<float*>(workspace) + off;
    if (t == 0) wgrad = W.dw != nullptr;
    STMP_REQUIRE((W.dw != nullptr) == wgrad, STMP_EINVAL, "stmp_hetero_lstm_bwd: dw must be given for every type or none");
    items += W.chunks * (wg.M / kWgTile) * W.tk;
    total += wg.M * (W.nb + 1);
    off += (size_t)W.chunks * wg.M * (W.nb + 1);
  }
  STMP_REQUIRE(!wgrad || workspace, STMP_EINVAL, "stmp_hetero_lstm_bwd: workspace is NULL");
  a.tiles = g.tiles = tiles;
  wg.items = items;
  constexpr int smem = 4 * CO * HgWd<NC>::P * 4;
  STMP_CUDA_OK(cudaFuncSetAttribute(k_hetero_lstm_bwd_rows<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const int cap = hg_cap(HgWd<NC>::CTAS);
  k_hetero_lstm_bwd_rows<NC><<<tiles < cap ? tiles : cap, kRowsThreads, smem, st>>>(a);
  STMP_LAUNCH_OK("k_hetero_lstm_bwd_rows");
  if (want_dh) {                               // the outgoing edge types of every source type, in metadata order
    for (int t = 0; t < num_types; ++t) {
      g.t[t].dh = a.t[t].dh; g.t[t].n = a.t[t].n; g.t[t].tile0 = a.t[t].tile0; g.t[t].nout = 0;
    }
    for (int rank = 0; rank < kHgMaxTypes * kHgMaxRel; ++rank)
      for (int e = 0; e < nedge; ++e) {
        const int t = order[e][0], r = order[e][1];
        const int64_t* d = desc + (size_t)t * STMP_HETERO_DESC;
        if (d[34 + r] != rank) continue;
        HgGatherType& S = g.t[d[30 + r]];
        STMP_REQUIRE(S.nout < kHgMaxOut, STMP_EUNSUPPORTED, "stmp_hetero_lstm_bwd: more than %d outgoing edge types of one type", kHgMaxOut);
        const stmp_plan* plan = pp(d[10 + r]);
        STMP_REQUIRE(plan && plan->n >= S.n, STMP_EINVAL, "stmp_hetero_lstm_bwd: type %d: plan %d has too few rows", t, r);
        S.rowptr[S.nout] = plan->bwd[0].rowptr; S.cv[S.nout] = plan->bwd[0].cv; S.q[S.nout] = a.t[t].q[r]; ++S.nout;
      }
    k_hetero_lstm_bwd_gather<NC><<<tiles < 2 * cap ? tiles : 2 * cap, kRowsThreads, 0, st>>>(g);
    STMP_LAUNCH_OK("k_hetero_lstm_bwd_gather");
  }
  if (wgrad) {
    k_hetero_wgrad<<<items, 256, 0, st>>>(wg);
    STMP_LAUNCH_OK("k_hetero_wgrad");
    k_hetero_wgrad_reduce<<<(total + 255) / 256, 256, 0, st>>>(wg, total);
    STMP_LAUNCH_OK("k_hetero_wgrad_reduce");
  }
  return STMP_OK;
}

extern "C" int stmp_hetero_lstm_bwd(int64_t out_channels, int64_t num_types, const int64_t* desc, int want_dh, void* workspace,
                                    void* stream) {
  if (int rc = hg_common("stmp_hetero_lstm_bwd", out_channels, num_types, desc)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  return out_channels == 32 ? hg_bwd<1>(desc, (int)num_types, want_dh, workspace, st)
                            : hg_bwd<2>(desc, (int)num_types, want_dh, workspace, st);
}
