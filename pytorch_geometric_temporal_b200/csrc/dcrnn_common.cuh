// dcrnn_common.cuh -- device helpers shared by the fused DCRNN sequence kernels (FFMA and wgmma variants).
#pragma once
#include "common.cuh"

namespace stmp {

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
// Two independent fp32 FMAs (round to nearest, as one fma.rn each).
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ void fma4(float4& acc, float w, const float4& x) {
  acc = make_float4(fmaf(w, x.x, acc.x), fmaf(w, x.y, acc.y), fmaf(w, x.z, acc.z), fmaf(w, x.w, acc.w));
}

// Shared-memory form of the two operators, built once per CTA from the plan's CSR:
//   * every (row, op) task's edge list is padded to a multiple of `pad` (4, or 2 = groups of 4 + one 2-edge tail)
//     with (self, 0.0f) entries, so the gather loop has no per-edge predication;
//   * the column index is pre-multiplied by LD (element offset of the source row in S);
//   * tasks are ordered by descending group count, so the quarter-warps of a warp (consecutive slots)
//     walk rows of equal length -- no divergence inside a warp pass.
struct GraphSmem {
  const int2* ce;      // padded (src_row*LD, val) entries
  const int* gstart;   // [2N+1] first padded entry of task
  const int* order;    // [2N] task ids (op*N + row) sorted by descending padded length
};

// sum over the padded edge list of one task for the float4 at S[src*LD + coff .. +3]
// (edge lists padded to a multiple of 4, or of 2 with a 2-edge tail group)
__device__ __forceinline__ float4 gather_row(const float* __restrict__ Sc, const int2* __restrict__ ce, int beg, int end) {
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  int k = beg;
  for (; k + 4 <= end; k += 4) {
    const int4 e01 = *reinterpret_cast<const int4*>(ce + k);      // two edges per 128-bit load
    const int4 e23 = *reinterpret_cast<const int4*>(ce + k + 2);
    const float4 x0 = ld4(Sc + e01.x);
    const float4 x1 = ld4(Sc + e01.z);
    const float4 x2 = ld4(Sc + e23.x);
    const float4 x3 = ld4(Sc + e23.z);
    fma4(acc, __int_as_float(e01.y), x0);
    fma4(acc, __int_as_float(e01.w), x1);
    fma4(acc, __int_as_float(e23.y), x2);
    fma4(acc, __int_as_float(e23.w), x3);
  }
  if (k < end) {   // 2-edge tail (pad == 2)
    const int4 e01 = *reinterpret_cast<const int4*>(ce + k);
    const float4 x0 = ld4(Sc + e01.x);
    const float4 x1 = ld4(Sc + e01.z);
    fma4(acc, __int_as_float(e01.y), x0);
    fma4(acc, __int_as_float(e01.w), x1);
  }
  return acc;
}


// Build the GraphSmem arrays from the plan's two CSR operators (global memory).  `pitch` = element pitch of
// a source row in the gather buffer.  Must be called by all NT threads; ends with the arrays complete after
// the caller's next __syncthreads().
template <int NT>
__device__ __forceinline__ void stage_graph(const int* __restrict__ grp0, const int* __restrict__ grp1, const int2* __restrict__ gcv0,
                                            const int2* __restrict__ gcv1, int N, int pitch, int2* s_ce, int* s_gstart, int* s_order,
                                            int tid, int split_row = 1 << 30, int n_ops = 2, int pad = 4) {
  const int NTASK = n_ops * N;
  int* s_len = s_order;  // scratch until the ranking pass writes it
  for (int task = tid; task < NTASK; task += NT) {
    const int op = task >= N ? 1 : 0, i = task - op * N;
    const int* rp = op ? grp1 : grp0;
    s_len[task] = (rp[i + 1] - rp[i] + pad - 1) & ~(pad - 1);
  }
  __syncthreads();
  if (tid == 0) {
    int run = 0;
    for (int task = 0; task < NTASK; ++task) { s_gstart[task] = run; run += s_len[task]; }
    s_gstart[NTASK] = run;
  }
  __syncthreads();
  for (int task = tid; task < NTASK; task += NT) {
    const int op = task >= N ? 1 : 0, i = task - op * N;
    const int* rp = op ? grp1 : grp0;
    const int2* cv = op ? gcv1 : gcv0;
    const int beg = rp[i], len = rp[i + 1] - beg, plen = s_gstart[task + 1] - s_gstart[task];
    int2* dst = s_ce + s_gstart[task];
    for (int k = 0; k < plen; ++k) {
      int2 e = k < len ? cv[beg + k] : make_int2(i, 0);
      e.x *= pitch;
      dst[k] = e;
    }
  }
  __syncthreads();
  // order tasks: rows >= split_row first (the second MMA row tile of the wgmma kernel), then by descending
  // padded length (rank = number of tasks that sort before this one)
  for (int task = tid; task < NTASK; task += NT) {
    const int len = s_gstart[task + 1] - s_gstart[task];
    const int hi = ((task >= N ? task - N : task) >= split_row) ? 1 : 0;
    int rank = 0;
    for (int o = 0; o < NTASK; ++o) {
      const int lo = s_gstart[o + 1] - s_gstart[o];
      const int ho = ((o >= N ? o - N : o) >= split_row) ? 1 : 0;
      rank += (ho > hi) || (ho == hi && ((lo > len) || (lo == len && o < task)));
    }
    s_order[rank] = task;
  }
}

}  // namespace stmp
