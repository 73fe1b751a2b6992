// common.cuh -- shared helpers for libstmp (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <atomic>
#include <cstdarg>
#include <cstdio>

#include "../../include/stmp.h"

namespace stmp {

// ---- error reporting (thread-local, no exceptions across the C ABI) ---------------------------------
char* err_buf();
int set_error(int code, const char* fmt, ...);
extern std::atomic<long long> g_launches;
inline void count_launch(int n = 1) { g_launches.fetch_add(n, std::memory_order_relaxed); }
// per-kernel launch counters ("which path served this call"): a call site registers its kernel name once and then bumps its slot
int path_slot(const char* name);
void count_path(int slot);

// ---- run-time switches (stmp_set_option, plan.cu) ----------------------------------------------------
// Each selects an independent implementation or a launch shape that a test compares the default against.
extern int g_dcrnn_tc;     // "dcrnn_tc": 1 wgmma forward (dcrnn_seq_tc.cu) / 0 exact-fp32 FFMA forward (dcrnn_seq.cu)
extern int g_fwd_split;    // "dcrnn_fwd_split": 1 a CTA pair per window for small batches / 0 one CTA per window (wgmma forward)
extern int g_bwd_split;    // "dcrnn_bwd_split": the same choice for the persistent backward (dcrnn_bwd.cu)
extern int g_wgrad_tc;     // "dcrnn_wgrad_tc": 1 wgmma weight-gradient contraction (wgrad_tc.cu) / 0 FFMA (train.cu)
extern int g_narrow_pack;  // "dcrnn_narrow_pack": windows per CTA of the narrow DCRNN kernels (dcrnn_narrow.cu), 0 = automatic

#define STMP_CUDA_OK(expr)                                                                    \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      (void)cudaGetLastError();  /* consumed here, so the next STMP_LAUNCH_OK does not report it */ \
      return stmp::set_error(STMP_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), \
                             __FILE__, __LINE__);                                             \
    }                                                                                         \
  } while (0)

#define STMP_LAUNCH_OK(name)                                                                  \
  do {                                                                                        \
    cudaError_t _e = cudaGetLastError();                                                      \
    if (_e != cudaSuccess)                                                                    \
      return stmp::set_error(STMP_ECUDA, "launch of %s failed: %s", name, cudaGetErrorString(_e)); \
    stmp::count_launch();                                                                     \
    static const int _path_slot = stmp::path_slot(name);                                      \
    stmp::count_path(_path_slot);                                                             \
  } while (0)

#define STMP_REQUIRE(cond, code, ...)                      \
  do {                                                     \
    if (!(cond)) return stmp::set_error(code, __VA_ARGS__); \
  } while (0)

// ---- plan layout -------------------------------------------------------------------------------------
// One sparse operator in CSR form.  `cv[k]` packs (column index, value bits) so one 64-bit load
// fetches an edge.  Entries of a row keep the reference's scatter order (stable sort).
struct Csr {
  int n = 0;
  int nnz = 0;
  int max_row_nnz = 0;
  int* rowptr = nullptr;  // [n+1]
  int2* cv = nullptr;     // [nnz] (col, __float_as_int(val))
  int* eid = nullptr;     // [nnz] position in the reference-order COO list
};

}  // namespace stmp

struct stmp_plan {
  int flavor = 0;
  int n = 0;
  long long e = 0;
  int n_ops = 0;
  int normalization = 0;
  unsigned flags = 0;
  float lambda_max = 0.f;
  bool nonfinite_vals = false;   // an operator holds a non-finite value (DConv: 1/deg_in = inf at a source of in-degree 0)
  stmp::Csr fwd[2];  // by destination
  stmp::Csr bwd[2];  // by source (transposed product)
  int device = 0;
  // Shared-memory image of the first n_ops operators for the fused tensor-core kernel (gstart | order | padded edge
  // entries, exactly as the kernel lays them out), built once at plan creation when the graph fits (N <= 207):
  // the kernel then fetches it with ONE TMA bulk copy instead of re-staging the CSR in every CTA.
  void* gimg[3] = {nullptr, nullptr, nullptr};   // index = n_ops (1, 2)
  int gimg_bytes[3] = {0, 0, 0};
  // Row image of the first n_ops operators for the one-CTA kernel (row_image.cuh): nodes mapped onto the MMA rows, gather lists
  // per (warp, operator, slot).  Its size follows from the number of group rows.
  void* rimg[3] = {nullptr, nullptr, nullptr};
  int rimg_groups[3] = {0, 0, 0};
  int aggr = 0;                  // STMP_FLAVOR_GATED: the stmp_aggr its operator was built for
};

namespace stmp {

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// ---- small PTX wrappers (sm_90a) ---------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Blocking wait.  try_wait suspends the thread in hardware until the phase completes or a time limit expires; with the default
// limit the loop re-polls about once a microsecond and the polls of waiting warps crowd the MIO queue that the working warps' LDS /
// MUFU instructions go through (round-2 profile: 13 % of all issued instructions were re-polls).  A long suspend-time hint keeps a
// waiting warp asleep until the barrier actually flips.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity), "r"(0x989680u)
        : "memory");
  } while (!ok);
}
// TMA 1-D bulk copy global -> shared, completion on an mbarrier (SASS: UBLKCP).
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// TMA 1-D bulk copy shared -> global (bulk async-group completion).
__device__ __forceinline__ void tma_bulk_s2g(void* dst_gmem, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem),
               "r"(smem_u32(src_smem)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ---- thread-block-cluster helpers (CTA pairs: the small-batch variants of the DCRNN sequence kernels) ------------------------------
__device__ __forceinline__ uint32_t cluster_rank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r)); return r; }
__device__ __forceinline__ void cluster_sync_all() {          // data barrier: my (remote) shared-memory stores are visible to the pair behind it
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// execution-only barrier, split: "I am done READING buf" is signalled right after the gather phase (relaxed: no memory ordering, so the
// phase's global stores are not drained -- the release form spent 14 % of the kernel in ERRBAR) and waited for only where the next GEMM is
// about to overwrite the partner's buf, i.e. behind its FFMA loop.
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t map_to_peer(const void* p, uint32_t peer) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(p)), "r"(peer));
  return r;
}
__device__ __forceinline__ void st4_cluster(uint32_t addr, float4 v) {
  asm volatile("st.shared::cluster.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void st2_cluster(uint32_t addr, float2 v) {
  asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(v.x), "f"(v.y) : "memory");
}

// 16-byte store into the partner CTA's shared memory that also completes 16 transaction bytes on an mbarrier THERE: the receiver waits on its
// own mbarrier for the expected byte count instead of meeting the sender at a release / acquire cluster barrier.
__device__ __forceinline__ void st4_async_cluster(uint32_t addr, float4 v, uint32_t remote_mbar) {
  asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(addr), "f"(v.x),
               "f"(v.y), "f"(v.z), "f"(v.w), "r"(remote_mbar)
               : "memory");
}
// 1/(1+e^-x): __frcp_rn is the correctly rounded reciprocal == IEEE 1.0f/y, without the division slow path.
__device__ __forceinline__ float sigmoidf_acc(float x) { return __frcp_rn(1.0f + expf(-x)); }

}  // namespace stmp
