// plan.cu -- device-side construction of the cached graph operators (K2 in SURVEY.md section 2a).
//
// The reference renormalises the static graph on every layer call (dense adjacency + nonzero() in
// nn/recurrent/dcrnn.py:59-77, PyG get_laplacian / gcn_norm inside ChebConv / GCNConv,
// nn/attention/astgcn.py:82-110).  Here the normalised operator is built ONCE per graph, on the GPU:
// a reference-order COO list (the order the reference's scatter_add_ visits entries) is produced per
// flavor and stable-radix-sorted into CSR by destination (forward) and by source (transposed product
// for the backward pass).  All value arithmetic mirrors the reference's op order with explicit
// round-to-nearest intrinsics (no FMA contraction) so plan values are bit-identical to the oracle.
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>
#include <numeric>
#include <vector>

#include <cstring>
#include <mutex>

#include "common.cuh"
#include "dcrnn_common.cuh"
#include "graph_image.cuh"
#include "row_image.cuh"

namespace stmp {

// ---------------------------------------------------------------------------------------------------------
// error plumbing
// ---------------------------------------------------------------------------------------------------------
std::atomic<long long> g_launches{0};

// run-time switches (common.cuh, stmp_set_option below)
int g_dcrnn_tc = 1;
int g_fwd_split = 1;       // 64 windows: 200 -> 171 us (H100 SXM, 700 W)
int g_bwd_split = 1;
int g_wgrad_tc = 1;
int g_narrow_pack = 0;

// ---- per-kernel launch counters (stmp_path_counters) ----------------------------------------------------
constexpr int kMaxPaths = 256;  // more than the library's distinct launch names: past the last slot, names would share one counter
static const char* g_path_names[kMaxPaths];
static std::atomic<long long> g_path_counts[kMaxPaths];
static std::atomic<int> g_n_paths{0};
static std::mutex g_path_mu;
int path_slot(const char* name) {
  std::lock_guard<std::mutex> lk(g_path_mu);
  const int n = g_n_paths.load();
  for (int i = 0; i < n; ++i)
    if (strcmp(g_path_names[i], name) == 0) return i;
  if (n >= kMaxPaths) return kMaxPaths - 1;
  g_path_names[n] = name;
  g_path_counts[n].store(0);
  g_n_paths.store(n + 1);
  return n;
}
void count_path(int slot) { g_path_counts[slot].fetch_add(1, std::memory_order_relaxed); }

char* err_buf() {
  static thread_local char buf[512] = {0};
  return buf;
}
int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(err_buf(), 512, fmt, ap);
  va_end(ap);
  return code;
}

namespace {

constexpr int kThreads = 256;
inline int blocks_for(long long n) { return (int)((n + kThreads - 1) / kThreads) > 0 ? (int)((n + kThreads - 1) / kThreads) : 1; }

// err flag bits
constexpr int kErrRange = 1;
constexpr int kErrDuplicate = 2;
constexpr int kNonFinite = 4;   // not an error: an operator holds a non-finite value (stmp_plan::nonfinite_vals)

struct Info {
  int err;
  int max_row[4];
  int count;  // compaction total
};

// ---------------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------------
__global__ void k_split_index(long long e, const long long* __restrict__ ei, int n, int* __restrict__ row,
                              int* __restrict__ col, Info* info) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= e) return;
  long long r = ei[i], c = ei[e + i];
  if (r < 0 || r >= n || c < 0 || c >= n) {
    atomicOr(&info->err, kErrRange);
    r = 0;
    c = 0;
  }
  row[i] = (int)r;
  col[i] = (int)c;
}

__global__ void k_iota(int n, int* out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = i;
}

__global__ void k_gather_int(int n, const int* __restrict__ src, const int* __restrict__ idx, int* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = src[idx[i]];
}

// rowptr[k] = first position in sorted keys with key >= k   (k in [0, n])
__global__ void k_rowptr(int n, int nnz, const int* __restrict__ keys_sorted, int* __restrict__ rowptr) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k > n) return;
  int lo = 0, hi = nnz;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (keys_sorted[mid] < k) lo = mid + 1; else hi = mid;
  }
  rowptr[k] = lo;
}

__global__ void k_max_row(int n, const int* __restrict__ rowptr, int* out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicMax(out, rowptr[i + 1] - rowptr[i]);
}

// out[i] = sum over the segment of w[perm[k]] in order (w == nullptr -> ones); sequential = the order
// of a CPU scatter_add_.
__global__ void k_segment_sum(int n, const int* __restrict__ rowptr, const int* __restrict__ perm,
                              const float* __restrict__ w, float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int k = rowptr[i]; k < rowptr[i + 1]; ++k) s = __fadd_rn(s, w ? w[perm[k]] : 1.0f);
  out[i] = s;
}

__global__ void k_fill_csr(int nnz, const int* __restrict__ perm, const int* __restrict__ src,
                           const float* __restrict__ val, int2* __restrict__ cv, int* __restrict__ eid, Info* info) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nnz) return;
  int p = perm[k];
  cv[k] = make_int2(src[p], __float_as_int(val[p]));
  eid[k] = p;
  if (!isfinite(val[p])) atomicOr(&info->err, kNonFinite);
}

// ---- DCONV ------------------------------------------------------------------------------------------
__global__ void k_dconv_out_vals(int e, const int* __restrict__ row, const float* __restrict__ deg_out,
                                 float* __restrict__ val) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < e) val[i] = __frcp_rn(deg_out[row[i]]);  // torch.reciprocal(deg_out)[row]   dcrnn.py:70,73
}

// p-th entry of the reverse list (sorted by (col,row)): dst=row[q], src=col[q], val = 1/deg_in[row[p]].
__global__ void k_dconv_in_coo(int e, const int* __restrict__ q, const int* __restrict__ row,
                               const int* __restrict__ col, const float* __restrict__ deg_in,
                               int* __restrict__ dst, int* __restrict__ src, float* __restrict__ val,
                               int allow_dup, Info* info) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= e) return;
  int qe = q[p];
  dst[p] = row[qe];
  src[p] = col[qe];
  val[p] = __frcp_rn(deg_in[row[p]]);  // deg_in_inv[row] paired positionally   dcrnn.py:71,74
  if (!allow_dup && p > 0) {
    int qp = q[p - 1];
    if (row[qp] == row[qe] && col[qp] == col[qe]) atomicOr(&info->err, kErrDuplicate);
  }
}

// ---- loop removal / compaction ------------------------------------------------------------------------
__global__ void k_flag_nonloop(int e, const int* __restrict__ row, const int* __restrict__ col, int* __restrict__ flag) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < e) flag[i] = row[i] != col[i];
}
__global__ void k_compact(int e, const int* __restrict__ flag, const int* __restrict__ pos,
                          const int* __restrict__ row, const int* __restrict__ col, const float* __restrict__ w,
                          int* __restrict__ r2, int* __restrict__ c2, float* __restrict__ w2, Info* info) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= e) return;
  if (flag[i]) {
    int p = pos[i];
    r2[p] = row[i];
    c2[p] = col[i];
    w2[p] = w ? w[i] : 1.0f;
  }
  if (i == e - 1) info->count = pos[i] + flag[i];
}

// ---- RGCN: relation-masked mean operators ------------------------------------------------------------
__global__ void k_flag_relation(int e, const long long* __restrict__ type, long long rel, int* __restrict__ flag) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < e) flag[i] = type[i] == rel;
}
// 1 / cnt_r(dst): every destination that holds an entry has a count >= 1 (the reference's clamp(min=1) never applies to one)
__global__ void k_mean_vals(int e, const int* __restrict__ dst, const float* __restrict__ cnt, float* __restrict__ val) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < e) val[i] = __frcp_rn(cnt[dst[i]]);
}

// ---- GATED: GatedGraphConv's aggregation operator ----------------------------------------------------
// add / max: the edge weight (1 without weights); mean: the weight divided by the destination's count of in-edges (>= 1 at every entry)
__global__ void k_gated_vals(int e, const int* __restrict__ dst, const float* __restrict__ w, const float* __restrict__ cnt,
                             float* __restrict__ val) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= e) return;
  const float v = w ? w[i] : 1.0f;
  val[i] = cnt ? __fdiv_rn(v, cnt[dst[i]]) : v;
}

// ---- Laplacian (PyG get_laplacian) -------------------------------------------------------------------
// entries [0,e2): non-loop edges; [e2, e2+n): loops.  Produces UNSCALED laplacian weights.
__global__ void k_laplacian_vals(int e2, int n, int normalization, const int* __restrict__ r2,
                                 const int* __restrict__ c2, const float* __restrict__ w2,
                                 const float* __restrict__ deg, float* __restrict__ val) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= e2 + n) return;
  if (k < e2) {
    float w = w2[k];
    float v;
    if (normalization == STMP_NORM_NONE) {
      v = w;
    } else if (normalization == STMP_NORM_SYM) {
      float dr = __fdiv_rn(1.0f, __fsqrt_rn(deg[r2[k]]));  // deg.pow(-0.5) == rsqrt on the CPU path
      float dc = __fdiv_rn(1.0f, __fsqrt_rn(deg[c2[k]]));
      if (isinf(dr)) dr = 0.f;
      if (isinf(dc)) dc = 0.f;
      v = __fmul_rn(__fmul_rn(dr, w), dc);
    } else {
      float di = __fdiv_rn(1.0f, deg[r2[k]]);
      if (isinf(di)) di = 0.f;
      v = __fmul_rn(di, w);
    }
    val[k] = -v;
  } else {
    val[k] = (normalization == STMP_NORM_NONE) ? deg[k - e2] : 1.0f;
  }
}

// w_hat = 2*w/lam ; inf -> 0 ; (cheb) loops -= 1.  lam read from device memory.
// lam_node (nullable): per-node lambda_max = lambda_max[batch[node]] of a multi-graph mini-batch; the entry's lambda is the one
// of its ROW node (PyG: lambda_max[batch[edge_index[0]]] on the get_laplacian list; loop entry k >= e2 has row (k - e2) % n).
__global__ void k_scale_lambda(int nnz, int e2, const float* __restrict__ lam, int sub_loops, float* __restrict__ val,
                               const float* __restrict__ lam_node = nullptr, const int* __restrict__ r2 = nullptr, int n = 1) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nnz) return;
  const float l = lam_node ? lam_node[k < e2 ? r2[k] : (k - e2) % n] : *lam;
  float v = __fdiv_rn(__fmul_rn(2.0f, val[k]), l);
  if (v == INFINITY) v = 0.f;  // masked_fill_(== inf): only +inf
  if (sub_loops && k >= e2) v = __fsub_rn(v, 1.0f);
  val[k] = v;
}
__global__ void k_times2(float* lam) { *lam = __fmul_rn(2.0f, *lam); }
__global__ void k_set(float* p, float v) { *p = v; }

// COO index arrays for "edges then loops" lists.  swap=1 -> dst=row, src=col (transposed propagate).
__global__ void k_edges_then_loops(int e2, int n, int nloops_sets, const int* __restrict__ r2, const int* __restrict__ c2,
                                   int swap, int* __restrict__ dst, int* __restrict__ src) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  int total = e2 + n * nloops_sets;
  if (k >= total) return;
  if (k < e2) {
    dst[k] = swap ? r2[k] : c2[k];
    src[k] = swap ? c2[k] : r2[k];
  } else {
    int i = (k - e2) % n;
    dst[k] = i;
    src[k] = i;
  }
}
__global__ void k_fill_tail(int begin, int count, float v, float* __restrict__ val) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < count) val[begin + k] = v;
}

// ---- GCN ---------------------------------------------------------------------------------------------
__global__ void k_fill_int(int n, int v, int* p) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
__global__ void k_gcn_loop_owner(int e, const int* __restrict__ row, const int* __restrict__ col, int* __restrict__ owner) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < e && row[i] == col[i]) atomicMax(&owner[row[i]], i);  // last existing loop wins
}
__global__ void k_gcn_loop_w(int n, int e2, const int* __restrict__ owner, const float* __restrict__ w, float fill,
                             float* __restrict__ wcoo) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int o = owner[i];
  wcoo[e2 + i] = (o >= 0) ? (w ? w[o] : 1.0f) : fill;
}
__global__ void k_copy_w(int e, const float* __restrict__ w, float* __restrict__ out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < e) out[i] = w ? w[i] : 1.0f;
}
__global__ void k_gcn_vals(int nnz, const int* __restrict__ dst, const int* __restrict__ src,
                           const float* __restrict__ wcoo, const float* __restrict__ deg, float* __restrict__ val) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nnz) return;
  float ds = __fdiv_rn(1.0f, __fsqrt_rn(deg[src[k]]));
  float dd = __fdiv_rn(1.0f, __fsqrt_rn(deg[dst[k]]));
  if (isinf(ds)) ds = 0.f;
  if (isinf(dd)) dd = 0.f;
  val[k] = __fmul_rn(__fmul_rn(ds, wcoo[k]), dd);  // dis[row] * w * dis[col]
}

__global__ void k_export(int nnz, const int2* __restrict__ cv, const int* __restrict__ eid_in, int* __restrict__ col,
                         float* __restrict__ val, int* __restrict__ eid) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nnz) return;
  int2 v = cv[k];
  if (col) col[k] = v.x;
  if (val) val[k] = __int_as_float(v.y);
  if (eid) eid[k] = eid_in[k];
}

// ---------------------------------------------------------------------------------------------------------
// host-side builder
// ---------------------------------------------------------------------------------------------------------
struct Builder {
  cudaStream_t st;
  std::vector<void*> tmp;
  Info* d_info = nullptr;
  int rc = 0;

  ~Builder() {
    for (void* p : tmp) cudaFree(p);
  }
  template <class T>
  T* talloc(size_t n) {
    T* p = nullptr;
    if (cudaMalloc(&p, (n ? n : 1) * sizeof(T)) != cudaSuccess) {
      rc = set_error(STMP_ENOMEM, "cudaMalloc of %zu bytes failed", n * sizeof(T));
      (void)cudaGetLastError();
      return nullptr;
    }
    tmp.push_back(p);
    return p;
  }
  static int bits_for(int n) {
    int b = 1;
    while ((1ll << b) < n) ++b;
    return b;
  }
  // stable sort (keys, iota) -> (keys_sorted, perm).  perm_in optional (defaults to iota).
  int sort_pairs(int num, int n_keys, const int* keys, const int* vals_in, int* keys_sorted, int* perm) {
    if (num == 0) return 0;
    int* iota = nullptr;
    if (!vals_in) {
      iota = talloc<int>(num);
      if (!iota) return rc;
      k_iota<<<blocks_for(num), kThreads, 0, st>>>(num, iota);
      STMP_LAUNCH_OK("k_iota");
      vals_in = iota;
    }
    size_t tb = 0;
    STMP_CUDA_OK(cub::DeviceRadixSort::SortPairs(nullptr, tb, keys, keys_sorted, vals_in, perm, num, 0, bits_for(n_keys), st));
    void* t = talloc<char>(tb);
    if (!t) return rc;
    STMP_CUDA_OK(cub::DeviceRadixSort::SortPairs(t, tb, keys, keys_sorted, vals_in, perm, num, 0, bits_for(n_keys), st));
    count_launch(3);
    return 0;
  }
  // CSR structure of `keys` over n segments: perm (stable) + rowptr (temporary buffers).
  int segments(int num, int n, const int* keys, int** perm_out, int** rowptr_out) {
    int* ks = talloc<int>(num);
    int* perm = talloc<int>(num);
    int* rowptr = talloc<int>(n + 1);
    if (!ks || !perm || !rowptr) return rc;
    int r = sort_pairs(num, n, keys, nullptr, ks, perm);
    if (r) return r;
    k_rowptr<<<blocks_for(n + 1), kThreads, 0, st>>>(n, num, ks, rowptr);
    STMP_LAUNCH_OK("k_rowptr");
    *perm_out = perm;
    *rowptr_out = rowptr;
    return 0;
  }
  int segment_sum(int num, int n, const int* keys, const float* w, float** out) {
    int *perm, *rowptr;
    int r = segments(num, n, keys, &perm, &rowptr);
    if (r) return r;
    float* o = talloc<float>(n);
    if (!o) return rc;
    k_segment_sum<<<blocks_for(n), kThreads, 0, st>>>(n, rowptr, perm, w, o);
    STMP_LAUNCH_OK("k_segment_sum");
    *out = o;
    return 0;
  }
  // Persistent CSR (owned by the plan) from a reference-order COO list.
  int build_csr(int n, int nnz, const int* dst, const int* src, const float* val, Csr* out, int info_slot) {
    out->n = n;
    out->nnz = nnz;
    STMP_CUDA_OK(cudaMalloc(&out->rowptr, (size_t)(n + 1) * sizeof(int)));
    STMP_CUDA_OK(cudaMalloc(&out->cv, (size_t)(nnz ? nnz : 1) * sizeof(int2)));
    STMP_CUDA_OK(cudaMalloc(&out->eid, (size_t)(nnz ? nnz : 1) * sizeof(int)));
    int* ks = talloc<int>(nnz);
    int* perm = talloc<int>(nnz);
    if (!ks || !perm) return rc;
    int r = sort_pairs(nnz, n, dst, nullptr, ks, perm);
    if (r) return r;
    k_rowptr<<<blocks_for(n + 1), kThreads, 0, st>>>(n, nnz, ks, out->rowptr);
    STMP_LAUNCH_OK("k_rowptr");
    if (nnz) {
      k_fill_csr<<<blocks_for(nnz), kThreads, 0, st>>>(nnz, perm, src, val, out->cv, out->eid, d_info);
      STMP_LAUNCH_OK("k_fill_csr");
    }
    k_max_row<<<blocks_for(n), kThreads, 0, st>>>(n, out->rowptr, &d_info->max_row[info_slot]);
    STMP_LAUNCH_OK("k_max_row");
    return 0;
  }
  int both_csr(stmp_plan* p, int op, int n, int nnz, const int* dst, const int* src, const float* val) {
    int r = build_csr(n, nnz, dst, src, val, &p->fwd[op], op * 2);
    if (r) return r;
    return build_csr(n, nnz, src, dst, val, &p->bwd[op], op * 2 + 1);
  }
  // remove self loops, keeping order: outputs r2,c2,w2 and the kept count (host sync).
  int compact_nonloops(int e, const int* row, const int* col, const float* w, int** r2, int** c2, float** w2, int* e2) {
    int* flag = e ? talloc<int>(e) : nullptr;
    if (e && !flag) return rc;
    if (e) {
      k_flag_nonloop<<<blocks_for(e), kThreads, 0, st>>>(e, row, col, flag);
      STMP_LAUNCH_OK("k_flag_nonloop");
    }
    return compact(e, flag, row, col, w, r2, c2, w2, e2);
  }
  // keep the edges whose flag is set, in order: outputs r2,c2,w2 and the kept count (host sync).
  int compact(int e, int* flag, const int* row, const int* col, const float* w, int** r2, int** c2, float** w2, int* e2) {
    *r2 = talloc<int>(e);
    *c2 = talloc<int>(e);
    *w2 = talloc<float>(e);
    if (!*r2 || !*c2 || !*w2) return rc;
    *e2 = 0;
    if (e == 0) return 0;
    int* pos = talloc<int>(e);
    if (!pos) return rc;
    size_t tb = 0;
    STMP_CUDA_OK(cub::DeviceScan::ExclusiveSum(nullptr, tb, flag, pos, e, st));
    void* t = talloc<char>(tb);
    if (!t) return rc;
    STMP_CUDA_OK(cub::DeviceScan::ExclusiveSum(t, tb, flag, pos, e, st));
    count_launch(2);
    k_compact<<<blocks_for(e), kThreads, 0, st>>>(e, flag, pos, row, col, w, *r2, *c2, *w2, d_info);
    STMP_LAUNCH_OK("k_compact");
    Info h;
    STMP_CUDA_OK(cudaMemcpyAsync(&h, d_info, sizeof(Info), cudaMemcpyDeviceToHost, st));
    STMP_CUDA_OK(cudaStreamSynchronize(st));
    *e2 = h.count;
    return 0;
  }
};

int build_dconv(Builder& b, stmp_plan* p, int n, int e, const int* row, const int* col, const float* w) {
  float *deg_out, *deg_in;
  int r;
  if ((r = b.segment_sum(e, n, row, w, &deg_out))) return r;  // dcrnn.py:61-64 / :279
  if ((r = b.segment_sum(e, n, col, w, &deg_in))) return r;   // dcrnn.py:65-68 / :280
  // op 0 (out): reference-order COO is the edge list itself.
  float* val0 = b.talloc<float>(e);
  if (!val0) return b.rc;
  if (e) {
    k_dconv_out_vals<<<blocks_for(e), kThreads, 0, b.st>>>(e, row, deg_out, val0);
    STMP_LAUNCH_OK("k_dconv_out_vals");
  }
  if ((r = b.both_csr(p, 0, n, e, col, row, val0))) return r;
  // op 1 (in): reverse list sorted by (col,row) = stable sort by row, then stable sort by col.
  int* ks = b.talloc<int>(e);
  int* perm_r = b.talloc<int>(e);
  int* key2 = b.talloc<int>(e);
  int* ks2 = b.talloc<int>(e);
  int* q = b.talloc<int>(e);
  int* dst1 = b.talloc<int>(e);
  int* src1 = b.talloc<int>(e);
  float* val1 = b.talloc<float>(e);
  if (!ks || !perm_r || !key2 || !ks2 || !q || !dst1 || !src1 || !val1) return b.rc;
  if (e) {
    if ((r = b.sort_pairs(e, n, row, nullptr, ks, perm_r))) return r;
    k_gather_int<<<blocks_for(e), kThreads, 0, b.st>>>(e, col, perm_r, key2);
    STMP_LAUNCH_OK("k_gather_int");
    if ((r = b.sort_pairs(e, n, key2, perm_r, ks2, q))) return r;
    k_dconv_in_coo<<<blocks_for(e), kThreads, 0, b.st>>>(e, q, row, col, deg_in, dst1, src1, val1,
                                                          (p->flags & STMP_DCONV_ALLOW_DUPLICATES) ? 1 : 0, b.d_info);
    STMP_LAUNCH_OK("k_dconv_in_coo");
  }
  if ((r = b.both_csr(p, 1, n, e, dst1, src1, val1))) return r;
  p->n_ops = 2;
  return 0;
}

// Shared by CHEB and CHEB_ATT: unscaled laplacian COO values for "E' edges then N loops".
int laplacian(Builder& b, int n, int e, const int* row, const int* col, const float* w, int normalization,
              int extra_loop_sets, int** r2o, int** c2o, float** valo, int* e2o) {
  int *r2, *c2;
  float* w2;
  int e2, r;
  if ((r = b.compact_nonloops(e, row, col, w, &r2, &c2, &w2, &e2))) return r;
  float* deg;
  if ((r = b.segment_sum(e2, n, r2, w2, &deg))) return r;  // deg = scatter_add(w, row)
  int total = e2 + n * (1 + extra_loop_sets);
  float* val = b.talloc<float>(total);
  if (!val) return b.rc;
  k_laplacian_vals<<<blocks_for(e2 + n), kThreads, 0, b.st>>>(e2, n, normalization, r2, c2, w2, deg, val);
  STMP_LAUNCH_OK("k_laplacian_vals");
  *r2o = r2;
  *c2o = c2;
  *valo = val;
  *e2o = e2;
  return 0;
}

int build_cheb(Builder& b, stmp_plan* p, int n, int e, const int* row, const int* col, const float* w, float lambda_max,
               const float* lam_node = nullptr) {
  int *r2, *c2, e2, r;
  float* val;
  if ((r = laplacian(b, n, e, row, col, w, p->normalization, 0, &r2, &c2, &val, &e2))) return r;
  int nnz = e2 + n;
  float* d_lam = b.talloc<float>(1);
  if (!d_lam) return b.rc;
  if (lambda_max > 0.f || lam_node) {
    k_set<<<1, 1, 0, b.st>>>(d_lam, lam_node ? 0.f : lambda_max);
    STMP_LAUNCH_OK("k_set");
  } else {
    // current PyG: lambda_max = 2 * edge_weight.max()   (SURVEY.md Appendix A.4)
    size_t tb = 0;
    STMP_CUDA_OK(cub::DeviceReduce::Max(nullptr, tb, val, d_lam, nnz, b.st));
    void* t = b.talloc<char>(tb);
    if (!t) return b.rc;
    STMP_CUDA_OK(cub::DeviceReduce::Max(t, tb, val, d_lam, nnz, b.st));
    count_launch(1);
    k_times2<<<1, 1, 0, b.st>>>(d_lam);
    STMP_LAUNCH_OK("k_times2");
  }
  k_scale_lambda<<<blocks_for(nnz), kThreads, 0, b.st>>>(nnz, e2, d_lam, 1, val, lam_node, r2, n);
  STMP_LAUNCH_OK("k_scale_lambda");
  STMP_CUDA_OK(cudaMemcpyAsync(&p->lambda_max, d_lam, sizeof(float), cudaMemcpyDeviceToHost, b.st));
  int* dst = b.talloc<int>(nnz);
  int* src = b.talloc<int>(nnz);
  if (!dst || !src) return b.rc;
  k_edges_then_loops<<<blocks_for(nnz), kThreads, 0, b.st>>>(e2, n, 1, r2, c2, 0, dst, src);
  STMP_LAUNCH_OK("k_edges_then_loops");
  if ((r = b.both_csr(p, 0, n, nnz, dst, src, val))) return r;
  p->n_ops = 1;
  return 0;
}

int build_cheb_att(Builder& b, stmp_plan* p, int n, int e, const int* row, const int* col, const float* w, float lambda_max,
                   const float* lam_node = nullptr) {
  int *r2, *c2, e2, r;
  float* val;
  if ((r = laplacian(b, n, e, row, col, w, p->normalization, 1, &r2, &c2, &val, &e2))) return r;
  int nnz = e2 + 2 * n;
  float* d_lam = b.talloc<float>(1);
  if (!d_lam) return b.rc;
  float lam = lambda_max > 0.f ? lambda_max : 2.0f;  // astgcn.py:141-142
  p->lambda_max = lam;
  k_set<<<1, 1, 0, b.st>>>(d_lam, lam);
  STMP_LAUNCH_OK("k_set");
  k_scale_lambda<<<blocks_for(e2 + n), kThreads, 0, b.st>>>(e2 + n, e2, d_lam, 0, val, lam_node, r2, n);
  STMP_LAUNCH_OK("k_scale_lambda");
  k_fill_tail<<<blocks_for(n), kThreads, 0, b.st>>>(e2 + n, n, -1.0f, val);  // add_self_loops(fill=-1)  astgcn.py:104-106
  STMP_LAUNCH_OK("k_fill_tail");
  int* dst = b.talloc<int>(nnz);
  int* src = b.talloc<int>(nnz);
  if (!dst || !src) return b.rc;
  k_edges_then_loops<<<blocks_for(nnz), kThreads, 0, b.st>>>(e2, n, 2, r2, c2, 1, dst, src);  // transposed index :167
  STMP_LAUNCH_OK("k_edges_then_loops");
  if ((r = b.both_csr(p, 0, n, nnz, dst, src, val))) return r;
  p->n_ops = 1;
  return 0;
}

int build_gcn(Builder& b, stmp_plan* p, int n, int e, const int* row, const int* col, const float* w) {
  int r, nnz;
  int *dst, *src;
  float* wcoo;
  if (p->flags & STMP_GCN_NO_SELF_LOOPS) {
    nnz = e;
    dst = b.talloc<int>(nnz);
    src = b.talloc<int>(nnz);
    wcoo = b.talloc<float>(nnz);
    if (!dst || !src || !wcoo) return b.rc;
    if (e) {
      STMP_CUDA_OK(cudaMemcpyAsync(dst, col, (size_t)e * sizeof(int), cudaMemcpyDeviceToDevice, b.st));
      STMP_CUDA_OK(cudaMemcpyAsync(src, row, (size_t)e * sizeof(int), cudaMemcpyDeviceToDevice, b.st));
      k_copy_w<<<blocks_for(e), kThreads, 0, b.st>>>(e, w, wcoo);
      STMP_LAUNCH_OK("k_copy_w");
    }
  } else {
    int *r2, *c2, e2;
    float* w2;
    if ((r = b.compact_nonloops(e, row, col, w, &r2, &c2, &w2, &e2))) return r;
    nnz = e2 + n;
    dst = b.talloc<int>(nnz);
    src = b.talloc<int>(nnz);
    wcoo = b.talloc<float>(nnz);
    int* owner = b.talloc<int>(n);
    if (!dst || !src || !wcoo || !owner) return b.rc;
    k_edges_then_loops<<<blocks_for(nnz), kThreads, 0, b.st>>>(e2, n, 1, r2, c2, 0, dst, src);
    STMP_LAUNCH_OK("k_edges_then_loops");
    if (e2) STMP_CUDA_OK(cudaMemcpyAsync(wcoo, w2, (size_t)e2 * sizeof(float), cudaMemcpyDeviceToDevice, b.st));
    k_fill_int<<<blocks_for(n), kThreads, 0, b.st>>>(n, -1, owner);
    STMP_LAUNCH_OK("k_fill_int");
    if (e) {
      k_gcn_loop_owner<<<blocks_for(e), kThreads, 0, b.st>>>(e, row, col, owner);
      STMP_LAUNCH_OK("k_gcn_loop_owner");
    }
    k_gcn_loop_w<<<blocks_for(n), kThreads, 0, b.st>>>(n, e2, owner, w, (p->flags & STMP_GCN_IMPROVED) ? 2.0f : 1.0f, wcoo);
    STMP_LAUNCH_OK("k_gcn_loop_w");
  }
  float* deg;
  if ((r = b.segment_sum(nnz, n, dst, wcoo, &deg))) return r;  // deg = scatter_add(w, col)
  float* val = b.talloc<float>(nnz);
  if (!val) return b.rc;
  if (nnz) {
    k_gcn_vals<<<blocks_for(nnz), kThreads, 0, b.st>>>(nnz, dst, src, wcoo, deg, val);
    STMP_LAUNCH_OK("k_gcn_vals");
  }
  if ((r = b.both_csr(p, 0, n, nnz, dst, src, val))) return r;
  p->n_ops = 1;
  return 0;
}

// PyG RGCNConv (aggr="mean"), relations rel0 .. rel0 + n_rel - 1: operator k holds the edges of type rel0 + k in edge order (the masked
// edge list the reference propagates), dst = col, src = row, val = 1 / (the destination's count of such edges).  Other types match none.
int build_rgcn(Builder& b, stmp_plan* p, int n, int e, const int* row, const int* col, const long long* type, long long rel0, int n_rel) {
  int* flag = b.talloc<int>(e);
  if (!flag) return b.rc;
  for (int k = 0; k < n_rel; ++k) {
    if (e) {
      k_flag_relation<<<blocks_for(e), kThreads, 0, b.st>>>(e, type, rel0 + k, flag);
      STMP_LAUNCH_OK("k_flag_relation");
    }
    int *src, *dst, ek, r;
    float *w2, *cnt;
    if ((r = b.compact(e, flag, row, col, nullptr, &src, &dst, &w2, &ek))) return r;
    if ((r = b.segment_sum(ek, n, dst, nullptr, &cnt))) return r;    // in-degree per relation: scatter(ones, dst)
    float* val = b.talloc<float>(ek);
    if (!val) return b.rc;
    if (ek) {
      k_mean_vals<<<blocks_for(ek), kThreads, 0, b.st>>>(ek, dst, cnt, val);
      STMP_LAUNCH_OK("k_mean_vals");
    }
    if ((r = b.both_csr(p, k, n, ek, dst, src, val))) return r;
  }
  p->n_ops = n_rel;
  return 0;
}

// PyG GatedGraphConv's propagate (aggr add / mean / max): one operator over every edge in edge order, dst = col, src = row, val = w_e
// (add, max) or w_e / cnt(dst) (mean, cnt = the destination's number of in-edges); a missing weight is 1.  No self loops are added.
int build_gated(Builder& b, stmp_plan* p, int n, int e, const int* row, const int* col, const float* w, int aggr) {
  float* cnt = nullptr;
  int r;
  if (aggr == STMP_AGGR_MEAN && (r = b.segment_sum(e, n, col, nullptr, &cnt))) return r;    // scatter(ones, dst)
  float* val = b.talloc<float>(e);
  if (!val) return b.rc;
  if (e) {
    k_gated_vals<<<blocks_for(e), kThreads, 0, b.st>>>(e, col, w, cnt, val);
    STMP_LAUNCH_OK("k_gated_vals");
  }
  if ((r = b.both_csr(p, 0, n, e, col, row, val))) return r;
  p->n_ops = 1;
  p->aggr = aggr;
  return 0;
}

// cost model of the static longest-first deal
constexpr int kLptHandicap = 24;
constexpr int kLptA = 2;
constexpr int kLptB = 3;

// ---- shared-memory graph image for the fused wgmma kernel (graph_image.cuh) ---------------------------------------
// One CTA.  Tasks (row, op) are rank-sorted per segment (destination row tile, operator) by descending group count, cut into
// warp-tasks of four, and dealt longest-first to the least loaded of the 16 warps (loads carry over between the segments,
// so the whole round is balanced, not each segment); then the padded edge groups are written.
__global__ void __launch_bounds__(512) k_build_graph_image(const int* rp0, const int* rp1, const int2* cv0, const int2* cv1, int N,
                                                           int n_ops, int nnz_total, unsigned char* image) {
  __shared__ int s_ng[2 * kImgMaxN], s_g0[2 * kImgMaxN + 1], s_sorted[2 * kImgMaxN];
  __shared__ unsigned char s_owner[2 * kImgMaxN / 4 + 8];
  __shared__ int s_segcount[kImgSegs], s_valid;
  const int NT = n_ops * N, tid = threadIdx.x;
  const GraphImageLayout L = graph_image_layout(NT, nnz_total);
  int* hdr = reinterpret_cast<int*>(image);
  uint16_t* wstart = reinterpret_cast<uint16_t*>(image + L.off_wstart);
  uint16_t* wcount = reinterpret_cast<uint16_t*>(image + L.off_wcount);
  uint32_t* wt = reinterpret_cast<uint32_t*>(image + L.off_wt);
  uint32_t* idx4 = reinterpret_cast<uint32_t*>(image + L.off_idx);
  float4* val4 = reinterpret_cast<float4*>(image + L.off_val);
  for (int task = tid; task < NT; task += blockDim.x) {
    const int op = task >= N ? 1 : 0, i = task - op * N;
    const int* rp = op ? rp1 : rp0;
    s_ng[task] = (rp[i + 1] - rp[i] + 3) >> 2;
  }
  if (tid == 0) s_valid = 1;
  __syncthreads();
  if (tid == 0) {
    int run = 0, ok = (N <= kImgMaxN) ? 1 : 0;
    for (int sg = 0; sg < kImgSegs; ++sg) s_segcount[sg] = 0;
    for (int task = 0; task < NT; ++task) {
      s_g0[task] = run;
      run += s_ng[task];
      if (s_ng[task] > 127) ok = 0;
      const int op = task >= N ? 1 : 0;
      ++s_segcount[((task - op * N) >= 128 ? 2 : 0) + op];
    }
    s_g0[NT] = run;
    if (run > 65535 || run + 1 > L.cap_groups) ok = 0;
    s_valid = ok;
  }
  __syncthreads();
  // rank sort: (segment asc, group count desc, task id asc)
  for (int task = tid; task < NT; task += blockDim.x) {
    const int seg = ((task >= N ? task - N : task) >= 128 ? 2 : 0) + (task >= N ? 1 : 0), ng = s_ng[task];
    int rank = 0;
    for (int o = 0; o < NT; ++o) {
      const int so = ((o >= N ? o - N : o) >= 128 ? 2 : 0) + (o >= N ? 1 : 0), no = s_ng[o];
      rank += (so < seg) || (so == seg && (no > ng || (no == ng && o < task)));
    }
    s_sorted[rank] = task;
  }
  __syncthreads();
  if (tid == 0) {
    int load[kImgWarps], cntw[kImgWarps], pos[kImgWarps];
    for (int w = 0; w < kImgWarps; ++w) load[w] = 0;
    load[0] = kLptHandicap;                              // warp 0 also issues the round's MMAs (~42 x 8 issue slots)
    int nwt = 0;
    int base = 0;
    for (int seg = 0; seg < kImgSegs; base += s_segcount[seg], ++seg) {
      const int cnt = s_segcount[seg], nw = (cnt + 3) >> 2;
      for (int w = 0; w < kImgWarps; ++w) cntw[w] = 0;
      for (int k = 0; k < nw; ++k) {                      // longest warp-task first onto the least loaded warp
        int best = 0;
        for (int w = 1; w < kImgWarps; ++w)
          if (load[w] < load[best]) best = w;
        s_owner[k] = (unsigned char)best;
        load[best] += kLptA * s_ng[s_sorted[base + 4 * k]] + kLptB;   // ~ issue slots: per group 6 loads + 8 FMA2, per task a split store
        ++cntw[best];
      }
      int run = nwt;
      for (int w = 0; w < kImgWarps; ++w) {
        wstart[w * kImgSegs + seg] = (uint16_t)run;
        wcount[w * kImgSegs + seg] = (uint16_t)cntw[w];
        pos[w] = run;
        run += cntw[w];
      }
      for (int k = 0; k < nw; ++k) {
        const int slot = pos[s_owner[k]]++;
        for (int qd = 0; qd < 4; ++qd) {
          uint32_t d = kImgNoTask;
          if (4 * k + qd < cnt) {
            const int task = s_sorted[base + 4 * k + qd];
            const int op = task >= N ? 1 : 0, i = task - op * N;
            d = (uint32_t)i | ((uint32_t)op << 8) | ((uint32_t)s_ng[task] << 9) | ((uint32_t)s_g0[task] << 16);
          }
          wt[slot * 4 + qd] = d;
        }
      }
      nwt = run;
    }
    hdr[0] = nwt;
    hdr[1] = s_g0[NT];
    hdr[2] = (s_valid && nwt <= L.cap_wt) ? 1 : 0;
    hdr[3] = 0;
  }
  if (!s_valid) return;
  // padded edge groups: pad entries read the all-zero row with value 0
  for (int task = tid; task < NT; task += blockDim.x) {
    const int op = task >= N ? 1 : 0, i = task - op * N;
    const int* rp = op ? rp1 : rp0;
    const int2* cv = op ? cv1 : cv0;
    const int beg = rp[i], len = rp[i + 1] - beg;
    for (int g = 0; g < s_ng[task]; ++g) {
      uint32_t u = 0;
      float v[4];
      for (int e = 0; e < 4; ++e) {
        const int k = 4 * g + e;
        const int2 c = k < len ? cv[beg + k] : make_int2(kImgZeroRow, 0);
        u |= ((uint32_t)c.x & 0xffu) << (8 * e);
        v[e] = __int_as_float(c.y);
      }
      idx4[s_g0[task] + g] = u;
      val4[s_g0[task] + g] = make_float4(v[0], v[1], v[2], v[3]);
    }
  }
  if (tid == 0) {   // the spare group the gather loop prefetches past the last task
    idx4[s_g0[NT]] = kImgZeroRow * 0x01010101u;
    val4[s_g0[NT]] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

int build_graph_images(Builder& b, stmp_plan* p) {
  if (p->n > kImgMaxN) return 0;
  const int N = p->n;
  int hdr[3][4] = {{0}};
  for (int n_ops = 1; n_ops <= p->n_ops; ++n_ops) {
    int nnz = 0;
    for (int op = 0; op < n_ops; ++op) nnz += p->fwd[op].nnz;
    const GraphImageLayout L = graph_image_layout(n_ops * N, nnz);
    if (L.bytes > tc_graph_image_budget()) continue;          // cannot fit beside the wgmma kernel's operand panels
    STMP_CUDA_OK(cudaMalloc(&p->gimg[n_ops], (size_t)L.bytes));
    STMP_CUDA_OK(cudaMemsetAsync(p->gimg[n_ops], 0, (size_t)L.bytes, b.st));
    const Csr& c1 = p->fwd[n_ops > 1 ? 1 : 0];
    k_build_graph_image<<<1, 512, 0, b.st>>>(p->fwd[0].rowptr, c1.rowptr, p->fwd[0].cv, c1.cv, N, n_ops, nnz,
                                             reinterpret_cast<unsigned char*>(p->gimg[n_ops]));
    STMP_LAUNCH_OK("k_build_graph_image");
    STMP_CUDA_OK(cudaMemcpyAsync(hdr[n_ops], p->gimg[n_ops], 16, cudaMemcpyDeviceToHost, b.st));
    p->gimg_bytes[n_ops] = L.bytes;
  }
  STMP_CUDA_OK(cudaStreamSynchronize(b.st));
  for (int n_ops = 1; n_ops <= p->n_ops; ++n_ops)
    if (p->gimg[n_ops] && !hdr[n_ops][2]) {                    // rows too long / too many groups for the compact format
      cudaFree(p->gimg[n_ops]);
      p->gimg[n_ops] = nullptr;
      p->gimg_bytes[n_ops] = 0;
    }
  // the one-CTA kernel's row image, built on the host from the forward CSR
  std::vector<int> rp[2], cl[2];
  std::vector<float> vl[2];
  for (int op = 0; op < p->n_ops; ++op) {
    const Csr& c = p->fwd[op];
    std::vector<int2> cv(c.nnz);
    rp[op].resize(N + 1);
    STMP_CUDA_OK(cudaMemcpyAsync(rp[op].data(), c.rowptr, (size_t)(N + 1) * sizeof(int), cudaMemcpyDeviceToHost, b.st));
    if (c.nnz) STMP_CUDA_OK(cudaMemcpyAsync(cv.data(), c.cv, (size_t)c.nnz * sizeof(int2), cudaMemcpyDeviceToHost, b.st));
    STMP_CUDA_OK(cudaStreamSynchronize(b.st));
    cl[op].resize(c.nnz);
    vl[op].resize(c.nnz);
    for (int k = 0; k < c.nnz; ++k) { cl[op][k] = cv[k].x; std::memcpy(&vl[op][k], &cv[k].y, 4); }
  }
  const int* rps[2] = {rp[0].data(), rp[1].data()};
  const int* cls[2] = {cl[0].data(), cl[1].data()};
  const float* vls[2] = {vl[0].data(), vl[1].data()};
  for (int n_ops = 1; n_ops <= p->n_ops; ++n_ops) {
    // which graphs get an image is decided by the by-total image, as it always was; the kernel gets the by-operator one when that fits
    int64_t bytes = build_row_image(N, n_ops, rps, cls, vls, ROW_ORDER_BY_TOTAL, nullptr, 0);
    if (bytes <= 0 || bytes > tc_row_image_budget()) continue;
    RowOrder order = ROW_ORDER_BY_OPERATOR;
    const int64_t by_op = build_row_image(N, n_ops, rps, cls, vls, order, nullptr, 0);
    if (by_op <= tc_row_image_budget()) bytes = by_op; else order = ROW_ORDER_BY_TOTAL;
    std::vector<unsigned char> img((size_t)bytes);
    build_row_image(N, n_ops, rps, cls, vls, order, img.data(), bytes);
    STMP_CUDA_OK(cudaMalloc(&p->rimg[n_ops], (size_t)bytes));
    STMP_CUDA_OK(cudaMemcpy(p->rimg[n_ops], img.data(), (size_t)bytes, cudaMemcpyHostToDevice));
    p->rimg_groups[n_ops] = reinterpret_cast<const int*>(img.data())[0];
  }
  return 0;
}

void free_csr(Csr& c) {
  if (c.rowptr) cudaFree(c.rowptr);
  if (c.cv) cudaFree(c.cv);
  if (c.eid) cudaFree(c.eid);
  c = Csr();
}

}  // namespace

// ---- row image for the one-CTA wgmma kernel (row_image.cuh) -------------------------------------------------------------
int64_t build_row_image(int N, int n_ops, const int* const rowptr[2], const int* const col[2], const float* const val[2], RowOrder order_by,
                        void* dst, int64_t capacity) {
  if (N < 1 || N > kRiMaxN || n_ops < 1 || n_ops > 2) return 0;
  std::vector<int> ng(2 * N, 0);   // groups of 4 entries per (operator, row)
  for (int op = 0; op < n_ops; ++op)
    for (int i = 0; i < N; ++i) {
      const int beg = rowptr[op][i], end = rowptr[op][i + 1];
      if (end < beg) return 0;
      for (int k = beg; k < end; ++k)
        if (col[op][k] < 0 || col[op][k] >= N) return 0;
      ng[op * N + i] = (end - beg + 3) / 4;
    }
  // nodes by descending group count -- of both operators together, or of operator 0 and then operator 1 (ties: node id) -- then the
  // empty positions
  std::vector<int> order(N);
  std::iota(order.begin(), order.end(), 0);
  if (order_by == ROW_ORDER_BY_OPERATOR)
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return ng[a] != ng[b] ? ng[a] > ng[b] : ng[N + a] > ng[N + b]; });
  else
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return ng[a] + ng[N + a] > ng[b] + ng[N + b]; });
  order.resize(kRiPos, -1);
  // bins of 8 consecutive nodes (one row per quad of a (warp, slot)); a bin's gather runs as long as its longest row per operator
  constexpr int kBins = kRiPos / 8;
  int bin_g[kBins][2] = {}, bin_cost[kBins];
  for (int k = 0; k < kBins; ++k) {
    for (int m = 0; m < 8; ++m) {
      const int node = order[8 * k + m];
      if (node >= 0)
        for (int op = 0; op < 2; ++op) bin_g[k][op] = std::max(bin_g[k][op], ng[op * N + node]);
    }
    bin_cost[k] = bin_g[k][0] + bin_g[k][1];
  }
  // longest processing time first: every bin onto the least loaded warp that has a free slot
  std::vector<int> bins(kBins);
  std::iota(bins.begin(), bins.end(), 0);
  std::stable_sort(bins.begin(), bins.end(), [&](int a, int b) { return bin_cost[a] > bin_cost[b]; });
  int load[kRiWarps] = {}, used[kRiWarps] = {}, bin_at[kRiWarps][2];
  for (int k : bins) {
    int best = -1;
    for (int w = 0; w < kRiWarps; ++w)
      if (used[w] < 2 && (best < 0 || load[w] < load[best])) best = w;
    bin_at[best][used[best]++] = k;
    load[best] += bin_cost[k];
  }
  std::vector<int16_t> perm(kRiPos, -1);
  std::vector<uint8_t> ipos(kRiPos, 0);
  int n_groups = 0;
  for (int w = 0; w < kRiWarps; ++w)
    for (int s = 0; s < 2; ++s) {
      for (int quad = 0; quad < 8; ++quad) {
        const int node = order[8 * bin_at[w][s] + quad], pos = 16 * w + 8 * s + quad;
        perm[pos] = (int16_t)node;
        if (node >= 0) ipos[node] = (uint8_t)pos;
      }
      for (int op = 0; op < n_ops; ++op) n_groups += bin_g[bin_at[w][s]][op];
    }
  int zero_pos = 0;
  while (perm[zero_pos] >= 0) ++zero_pos;   // N <= 255: there is an empty position
  const RowImageLayout L = row_image_layout(n_groups);
  if (!dst || capacity < L.bytes) return L.bytes;

  unsigned char* img = static_cast<unsigned char*>(dst);
  std::memset(img, 0, (size_t)L.bytes);
  int* hdr = reinterpret_cast<int*>(img);
  hdr[0] = n_groups; hdr[1] = zero_pos; hdr[2] = N; hdr[3] = n_ops;
  std::memcpy(img + kRiOffPerm, perm.data(), 2 * kRiPos);
  std::memcpy(img + kRiOffIpos, ipos.data(), kRiPos);
  uint16_t* gstart = reinterpret_cast<uint16_t*>(img + kRiOffGstart);
  uint16_t* gcount = reinterpret_cast<uint16_t*>(img + kRiOffGcount);
  uint32_t* idx = reinterpret_cast<uint32_t*>(img + kRiOffIdx);
  float* vals = reinterpret_cast<float*>(img + L.off_val);
  int run = 0;
  for (int w = 0; w < kRiWarps; ++w)
    for (int op = 0; op < n_ops; ++op)
      for (int s = 0; s < 2; ++s) {
        const int G = bin_g[bin_at[w][s]][op];
        gstart[ri_list(w, op, s)] = (uint16_t)run;
        gcount[ri_list(w, op, s)] = (uint16_t)G;
        for (int g = 0; g < G; ++g)
          for (int quad = 0; quad < 8; ++quad) {
            const int node = perm[16 * w + 8 * s + quad];
            const int beg = node >= 0 ? rowptr[op][node] : 0, len = node >= 0 ? rowptr[op][node + 1] - beg : 0;
            uint32_t u = 0;
            for (int e = 0; e < 4; ++e) {
              const int k = 4 * g + e;
              u |= (uint32_t)(k < len ? ipos[col[op][beg + k]] : zero_pos) << (8 * e);
              vals[((run + g) * 8 + quad) * 4 + e] = k < len ? val[op][beg + k] : 0.f;
            }
            idx[(run + g) * 8 + quad] = u;
          }
        run += G;
      }
  for (int quad = 0; quad < 8; ++quad) idx[run * 8 + quad] = (uint32_t)zero_pos * 0x01010101u;   // the spare group row
  return L.bytes;
}

}  // namespace stmp

using namespace stmp;

static int plan_create_impl(int flavor, int64_t num_nodes, int64_t num_edges, const int64_t* edge_index,
                            const float* edge_weight, int normalization, float lambda_max, const float* lambda_node,
                            uint32_t flags, void* stream, stmp_plan** out, const int64_t* edge_type = nullptr, int64_t rel0 = 0,
                            int n_rel = 0, int aggr = 0);

extern "C" int stmp_plan_create(int flavor, int64_t num_nodes, int64_t num_edges, const int64_t* edge_index,
                                const float* edge_weight, int normalization, float lambda_max, uint32_t flags,
                                void* stream, stmp_plan** out) {
  STMP_REQUIRE(flavor != STMP_FLAVOR_RGCN, STMP_EINVAL, "stmp_plan_create: the RGCN flavor is built by stmp_plan_create_rgcn");
  STMP_REQUIRE(flavor != STMP_FLAVOR_GATED, STMP_EINVAL, "stmp_plan_create: the GATED flavor is built by stmp_plan_create_gated");
  return plan_create_impl(flavor, num_nodes, num_edges, edge_index, edge_weight, normalization, lambda_max, nullptr, flags, stream, out);
}

extern "C" int stmp_plan_create_rgcn(int64_t num_nodes, int64_t num_edges, const int64_t* edge_index, const int64_t* edge_type,
                                     int64_t rel0, int n_rel, void* stream, stmp_plan** out) {
  STMP_REQUIRE(n_rel >= 1 && n_rel <= 2, STMP_EINVAL, "stmp_plan_create_rgcn: a plan holds 1 or 2 relations (got %d)", n_rel);
  STMP_REQUIRE(edge_type != nullptr || num_edges == 0, STMP_EINVAL, "stmp_plan_create_rgcn: edge_type is NULL");
  return plan_create_impl(STMP_FLAVOR_RGCN, num_nodes, num_edges, edge_index, nullptr, STMP_NORM_NONE, 0.f, nullptr, 0u, stream, out,
                          edge_type, rel0, n_rel);
}

extern "C" int stmp_plan_create_gated(int64_t num_nodes, int64_t num_edges, const int64_t* edge_index, const float* edge_weight,
                                      int aggr, void* stream, stmp_plan** out) {
  STMP_REQUIRE(aggr >= STMP_AGGR_ADD && aggr <= STMP_AGGR_MAX, STMP_EINVAL, "stmp_plan_create_gated: unknown aggregation %d", aggr);
  return plan_create_impl(STMP_FLAVOR_GATED, num_nodes, num_edges, edge_index, edge_weight, STMP_NORM_NONE, 0.f, nullptr, 0u, stream, out,
                          nullptr, 0, 0, aggr);
}

extern "C" int stmp_plan_create_pergraph(int flavor, int64_t num_nodes, int64_t num_edges, const int64_t* edge_index,
                                         const float* edge_weight, int normalization, const float* lambda_node, uint32_t flags,
                                         void* stream, stmp_plan** out) {
  STMP_REQUIRE(lambda_node != nullptr, STMP_EINVAL, "stmp_plan_create_pergraph: lambda_node is NULL");
  STMP_REQUIRE(flavor == STMP_FLAVOR_CHEB || flavor == STMP_FLAVOR_CHEB_ATT, STMP_EINVAL,
               "per-graph lambda_max applies to the Chebyshev flavors only (got flavor %d)", flavor);
  return plan_create_impl(flavor, num_nodes, num_edges, edge_index, edge_weight, normalization, 0.f, lambda_node, flags, stream, out);
}

static int plan_create_impl(int flavor, int64_t num_nodes, int64_t num_edges, const int64_t* edge_index,
                            const float* edge_weight, int normalization, float lambda_max, const float* lambda_node,
                            uint32_t flags, void* stream, stmp_plan** out, const int64_t* edge_type, int64_t rel0, int n_rel,
                            int aggr) {
  STMP_REQUIRE(out != nullptr, STMP_EINVAL, "stmp_plan_create: out is NULL");
  *out = nullptr;
  STMP_REQUIRE(flavor >= STMP_FLAVOR_DCONV && flavor <= STMP_FLAVOR_GATED, STMP_EINVAL, "unknown flavor %d", flavor);
  STMP_REQUIRE(normalization >= STMP_NORM_NONE && normalization <= STMP_NORM_RW, STMP_EINVAL,
               "Invalid normalization %d", normalization);
  STMP_REQUIRE(num_nodes > 0 && num_nodes < (1ll << 30), STMP_EINVAL, "num_nodes=%lld out of range", (long long)num_nodes);
  STMP_REQUIRE(num_edges >= 0 && num_edges < (1ll << 30), STMP_EINVAL, "num_edges=%lld out of range", (long long)num_edges);
  STMP_REQUIRE(edge_index != nullptr || num_edges == 0, STMP_EINVAL, "edge_index is NULL");
  if (!(lambda_max > 0.f)) lambda_max = 0.f;  // NaN / <=0 -> default

  stmp_plan* p = new stmp_plan();
  p->flavor = flavor;
  p->n = (int)num_nodes;
  p->e = num_edges;
  p->normalization = normalization;
  p->flags = flags;
  cudaGetDevice(&p->device);

  Builder b;
  b.st = (cudaStream_t)stream;
  int n = (int)num_nodes, e = (int)num_edges;
  int rc = 0;
  do {
    b.d_info = b.talloc<Info>(1);
    int* row = b.talloc<int>(e);
    int* col = b.talloc<int>(e);
    if (!b.d_info || !row || !col) { rc = b.rc; break; }
    if (cudaMemsetAsync(b.d_info, 0, sizeof(Info), b.st) != cudaSuccess) { rc = set_error(STMP_ECUDA, "memset failed"); break; }
    if (e) {
      k_split_index<<<blocks_for(e), kThreads, 0, b.st>>>(e, (const long long*)edge_index, n, row, col, b.d_info);
      if (cudaGetLastError() != cudaSuccess) { rc = set_error(STMP_ECUDA, "k_split_index launch failed"); break; }
      count_launch();
    }
    switch (flavor) {
      case STMP_FLAVOR_DCONV: rc = build_dconv(b, p, n, e, row, col, edge_weight); break;
      case STMP_FLAVOR_CHEB: rc = build_cheb(b, p, n, e, row, col, edge_weight, lambda_max, lambda_node); break;
      case STMP_FLAVOR_GCN: rc = build_gcn(b, p, n, e, row, col, edge_weight); break;
      case STMP_FLAVOR_CHEB_ATT: rc = build_cheb_att(b, p, n, e, row, col, edge_weight, lambda_max, lambda_node); break;
      case STMP_FLAVOR_RGCN: rc = build_rgcn(b, p, n, e, row, col, (const long long*)edge_type, rel0, n_rel); break;
      case STMP_FLAVOR_GATED: rc = build_gated(b, p, n, e, row, col, edge_weight, aggr); break;
    }
    if (rc) break;
    Info h;
    cudaError_t ce = cudaMemcpyAsync(&h, b.d_info, sizeof(Info), cudaMemcpyDeviceToHost, b.st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(b.st);
    if (ce != cudaSuccess) { rc = set_error(STMP_ECUDA, "plan build failed: %s", cudaGetErrorString(ce)); break; }
    if (h.err & kErrRange) { rc = set_error(STMP_EGRAPH, "edge_index has entries outside [0, %d)", n); break; }
    if (h.err & kErrDuplicate) {
      rc = set_error(STMP_EGRAPH, "duplicate edges: DConv's dense adjacency merges them and the reference fails "
                                  "on the norm/reverse-index length mismatch (dcrnn.py:59-77,87)");
      break;
    }
    p->nonfinite_vals = (h.err & kNonFinite) != 0;
    for (int op = 0; op < p->n_ops; ++op) {
      p->fwd[op].max_row_nnz = h.max_row[op * 2];
      p->bwd[op].max_row_nnz = h.max_row[op * 2 + 1];
    }
    rc = build_graph_images(b, p);
    if (rc) break;
  } while (0);
  if (rc) {
    stmp_plan_destroy(p);
    return rc;
  }
  *out = p;
  return STMP_OK;
}

extern "C" void stmp_plan_destroy(stmp_plan* p) {
  if (!p) return;
  for (int i = 0; i < 2; ++i) {
    free_csr(p->fwd[i]);
    free_csr(p->bwd[i]);
  }
  for (int i = 0; i < 3; ++i) {
    if (p->gimg[i]) cudaFree(p->gimg[i]);
    if (p->rimg[i]) cudaFree(p->rimg[i]);
  }
  delete p;
}

extern "C" int stmp_plan_num_ops(const stmp_plan* p) { return p ? p->n_ops : 0; }
extern "C" int64_t stmp_plan_num_nodes(const stmp_plan* p) { return p ? p->n : 0; }
extern "C" int64_t stmp_plan_nnz(const stmp_plan* p, int op) {
  if (!p || op < 0 || op >= p->n_ops) return -1;
  return p->fwd[op].nnz;
}

extern "C" int stmp_plan_export(const stmp_plan* p, int op, int transposed, int32_t* rowptr, int32_t* col, float* val,
                                int32_t* eid, void* stream) {
  STMP_REQUIRE(p != nullptr, STMP_EINVAL, "plan is NULL");
  STMP_REQUIRE(op >= 0 && op < p->n_ops, STMP_EINVAL, "op %d out of range (plan has %d)", op, p->n_ops);
  const Csr& c = transposed ? p->bwd[op] : p->fwd[op];
  cudaStream_t st = (cudaStream_t)stream;
  if (rowptr) STMP_CUDA_OK(cudaMemcpyAsync(rowptr, c.rowptr, (size_t)(c.n + 1) * sizeof(int), cudaMemcpyDeviceToDevice, st));
  if (c.nnz && (col || val || eid)) {
    k_export<<<blocks_for(c.nnz), kThreads, 0, st>>>(c.nnz, c.cv, c.eid, col, val, eid);
    STMP_LAUNCH_OK("k_export");
  }
  return STMP_OK;
}

extern "C" int64_t stmp_plan_graph_image(const stmp_plan* p, int n_ops, void* dst, int64_t capacity) {
  if (!p || n_ops < 1 || n_ops > 2 || !p->gimg[n_ops]) return 0;
  const int64_t bytes = p->gimg_bytes[n_ops];
  if (dst && capacity >= bytes && cudaMemcpy(dst, p->gimg[n_ops], (size_t)bytes, cudaMemcpyDefault) != cudaSuccess) {
    (void)cudaGetLastError();
    return -set_error(STMP_ECUDA, "stmp_plan_graph_image: copy of %lld bytes failed", (long long)bytes);
  }
  return bytes;
}

extern "C" int64_t stmp_row_image_build(int64_t num_nodes, int n_ops, const int32_t* rowptr0, const int32_t* col0, const float* val0,
                                        const int32_t* rowptr1, const int32_t* col1, const float* val1, void* dst, int64_t capacity) {
  if (num_nodes < 1 || num_nodes > kRiMaxN || n_ops < 1 || n_ops > 2 || !rowptr0 || (n_ops > 1 && !rowptr1)) return 0;
  const int* rp[2] = {rowptr0, rowptr1};
  const int* cl[2] = {col0, col1};
  const float* vl[2] = {val0, val1};
  return build_row_image((int)num_nodes, n_ops, rp, cl, vl, ROW_ORDER_BY_TOTAL, dst, capacity);
}

extern "C" int64_t stmp_row_image_build_by_operator(int64_t num_nodes, int n_ops, const int32_t* rowptr0, const int32_t* col0,
                                                    const float* val0, const int32_t* rowptr1, const int32_t* col1, const float* val1,
                                                    void* dst, int64_t capacity) {
  if (num_nodes < 1 || num_nodes > kRiMaxN || n_ops < 1 || n_ops > 2 || !rowptr0 || (n_ops > 1 && !rowptr1)) return 0;
  const int* rp[2] = {rowptr0, rowptr1};
  const int* cl[2] = {col0, col1};
  const float* vl[2] = {val0, val1};
  return build_row_image((int)num_nodes, n_ops, rp, cl, vl, ROW_ORDER_BY_OPERATOR, dst, capacity);
}

/* Test hook: select, at run time, the implementation or launch shape a test cross-checks against the default (common.cuh). */
extern "C" int stmp_set_option(const char* name, int value) {
  STMP_REQUIRE(name != nullptr, STMP_EINVAL, "stmp_set_option: NULL name");
  if (strcmp(name, "dcrnn_tc") == 0) { g_dcrnn_tc = value ? 1 : 0; return STMP_OK; }
  if (strcmp(name, "dcrnn_fwd_split") == 0) { g_fwd_split = value ? 1 : 0; return STMP_OK; }
  if (strcmp(name, "dcrnn_bwd_split") == 0) { g_bwd_split = value ? 1 : 0; return STMP_OK; }
  if (strcmp(name, "dcrnn_wgrad_tc") == 0) { g_wgrad_tc = value ? 1 : 0; return STMP_OK; }
  if (strcmp(name, "dcrnn_narrow_pack") == 0) {
    STMP_REQUIRE(value >= 0 && value <= 8, STMP_EINVAL, "stmp_set_option: dcrnn_narrow_pack must be 0 (automatic) .. 8");
    g_narrow_pack = value;
    return STMP_OK;
  }
  return set_error(STMP_EINVAL, "stmp_set_option: unknown option '%s'", name);
}

extern "C" const char* stmp_last_error(void) { return err_buf(); }
extern "C" const char* stmp_version(void) { return "stmp 0.1.0 sm_90a"; }
extern "C" int64_t stmp_launch_count(void) { return g_launches.load(); }
extern "C" int stmp_path_counters(const char** names, int64_t* counts, int max_entries) {
  const int n = stmp::g_n_paths.load();
  for (int i = 0; i < n && i < max_entries; ++i) {
    if (names) names[i] = stmp::g_path_names[i];
    if (counts) counts[i] = stmp::g_path_counts[i].load();
  }
  return n;
}
