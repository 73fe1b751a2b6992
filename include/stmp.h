/*
 * stmp.h -- C ABI of libstmp.so, the sm_90a (H100) spatiotemporal message-passing engine.
 *
 * The reference (benedekrozemberczki/pytorch_geometric_temporal @ adefe44) is pure Python and has no
 * FFI layer: its hot path is `torch.nn.Module.forward` -> torch_geometric `MessagePassing.propagate`
 * (index_select + scatter_add_) + ATen matmul/pointwise.  This header is therefore the boundary a
 * maintainer would bind with ctypes from those modules (INTEGRATION.md shows the stub).  Each entry
 * point cites the reference code it replaces, relative to /root/reference/torch_geometric_temporal/.
 *
 * Conventions
 *  - plain C types only; all data pointers are DEVICE pointers unless a name ends in `_host`;
 *  - tensors are fp32, row-major, indices int64 on input (torch LongTensor) and int32 inside a plan;
 *  - every call enqueues on the caller's `stream` (a cudaStream_t passed as void*), never
 *    synchronises the device and never allocates, except stmp_plan_create/destroy/export (setup path);
 *  - return value: 0 = STMP_OK, otherwise an stmp_status code; the message is available from
 *    stmp_last_error() (thread-local);
 *  - entry points are re-entrant (autograd / DDP call backward from worker threads); a plan is
 *    immutable after creation.
 */
#ifndef STMP_H_
#define STMP_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct stmp_plan stmp_plan;

enum stmp_status {
  STMP_OK = 0,
  STMP_EINVAL = 1,       /* bad argument (null pointer, negative size, unknown enum)  -> ValueError   */
  STMP_ESHAPE = 2,       /* shape/stride/alignment the kernels cannot take            -> RuntimeError */
  STMP_EGRAPH = 3,       /* edge_index out of range / duplicate edges where the reference would fail */
  STMP_ECUDA = 4,        /* CUDA runtime error (message carries cudaGetErrorString)                   */
  STMP_EUNSUPPORTED = 5, /* configuration does not fit the fused kernel; caller must use the tiled path */
  STMP_ENOMEM = 6
};

/* Which normalised operator(s) a plan holds. */
enum stmp_flavor {
  /* DConv / BatchedDConv (nn/recurrent/dcrnn.py:59-77, :277-290): two operators,
   *   op 0 "out": dst=col[e], src=row[e], val = 1/deg_out[row[e]]
   *   op 1 "in" : p-th entry of the (col,row)-sorted reverse list: dst=row[q_p], src=col[q_p],
   *               val = 1/deg_in[row[p]]   (positional pairing, quirk preserved)
   * degrees are weighted sums; messages never multiply by edge_weight. */
  STMP_FLAVOR_DCONV = 0,
  /* PyG ChebConv.__norm__ (used by gconv_gru.py:57-107, gconv_lstm.py:62-138): scaled Laplacian
   *   2L/lambda_max - I, self-loop entries appended after the non-loop edges. */
  STMP_FLAVOR_CHEB = 1,
  /* PyG gcn_norm (used by temporalgcn.py:38-68,162-173): D^-1/2 (A+I) D^-1/2 with remaining self loops. */
  STMP_FLAVOR_GCN = 2,
  /* ChebConvAttention.__norm__ (nn/attention/astgcn.py:82-110), propagated on the TRANSPOSED index
   * (:167): dst=row', src=col', E'+2N entries. */
  STMP_FLAVOR_CHEB_ATT = 3,
  /* PyG RGCNConv's mean aggregation (LRGCN, nn/recurrent/lrgcn.py), built by stmp_plan_create_rgcn only: operator k holds the
   * edges of type rel0 + k in edge order, dst=col, src=row, val = 1/(the destination's count of such edges).  No self loops are
   * added; duplicates and self loops count as ordinary edges; a node without such an in-edge has an empty row. */
  STMP_FLAVOR_RGCN = 4,
  /* PyG GatedGraphConv's propagate (DyGrEncoder, nn/recurrent/dygrae.py), built by stmp_plan_create_gated only: one operator over every
   * edge in edge order, dst=col, src=row, val = w_e for STMP_AGGR_ADD and STMP_AGGR_MAX, w_e / (the destination's count of in-edges) for
   * STMP_AGGR_MEAN (the count is of edges, not of weights); w_e = 1 without weights.  No self loops are added; duplicates and self loops
   * are ordinary edges; a node without an in-edge has an empty row. */
  STMP_FLAVOR_GATED = 5
};

/* GatedGraphConv's aggregation (stmp_plan_create_gated, stmp_ggc_rows_*). */
enum stmp_aggr { STMP_AGGR_ADD = 0, STMP_AGGR_MEAN = 1, STMP_AGGR_MAX = 2 };

enum stmp_norm { STMP_NORM_NONE = 0, STMP_NORM_SYM = 1, STMP_NORM_RW = 2 };

enum stmp_plan_flags {
  STMP_GCN_IMPROVED = 1u << 0,      /* GCNConv(improved=True): self-loop fill 2 instead of 1 */
  STMP_GCN_NO_SELF_LOOPS = 1u << 1, /* GCNConv(add_self_loops=False) */
  STMP_DCONV_ALLOW_DUPLICATES = 1u << 2 /* BatchedDConv semantics (scatter degrees, no dense adjacency):
                                           duplicate edges are legal; DConv proper raises on them */
};

/* ---- plan ------------------------------------------------------------------------------------ */

/* Build the cached operator(s) for a static graph on the device (stable radix sort to CSR by
 * destination + CSR by source for the transposed/backward product, degree/Laplacian/GCN norms).
 * Replaces the per-call renormalisation of dcrnn.py:59-77, PyG get_laplacian / gcn_norm and
 * astgcn.py:82-110.  edge_index: int64 [2,E] row-major; edge_weight: [E] or NULL (=> ones).
 * lambda_max: >0 to use it, <=0 / NaN => PyG default (CHEB: 2*max(w_hat); CHEB_ATT: 2.0).
 * Setup path: allocates, and synchronises `stream` once to read validation flags. */
int stmp_plan_create(int flavor, int64_t num_nodes, int64_t num_edges, const int64_t* edge_index,
                     const float* edge_weight, int normalization, float lambda_max, uint32_t flags,
                     void* stream, stmp_plan** out);
/* Multi-graph mini-batches (StaticGraphTemporalSignalBatch; PyG ChebConv `lambda_max[batch[edge_index[0]]]`, and
 * ChebConvAttention.__norm__, astgcn.py:98-99; exercised by the reference's test/attention_test.py:205-218): the scaling
 * 2 w / lambda uses the lambda_max of the entry's ROW node.  lambda_node: device float [num_nodes] = lambda_max[batch].
 * Flavors CHEB and CHEB_ATT only. */
int stmp_plan_create_pergraph(int flavor, int64_t num_nodes, int64_t num_edges, const int64_t* edge_index,
                              const float* edge_weight, int normalization, const float* lambda_node, uint32_t flags,
                              void* stream, stmp_plan** out);
/* Relation-masked mean operators (STMP_FLAVOR_RGCN) of relations rel0 .. rel0 + n_rel - 1 (n_rel 1 or 2): edge_type is a device
 * int64 [E]; a type outside that range matches no operator.  edge_index is validated as stmp_plan_create validates it (STMP_EGRAPH).
 * More relations take ceil(R / 2) plans.  Setup path: synchronises `stream` once per relation and once to read validation flags. */
int stmp_plan_create_rgcn(int64_t num_nodes, int64_t num_edges, const int64_t* edge_index, const int64_t* edge_type, int64_t rel0,
                          int n_rel, void* stream, stmp_plan** out);
/* GatedGraphConv's aggregation operator (STMP_FLAVOR_GATED) for `aggr` (stmp_aggr): edge_weight is a device float [E] or NULL (ones).
 * edge_index is validated as stmp_plan_create validates it (STMP_EGRAPH).  Setup path: synchronises `stream` to read validation flags. */
int stmp_plan_create_gated(int64_t num_nodes, int64_t num_edges, const int64_t* edge_index, const float* edge_weight, int aggr,
                           void* stream, stmp_plan** out);
void stmp_plan_destroy(stmp_plan* plan);

/* Introspection (tests, bit-exact index parity): number of operators, nodes, entries of operator `op`. */
int stmp_plan_num_ops(const stmp_plan* plan);
int64_t stmp_plan_num_nodes(const stmp_plan* plan);
int64_t stmp_plan_nnz(const stmp_plan* plan, int op);
/* Copy operator `op` (transposed=0: CSR by destination; 1: CSR by source) into caller device buffers:
 * rowptr[N+1], col[nnz], val[nnz], eid[nnz] (eid = position of the entry in the reference-order
 * COO list, i.e. the order the reference's scatter_add_ visits it).  Any output may be NULL. */
int stmp_plan_export(const stmp_plan* plan, int op, int transposed, int32_t* rowptr, int32_t* col,
                     float* val, int32_t* eid, void* stream);
/* The compact shared-memory image of the first n_ops (1 or 2) forward operators that the wgmma graph-GRU kernel
 * gathers from (layout: csrc/graph_image.cuh).  Returns its size in bytes, or 0 when the plan has none for n_ops
 * (N > 207, a row of more than 508 entries, or too dense for the kernel's shared memory).  When dst is non-NULL and
 * capacity >= that size, the image is copied to dst (host or device memory).  Setup path: synchronous.  A failed copy
 * returns -STMP_ECUDA. */
int64_t stmp_plan_graph_image(const stmp_plan* plan, int n_ops, void* dst, int64_t capacity);
/* The row image the one-CTA wgmma graph-GRU kernel gathers from (layout: csrc/row_image.cuh), built on the host from host CSR
 * arrays of n_ops (1 or 2) operators (rowptr [N+1], col / val [nnz]; the second set is ignored for n_ops = 1).  Returns its size
 * in bytes, or 0 for a graph the format cannot hold (N outside 1..255, a column outside [0, N)).  When dst is non-NULL and
 * capacity >= that size, the image is written to dst (host memory).  Needs no GPU. */
int64_t stmp_row_image_build(int64_t num_nodes, int n_ops, const int32_t* rowptr0, const int32_t* col0, const float* val0,
                             const int32_t* rowptr1, const int32_t* col1, const float* val1, void* dst, int64_t capacity);
/* The same image with the nodes sorted by operator 0's group count, then operator 1's: the image a plan gives the kernel whenever it
 * fits (stmp_row_image_build's nodes are sorted by the sum of both, which decides whether a plan has an image at all).  Arguments
 * and return value as stmp_row_image_build. */
int64_t stmp_row_image_build_by_operator(int64_t num_nodes, int n_ops, const int32_t* rowptr0, const int32_t* col0, const float* val0,
                                         const int32_t* rowptr1, const int32_t* col1, const float* val1, void* dst, int64_t capacity);

/* ---- K1/K3: gather -> weighted scatter-add (SpMM) with fused Chebyshev axpby -------------------
 * y[b,i,:] = alpha * sum_k val_k * x[b, col_k, :] + beta * z[b,i,:]        (z may be NULL)
 * Replaces MessagePassing.propagate (x_j = index_select; norm*x_j; scatter_add_) at
 * dcrnn.py:86-87,95-99,300-313, astgcn.py:169-175 and inside ChebConv/GCNConv, plus the
 * `2*prop - T0` recurrence (dcrnn.py:96,100; astgcn.py:176).  Per destination the products are summed
 * in the reference's edge order with separate multiply and add (no FMA), so results are bit-identical
 * to the CPU scatter_add_ path.  x,y,z: [batch, N, f] with row strides ld* and batch strides bs*
 * (elements).  att (nullable): [batch, N, N] spatial attention; the entry value becomes
 * val * att[b, dst, src] (astgcn.py:156-157, first hop only).  transposed=1 applies A^T (backward). */
int stmp_spmm(const stmp_plan* plan, int op, int transposed, int64_t batch, int64_t f,
              const float* x, int64_t ldx, int64_t bsx, float* y, int64_t ldy, int64_t bsy,
              float alpha, const float* z, int64_t ldz, int64_t bsz, float beta,
              const float* att, void* stream);

/* The forward product with the attention handed in TRANSPOSED and row-padded: entry (dst, src) uses attT[b, src, dst], rows att_ld
 * floats apart (the layout stmp_spatial_attention_fwd writes: softmax over dim 1 of S is a row softmax of S^T). */
int stmp_spmm_att_t(const stmp_plan* plan, int op, int64_t batch, int64_t f, const float* x, int64_t ldx, int64_t bsx, float* y,
                   int64_t ldy, int64_t bsy, float alpha, const float* z, int64_t ldz, int64_t bsz, float beta, const float* attT,
                   int64_t att_ld, void* stream);

/* d(att)[b,dst,src] += val * <gy[b,dst,:], x[b,src,:]> for every entry of `op` (backward of the
 * attention-weighted first hop, astgcn.py:156-170).  datt must be zero-initialised by the caller. */
int stmp_spmm_att_grad(const stmp_plan* plan, int op, int64_t batch, int64_t f, const float* gy,
                       int64_t ldg, int64_t bsg, const float* x, int64_t ldx, int64_t bsx, float* datt,
                       void* stream);

/* ---- K1-K5 fused: the DCRNN recurrence ---------------------------------------------------------
 * For each window b: H_0 = h0[b] (or 0); for t in [0,T): H_t = DCRNN_cell(X[b,t], H_{t-1});
 * out[b,t] = H_t.  One persistent CTA per window keeps graph, weights, [X|H] and both diffusion
 * products in shared memory across all T steps.  Replaces BatchedDCRNN.forward (dcrnn.py:429-475)
 * and, with B=T=1, DCRNN.forward (:194-219).  plan: STMP_FLAVOR_DCONV.
 *   x: window b, step t starts at x + (win_start ? win_start[b] : b*x_bstride) ... see x_tstride:
 *      addr = x + base_b + t*x_tstride, base_b = win_start ? win_start[b]*x_tstride : b*x_bstride
 *      (win_start: int64 [B] device, index-batching over a resident series, signal/index_dataset.py:49-57)
 *   w_z,w_r,w_h: DConv.weight [2,K,cin+cout,cout]; b_*: [cout] or NULL (dcrnn.py:26-37)
 *   h0: [B,N,cout] or NULL; out: [B,T,N,cout]
 *   stash (nullable): [B,T,3,N,cout] receives (Z,R,Htilde) per step for the backward pass.
 * Kernels: cout = 32, K = 2 the wgmma kernel; cout in {16, 32} the FFMA kernel; cout in 1..4 (cin in 1..4, K in 1..4: the
 * reference's BatchedDCRNN(F, F, K=3) training model) the narrow-state kernel, whose CTAs serve up to 8 windows side by side
 * ("dcrnn_narrow_pack", stmp_set_option; fewer where N * P would exceed 1024 in the forward or 512 in the backward) and which ignores
 * wimage / workspace.
 * Returns STMP_EUNSUPPORTED when (N, nnz, cin, cout, K) do not fit the fused kernel. */
int stmp_dcrnn_seq_fwd(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K,
                       const float* x, const int64_t* win_start, int64_t x_bstride, int64_t x_tstride,
                       const float* w_z, const float* w_r, const float* w_h, const float* b_z,
                       const float* b_r, const float* b_h, const float* h0, float* out, float* stash,
                       const void* wimage, void* workspace, void* stream);
/* 1 if stmp_dcrnn_seq_fwd can take this configuration on the current device, else 0. */
int stmp_dcrnn_seq_supported(const stmp_plan* plan, int64_t cin, int64_t cout, int64_t K);

/* Generic fused graph-GRU recurrence on the tensor cores (wgmma, fp16 hi/lo operand split = fp32-class accuracy):
 *   pre_g = [H' | Op0 H' | Op1 H' | X | Op0 X | Op1 X] @ wcat_g^T + bcat_g      g in {z, r, h};  H' = H (z, r) or H*R (h)
 *   Z = sigmoid(pre_z); R = sigmoid(pre_r); Ht = tanh(pre_h); H_t = Z*H + (1-Z)*Ht
 * with the first `n_ops` (0..2) operators of `plan` (any flavor).  This one kernel serves DCRNN K=2 (DConv plan, 2 ops),
 * GConvGRU K<=2 (gconv_gru.py:119-139; CHEB plan, 1 op) and TGCN / A3TGCN(2) (temporalgcn.py:82-102; GCN plan, 1 op:
 * the GCNConv weight and the gate Linear are folded into wcat on the host side).  Cout = 32, cin <= 4, N <= 207.
 *   wcat: [96][112] fp32, row = gate*32 + out channel, columns = H(32) | Op0 H(32) | Op1 H(32) | X(4) | Op0 X(4) | Op1 X(4) | 0(4)
 *   bcat: [96];  h0: [B,N,32] (h0_bstride = N*32), one shared [N,32] (h0_bstride = 0) or NULL (zeros)
 * x / win_start / strides / out / stash as stmp_dcrnn_seq_fwd.  STMP_EUNSUPPORTED outside the envelope. */
int stmp_gru_seq_fwd(const stmp_plan* plan, int n_ops, int64_t B, int64_t T, int64_t cin, const float* x,
                     const int64_t* win_start, int64_t x_bstride, int64_t x_tstride, const float* wcat,
                     const float* bcat, const float* h0, int64_t h0_bstride, float* out, float* stash,
                     const void* wimage, void* workspace, void* stream);
/* Optional weight image for the wgmma kernel: the B operand (fp16 hi/lo halves, SWIZZLE_128B, + biases) exactly as the kernel
 * holds it in shared memory, so every CTA fetches it with one TMA bulk copy instead of converting the fp32 weights itself.
 * Build it once per weight update into a device buffer of stmp_gru_weight_image_bytes() bytes and pass it as `wimage`
 * (NULL => the kernel converts in place).  The plan carries the analogous graph image. */
int64_t stmp_gru_weight_image_bytes(void);
/* Optional workspace of the wgmma kernel (both entries): stmp_seq_workspace_bytes(plan, T, cin) bytes of device memory, reusable across
 * calls on one stream.  The window prologue parks P_o X_t / P_i X_t of all steps there (per-CTA rows, rewritten every window => L2-resident,
 * full-sector stores).  NULL => they are parked in the window's own not-yet-written output rows instead (same results; partial-sector
 * writes cost extra DRAM traffic). */
int64_t stmp_seq_workspace_bytes(const stmp_plan* plan, int64_t T, int64_t cin);
int stmp_dcrnn_pack_weights(int64_t cin, int64_t cout, int64_t K, const float* w_z, const float* w_r, const float* w_h,
                            const float* b_z, const float* b_r, const float* b_h, void* image, void* stream);
int stmp_gru_pack_weights(const float* wcat, const float* bcat, void* image, void* stream);
int stmp_gru_seq_supported(const stmp_plan* plan, int n_ops, int64_t cin, int64_t cout);

/* ---- fused temporal-attention + GCN-GRU: A3TGCN / A3TGCN2 (attentiontemporalgcn.py:51-79,130-157) and, with periods = 1 and
 * probs = NULL, a TGCN / TGCN2 cell (temporalgcn.py:104-130,212-233) -- graphs of any size, out_channels = 32.
 *   out[b,n,:] = sum_t probs[t] * GRU(A^ X[b,:,:,t], H[b])        A^ = operator 0 of `plan` (GCN flavor: gcn_norm)
 * with GCNConv's Linear and the gate Linear folded on the host:  pre_g = (A^X_t) A[:, g] + H' Bm[:, g] + c[g],  g in z|r|h
 *   x: [B][N][fin][periods] contiguous;  h: [B][N][32] with batch stride h_bstride (0: one state shared by all rows) or NULL (zeros)
 *   A: [fin][96], Bm: [32][96], c: [96] (columns z | r | h);  probs: [periods] = softmax(attention) or NULL;  out: [B][N][32]
 * One gather per node serves every period (A^(XW) = (A^X)W); X[b] is staged in shared memory by one TMA bulk copy per CTA.
 * STMP_EUNSUPPORTED unless fin <= 4 and fin * periods <= 128. */
int stmp_tgcn_attn_fwd(const stmp_plan* plan, int64_t B, int64_t fin, int64_t periods, const float* x, const float* h,
                       int64_t h_bstride, const float* A, const float* Bm, const float* c, const float* probs, float* out,
                       void* stream);

/* ---- K5: gate epilogues for the tiled path -------------------------------------------------------
 * GRU (dcrnn.py:172-192, gconv_gru.py:119-139, temporalgcn.py:82-102), n = number of elements:
 *   stmp_gru_zr:   z = sigmoid(pz); r = sigmoid(pr); hr = h * r
 *   stmp_gru_out:  ht = tanh(ph); hnew = z*h + (1-z)*ht
 * LSTM with peepholes (gconv_lstm.py:168-202), rows x cout, w_c*, b_* are [cout]:
 *   stmp_lstm_ifc: i = sig(pi + wci*c + bi); f = sig(pf + wcf*c + bf); t = tanh(pc + bc); cnew = f*c + i*t
 *   stmp_lstm_oh:  o = sig(po + wco*cnew + bo); hnew = o * tanh(cnew)
 */
int stmp_gru_zr(int64_t n, const float* pz, const float* pr, const float* h, float* z, float* r, float* hr,
                void* stream);
int stmp_gru_out(int64_t n, const float* ph, const float* z, const float* h, float* ht, float* hnew,
                 void* stream);
int stmp_lstm_ifc(int64_t rows, int64_t cout, const float* pi, const float* pf, const float* pc,
                  const float* c, const float* wci, const float* wcf, const float* bi, const float* bf,
                  const float* bc, float* i, float* f, float* t, float* cnew, void* stream);
int stmp_lstm_oh(int64_t rows, int64_t cout, const float* po, const float* cnew, const float* wco,
                 const float* bo, float* o, float* hnew, void* stream);

/* Backward of the peephole-LSTM gate chain (what autograd records for gconv_lstm.py:168-202): pre [rows][4*cout] = i|f|c|o pre-activations
 * of the contraction incl. the ChebConv biases, c_old / c_new [rows][cout], gh = dL/dH', gc = dL/dC' (either may be NULL = zeros)
 * -> dpre [rows][4*cout], dc_old [rows][cout].  The gates are recomputed from `pre` (nothing but S, C_{t-1}, C_t is kept by the forward). */
int stmp_lstm_gate_bwd(int64_t rows, int64_t cout, const float* pre, const float* c_old, const float* c_new, const float* gh,
                       const float* gc, const float* wci, const float* wcf, const float* wco, const float* bi, const float* bf,
                       const float* bc, const float* bo, float* dpre, float* dc_old, void* stream);

/* ---- backward of the fused DCRNN sequence (what autograd replays for dcrnn.py:429-475 / :172-219), small graphs ----
 * Served when stmp_dcrnn_bwd_supported(plan, cin, cout, K) != 0 (DCONV plan, K = 2, cout = 32, cin <= 4, graph + tiles
 * fit one SM's shared memory: N <= ~235); otherwise callers use the per-step path (stmp_gru_bwd_* + stmp_spmm).
 *   stmp_dcrnn_bwd_basis: for every (t, b) rebuild S1[t*B+b] = [U | P_o U | P_i U], U = [X_t | H_{t-1}] and S2 with
 *                         U = [X_t | H_{t-1} * R_t] (row pitch ld >= 3(cin+cout)) from x, the forward output `out`
 *                         (B,T,N,cout), h0 (nullable) and the gate stash (B,T,3,N,cout).  One launch.
 *   stmp_dcrnn_bwd_seq:   the reverse-time recurrence, one CTA per window: consumes gout (B,T,N,cout), whsT (cout, 3C),
 *                         wzrT (2cout, 3C) [transposed stacked weights]; writes d pre-activations dph_all (T,B,N,cout),
 *                         dpzr_all (T,B,N,2cout) for the weight-gradient GEMMs, dx (B,T,N,cin; nullable), dh0 (B,N,cout).
 */
int stmp_dcrnn_bwd_supported(const stmp_plan* plan, int64_t cin, int64_t cout, int64_t K);
int stmp_dcrnn_bwd_basis(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, const float* x,
                         int64_t x_bstride, int64_t x_tstride, const float* out, const float* h0, const float* stash,
                         float* S1, float* S2, int64_t ld, void* stream);
int stmp_dcrnn_bwd_seq(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, const float* gout,
                       const float* out, const float* h0, const float* stash, const float* whsT, const float* wzrT,
                       float* dph_all, float* dpzr_all, float* dx, float* dh0, void* stream);

/* ---- backward of the generic graph-GRU recurrence (the twin of stmp_gru_seq_fwd: what autograd records for gconv_gru.py:119-139, and
 * for the DCRNN cell on any n_ops <= 2 operators of `plan`), graphs that fit one SM -- the kernels of stmp_dcrnn_bwd_* for n_ops operators:
 * the basis of U = [X | H] is [U | Op0 U | .. | Op_{n_ops-1} U] (width (n_ops+1)(cin+32)), its adjoint dU = dS_0 + sum_op Op^T dS_{1+op}
 * (the plan's transposed CSRs).  Envelope: cout = 32, cin 1..4, n_ops <= plan's operators, graph and per-window buffers fit one SM's shared
 * memory (stmp_gru_bwd_supported).  B windows x T steps; x, out (B,T,N,32) and stash (B,T,3,N,32) are those of the forward
 * (stmp_gru_seq_fwd with a stash); h0 (B,N,32) dense (h0_bstride = N*32) or NULL (zeros).  A shared h0 (h0_bstride = 0) returns
 * STMP_EUNSUPPORTED.  Deterministic: no atomics, fixed reduction order.
 *   stmp_gru_pack_bwd_weights: the transposed stacked weights of the backward GEMMs from the forward's wcat [96][112], basis order
 *                              [X | H] per block: whsT (32, (n_ops+1)(cin+32)) from the h rows, wzrT (64, ..) from the z | r rows.  One launch.
 *   stmp_gru_bwd_basis:        S1[t*B+b] = basis of [X_t | H_{t-1}], S2 = basis of [X_t | H_{t-1} * R_t], row pitch
 *                              ld = (n_ops+1)(cin+32) rounded up to 8.  One launch.
 *   stmp_gru_bwd_seq:          the reverse-time recurrence, one CTA (or a 2-CTA cluster) per window: gout = dL/dout (B,T,N,32) ->
 *                              dph_all (T,B,N,32), dpzr_all (T,B,N,64), dx (B,T,N,cin; nullable), dh0 (B,N,32).  One launch.
 *   stmp_gru_bwd_wgrad:        dwcat [96][112] in wcat's layout (columns of absent operators / channels and the padding zero) and dbcat [96]
 *                              (nullable) over all T*B*N = rows rows: TF32 wgmma per-CTA partials + a fixed-order sum (two launches);
 *                              workspace of stmp_gru_bwd_wgrad_workspace_bytes(n_ops, cin) bytes.
 * STMP_EINVAL for NULL tensors, STMP_ESHAPE for bad sizes, pitches or alignment, STMP_EUNSUPPORTED outside the envelope. */
int stmp_gru_bwd_supported(const stmp_plan* plan, int n_ops, int64_t cin, int64_t cout);
int stmp_gru_pack_bwd_weights(int n_ops, int64_t cin, const float* wcat, float* whsT, float* wzrT, void* stream);
int stmp_gru_bwd_basis(const stmp_plan* plan, int n_ops, int64_t B, int64_t T, int64_t cin, const float* x, int64_t x_bstride,
                       int64_t x_tstride, const float* out, const float* h0, int64_t h0_bstride, const float* stash, float* S1,
                       float* S2, int64_t ld, void* stream);
int stmp_gru_bwd_seq(const stmp_plan* plan, int n_ops, int64_t B, int64_t T, int64_t cin, const float* gout, const float* out,
                     const float* h0, int64_t h0_bstride, const float* stash, const float* whsT, const float* wzrT, float* dph_all,
                     float* dpzr_all, float* dx, float* dh0, void* stream);
int64_t stmp_gru_bwd_wgrad_workspace_bytes(int n_ops, int64_t cin);
int stmp_gru_bwd_wgrad(int n_ops, int64_t cin, int64_t rows, int64_t ld, const float* S1, const float* S2, const float* dpzr,
                       const float* dph, void* workspace, float* dwcat, float* dbcat, void* stream);

/* ---- the generic graph-GRU cell on graphs of ANY size, split over CTAs by destination rows (gru_rows.cu): GConvGRU K <= 2 on a
 * Chebyshev plan (gconv_gru.py:119-139), one graph and one step per call.  Envelope: cout = 32, cin 1..16, n_ops 0..1 and at most the
 * plan's operators (stmp_gru_rows_supported), any number of nodes and any degree.  Exact fp32 FFMA; deterministic (no atomics, every
 * reduction in a fixed order); no host sync and no allocation: scratch and workspace come from the caller, so a call can be captured.
 *   packed weights w [96][nb], nb = (n_ops+1)(cin+32): row gate*32 + o (gates z | r | h), column m of the basis [X | H | Op X | Op H]
 *   (X channels first in each block); b [96] = the sum of a gate's two biases (zeros without biases).
 *   stmp_gru_rows_pack_weights: w, b from the parameters' layout: wx [3][n_ops+1][32][cin], wh [3][n_ops+1][32][32] (gate, Chebyshev
 *                               order, out, in), bx / bh [3][32] (both or neither).  One launch.
 *   stmp_gru_rows_fwd:          x (N,cin), h (N,32) or NULL (H = None) -> out (N,32).  H given: two launches (Op[X | H] -> Z, R, H*R;
 *                               Op(H*R) -> H'), scratch of N*96 floats; H = None: one launch, no scratch.  Training adds (all nullable)
 *                               stash (3,N,32) = Z | R | Ht (R unwritten for H = None) and the weight-gradient bases S1 = [U | Op U],
 *                               S2 = [X | H*R | Op X | Op(H*R)] (N, ld), ld = nb rounded up to 8, 16-byte aligned; for H = None S1 = S2
 *                               (pass S2 = NULL).  The output does not depend on which of them are given.
 *   stmp_gru_rows_bwd:          gout = dL/dH' (N,32), h, stash and w of the forward -> dph (N,32), dpzr (N,64) (the weight-gradient
 *                               operands; dpr = 0 for H = None), dx (N,cin; nullable), dh (N,32; nullable, NULL for H = None).  H given:
 *                               rowwise dS2 = dph W_h^T; Op^T of dS2's H*R block -> dpr, dS1 = [dpz | dpr] W_zr^T; Op^T of the operator
 *                               blocks -> dH, dX (skipped when neither is asked for or n_ops = 0).  H = None: one rowwise launch, plus
 *                               one Op^T gather for dx.  scratch of stmp_gru_rows_scratch_bytes(plan) bytes (N*192 floats).
 *   stmp_gru_rows_wgrad:        dw [96][nb] (the packed layout) and db [96] (nullable) = S1^T [dpz | dpr], S2^T dph and the column sums
 *                               over `rows` rows: fp32 FFMA per-CTA partials + a fixed-order sum (two launches); workspace of
 *                               stmp_gru_rows_wgrad_workspace_bytes(n_ops, cin) bytes, 16-byte aligned operands.
 * STMP_EINVAL for NULL tensors, STMP_ESHAPE for bad sizes, pitches or alignment, STMP_EUNSUPPORTED for cin > 16, n_ops > 1, cout != 32
 * or n_ops above the plan's operators.  stmp_gru_rows_supported also answers 1 for cout = 64 (the stmp_gru_wide_rows_* entries below). */
int stmp_gru_rows_supported(const stmp_plan* plan, int n_ops, int64_t cin, int64_t cout);
int stmp_gru_rows_pack_weights(int n_ops, int64_t cin, const float* wx, const float* wh, const float* bx, const float* bh, float* w,
                               float* b, void* stream);
int stmp_gru_rows_fwd(const stmp_plan* plan, int n_ops, int64_t cin, const float* x, const float* h, const float* w, const float* b,
                      float* scratch, float* out, float* stash, float* S1, float* S2, int64_t ld, void* stream);
int64_t stmp_gru_rows_scratch_bytes(const stmp_plan* plan);
int stmp_gru_rows_bwd(const stmp_plan* plan, int n_ops, int64_t cin, const float* gout, const float* h, const float* stash,
                      const float* w, float* scratch, float* dph, float* dpzr, float* dx, float* dh, void* stream);
int64_t stmp_gru_rows_wgrad_workspace_bytes(int n_ops, int64_t cin);
int stmp_gru_rows_wgrad(int n_ops, int64_t cin, int64_t rows, int64_t ld, const float* S1, const float* S2, const float* dpzr,
                        const float* dph, void* workspace, float* dw, float* db, void* stream);

/* ---- the same cell at 64 hidden channels (gru_rows.cu, the width-2 instance of its kernels): GConvGRU(cin, 64, K <= 2).  Envelope: cout =
 * 64, cin 1..16, n_ops 0..1 and at most the plan's operators (stmp_gru_rows_supported(plan, n_ops, cin, 64)), any number of nodes and any
 * degree.  Same argument lists, launch chain and guarantees as the stmp_gru_rows_* entries, with 32 -> 64 throughout:
 *   packed weights w [192][nb], nb = (n_ops+1)(cin+64): row gate*64 + o, column m of the basis [X | H | Op X | Op H]; b [192].
 *   stmp_gru_wide_rows_pack_weights: wx [3][n_ops+1][64][cin], wh [3][n_ops+1][64][64], bx / bh [3][64] (both or neither).
 *   stmp_gru_wide_rows_fwd:          x (N,cin), h (N,64) or NULL -> out (N,64); scratch of N*192 floats when h is given; stash (3,N,64);
 *                                    S1 / S2 (N, ld), ld = nb rounded up to 8, 16-byte aligned.
 *   stmp_gru_wide_rows_bwd:          gout (N,64) -> dph (N,64), dpzr (N,128), dx (N,cin), dh (N,64); scratch of
 *                                    stmp_gru_wide_rows_scratch_bytes(plan) bytes (N*320 floats).
 *   stmp_gru_wide_rows_wgrad:        dw [192][nb], db [192] (nullable): fp32 FFMA per-CTA partials of each gate's product over strided
 *                                    32-row tiles + a fixed-order sum (two launches); workspace of
 *                                    stmp_gru_wide_rows_wgrad_workspace_bytes(n_ops, cin) bytes, 16-byte aligned operands.
 * STMP_EINVAL for NULL tensors, STMP_ESHAPE for bad sizes, pitches or alignment, STMP_EUNSUPPORTED for cin > 16, n_ops > 1 or n_ops above
 * the plan's operators. */
int stmp_gru_wide_rows_pack_weights(int n_ops, int64_t cin, const float* wx, const float* wh, const float* bx, const float* bh, float* w,
                                    float* b, void* stream);
int stmp_gru_wide_rows_fwd(const stmp_plan* plan, int n_ops, int64_t cin, const float* x, const float* h, const float* w, const float* b,
                           float* scratch, float* out, float* stash, float* S1, float* S2, int64_t ld, void* stream);
int64_t stmp_gru_wide_rows_scratch_bytes(const stmp_plan* plan);
int stmp_gru_wide_rows_bwd(const stmp_plan* plan, int n_ops, int64_t cin, const float* gout, const float* h, const float* stash,
                           const float* w, float* scratch, float* dph, float* dpzr, float* dx, float* dh, void* stream);
int64_t stmp_gru_wide_rows_wgrad_workspace_bytes(int n_ops, int64_t cin);
int stmp_gru_wide_rows_wgrad(int n_ops, int64_t cin, int64_t rows, int64_t ld, const float* S1, const float* S2, const float* dpzr,
                             const float* dph, void* workspace, float* dw, float* db, void* stream);

/* ---- BatchedDCRNN at 32 hidden channels on graphs of ANY size, split over CTAs by destination rows (dcrnn_rows.cu): the reference's
 * BatchedDCRNN (dcrnn.py:328-475) with H_0 = 0, all B windows of a step in each launch.  Envelope: a DConv plan, cout = 32, K = 2, cin 1..4
 * (stmp_dcrnn_rows_supported), any number of nodes and any degree.  Exact fp32 FFMA; deterministic (no atomics, every sum in a fixed
 * order); no host sync and no allocation: scratch comes from the caller, so a training step can be captured.
 *   weights: wzrT (64, 3C) and whsT (32, 3C), C = cin + 32, from stmp_dcrnn_pack_bwd_weights (rows are outputs, columns the basis
 *   [X | H | P_o X | P_o H | P_i X | P_i H]); bz / br / bh (32) each nullable.
 *   stmp_dcrnn_rows_fwd:  x as stmp_dcrnn_seq_fwd (windows (B,T,N,cin) at strides x_bstride / x_tstride, or the resident series read at
 *                         win_start) -> out (B,T,N,32).  2T - 1 launches: two per step, one for step 0 (a plan holding a non-finite
 *                         operator value runs step 0 as two, so the non-finite values spread as in the reference).  Training adds
 *                         stash (T,B,N,96) = Z | R | Ht and the weight-gradient bases S1 / S2 (T*B, N, ld), ld = 3C rounded up to 8,
 *                         16-byte aligned (the layout stmp_dcrnn_bwd_wgrad reads); give all three or none.  The output does not depend
 *                         on whether they are given.
 *   stmp_dcrnn_rows_bwd:  gout = dL/dout (B,T,N,32), out and stash of the forward -> dph_all (T,B,N,32), dpzr_all (T,B,N,64) (the operands
 *                         of stmp_dcrnn_bwd_wgrad) and dx (B,T,N,cin; nullable).  Reverse time: a rowwise launch, then per step t >= 1 the
 *                         transposed gathers of dS2's and of dS1's operator blocks (the second also starts step t - 1), and one more
 *                         gather for step 0's dX: 2T - 1 launches, 2T with dx.
 *   Both take scratch of stmp_dcrnn_rows_scratch_bytes(plan, B) bytes.
 * STMP_EINVAL for a NULL plan or tensor, a non-DConv plan or negative B / T, STMP_ESHAPE for a bad pitch, alignment or B * N >= 2^31,
 * STMP_EUNSUPPORTED outside the envelope. */
int stmp_dcrnn_rows_supported(const stmp_plan* plan, int64_t cin, int64_t cout, int64_t K);
int64_t stmp_dcrnn_rows_scratch_bytes(const stmp_plan* plan, int64_t B);
int stmp_dcrnn_rows_fwd(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, const float* x, const int64_t* win_start,
                        int64_t x_bstride, int64_t x_tstride, const float* wzrT, const float* whsT, const float* bz, const float* br,
                        const float* bh, float* scratch, float* out, float* stash, float* S1, float* S2, int64_t ld, void* stream);
int stmp_dcrnn_rows_bwd(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, const float* gout, const float* out, const float* stash,
                        const float* wzrT, const float* whsT, float* scratch, float* dph_all, float* dpzr_all, float* dx, void* stream);

/* ---- BatchedDCRNN for narrow states on graphs of ANY size, split over CTAs by destination rows (dcrnn_narrow_rows.cu): the reference's
 * BatchedDCRNN (dcrnn.py:328-475) with H_0 = 0 at cout 1..4, cin 1..4, K 1..4 (stmp_dcrnn_narrow_rows_supported) -- the index-batching
 * training model BatchedDCRNN(F, F, K=3) on graphs the one-SM kernels (stmp_dcrnn_seq_*) cannot hold.  All B windows of a step in each
 * launch; the state lives node-major in the scratch.  Exact fp32; deterministic (no atomics, every sum in a fixed order); no host sync and
 * no allocation: scratch comes from the caller, so a training step can be captured.  C = cin + cout, nbc = (2K-1) C, cp = cout padded to
 * 1, 2 or 4 (cout 3 -> 4).
 *   weights: wzrT (2 cout, nbc) and whsT (cout, nbc) from stmp_dcrnn_pack_bwd_weights; bz / br / bh (cout) each nullable.
 *   stmp_dcrnn_narrow_rows_fwd: x = the X blocks [X | P_o X | P_i X | 2 P_o T_1o - X | ...] of every (t, b): block j of row n at
 *                         x + t * x_tstride + b * x_bstride + n * x_ld + j * x_blk (the caller builds them with stmp_spmm; for K = 1 they
 *                         are X itself) -> out (B,T,N,cout).  K >= 2: 2(K-1) launches per step, one for step 0 (a plan holding a
 *                         non-finite operator value runs step 0 as 2(K-1) on a zero state, so the non-finite values spread as in the
 *                         reference); K = 1: one launch.  Training gives stash (T,N,B,3cp) = Z | R | Ht and the weight-gradient bases
 *                         S1 / S2 (T*B, N, nbc) (all three or none); x is then NULL and the X blocks are read from S1's X columns (block j
 *                         at column j C), which the caller has filled; the kernels write every other column of S1 and S2.  The output
 *                         does not depend on whether they are given.
 *   stmp_dcrnn_narrow_rows_bwd: gout = dL/dout (B,T,N,cout), out and stash of the forward -> dph_all (T,B,N,cout), dpzr_all
 *                         (T,B,N,2cout) (the operands of the weight-gradient contraction) and dsx (T*B, N, dsx_ld; nullable): the X
 *                         columns of dS1 + dS2, block j at column j cin, to which the caller applies the transposed basis adjoint for dX.
 *                         K >= 2: 1 + 2(K-1)(T-1) launches; K = 1: one.
 *   Both take scratch of stmp_dcrnn_narrow_rows_scratch_bytes(plan, B, cout, K) bytes (0 for K = 1: scratch may be NULL), 16-byte aligned.
 * STMP_EINVAL for a NULL plan or tensor, a non-DConv plan or negative B / T, STMP_ESHAPE for a bad stride or alignment or (B + 31) N >= 2^31,
 * STMP_EUNSUPPORTED outside the envelope. */
int stmp_dcrnn_narrow_rows_supported(const stmp_plan* plan, int64_t cin, int64_t cout, int64_t K);
int64_t stmp_dcrnn_narrow_rows_scratch_bytes(const stmp_plan* plan, int64_t B, int64_t cout, int64_t K);
int stmp_dcrnn_narrow_rows_fwd(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K, const float* x,
                               int64_t x_bstride, int64_t x_tstride, int64_t x_ld, int64_t x_blk, const float* wzrT, const float* whsT,
                               const float* bz, const float* br, const float* bh, float* scratch, float* out, float* stash, float* S1,
                               float* S2, void* stream);
int stmp_dcrnn_narrow_rows_bwd(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K, const float* gout,
                               const float* out, const float* stash, const float* wzrT, const float* whsT, float* scratch, float* dph_all,
                               float* dpzr_all, float* dsx, int64_t dsx_ld, void* stream);

/* ---- BatchedDCRNN at 64 hidden channels on graphs of ANY size, split over CTAs by destination rows (dcrnn_wide_rows.cu): the reference's
 * BatchedDCRNN (dcrnn.py:328-475) with H_0 = 0 at cout = 64, K = 2 or 3, cin 1..4 (stmp_dcrnn_wide_rows_supported) -- the DCRNN paper's
 * 64 recurrent units with one or two diffusion steps, which no one-SM kernel holds.  All B windows of a step in each launch; rows are
 * window-major (b N + n).  Exact fp32 FFMA; deterministic (no atomics, every sum in a fixed order); no host sync and no allocation: scratch
 * comes from the caller, so a training step can be captured.  C = cin + 64, nbc = (2K-1) C.  Arguments as stmp_dcrnn_narrow_rows_*:
 *   weights: wzrT (128, nbc) and whsT (64, nbc) from stmp_dcrnn_pack_bwd_weights; bz / br / bh (64) each nullable.
 *   stmp_dcrnn_wide_rows_fwd: x = the X blocks of every (t, b) (block j of row n at x + t * x_tstride + b * x_bstride + n * x_ld +
 *                         j * x_blk) -> out (B,T,N,64), 16-byte aligned.  One launch builds the kernels' weight image, then 2(K-1) launches
 *                         per step and one for step 0 (a plan holding a non-finite operator value runs step 0 as 2(K-1) on a zero state).
 *                         Training gives stash (T,B,N,192) = Z | R | Ht and the weight-gradient bases S1 / S2 (T*B, N, nbc) (all three or
 *                         none); x is then NULL and the X blocks are read from S1's X columns (block j at column j C), which the caller
 *                         has filled.  The output does not depend on whether they are given.
 *   stmp_dcrnn_wide_rows_bwd: gout = dL/dout (B,T,N,64), out and stash of the forward -> dph_all (T,B,N,64), dpzr_all (T,B,N,128) and
 *                         dsx (T*B, N, dsx_ld; nullable): the X columns of dS1 + dS2, block j at column j cin.  2 + 2(K-1)(T-1) launches.
 *   Both take scratch of stmp_dcrnn_wide_rows_scratch_bytes(plan, B, cout, K) bytes, 16-byte aligned.
 * STMP_EINVAL for a NULL plan or tensor, a non-DConv plan or negative B / T, STMP_ESHAPE for a bad stride or alignment or B N >= 2^40,
 * STMP_EUNSUPPORTED outside the envelope. */
int stmp_dcrnn_wide_rows_supported(const stmp_plan* plan, int64_t cin, int64_t cout, int64_t K);
int64_t stmp_dcrnn_wide_rows_scratch_bytes(const stmp_plan* plan, int64_t B, int64_t cout, int64_t K);
int stmp_dcrnn_wide_rows_fwd(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K, const float* x,
                             int64_t x_bstride, int64_t x_tstride, int64_t x_ld, int64_t x_blk, const float* wzrT, const float* whsT,
                             const float* bz, const float* br, const float* bh, float* scratch, float* out, float* stash, float* S1,
                             float* S2, void* stream);
int stmp_dcrnn_wide_rows_bwd(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K, const float* gout,
                             const float* out, const float* stash, const float* wzrT, const float* whsT, float* scratch, float* dph_all,
                             float* dpzr_all, float* dsx, int64_t dsx_ld, void* stream);

/* ---- the peephole graph-LSTM cell on graphs of ANY size, split over CTAs by destination rows (lstm_rows.cu): GConvLSTM
 * (gconv_lstm.py:168-238) and GCLSTM (gc_lstm.py:139-205) at K <= 2 on a Chebyshev plan, one graph and one step per call.  `variant`
 * selects the basis: STMP_LSTM_GCONV [X | H | Op X | Op H], STMP_LSTM_GC [X | H | Op H] (X is not diffused); nb basis columns, X channels
 * first; with n_ops = 0 both are [X | H].  Peepholes are the nullable `peep` (3, 32) = w_c_i | w_c_f | w_c_o (NULL: none, as GCLSTM).
 * Envelope: cout = 32, cin 1..16, n_ops 0..1 and at most the plan's operators (stmp_lstm_rows_supported), any number of nodes and any
 * degree.  Exact fp32 FFMA; deterministic (no atomics, every reduction in a fixed order); no host sync and no allocation: scratch and
 * workspace come from the caller, so a call can be captured.
 *   packed weights w [128][nb]: row gate*32 + o (gates i | f | c | o), column m of the basis; b [128] = the sum of every bias of a gate.
 *   stmp_lstm_rows_pack_weights: w, b from the parameters' layout in one launch.  GConvLSTM: wx [4][n_ops+1][32][cin], wh
 *                                [4][n_ops+1][32][32] (gate, Chebyshev order, out, in), bx / bh [4][32] (both or neither), bg [4][32];
 *                                GCLSTM: wx [4][cin][32] (W_g, in x out), wh as above, bx NULL, bh [4][32] or NULL, bg [4][32].
 *   stmp_lstm_rows_fwd:          x (N,cin), h and c (N,32) or NULL (zeros) -> hout, cout (N,32).  One launch.  Training adds (nullable)
 *                                stash (4,N,32) = I | F | T | O and the weight-gradient basis S (N, ld), ld = nb rounded up to 8,
 *                                16-byte aligned.  The outputs do not depend on which of them are given.
 *   stmp_lstm_rows_bwd:          gh = dL/dH', gc = dL/dC' (N,32; either NULL), c, cn = C' and stash of the forward -> dpre (2,N,64) =
 *                                [dpi | dpf], [dpc | dpo] (16-byte aligned), dx (N,cin), dh (N,32), dc (N,32) (nullable; dh / dc only
 *                                with h / c given).  A rowwise launch (dpre, dC, dS = dpre W: own-row block -> dX, dH), then for n_ops = 1
 *                                an Op^T gather of dS's operator block into dH (and dX for GConvLSTM) when one of them is asked for.
 *                                scratch of stmp_lstm_rows_scratch_bytes(plan) bytes; with peep it also carries the per-CTA peephole sums
 *                                to stmp_lstm_rows_wgrad.
 *   stmp_lstm_rows_wgrad:        dw [128][nb] (the packed layout) = dpre^T S, db [128] = 1^T dpre and dpeep [96] = the sums of dpi*C,
 *                                dpf*C and dpo*C' (db, dpeep nullable; dpeep reads the backward's scratch, rows = the plan's nodes):
 *                                fp32 FFMA per-CTA partials + a fixed-order sum (two launches); workspace of
 *                                stmp_lstm_rows_wgrad_workspace_bytes(variant, n_ops, cin) bytes, 16-byte aligned.
 * STMP_EINVAL for NULL tensors or an unknown variant, STMP_ESHAPE for a bad pitch or alignment, STMP_EUNSUPPORTED for cin > 16,
 * n_ops > 1, cout != 32 or n_ops above the plan's operators.  stmp_lstm_rows_supported also answers 1 for cout = 64 (the
 * stmp_lstm_wide_rows_* entries below). */
enum stmp_lstm_basis { STMP_LSTM_GCONV = 0, STMP_LSTM_GC = 1 };
int stmp_lstm_rows_supported(const stmp_plan* plan, int variant, int n_ops, int64_t cin, int64_t cout);
int stmp_lstm_rows_pack_weights(int variant, int n_ops, int64_t cin, const float* wx, const float* wh, const float* bx, const float* bh,
                                const float* bg, float* w, float* b, void* stream);
int stmp_lstm_rows_fwd(const stmp_plan* plan, int variant, int n_ops, int64_t cin, const float* x, const float* h, const float* c,
                       const float* w, const float* b, const float* peep, float* hout, float* cout, float* stash, float* S, int64_t ld,
                       void* stream);
int64_t stmp_lstm_rows_scratch_bytes(const stmp_plan* plan);
int stmp_lstm_rows_bwd(const stmp_plan* plan, int variant, int n_ops, int64_t cin, const float* gh, const float* gc, const float* c,
                       const float* cn, const float* stash, const float* w, const float* peep, float* scratch, float* dpre, float* dx,
                       float* dh, float* dc, void* stream);
int64_t stmp_lstm_rows_wgrad_workspace_bytes(int variant, int n_ops, int64_t cin);
int stmp_lstm_rows_wgrad(int variant, int n_ops, int64_t cin, int64_t rows, int64_t ld, const float* S, const float* dpre,
                         const float* scratch, void* workspace, float* dw, float* db, float* dpeep, void* stream);

/* ---- the two-operator GConvLSTM basis at 32 channels (LRGCN with two relations, nn/recurrent/lrgcn.py): n_ops = 2 on a plan with two
 * operators (STMP_FLAVOR_RGCN), basis [X | H | Op0 X | Op0 H | Op1 X | Op1 H], nb = 3 (cin + 32) <= 144.  The two operators are two
 * independent one-hop products (one per relation), not Chebyshev order 2: ChebConv plans hold one operator, so K = 3 never reaches it.
 * stmp_lstm_rows_supported answers 1 for (STMP_LSTM_GCONV, n_ops = 2, cin 1..16, cout = 32) on such a plan, 0 at cout = 64.
 * stmp_lstm_rows_pack_weights, _fwd, _scratch_bytes and _bwd take n_ops = 2 with the layouts above, wx [4][3][32][cin], wh [4][3][32][32]
 * (block k + 1 = operator k); the backward's gather covers both operators in one launch.  Its weight gradient has its own entry:
 *   stmp_lstm_rows_wgrad2: dw [128][nb] = dpre^T S and db [128] = 1^T dpre (db nullable; no peepholes) for the basis S (rows, ld),
 *                          ld = nb rounded up to 8: fp32 FFMA per-CTA partials of the two 64-row halves [dpi | dpf], [dpc | dpo] + a
 *                          fixed-order sum (two launches); workspace of stmp_lstm_rows_wgrad2_workspace_bytes(cin) bytes, 16-byte aligned
 *                          S, dpre and workspace.  STMP_EUNSUPPORTED for cin outside 1..16. */
int64_t stmp_lstm_rows_wgrad2_workspace_bytes(int64_t cin);
int stmp_lstm_rows_wgrad2(int64_t cin, int64_t rows, int64_t ld, const float* S, const float* dpre, void* workspace, float* dw, float* db,
                          void* stream);

/* ---- PyG GatedGraphConv(C, L, aggr, bias=True) -- the convolution of DyGrEncoder (nn/recurrent/dygrae.py) -- on graphs of ANY size, split
 * over CTAs by destination rows (ggc_rows.cu): x^0 = X padded with zeros to C channels, then for l < L: m = x^l W_l, m = aggr over the
 * in-edges of w_e m_j, x^{l+1} = GRUCell(m, x^l) with ONE GRU weight set for every layer; the result is x^L.  On a STMP_FLAVOR_GATED plan,
 * whose aggregation the kernels take from the plan.  add / mean gather a = Op x^l and contract m = a W_l (the aggregation is linear);
 * max needs the message of every source first, so each launch also writes the next layer's m^{l+1} = x^{l+1} W_{l+1}.  max takes
 * max_e (w_e m_j) per channel (w_e m_j rounded as the reference's message), 0 for a node without in-edges; its backward splits a
 * channel's gradient evenly among the messages equal to the maximum, counting the zero-initialised output as one more when the maximum
 * is exactly 0 (torch's scatter_reduce "amax", include_self=False).  Envelope (stmp_ggc_rows_supported): C 1..32, cin 1..C, L 1..1024, any
 * number of nodes and edges.  Exact fp32 (separate multiply and add in the gathers, FFMA in the contractions); deterministic (no
 * atomics, every sum in a fixed order); no host sync and no allocation: scratch and workspace come from the caller, so a call can be
 * captured.  Weights in PyG's layouts: W (L, C, C) with m = x W_l, W_ih / W_hh (3C, C) in gate order r | z | n, b_ih / b_hh (3C).
 *   stmp_ggc_rows_fwd:   x (N, cin) -> out (N, C).  L launches for add / mean, L + 1 for max.  Inference passes stash NULL and scratch
 *                        of stmp_ggc_rows_scratch_bytes(plan, C) bytes; training passes stash (L, 8, N, C): per layer x^l | a^l (add,
 *                        mean) or m^l (max) | the GRU input | r | z | n | W_hn x^l + b_hn | the max's tie count (scratch may then be
 *                        NULL).  The output does not depend on which is given.
 *   stmp_ggc_rows_bwd:   gout = dL/dout (N, C) and the stash -> dG (L, N, 4C) = the GRU pre-activation gradients [dr | dz | dn | r dn] and
 *                        dM (L, N, C) = the gradient at m (add, mean: per destination) or at the messages m^l (max: per source), the
 *                        operands of stmp_ggc_rows_wgrad, and dx (N, cin; nullable).  One launch per layer (the transposed gather of
 *                        layer l + 1 fused with the rowwise GRUCell backward of layer l), plus one when dx is asked for (add, mean)
 *                        or always (max).  scratch of stmp_ggc_rows_scratch_bytes(plan, C) bytes.
 *   stmp_ggc_rows_wgrad: dW (L, C, C), dW_ih, dW_hh (3C, C), db_ih, db_hh (3C) from the stash, dG and dM: the GRU's sums run over all
 *                        L N rows, dW_l's over its layer's N.  fp32 FFMA per-CTA partials + a fixed-order sum (two launches); workspace
 *                        of stmp_ggc_rows_wgrad_workspace_bytes(L, C) bytes.
 * STMP_EINVAL for a NULL plan or tensor or a plan of another flavor, STMP_ESHAPE for a misaligned tensor, STMP_EUNSUPPORTED outside the
 * envelope. */
int stmp_ggc_rows_supported(const stmp_plan* plan, int64_t num_layers, int64_t cin, int64_t channels);
int64_t stmp_ggc_rows_scratch_bytes(const stmp_plan* plan, int64_t channels);
int stmp_ggc_rows_fwd(const stmp_plan* plan, int64_t num_layers, int64_t cin, int64_t channels, const float* x, const float* W,
                      const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, float* scratch, float* out, float* stash,
                      void* stream);
int stmp_ggc_rows_bwd(const stmp_plan* plan, int64_t num_layers, int64_t cin, int64_t channels, const float* gout, const float* stash,
                      const float* W, const float* w_ih, const float* w_hh, float* scratch, float* dG, float* dM, float* dx, void* stream);
int64_t stmp_ggc_rows_wgrad_workspace_bytes(int64_t num_layers, int64_t channels);
int stmp_ggc_rows_wgrad(const stmp_plan* plan, int64_t num_layers, int64_t channels, const float* stash, const float* dG, const float* dM,
                        void* workspace, float* dW, float* dw_ih, float* dw_hh, float* db_ih, float* db_hh, void* stream);

/* ---- EvolveGCN-O and EvolveGCN-H (nn/recurrent/evolvegcno.py, evolvegcnh.py) on graphs of ANY size, split over CTAs by destination rows
 * (evolvegcn_rows.cu).  One call replaces the reference's step: the torch GRU over the C rows of the weight (evolvegcno.py:186-189,
 * evolvegcnh.py:97-100), TopKPooling for -H (evolvegcnh.py:95-96: PyG SelectTopK's score, stable sort and gather) and
 * GCNConv_Fixed_W (evolvegcno.py:86-97, :190: gcn_norm, matmul and propagate).  The plan holds Op: STMP_FLAVOR_GCN (normalize=True, with
 * STMP_GCN_IMPROVED / STMP_GCN_NO_SELF_LOOPS) or STMP_FLAVOR_GATED with STMP_AGGR_ADD (normalize=False: the raw edge weights, no self
 * loops).  Envelope (stmp_evolvegcn_rows_supported): C 1..32, any number of nodes and edges; -H needs N >= C.  Exact fp32 (separate
 * multiply and add in the gathers, FFMA in the contractions); deterministic (no atomics, every sum in a fixed order); no host sync and no
 * allocation, so a call can be captured.  Weights in torch.nn.GRU's layouts: W_ih / W_hh (3C, C) in gate order r | z | n, b_ih / b_hh
 * (3C); the evolving weight W (C, C), row r = batch entry r of the GRU; p (C) = TopKPooling's select.weight.
 *   stmp_evolvegcn_rows_fwd:   x (N, C), w_prev = W_{t-1} -> w_new = W_t, out = Op x W_t (N, C).  p NULL: -O, W_t = GRU(W_{t-1},
 *                              W_{t-1}), one launch.  p given: -H, two launches: s = tanh((x p) / |p|), perm = the C nodes of highest s
 *                              (the lower index first on equal scores), W_t = GRU(x[perm] s[perm], W_{t-1}); perm (int32, C) and
 *                              score = s[perm] (C) are written, and scratch of stmp_evolvegcn_rows_scratch_bytes(plan, C) bytes is used.
 *                              Training passes stash (N, C) = Op x, the operand of the backward (NULL for inference); the outputs do not
 *                              depend on it.
 *   stmp_evolvegcn_rows_bwd:   gout = dL/dout (N, C) and the stash -> dx = Op^T gout W_t^T (N, C; nullable) and per-CTA partials of
 *                              (Op x)^T gout in the workspace (stmp_evolvegcn_rows_workspace_bytes(plan, C) bytes).  One launch.
 *   stmp_evolvegcn_rows_wgrad: one launch of one CTA after stmp_evolvegcn_rows_bwd on the same workspace: dL/dW_t = the fixed-order sum of
 *                              the partials + g_wnew (dL/dW_t from later calls; NULL for none), then the GRU backward over the C rows ->
 *                              dw_prev (-O: the input's and the hidden state's gradients added), dw_ih, dw_hh, db_ih, db_hh; -H (p given,
 *                              with x, perm and score of the forward): dp and, when dx is given, the TopK term added to dx's rows perm.
 * STMP_EINVAL for a NULL plan or tensor or a plan of another flavor, STMP_ESHAPE for a misaligned tensor, STMP_EUNSUPPORTED outside the
 * envelope (C outside 1..32, a GatedGraphConv plan that is not add, -H on fewer than C nodes). */
int stmp_evolvegcn_rows_supported(const stmp_plan* plan, int64_t channels);
int64_t stmp_evolvegcn_rows_scratch_bytes(const stmp_plan* plan, int64_t channels);
int stmp_evolvegcn_rows_fwd(const stmp_plan* plan, int64_t channels, const float* x, const float* w_prev, const float* w_ih, const float* w_hh,
                            const float* b_ih, const float* b_hh, const float* p, void* scratch, float* out, float* w_new, int32_t* perm,
                            float* score, float* stash, void* stream);
int64_t stmp_evolvegcn_rows_workspace_bytes(const stmp_plan* plan, int64_t channels);
int stmp_evolvegcn_rows_bwd(const stmp_plan* plan, int64_t channels, const float* gout, const float* stash, const float* w_new,
                            void* workspace, float* dx, void* stream);
int stmp_evolvegcn_rows_wgrad(const stmp_plan* plan, int64_t channels, void* workspace, const float* g_wnew, const float* x,
                              const float* w_prev, const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh, const float* p,
                              const int32_t* perm, const float* score, float* dw_prev, float* dw_ih, float* dw_hh, float* db_ih,
                              float* db_hh, float* dp, float* dx, void* stream);

/* ---- MPNN-LSTM (nn/recurrent/mpnn_lstm.py) on graphs of ANY size, split over CTAs by destination rows (mpnn_rows.cu).  One call replaces
 * the reference's forward (mpnn_lstm.py:60-105): gcn_norm and two GCNConvs (shared: the plan's operator 0), ReLU, BatchNorm1d and
 * dropout after each, the concatenation and transposes, and two cuDNN LSTMs over `window` steps.  The plan is STMP_FLAVOR_GCN with flags 0
 * (remaining self loops of fill 1, as GCNConv's defaults) built on all R = B * window * num_nodes rows of x.  Envelope
 * (stmp_mpnn_rows_supported): hidden = 32, cin 1..64, window >= 1 dividing R; any number of nodes and edges.  Exact fp32 (separate
 * multiply and add in the gathers, FFMA in the contractions); deterministic (no atomics; BatchNorm's batch statistics are per-CTA
 * Welford partials merged with Chan's formula in one fixed order by every CTA of the next launch); no host sync and no allocation, so a
 * call can be captured.  Weights in the reference's layouts: w1 (32, cin), w2 (32, 32), b1 / b2 (32); BatchNorm weight / bias / running
 * mean / running var (32) and num_batches_tracked (int64, 8-byte aligned); LSTM w_ih1 (128, 64), w_hh1 / w_ih2 / w_hh2 (128, 32), biases
 * (128), gate order i | f | g | o.
 *   stmp_mpnn_rows_fwd: x (R, cin) -> out (B num_nodes, 64 + cin + window - 1) = [h1 | h2 | S], S = every feature of step 0 and the last
 *                       feature of steps 1 .. window-1.  training != 0: BatchNorm normalises with the batch mean and biased variance and
 *                       updates the running statistics (unbiased variance) and num_batches_tracked in place; a negative momentum means
 *                       None (1 / num_batches_tracked).  training = 0: the running statistics.  u (2, R, 32) or NULL: the dropout
 *                       uniforms of both layers, kept where u >= p and scaled by 1 / (1 - p) (0 < p < 1; BatchNorm's mode aside).  Scratch of
 *                       stmp_mpnn_rows_scratch_bytes(plan, cin, 32, window) bytes.  Three launches.
 *                       Training passes stash (stmp_mpnn_rows_stash_bytes, 16-byte aligned): the convolutions' gathers, the LSTMs'
 *                       gates and cell states, z2 and BatchNorm's statistics; NULL for inference.  The outputs do not depend on it.
 *   stmp_mpnn_rows_bwd: after a training forward, with its scratch and stash (both kept) and gout = dL/dout: dx (R, cin; nullable) and
 *                       dbn (4, 32) = dbeta1 | dgamma1 | dbeta2 | dgamma2; the other gradients' operands go to the workspace
 *                       (stmp_mpnn_rows_workspace_bytes, 16-byte aligned).  training and p are the forward's (p = 0: it had no
 *                       dropout).  Four launches, five with dx.
 *   stmp_mpnn_rows_wgrad: after stmp_mpnn_rows_bwd on the same workspace: dw (320, 96) and db (320): rows 0..127 LSTM-1 ([dW_ih | dW_hh]
 *                       in columns 0..95; db = db_ih = db_hh), rows 128..255 LSTM-2 (dW_ih columns 0..31, dW_hh 32..63), rows
 *                       256..287 dW1 (columns 0..cin-1) and db1, rows 288..319 dW2 (columns ld1 .. ld1 + 31, ld1 = cin rounded up to 8)
 *                       and db2.  Two launches; every sum in a fixed order.
 * STMP_EINVAL for a NULL plan or tensor, a plan of another flavor, uniforms with p outside (0, 1), or one row in training mode; STMP_ESHAPE for a misaligned tensor or R not a multiple of window * num_nodes; STMP_EUNSUPPORTED outside the envelope (a GCN
 * plan with flags included). */
int stmp_mpnn_rows_supported(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window);
int64_t stmp_mpnn_rows_scratch_bytes(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window);
int stmp_mpnn_rows_fwd(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window, int64_t num_nodes, const float* x, const float* w1,
                       const float* b1, const float* w2, const float* b2, const float* bn1_weight, const float* bn1_bias, float* bn1_mean,
                       float* bn1_var, int64_t* bn1_count, float bn1_eps, float bn1_momentum, const float* bn2_weight,
                       const float* bn2_bias, float* bn2_mean, float* bn2_var, int64_t* bn2_count, float bn2_eps, float bn2_momentum,
                       const float* w_ih1, const float* w_hh1, const float* b_ih1, const float* b_hh1, const float* w_ih2,
                       const float* w_hh2, const float* b_ih2, const float* b_hh2, int training, float p, const float* u,
                       void* scratch, void* stash, float* out, void* stream);
int64_t stmp_mpnn_rows_stash_bytes(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window);
int64_t stmp_mpnn_rows_workspace_bytes(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window);
int stmp_mpnn_rows_bwd(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window, int64_t num_nodes, const float* gout,
                       const float* w1, const float* w2, const float* bn1_weight, const float* bn2_weight, const float* w_ih1,
                       const float* w_hh1, const float* w_ih2, const float* w_hh2, int training, float p, void* scratch, void* stash,
                       void* workspace, float* dx, float* dbn, void* stream);
int stmp_mpnn_rows_wgrad(const stmp_plan* plan, int64_t cin, int64_t hidden, int64_t window, void* stash, void* workspace, float* dw,
                         float* db, void* stream);

/* ---- AGCRN (nn/recurrent/agcrn.py), the adaptive graph convolutional recurrent cell (agcrn.cu).  One call replaces the reference's
 * AGCRN.forward with its two AVWGCNs (agcrn.py:40-56, 118-127): S = softmax(relu(E E^T)) and its Chebyshev supports, the node weights
 * E weights_pool and biases E bias_pool of both AVWGCNs, the support products, the per-node contractions and the GRU gates (Z gates the
 * state inside the candidate, R is the update gate; at K = 1 the single weight block multiplies Y + S Y, as the reference's einsum
 * broadcast does).  No graph plan: the operator is learned from E.  Envelope (stmp_agcrn_supported): 1 <= N <= 4096, in >= 1,
 * 1 <= out <= 64, in + out <= 128, 1 <= K <= 3, 1 <= d <= 64, 0 <= B <= 8388607 (B = 0: no launch).  Exact fp32 (FFMA products, one
 * fixed order per sum), deterministic (no atomics); no host sync and no allocation, so a call can be captured.  Tensors contiguous
 * float32: x (B, N, in), e (N, d), h (B, N, out) or NULL (zeros), weights_pool (d, K, in + out, Co), bias_pool (d, Co), Co = 2 out for
 * the gate and out for the update.
 *   stmp_agcrn_fwd: -> hout (B, N, out).  Scratch of stmp_agcrn_scratch_bytes(B, N, in, out, K) bytes (the supports, both AVWGCNs' node
 *                   weights, the support products and the gates).  Training passes stash (stmp_agcrn_stash_bytes); NULL for inference.
 *                   Six launches, seven at K = 3.
 *   stmp_agcrn_bwd: after a training forward, with its scratch and stash (both kept) and gh = dL/dhout: dx, dh (only with h), de and the
 *                   pools' gradients dwp_* (d, K, in + out, Co) and dbp_* (d, Co), each nullable; workspace of stmp_agcrn_workspace_bytes.
 *                   Every sum over the batch or the nodes runs in one fixed order; long dT / dE products are split over k in chunks
 *                   that depend on the shapes alone, summed in chunk order.  Eight to fifteen launches (B = 0: none, the requested
 *                   gradients zeroed).
 * STMP_EINVAL for a NULL required tensor or B < 0; STMP_ESHAPE for a misaligned tensor; STMP_EUNSUPPORTED outside the envelope
 * (B > 8388607 included). */
int stmp_agcrn_supported(int64_t b, int64_t n, int64_t in, int64_t out, int64_t K, int64_t d);
int64_t stmp_agcrn_scratch_bytes(int64_t b, int64_t n, int64_t in, int64_t out, int64_t K);
int64_t stmp_agcrn_stash_bytes(int64_t b, int64_t n, int64_t in, int64_t out, int64_t K);
int64_t stmp_agcrn_workspace_bytes(int64_t b, int64_t n, int64_t in, int64_t out, int64_t K);
int stmp_agcrn_fwd(int64_t b, int64_t n, int64_t in, int64_t out, int64_t K, int64_t d, const float* x, const float* e, const float* h,
                   const float* wp_gate, const float* bp_gate, const float* wp_update, const float* bp_update, void* scratch, void* stash,
                   float* hout, void* stream);
/* ---- HeteroGCLSTM (nn/hetero/heterogclstm.py), the heterogeneous graph LSTM (hetero_rows.cu): every destination node type of one call in
 * ONE launch.  Per type t with incoming edge types e_1 .. e_R (sources s_r): pre = S w^T + b on the basis
 * S = [X_t | H_t | mean_{e_1}(H_{s_1}) | ... | mean_{e_R}(H_{s_R})], packed weight w (4 out, nb), nb = in + out (1 + R), per gate the rows
 * [W_g^T | sum_r lin_r^{g,e_r} | lin_l^{g,e_1} | ...] and b = b_g + sum_r lin_l^{g,e_r}.bias; then I, F, O sigmoids, T tanh,
 * C' = F C + I T, H' = O tanh(C') (no peepholes).  mean_e is an STMP_FLAVOR_RGCN plan of one relation over at least N_t nodes whose
 * columns index the source type's rows (the caller checks them against N_s when it makes the plan).  Exact fp32, deterministic, no host
 * sync and no allocation, so a call can be captured.
 * Envelope (stmp_hetero_lstm_supported, per type): 1 <= in <= 32 and out 32 with 1 <= R <= 4, or out 64 with R = 1; at most
 * STMP_HETERO_MAX_TYPES destination types per call, each with 1 <= N.
 *   stmp_hetero_lstm_fwd: desc holds num_types rows of STMP_HETERO_DESC int64 fields: N, in, R, then device pointers x (N, in),
 *                         h (N, out) or 0, c (N, out) or 0 (zeros), w (4 out, nb), b (4 out), hout (N, out), cout (N, out), then
 *                         STMP_HETERO_MAX_REL plan handles and STMP_HETERO_MAX_REL source states H_{s_r} (N_{s_r}, out) (entries past R
 *                         ignored), fields 18.. below.  has_h = 0 means H = 0 for every type: no H loads and no gathers.  One launch.
 * STMP_EINVAL for a NULL required pointer or a plan of another flavor or too few rows; STMP_ESHAPE for a misaligned tensor;
 * STMP_EUNSUPPORTED outside the envelope.
 * Training: fields 18 stash (4 planes of N x out: I, F, T, O) and 19 S (N x nb, the basis rows) make the forward write both (the same
 * launch and arithmetic, so H' and C' equal the inference call's bit for bit); NULL for inference.
 *   stmp_hetero_lstm_bwd: after a training forward, with fields 20 gh, 21 gc (dL/dH', dL/dC', each nullable), 22 dpre (N x 4 out,
 *                         scratch), 23 dx, 25 dc (nullable), 24 dh and 26.. Q_r (N x out, scratch) when want_dh, 30.. the table index of
 *                         each incoming edge type's source type, 34.. its rank in metadata order, 38 dw ((4 out) x (nb + 1): [dw | db],
 *                         nullable for no weight gradient) and workspace of stmp_hetero_lstm_workspace_bytes.  Launches: the rowwise
 *                         backward (dpre, dC, dX, the own-row dH and Q_r = dpre lin_l^{e_r}); with want_dh one transposed gather over
 *                         every source type (own term, then its outgoing edge types in metadata order, then CSR entries); with dw the
 *                         contraction dpre^T [S | 1] over fixed row chunks and its chunk-order reduce: at most four, whatever the number
 *                         of types.  At most 8 outgoing edge types per source type (STMP_EUNSUPPORTED beyond). */
enum { STMP_HETERO_MAX_TYPES = 8, STMP_HETERO_MAX_REL = 4, STMP_HETERO_DESC = 39 };
int stmp_hetero_lstm_supported(int64_t out, int64_t in, int64_t num_rel);
int stmp_hetero_lstm_fwd(int64_t out, int64_t num_types, const int64_t* desc, int has_h, void* stream);
int64_t stmp_hetero_lstm_workspace_bytes(int64_t out, int64_t num_types, const int64_t* desc);
int stmp_hetero_lstm_bwd(int64_t out, int64_t num_types, const int64_t* desc, int want_dh, void* workspace, void* stream);

int stmp_agcrn_bwd(int64_t b, int64_t n, int64_t in, int64_t out, int64_t K, int64_t d, const float* x, const float* e, const float* h,
                   const float* wp_gate, const float* bp_gate, const float* wp_update, const float* bp_update, void* scratch, void* stash,
                   const float* gh, void* workspace, float* dx, float* dh, float* de, float* dwp_gate, float* dbp_gate,
                   float* dwp_update, float* dbp_update, void* stream);

/* ---- GMAN's multi-head attention (nn/attention/gman.py), gman_attention.cu.  One call replaces the attention core of the reference's
 * SpatialAttention, TemporalAttention or TransformAttention.forward (gman.py:235-242, 297-319, 463-474: the split into heads, Q K^T,
 * the division by sqrt(d), the optional tril mask, softmax, the product with V and the concatenation of the heads), read and written
 * in place in the channels-last activations.  A call serves p0 x p1 problems of `heads` heads of width `width`; element (i0, i1, row r,
 * head h, channel c) of tensor t sits at t + i0 s0 + i1 s1 + r sl + h width + c, with strides[12] = host array of (s0, s1, sl) for Q,
 * K, V and O in that order (elements).  The backward's dQ, dK, dV take Q's, K's and V's strides and dO takes O's.
 *   S = scale Q K^T; with mask, S[i][j] = -32767 for j > i, still inside the softmax sum (the reference's torch.where); O = softmax(S) V.
 *   long_kernel = 1: any Lq, Lk, no mask (the spatial attention): online softmax over key tiles, one launch; backward two launches
 *                    (dQ and D = rowsum(dO . O) over query rows, then dK and dV over key rows), workspace of
 *                    stmp_gman_attn_workspace_bytes (D).
 *   long_kernel = 0: Lq, Lk <= 64, a mask needs Lq == Lk (temporal and transform): one warp per (problem, head), exact two-pass
 *                    softmax; backward one launch.
 *   stmp_gman_attn_fwd: -> O.  stash (stmp_gman_attn_stash_bytes: the per-row log-sum-exp, (p0, p1, heads, Lq) floats) for a
 *                       training call, NULL for inference.
 *   stmp_gman_attn_bwd: after a training forward, with its O and stash and dout = dL/dO: dq, dk, dv, each nullable (none: no launch).
 * Envelope (stmp_gman_attn_supported): 1 <= width <= 16, Lq, Lk >= 1, heads >= 1, p0, p1 >= 0 (p0 p1 = 0: no launch) and every grid
 * below 2^31 CTAs.  Exact fp32 (FFMA, every sum in one fixed order), deterministic (no atomics), no host sync and no allocation.
 * STMP_EINVAL for a NULL required tensor or a negative count; STMP_EUNSUPPORTED outside the envelope. */
int stmp_gman_attn_supported(int64_t p0, int64_t p1, int64_t heads, int64_t width, int64_t lq, int64_t lk, int mask, int long_kernel);
int64_t stmp_gman_attn_stash_bytes(int64_t p0, int64_t p1, int64_t heads, int64_t lq);
int64_t stmp_gman_attn_workspace_bytes(int64_t p0, int64_t p1, int64_t heads, int64_t lq, int long_kernel);
int stmp_gman_attn_fwd(int64_t p0, int64_t p1, int64_t heads, int64_t width, int64_t lq, int64_t lk, int mask, int long_kernel,
                       float scale, const int64_t* strides, const float* q, const float* k, const float* v, float* o, float* stash,
                       void* stream);
int stmp_gman_attn_bwd(int64_t p0, int64_t p1, int64_t heads, int64_t width, int64_t lq, int64_t lk, int mask, int long_kernel,
                       float scale, const int64_t* strides, const float* q, const float* k, const float* v, const float* o,
                       const float* stash, const float* dout, void* workspace, float* dq, float* dk, float* dv, void* stream);

/* ---- MTGNN's graph work (nn/attention/mtgnn.py), mtgnn.cu: the top-k graph of GraphConstructor and the mix-hop propagation of the two
 * MixProps of a layer (operators (A + I) / rowsum and (A^T + I) / rowsum), with their backward.  A graph of N nodes and row width W
 * (W = k for a learned graph, the widest row for a predefined one) lives in three caller-owned buffers:
 *   pattern int32 [N W | N | N + 1 | N W | N W]: col1, cnt1 (the entries of each row of A), ptr2, row2 (the rows of each column of A,
 *           ascending) and pos2 (where each column entry sits in the row arrays);
 *   state   fp32  [N W | N | N]: the raw entries a of A, d1 = 1 + row sums, d2 = 1 + column sums;
 *   values  fp32  [N W | N W | N | N]: v1 = a / d1[row], v2 = a / d2[column] (both at the row position of entry (i, j)), diag1 = 1 / d1,
 *           diag2 = 1 / d2.  Unused row slots hold zero values.
 *   stmp_mtgnn_graph_fwd:   m1, m2 (N, dim) -> A = relu(tanh(alpha (m1 m2^T - m2 m1^T))) keeping the k largest entries of each row
 *                           (equal values: the lower column first; zero entries dropped); workspace: stmp_mtgnn_graph_workspace_bytes.
 *   stmp_mtgnn_graph_dense: the same structures from the nonzeros of a dense (N, N) A, W >= its widest row (a wider row keeps its
 *                           first W nonzeros: nothing is written past a row's slots).
 *   stmp_mtgnn_graph_bwd:   dvals (the values' layout) -> dm1, dm2 through both normalisations, the mask, relu and tanh;
 *                           workspace: stmp_mtgnn_graph_bwd_workspace_bytes.
 *   stmp_mtgnn_prop_fwd:    x (B, C, N, T) contiguous -> hops (B, 2 depth C, N, T): channel block o depth + k - 1 = hop k of operator o,
 *                           H_k = alpha x + (1 - alpha) S_o H_{k-1}, H_0 = x.  2 depth launches.
 *   stmp_mtgnn_prop_bwd:    dhops = dL/dhops (overwritten), dx = the direct gradient of x (accumulated in place) -> dx, and dvals
 *                           (nullable) the gradient of the values.  2 depth + 1 launches.
 * Envelope (stmp_mtgnn_supported returns STMP_OK or STMP_EUNSUPPORTED): 1 <= N <= 4096, 1 <= k <= min(N, 64), 1 <= dim <= 64,
 * 1 <= C <= 64, 1 <= depth <= 4, B >= 0 (B = 0: no launch), T >= 1, every grid below 2^31 CTAs.  Exact fp32 (FFMA, every sum in one
 * fixed order), deterministic (no atomics), no host sync and no allocation. */
int stmp_mtgnn_supported(int64_t n, int64_t k, int64_t dim, int64_t channels, int64_t depth, int64_t batch, int64_t steps);
int64_t stmp_mtgnn_graph_workspace_bytes(int64_t n);
int stmp_mtgnn_graph_fwd(int64_t n, int64_t k, int64_t dim, float alpha, const float* m1, const float* m2, void* workspace, int* pattern,
                         float* state, float* vals, void* stream);
int stmp_mtgnn_graph_dense(int64_t n, int64_t w, const float* A, void* workspace, int* pattern, float* state, float* vals, void* stream);
int64_t stmp_mtgnn_graph_bwd_workspace_bytes(int64_t n);
int stmp_mtgnn_graph_bwd(int64_t n, int64_t k, int64_t dim, float alpha, const float* m1, const float* m2, const int* pattern,
                         const float* state, const float* vals, const float* dvals, void* workspace, float* dm1, float* dm2, void* stream);
int stmp_mtgnn_prop_fwd(int64_t B, int64_t C, int64_t N, int64_t T, int64_t W, int64_t depth, float alpha, const float* x,
                        const int* pattern, const float* vals, float* hops, void* stream);
int stmp_mtgnn_prop_bwd(int64_t B, int64_t C, int64_t N, int64_t T, int64_t W, int64_t depth, float alpha, const float* x,
                        const int* pattern, const float* vals, const float* hops, float* dhops, float* dx, float* dvals, void* stream);

/* ---- the same cell at 64 hidden channels (lstm_rows.cu, the width-2 instance of its kernels): GConvLSTM / GCLSTM(cin, 64, K <= 2).
 * Envelope: cout = 64, cin 1..16, n_ops 0..1 and at most the plan's operators (stmp_lstm_rows_supported(plan, variant, n_ops, cin, 64)),
 * any number of nodes and any degree.  Same argument lists, launch chain and guarantees as the stmp_lstm_rows_* entries, with 32 -> 64
 * throughout:
 *   packed weights w [256][nb]: row gate*64 + o, column m of the basis; nb = (n_ops+1)(cin+64) (GConvLSTM) or cin + 64(n_ops+1) (GCLSTM);
 *                                     b [256]; peep (3, 64) or NULL.
 *   stmp_lstm_wide_rows_pack_weights: wx [4][n_ops+1][64][cin] (GCLSTM: [4][cin][64]), wh [4][n_ops+1][64][64], bx / bh / bg [4][64].
 *   stmp_lstm_wide_rows_fwd:          x (N,cin), h and c (N,64) or NULL -> hout, cout (N,64); stash (4,N,64); S (N, ld), ld = nb
 *                                     rounded up to 8, 16-byte aligned.
 *   stmp_lstm_wide_rows_bwd:          gh, gc (N,64) -> dpre (2,N,128) = [dpi | dpf], [dpc | dpo], dx (N,cin), dh (N,64), dc (N,64);
 *                                     scratch of stmp_lstm_wide_rows_scratch_bytes(plan) bytes (N*80 floats + 192 per CTA).
 *   stmp_lstm_wide_rows_wgrad:        dw [256][nb], db [256], dpeep [192] (db, dpeep nullable): fp32 FFMA per-CTA partials of each gate's
 *                                     product over strided 32-row tiles + a fixed-order sum (two launches); workspace of
 *                                     stmp_lstm_wide_rows_wgrad_workspace_bytes(variant, n_ops, cin) bytes, 16-byte aligned operands.
 * STMP_EINVAL for NULL tensors or an unknown variant, STMP_ESHAPE for a bad pitch or alignment, STMP_EUNSUPPORTED for cin > 16,
 * n_ops > 1 or n_ops above the plan's operators. */
int stmp_lstm_wide_rows_pack_weights(int variant, int n_ops, int64_t cin, const float* wx, const float* wh, const float* bx,
                                     const float* bh, const float* bg, float* w, float* b, void* stream);
int stmp_lstm_wide_rows_fwd(const stmp_plan* plan, int variant, int n_ops, int64_t cin, const float* x, const float* h, const float* c,
                            const float* w, const float* b, const float* peep, float* hout, float* cout, float* stash, float* S,
                            int64_t ld, void* stream);
int64_t stmp_lstm_wide_rows_scratch_bytes(const stmp_plan* plan);
int stmp_lstm_wide_rows_bwd(const stmp_plan* plan, int variant, int n_ops, int64_t cin, const float* gh, const float* gc, const float* c,
                            const float* cn, const float* stash, const float* w, const float* peep, float* scratch, float* dpre,
                            float* dx, float* dh, float* dc, void* stream);
int64_t stmp_lstm_wide_rows_wgrad_workspace_bytes(int variant, int n_ops, int64_t cin);
int stmp_lstm_wide_rows_wgrad(int variant, int n_ops, int64_t cin, int64_t rows, int64_t ld, const float* S, const float* dpre,
                              const float* scratch, void* workspace, float* dw, float* db, float* dpeep, void* stream);

/* ---- backward of the fused DCRNN sequence for narrow states (cout <= 4): the reference's training model BatchedDCRNN(F, F, K=3) ----
 * Served when stmp_dcrnn_narrow_bwd_supported(plan, cin, cout, K) != 0 (DCONV plan, cin and cout in 1..4, K in 1..4, graph and state
 * buffers fit one SM's shared memory: PEMS-BAY's 325 nodes at K = 3 do).  stmp_dcrnn_narrow_bwd_seq is the reverse-time recurrence in
 * one persistent launch, with the contract of stmp_dcrnn_bwd_seq plus K: gout (B,T,N,cout), out and stash (B,T,3,N,cout) of the
 * forward, h0 (B,N,cout; nullable), whsT (cout, (2K-1)C) / wzrT (2cout, (2K-1)C) from stmp_dcrnn_pack_bwd_weights -> dph_all
 * (T,B,N,cout), dpzr_all (T,B,N,2cout), dx (B,T,N,cin; nullable), dh0 (B,N,cout).  Deterministic, no atomics; the results do not
 * depend on how many windows a CTA serves ("dcrnn_narrow_pack"). */
int stmp_dcrnn_narrow_bwd_supported(const stmp_plan* plan, int64_t cin, int64_t cout, int64_t K);
int stmp_dcrnn_narrow_bwd_seq(const stmp_plan* plan, int64_t B, int64_t T, int64_t cin, int64_t cout, int64_t K, const float* gout,
                              const float* out, const float* h0, const float* stash, const float* whsT, const float* wzrT,
                              float* dph_all, float* dpzr_all, float* dx, float* dh0, void* stream);

/* Backward of stmp_tgcn_attn_fwd for H = NULL (the training configuration of the reference's A3TGCN2 example; what autograd records for
 * attentiontemporalgcn.py:130-157 / temporalgcn.py:187-233 over all periods): given gout (B, N, 32) it recomputes A^X and the gates and
 * reduces dA (fin, 96; the r-gate columns are zero: R multiplies H = 0), dc (96) and dprobs (periods; nullable when probs is NULL) over all
 * (batch row, node, period).  The gradients of the module parameters follow from the (differentiable, host-side) folding A = (L1 W)^T,
 * c = L1 b + l and probs = softmax(attention).  No gradient w.r.t. X.  Two launches (per-CTA partials, fixed-order reduction);
 * workspace of stmp_tgcn_attn_bwd_workspace_bytes(plan, B) bytes. */
int64_t stmp_tgcn_attn_bwd_workspace_bytes(const stmp_plan* plan, int64_t B);
int stmp_tgcn_attn_bwd(const stmp_plan* plan, int64_t B, int64_t fin, int64_t periods, const float* x, const float* A,
                       const float* c, const float* probs, const float* gout, void* workspace, float* dA, float* dc,
                       float* dprobs, void* stream);

/* Backward of ONE TGCN cell step with an incoming state: stmp_tgcn_attn_fwd with periods = 1, probs = NULL and h != NULL (what autograd
 * records for temporalgcn.py:104-130 / :212-233 on the steps t >= 1 of the reference's BatchedTGCN loop, H carried).  x (B, N, fin), h
 * (B, N, 32) at batch stride h_bstride, A (fin, 96), Bm (32, 96), c (96) are the forward's operands, gout = dL/dH_new (B, N, 32).  It
 * recomputes A^X and the gates and writes dh = dL/dH (B, N, 32, contiguous; skipped when dh is NULL) and the folded-weight gradients
 * dA (fin, 96), dBm (32, 96) and dc (96), reduced over all (batch row, node).  No gradient w.r.t. X.  Two launches (k_tgcn_cell_bwd:
 * per-CTA partials; k_tgcn_cell_bwd_reduce: fixed-order sum), deterministic; workspace of stmp_tgcn_cell_bwd_workspace_bytes(plan, B)
 * bytes.  STMP_EUNSUPPORTED for fin outside 1..4, STMP_EINVAL for a NULL tensor or B < 1, STMP_ESHAPE for B >= 65536. */
int64_t stmp_tgcn_cell_bwd_workspace_bytes(const stmp_plan* plan, int64_t B);
int stmp_tgcn_cell_bwd(const stmp_plan* plan, int64_t B, int64_t fin, const float* x, const float* h, int64_t h_bstride, const float* A,
                       const float* Bm, const float* c, const float* gout, void* workspace, float* dh, float* dA, float* dBm, float* dc,
                       void* stream);

/* The three entries above at out_channels = 64, with the same argument lists and answers: A (fin, 192), Bm (64, 192), c (192) in
 * columns z | r | h of 64 each; h, out, gout and dh (B, N, 64); dA (fin, 192), dBm (64, 192), dc (192).  The forward stages Bm in shared
 * memory next to X[b].  stmp_tgcn_wide_cell_bwd writes dH, the per-row gate gradients and the bases [A^X | H], [A^X | H*R] into the
 * workspace, contracts them with the 64-wide weight-gradient kernels of the row-split GConvGRU cell (fixed-order sums, no atomics) and
 * unpacks the result into dA and dBm: four launches, deterministic; the workspace (16-byte aligned) grows with B * N. */
int stmp_tgcn_wide_attn_fwd(const stmp_plan* plan, int64_t B, int64_t fin, int64_t periods, const float* x, const float* h,
                            int64_t h_bstride, const float* A, const float* Bm, const float* c, const float* probs, float* out,
                            void* stream);
int64_t stmp_tgcn_wide_attn_bwd_workspace_bytes(const stmp_plan* plan, int64_t B);
int stmp_tgcn_wide_attn_bwd(const stmp_plan* plan, int64_t B, int64_t fin, int64_t periods, const float* x, const float* A,
                            const float* c, const float* probs, const float* gout, void* workspace, float* dA, float* dc,
                            float* dprobs, void* stream);
int64_t stmp_tgcn_wide_cell_bwd_workspace_bytes(const stmp_plan* plan, int64_t B);
int stmp_tgcn_wide_cell_bwd(const stmp_plan* plan, int64_t B, int64_t fin, const float* x, const float* h, int64_t h_bstride,
                            const float* A, const float* Bm, const float* c, const float* gout, void* workspace, float* dh, float* dA,
                            float* dBm, float* dc, void* stream);

/* Weight / bias gradients of the three DCRNN gates over all (t, b, n) rows (what autograd accumulates for the `matmul(basis, W)` and
 * `+ bias` of dcrnn.py:86-111 across steps, gates and hops): S1 / S2 (rows, ld) are stmp_dcrnn_bwd_basis' bases (ld = 3(cin+cout) rounded
 * up to 8), dpzr (rows, 2cout) / dph (rows, cout) stmp_dcrnn_bwd_seq's d pre-activations.  Writes gz / gr / gh in the module's
 * (2, K, cin+cout, cout) layout and the bias gradients (nullable).  Two launches (per-CTA partials, fixed-order reduction: deterministic);
 * the contraction runs on wgmma (TF32, K-major operands transposed as they are staged, TF32 hi/lo split; stmp_set_option("dcrnn_wgrad_tc", 0) selects the
 * fp32 FFMA kernel).  Workspace of stmp_dcrnn_bwd_wgrad_workspace_bytes(cin) bytes.  K = 2, cout = 32, cin <= 4. */
int64_t stmp_dcrnn_bwd_wgrad_workspace_bytes(int64_t cin);
int stmp_dcrnn_bwd_wgrad(int64_t cin, int64_t cout, int64_t K, int64_t rows, int64_t ld, const float* S1, const float* S2,
                         const float* dpzr, const float* dph, void* workspace, float* gz, float* gr, float* gh, float* gbz,
                         float* gbr, float* gbh, void* stream);

/* torch.optim.Adam's update (the optimizer of examples/indexBatching/DCRNN/pems_ddp.py:90) over ONE flat fp32 buffer of n parameters:
 * g' = grad * grad_scale (+ weight_decay * param); exp_avg.lerp(g', 1-beta1); exp_avg_sq = beta2 exp_avg_sq + (1-beta2) g'^2;
 * param -= lr / (1-beta1^t) * exp_avg / (sqrt(exp_avg_sq) / sqrt(1-beta2^t) + eps), t = *step + 1.  `step` (one float) and `ticket`
 * (one zero-initialised uint32) live on the device: the last block to finish bumps the counter, so a captured CUDA graph replays
 * correctly.  zero_grad != 0 clears the gradient buffer in the same pass.  One launch. */
int stmp_adam_flat(int64_t n, float* param, float* grad, float* exp_avg, float* exp_avg_sq, float* step, void* ticket, float lr,
                   float beta1, float beta2, float eps, float weight_decay, float grad_scale, int zero_grad, void* stream);

/* Transposed stacked DConv weights for the backward kernels, one launch: whsT (cout, (2K-1)C) from wh, wzrT (2cout, (2K-1)C)
 * from wz | wr; C = cin + cout; stacked block 0 = W[0,0] + W[1,0], block 1+2(k-1)+o = W[o,k] (the order of the basis). */
int stmp_dcrnn_pack_bwd_weights(int64_t cin, int64_t cout, int64_t K, const float* wz, const float* wr, const float* wh,
                                float* whsT, float* wzrT, void* stream);

/* Masked MAE of the index-batching training loops (examples/indexBatching/DCRNN/utils.py:10-18, used at pems_ddp.py:104-121):
 * loss = mean(nan_to_zero(|pred - y| * mask / mean(mask))), mask = (y != 0) == sum_i nz(|p_i - y_i| m_i) / sum_i m_i.
 * fwd writes the scalar loss and s0 = sum(mask) (device scalars; deterministic two-stage reduction, workspace of
 * stmp_masked_mae_workspace_floats() floats); bwd writes gpred = gout * sign(pred - y) * mask / s0. */
int64_t stmp_masked_mae_workspace_floats(void);
int stmp_masked_mae_fwd(int64_t n, const float* pred, const float* target, float* workspace, float* loss, float* s0, void* stream);
int stmp_masked_mae_bwd(int64_t n, const float* pred, const float* target, const float* s0, const float* gout, float* gpred,
                        void* stream);

/* GRU reverse-time gate derivatives: the pointwise part of the hand-written backward of the DCRNN sequence (what
 * autograd records for dcrnn.py:172-192, once per step).  Tensors are (B, N, cout) with a batch stride in elements
 * (slices of gout (B,T,N,cout) and of the forward stash (B,T,3,N,cout)); du2/du1 are (B, N, du_ld) buffers whose
 * first cin+cout columns hold dL/d[X | H*R] and dL/d[X | H_{t-1}] of the step being closed.
 *   stmp_gru_bwd_carry: close step t+1 (all of g_prev.. or none): dH = g_prev*Z + dU2[...,cin:]*R + dU1[...,cin:],
 *                       dX_{t+1} = dU2[...,:cin] + dU1[...,:cin] (dx nullable), dh_out = dH (nullable);
 *                       open step t (gout.. or none): g = gout_t + dH, dph = g (1-Z_t)(1-Ht_t^2).
 *   stmp_gru_bwd_zr:    dpzr[..., :cout] = g (H_{t-1} - Ht) Z (1-Z);  dpzr[..., cout:] = dU2[...,cin:] H_{t-1} R (1-R);
 *                       hprev NULL = zeros (first step without H0).
 */
int stmp_gru_bwd_carry(int64_t B, int64_t N, int64_t cin, int64_t cout, int64_t du_ld, const float* g_prev,
                       const float* z_prev, const float* r_prev, const float* du2, const float* du1, float* dx,
                       int64_t dx_bstride, const float* gout, int64_t gout_bstride, const float* z, const float* ht,
                       int64_t stash_bstride, float* g, float* dph, float* dh_out, void* stream);
int stmp_gru_bwd_zr(int64_t B, int64_t N, int64_t cin, int64_t cout, int64_t du_ld, const float* g, const float* hprev,
                    int64_t hprev_bstride, const float* z, const float* r, const float* ht, int64_t stash_bstride,
                    const float* du2, float* dpzr, void* stream);

/* ---- K4: dense node-feature x weight contraction on the tensor cores (wgmma), fp32 in / fp32 out ------------------
 * C[M,N] = A[M,K] @ W[K,N] + bias.  Replaces `torch.matmul(Tx_k, weight[..][k])` / ChebConv `lins[k](Tx_k)` / GCNConv
 * `lin(x)` (dcrnn.py:81-105; PyG) for the large-graph (tiled) path.  Operands are split into fp16 hi = fp16(v), lo = fp16(v - hi)
 * and multiplied in three wgmma passes (lo*hi + hi*lo + hi*hi) with fp32 register accumulators.  Accuracy envelope (also of
 * stmp_gemm_blocks_f32): |C - A W| <= ~8 (2^-22 (|A||W|)_mn + 2^-25 (sum_k |A_mk| + sum_k |W_kn|)),
 * i.e. fp32-class relative accuracy only while |operands| lie between about 2^-3 and 2^15; below that an absolute floor of about
 * 2^-25 per operand element (elements under 3e-8 become zero).  Callers must keep |operands| < 65504 (larger overflow the hi half
 * to inf) and prescale small operands such as gradients by an exact power of two (see nn/recurrent/gconv_lstm.py::_split_prescale).
 *   stmp_gemm_packed_elems(K,N): number of fp16 elements of the packed weight buffer
 *   stmp_gemm_prepack: W [K,N] row-major (row stride ldw) -> packed (hi/lo, K-major, K padded to 64); once per weight update
 *   stmp_gemm_f32: A row-major (row stride lda), C row-major (ldc); needs N <= 256, N % 32 == 0, K % 4 == 0, 16-byte aligned
 *                  rows; otherwise STMP_EUNSUPPORTED (callers use cuBLAS)
 *   stmp_gemm_lstm_f32: same contraction with N = 4*cout (column blocks i|f|c|o) fused with the peephole-LSTM gate epilogue
 *                  of GConvLSTM (gconv_lstm.py:168-202): conv_bias [4*cout] (ChebConv biases), cell C_{t-1} [M,cout],
 *                  peepholes w_c{i,f,o} [cout], gate biases b_{i,f,c,o} [cout] -> h_out, c_out [M,cout]; cout in {32, 64}. */
int64_t stmp_gemm_packed_elems(int64_t K, int64_t N);
int stmp_gemm_prepack(const float* W, int64_t ldw, int64_t K, int64_t N, void* packed, void* stream);
int stmp_gemm_f32(const float* A, int64_t lda, int64_t M, int64_t K, int64_t N, const void* packed, const float* bias,
                  float* C, int64_t ldc, void* stream);
int stmp_gemm_lstm_f32(const float* A, int64_t lda, int64_t M, int64_t K, int64_t cout, const void* packed,
                       const float* conv_bias, const float* cell, const float* wci, const float* wcf, const float* wco,
                       const float* bi, const float* bf, const float* bc, const float* bo, float* h_out, float* c_out,
                       void* stream);

/* ---- ASTGCN block (nn/attention/astgcn.py:408-481): the dense products on wgmma with their operand gathers and pointwise tails fused
 * stmp_gemm_blocks_f32:  C[m, 0:ncols] = epilogue( sum_i A_i[m + shift_i, 0:width_i] @ W_i + bias )
 *   the A operand is a list of nblk (<= 12) K-blocks of <= 64 columns: blk_ptr[i] (device pointer, HOST array), row stride blk_ld[i],
 *   valid columns blk_width[i], row shift blk_shift[i] inside sequences of `seq` consecutive rows (rows shifted out of their sequence read
 *   as zero).  packed = stmp_gemm_prepack of the stacked weight [nblk*64][N] (rows of a block beyond its width are zero), N % 16 == 0,
 *   N <= 320.  epilogue 0: + bias; 1: + bias, ReLU; 2: + bias, ReLU, LayerNorm(gamma, beta, eps) over the row (N == ncols == 64).
 *   With channels-last activations (B, nodes, T, F) this is: the Chebyshev contraction sum_k T_k W_k + ReLU (astgcn.py:166-178,448) with
 *   blocks T_0|T_1|T_2; time convolution (1x3, padding 1) + residual 1x1 convolution + ReLU + LayerNorm (:473-480) with blocks
 *   X^[t-1] | X^[t] | X^[t+1] | X[t], seq = T; the final (1 x F) convolution (:604-610) with the T blocks of a row.
 * stmp_spatial_attention_fwd:  S = softmax_dim1(Vs @ sigmoid(LHS @ RHS + bs)) (astgcn.py:245-262), written TRANSPOSED:
 *   st_out[b, j, i] = S[b, i, j], rows ld_out (>= nodes rounded up to 64, % 4 == 0) floats apart, padding columns zero.
 *   lhs [B][nodes][T] = (X~ W1) W2, rhs [B][T][nodes] = (W3 X~)^T, bsT [nodes][nodes] = bs^T, vsT_packed = stmp_gemm_prepack of Vs^T
 *   zero-padded to [P][P], P = nodes rounded up to 64 (<= 320).  The N x N sigmoid is generated inside the GEMM's operand stage and the
 *   softmax is the GEMM epilogue: neither ever reaches HBM.
 *   nodes <= 320, T <= 12.  At T == 12 lhs must be 16-byte aligned (its rows are read as float4): EINVAL otherwise.  NULL pointers are
 *   EINVAL when B > 0; B == 0 launches nothing.
 * Optional weight IMAGE (both entries; NULL = the kernel swizzles the packed weights itself): stmp_gemm_blocks_image rewrites a packed weight
 * into the per-k-block shared-memory image (hi | lo tile, SWIZZLE_128B) of stmp_gemm_blocks_image_bytes(N, nblk) bytes, which every CTA then
 * fetches with ONE TMA bulk copy per k-block while it loads / generates its A tile. */
int stmp_gemm_blocks_f32(int64_t M, int64_t N, int64_t ncols, int64_t nblk, const float* const* blk_ptr, const int64_t* blk_ld,
                         const int32_t* blk_width, const int32_t* blk_shift, int64_t seq, const void* packed, const void* image,
                         const float* bias, int epilogue, const float* gamma, const float* beta, float eps, float* C, int64_t ldc, void* stream);
int stmp_spatial_attention_fwd(int64_t B, int64_t n_nodes, int64_t n_steps, const float* lhs, const float* rhs, const float* bsT,
                               const void* vsT_packed, const void* vsT_image, float* st_out, int64_t ld_out, void* stream);
/* stmp_spatial_attention_tiled_fwd:  the same st_out as stmp_spatial_attention_fwd, same inputs (vsT_packed only: no image), for
 *   1 <= nodes <= 1024 (PeMS03 / PeMS07-sized graphs), T <= 12.  Two launches: k_spatt_tiles tiles the columns as well as the rows (<= 256
 *   columns per CTA, the sigmoid operand regenerated per column tile), writes the unnormalised logits into st_out and one (max, sum) pair per
 *   (row, column tile) into `workspace`; k_spatt_norm combines a row's pairs in a fixed order and normalises the row in place.
 *   Deterministic (no atomics), no allocation, no host synchronisation: capturable into a CUDA graph.
 *   workspace: >= stmp_spatial_attention_tiled_workspace_bytes(B, nodes) bytes, 8-byte aligned, given as `workspace_bytes`.
 *   EUNSUPPORTED beyond 1024 nodes or 12 timesteps; ESHAPE for ld_out < nodes rounded up to 64, ld_out % 4 != 0 or st_out not 16-byte
 *   aligned; EINVAL for NULL pointers (B > 0) or a short / misaligned workspace.  B == 0 launches nothing.
 * stmp_spatial_attention_tiled_workspace_bytes: -1 outside the envelope. */
int stmp_spatial_attention_tiled_fwd(int64_t B, int64_t n_nodes, int64_t n_steps, const float* lhs, const float* rhs, const float* bsT,
                                     const void* vsT_packed, float* st_out, int64_t ld_out, void* workspace, int64_t workspace_bytes,
                                     void* stream);
int64_t stmp_spatial_attention_tiled_workspace_bytes(int64_t B, int64_t n_nodes);
/* The small-matrix front of an ASTGCN block in one launch (astgcn.py:311-328 temporal attention, :427-430 X~ = X E, :245-256 the spatial
 * attention factors): x [B][nodes][T][F] channels-last; TemporalAttention parameters U1 [nodes], U2 [F][nodes], U3 [F], be [T][T],
 * Ve [T][T]; SpatialAttention parameters W1 [T], W2 [F][T], W3 [F]  ->  lhs_s [B][nodes][T] = (X~ W1) W2, rhs_s [B][T][nodes] = (W3 X~)^T
 * (the inputs of stmp_spatial_attention_fwd) and optionally E [B][T][T].  X~ is never materialised.  T <= 12, F in {1,2,4,...,64}
 * (F >= 32 needs x 16-byte aligned), B <= 65535 and 4 (3 nodes T + T F + 2 T^2 + T + 16) <= 200 KB: EUNSUPPORTED otherwise.  B == 0
 * launches nothing. */
int stmp_astgcn_factors_fwd(int64_t B, int64_t n_nodes, int64_t n_steps, int64_t f_in, const float* x, const float* U1, const float* U2,
                            const float* U3, const float* be, const float* Ve, const float* W1, const float* W2, const float* W3,
                            float* lhs_s, float* rhs_s, float* E_out, void* stream);
int64_t stmp_gemm_blocks_image_bytes(int64_t N, int64_t nblk);
int stmp_gemm_blocks_image(const void* packed, int64_t N, int64_t nblk, void* image, void* stream);

/* ---- K8: index-batching window gather -----------------------------------------------------------
 * x[b] = series[start[b] : start[b]+h], y[b] = series[start[b]+h : start[b]+2h]   (index_dataset.py:49-57
 * + DataLoader default collate), series [T_total, row_elems] resident on the device.  y may be NULL. */
int stmp_window_gather(const float* series, int64_t t_total, int64_t row_elems, const int64_t* start,
                       int64_t B, int64_t horizon, float* x, float* y, void* stream);

/* Run-time switches for tests, each selecting an implementation or launch shape that a test compares the default against:
 * "dcrnn_tc" = 1 (wgmma kernel, default) / 0 (FFMA kernel) behind stmp_dcrnn_seq_fwd; "dcrnn_fwd_split" = 1 (default: the fused
 * forward runs on a 2-CTA cluster per window when 2 B <= SM count and N > 128) / 0 (one CTA per window); "dcrnn_bwd_split" = 1
 * (default: a 2-CTA cluster per window when 2 B <= SM count) / 0 (one CTA per window); "dcrnn_wgrad_tc" = 1 (default, wgmma) /
 * 0 (FFMA); "dcrnn_narrow_pack" = 0 (default: automatic) / P in 1..8, the number of windows one CTA of the narrow-state DCRNN kernels
 * serves side by side (lowered if the layout does not fit; outputs do not depend on it).  Any other name returns STMP_EINVAL. */
int stmp_set_option(const char* name, int value);

/* ---- misc ---------------------------------------------------------------------------------------- */
const char* stmp_last_error(void);
/* "stmp <version> sm_90a" */
const char* stmp_version(void);
/* Number of kernels this library has launched in the calling process (bench.py's gpu_launches). */
int64_t stmp_launch_count(void);
/* Which kernels served the calls so far ("did the fused wgmma path run, or the tiled one?" -- the dispatchers fall back
 * silently on STMP_EUNSUPPORTED, e.g. dcrnn.py:429-475 at N > 207).  Fills up to max_entries (kernel name, launches) pairs,
 * names are static strings such as "k_dcrnn_seq_tc"; returns the number of distinct kernels launched. */
int stmp_path_counters(const char** names, int64_t* counts, int max_entries);

#ifdef __cplusplus
}
#endif
#endif /* STMP_H_ */
