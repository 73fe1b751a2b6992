// gemm_blocks.cu -- the dense products of an ASTGCN block (nn/attention/astgcn.py) on the Hopper tensor cores (wgmma), fp32 in / fp32 out,
// with the operand GATHER and the pointwise tail of each product fused into one kernel:
//
//   C[m, :] = epilogue( sum_blocks  A_blk[row(m) + shift_blk, 0:width_blk] @ W_blk  + bias )
//
// * the A operand is a list of up to 12 K-blocks (<= 64 columns each) that may come from DIFFERENT tensors and may be SHIFTED by
//   whole rows inside sequences of `seq` rows (out-of-sequence rows read as zero).  With activations kept channels-last
//   (B, N, T, F) this expresses, without any im2col / cat / permute in HBM:
//     - the Chebyshev contraction  sum_k T_k W_k            (astgcn.py:166-178)      blocks = T_0 | T_1 | T_2, epilogue ReLU (:448)
//     - time convolution (1x3, pad 1) + residual 1x1 convolution + ReLU + LayerNorm   (:473-480)
//                                                            blocks = X^[t-1] | X^[t] | X^[t+1] | X[t], epilogue ReLU + LayerNorm
//     - the final (1 x F_t) convolution over (T, F_t)        (:604-610)               blocks = the T*F_t columns of a row
// * MODE_SPATT generates the A operand instead of loading it: spatial attention (astgcn.py:245-262)
//     S = softmax_dim1( Vs @ sigmoid(LHS @ RHS + bs) )   is computed TRANSPOSED,  S^T[b] = sigmoid(...)^T @ Vs^T, rows (b, j):
//     A[(b,j)][k] = sigmoid( sum_t LHS[b,k,t] RHS[b,t,j] + bs[k][j] )  is formed on the fly from the two (B,N,T) factors, and the
//     softmax over dim 1 of S becomes a softmax over the COLUMNS of each output row -- thread-local in the epilogue (the accumulators are
//     staged in shared memory, one thread per row).  2 B N^3 FLOPs, the one GEMM of the model SURVEY calls a tensor-core target, never materialises the N x N sigmoid.
// * fp32-class accuracy from fp16 tensor cores: operands split into hi = fp16(v), lo = fp16(v - hi), three wgmma f16 passes
//   lo*hi + hi*lo + hi*hi into fp32 register accumulators (as gemm_tc.cu / dcrnn_seq_tc.cu).
// One CTA = 128 rows x all N (<= 320) columns; N > 256 runs as two MMA column halves.  2-stage pipeline: the tile of k-block i+1 is
// loaded / generated / converted while the MMAs of k-block i run.
#include "common.cuh"
#include "tc_common.cuh"

namespace stmp {
namespace {

constexpr int GB_NT = 256;
constexpr int GB_BM = 128;
constexpr int GB_A_BYTES = GB_BM * 128;   // one K-block of A (hi or lo): 128 rows x 64 fp16
constexpr int GB_MAXBLK = 12;
constexpr int GB_MAXN = 320;

enum { EPI_BIAS = 0, EPI_RELU = 1, EPI_RELU_LN = 2, EPI_SOFTMAX = 3 };

struct KBlock {
  const float* ptr;
  long long ld;     // row stride (floats)
  int width;        // valid columns (<= 64); the rest of the k-block is zero
  int shift;        // row shift inside a sequence of `seq` rows
};

struct GbParams {
  KBlock blk[GB_MAXBLK];
  int nblk;
  int M, N;                 // N % 16 == 0, N <= 320
  int seq;                  // rows per sequence for shifted blocks (>= 1)
  const __half* w_hi;       // [N][nblk*64]
  const __half* w_lo;
  const unsigned char* w_img;   // optional: per k-block the B tile exactly as it sits in shared memory (hi | lo, swizzled): one TMA bulk copy
  const float* bias;        // [N] or null
  float* C; long long ldc;
  int ncols;                // columns written (<= N)
  // EPI_RELU_LN (N == 64): LayerNorm over the row
  const float* gamma; const float* beta; float eps;
  // MODE_SPATT
  int spatt;                // 1: generate A
  int Nn, Tn;               // nodes, timesteps
  const float* lhs;         // [B][Nn][Tn]
  const float* rhs;         // [B][Tn][Nn]
  const float* bsT;         // [Nn][Nn]  bs transposed: bsT[j][k] = bs[k][j]
};

__device__ __forceinline__ float sigmoid_g(float x) { return __fdividef(1.0f, 1.0f + __expf(-x)); }

// NCH: accumulator column chunks of 16 compiled in (N <= 16 NCH); the small-N instance keeps two CTAs per SM
template <int EPI, int NCH>
__global__ void __launch_bounds__(GB_NT, (EPI == EPI_SOFTMAX || NCH > 4) ? 1 : 2) k_gemm_blocks(const GbParams p) {
  constexpr bool SPATT = EPI == EPI_SOFTMAX;         // spatial attention: generated A operand + row-softmax epilogue
  extern __shared__ __align__(1024) unsigned char smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int N = p.N;
  const int b_bytes = N * 128;                       // one K-block of B (hi or lo)
  const int stage_bytes = 2 * GB_A_BYTES + 2 * b_bytes;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 2 * stage_bytes);   // [2,3] B tile of a stage landed (TMA)
  float* red = reinterpret_cast<float*>(bars + 6);     // [2][128] epilogue exchange (EPI_SOFTMAX)

  if (tid == 0) {
    for (int i = 0; i < 4; ++i) mbar_init(&bars[i], 1);
    fence_mbar_init();
  }
  __syncthreads();
  // warpgroup g owns rows [64 g, 64 g + 64) of the tile and all N columns, as N / 16 accumulators of m64n16
  const int wg = warp >> 2, wt = tid & 127;
  float acc[NCH][8];
  // row tiles: plain GEMMs tile M; spatial attention tiles every batch element separately (ceil(Nn/128) tiles each), so all rows of
  // a tile share their batch index (warp-uniform LHS addresses, no divergence at batch boundaries)
  const int sp_tiles = SPATT ? (p.Nn + GB_BM - 1) / GB_BM : 1;
  const int sp_bt = SPATT ? (int)(blockIdx.x / sp_tiles) : 0;                       // batch element of this tile
  const int sp_j0 = SPATT ? (int)(blockIdx.x % sp_tiles) * GB_BM : 0;              // first node of this tile
  const long long m0 = SPATT ? (long long)sp_bt * p.Nn + sp_j0 : (long long)blockIdx.x * GB_BM;
  const int rows_here = SPATT ? min(GB_BM, p.Nn - sp_j0) : (int)min((long long)GB_BM, (long long)p.M - m0);
  const int nkb = p.nblk, Kpad = p.nblk * 64;

  // MODE_SPATT register tile: thread = 4 consecutive rows (b, j..j+3) x 8 k of every k-block.  RHS columns of my rows live in
  // registers for the whole tile; LHS rows are warp-uniform addresses (a warp shares k and the tile shares b): broadcast 16-byte loads.
  float rj[4][12];
  int sp_j[4];
  const int sp_r0 = (tid & 31) * 4, sp_k8 = (tid >> 5) * 8;
  if (SPATT) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int jr = sp_j0 + sp_r0 + r;
      sp_j[r] = jr < p.Nn ? jr : p.Nn - 1;
#pragma unroll
      for (int t = 0; t < 12; ++t) rj[r][t] = t < p.Tn ? __ldg(p.rhs + ((long long)sp_bt * p.Tn + t) * p.Nn + sp_j[r]) : 0.f;
    }
  }

  // my 8 (row, 16-byte column) slots of an A tile are the same for every k-block: position of each row inside its sequence once
  // (one 64-bit modulo per slot per CTA instead of one per slot per k-block: it was 22 % of the issued instructions)
  float4 av[SPATT ? 1 : 8];
  int tseq[SPATT ? 1 : 8];
  if (!SPATT) {
#pragma unroll
    for (int jj = 0; jj < (SPATT ? 1 : 8); ++jj) {
      const int r = (tid + jj * GB_NT) >> 4;
      tseq[jj] = r < rows_here ? (int)((m0 + r) % p.seq) : -(1 << 20);      // rows past the end never fall inside a sequence
    }
  }
  auto load_a = [&](int kb, float4 (&v)[SPATT ? 1 : 8]) {
    if (SPATT) return;
    const KBlock blk = p.blk[kb];
    const bool vec = (blk.width % 4 == 0) && (blk.ld % 4 == 0) && ((reinterpret_cast<uintptr_t>(blk.ptr) & 15) == 0);
    const float* base = blk.ptr + (m0 + blk.shift) * blk.ld;
#pragma unroll
    for (int jj = 0; jj < (SPATT ? 1 : 8); ++jj) {
      const int idx = tid + jj * GB_NT;
      const int r = idx >> 4, k = 4 * (idx & 15);
      v[jj] = make_float4(0.f, 0.f, 0.f, 0.f);
      const int tt = tseq[jj] + blk.shift;
      if (k < blk.width && tt >= 0 && tt < p.seq) {
        const float* src = base + (long long)r * blk.ld + k;
        if (vec) {
          v[jj] = __ldg(reinterpret_cast<const float4*>(src));
        } else {
          v[jj].x = __ldg(src);
          if (k + 1 < blk.width) v[jj].y = __ldg(src + 1);
          if (k + 2 < blk.width) v[jj].z = __ldg(src + 2);
          if (k + 3 < blk.width) v[jj].w = __ldg(src + 3);
        }
      }
    }
  };

  for (int kb = 0; kb < nkb; ++kb) {
    const int s = kb & 1;
    unsigned char* a_hi = smem + s * stage_bytes;
    unsigned char* a_lo = a_hi + GB_A_BYTES;
    unsigned char* b_hi = a_lo + GB_A_BYTES;
    unsigned char* b_lo = b_hi + b_bytes;
    if (kb >= 2) {  // the MMAs of k-block kb-2 (both warpgroups) must have drained this stage; those of kb-1 keep running
      wgmma_wait<1>();
      __syncthreads();
    }
    const int k0 = kb * 64;
    if (p.w_img && tid == 0) {
      mbar_arrive_expect_tx(&bars[2 + s], 2u * (uint32_t)b_bytes);
      tma_bulk_g2s(b_hi, p.w_img + (size_t)kb * 2 * b_bytes, 2u * (uint32_t)b_bytes, &bars[2 + s]);
    }
    if (!SPATT) {
      // A: 128 x 64 fp32 of block kb (row-shifted, zero outside the sequence / beyond `width`) -> hi/lo fp16, swizzled.  The loads of
      // block kb+1 are issued (into registers) before this block's barrier and MMAs, so a k-block does not cost a full HBM round trip.
      if (kb == 0) load_a(0, av);
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int idx = tid + jj * GB_NT;
        store_split4(a_hi, a_lo, idx >> 4, 4 * (idx & 15), av[jj]);
      }
      if (kb + 1 < nkb) load_a(kb + 1, av);
    } else {
      // A generated: A[(b,j)][k] = sigmoid(sum_t LHS[b,k,t] RHS[b,t,j] + bsT[j][k]).  The 32 bs values of the thread are requested
      // first so that their (row-strided, uncoalesced) loads are in flight under the FMA loops.
      const int Tn = p.Tn;
      float o[4][8];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const float* bsr = p.bsT + (long long)sp_j[r] * p.Nn + k0 + sp_k8;
#pragma unroll
        for (int e = 0; e < 8; ++e) o[r][e] = (k0 + sp_k8 + e < p.Nn) ? __ldg(bsr + e) : 0.f;
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const int k = k0 + sp_k8 + e;
        float l[12];
#pragma unroll
        for (int t = 0; t < 12; ++t) l[t] = 0.f;
        if (k < p.Nn) {
          const float* lk = p.lhs + ((long long)sp_bt * p.Nn + k) * Tn;
          if (Tn == 12) {                              // 48-byte rows: three 16-byte broadcast loads
#pragma unroll
            for (int q4 = 0; q4 < 3; ++q4) {
              const float4 v4 = __ldg(reinterpret_cast<const float4*>(lk) + q4);
              l[4 * q4] = v4.x; l[4 * q4 + 1] = v4.y; l[4 * q4 + 2] = v4.z; l[4 * q4 + 3] = v4.w;
            }
          } else {
#pragma unroll
            for (int t = 0; t < 12; ++t)
              if (t < Tn) l[t] = __ldg(lk + t);
          }
        }
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          float acc = o[r][e];
#pragma unroll
          for (int t = 0; t < 12; ++t) acc = fmaf(l[t], rj[r][t], acc);
          o[r][e] = acc;
        }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
#pragma unroll
        for (int e = 0; e < 8; ++e) o[r][e] = (k0 + sp_k8 + e < p.Nn) ? sigmoid_g(o[r][e]) : 0.f;
        store_split4(a_hi, a_lo, sp_r0 + r, sp_k8, make_float4(o[r][0], o[r][1], o[r][2], o[r][3]));
        store_split4(a_hi, a_lo, sp_r0 + r, sp_k8 + 4, make_float4(o[r][4], o[r][5], o[r][6], o[r][7]));
      }
    }
    // B: the k-block's tile.  With a pre-swizzled image it is ONE TMA bulk copy issued before the A tile is formed (it lands while the
    // threads load / generate A); otherwise N x 64 fp16 (already split, L2-resident) -> swizzled by hand.
    for (int base = 0; base < (p.w_img ? 0 : N * 8); base += 4 * GB_NT) {
      uint4 h[4], l[4];
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int idx = base + tid + jj * GB_NT;
        if (idx < N * 8) {
          const long long g = (long long)(idx >> 3) * Kpad + k0 + 8 * (idx & 7);
          h[jj] = __ldg(reinterpret_cast<const uint4*>(p.w_hi + g));
          l[jj] = __ldg(reinterpret_cast<const uint4*>(p.w_lo + g));
        }
      }
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int idx = base + tid + jj * GB_NT;
        if (idx < N * 8) {
          const int n = idx >> 3, c = idx & 7;
          const int off = n * 128 + ((c ^ (n & 7)) << 4);
          *reinterpret_cast<uint4*>(b_hi + off) = h[jj];
          *reinterpret_cast<uint4*>(b_lo + off) = l[jj];
        }
      }
    }
    fence_proxy_async();        // generic-proxy operand stores -> visible to the tensor core (async proxy)
    __syncthreads();
    if (p.w_img) mbar_wait(&bars[2 + s], (uint32_t)(kb >> 1) & 1u);
    const uint32_t ah = smem_u32(a_hi) + wg * 64 * 128, al = smem_u32(a_lo) + wg * 64 * 128, bh = smem_u32(b_hi), bl = smem_u32(b_lo);
    wgmma_fence();
#pragma unroll
    for (int pass = 0; pass < 3; ++pass) {          // lo*hi, hi*lo, hi*hi
      const uint32_t ab = pass == 0 ? al : ah, bb = pass == 1 ? bl : bh;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
        for (int c = 0; c < NCH; ++c)
          if (16 * c < N)
            wgmma_f16_n16(acc[c], gmma_desc_sw128(ab + ks * 32), gmma_desc_sw128(bb + c * 16 * 128 + ks * 32), (kb | pass | ks) ? 1u : 0u);
      }
    }
    wgmma_commit();
  }
  wgmma_wait<0>();
#pragma unroll
  for (int c = 0; c < NCH; ++c) acc_fence(acc[c]);
  // the accumulators go to a row-major fp32 tile over the (now idle) operand stages, so that the epilogue walks rows
  __syncthreads();              // the other warpgroup's MMAs have read the stages too
  float* ct = reinterpret_cast<float*>(smem);
  const int cp = N + 8;         // row pitch (floats): the fragment's 8-row float2 stores hit 2 bank wavefronts per warp
#pragma unroll
  for (int c = 0; c < NCH; ++c)
    if (16 * c < N) acc_store(ct, cp, 64 * wg, 16 * c, wt, acc[c]);
  __syncthreads();

  // ---- epilogue: thread == row ---------------------------------------------------------------------------------------------
  const int q = warp & 3, half = warp >> 2;
  const int trow = q * 32 + lane;
  const long long row = m0 + trow;
  const bool live = trow < rows_here;
  if (EPI == EPI_BIAS || EPI == EPI_RELU) {
    // warps 0-3 / 4-7 split the 16-column chunks
    const int nchunk = N / 16;
    for (int ch = half; ch < nchunk; ch += 2) {
      const int c0 = ch * 16;
      uint32_t v[16];
      acc_ld<16>(ct, cp, trow, c0, v);
      if (live) {
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const int c = c0 + jj;
          if (c < p.ncols) {
            float o = __uint_as_float(v[jj]) + (p.bias ? __ldg(p.bias + c) : 0.f);
            if (EPI == EPI_RELU) o = fmaxf(o, 0.f);
            v[jj] = __float_as_uint(o);
          }
        }
        float* dst = p.C + row * p.ldc + c0;
        if (c0 + 16 <= p.ncols && (p.ldc % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0)) {
#pragma unroll
          for (int jj = 0; jj < 4; ++jj)
            *reinterpret_cast<float4*>(dst + 4 * jj) = make_float4(__uint_as_float(v[4 * jj]), __uint_as_float(v[4 * jj + 1]),
                                                                   __uint_as_float(v[4 * jj + 2]), __uint_as_float(v[4 * jj + 3]));
        } else {
#pragma unroll
          for (int jj = 0; jj < 16; ++jj)
            if (c0 + jj < p.ncols) dst[jj] = __uint_as_float(v[jj]);
        }
      }
    }
  } else if (EPI == EPI_RELU_LN) {
    // y = LayerNorm(relu(acc + bias)) over the row's 64 columns (torch: biased variance, eps inside the sqrt); warps 0-3 own the rows
    if (half == 0) {
      // pass 1: mean and (two-pass) variance from the staged accumulator tile; pass 2: normalise and store -- 16 values live at a time, so the
      // kernel fits two CTAs per SM
      float mean = 0.f;
#pragma unroll
      for (int ch = 0; ch < 4; ++ch) {
        uint32_t v[16];
        acc_ld<16>(ct, cp, trow, 16 * ch, v);
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) mean += fmaxf(__uint_as_float(v[jj]) + (p.bias ? __ldg(p.bias + 16 * ch + jj) : 0.f), 0.f);
      }
      mean *= (1.0f / 64.0f);
      float var = 0.f;
#pragma unroll
      for (int ch = 0; ch < 4; ++ch) {
        uint32_t v[16];
        acc_ld<16>(ct, cp, trow, 16 * ch, v);
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const float d = fmaxf(__uint_as_float(v[jj]) + (p.bias ? __ldg(p.bias + 16 * ch + jj) : 0.f), 0.f) - mean;
          var = fmaf(d, d, var);
        }
      }
      const float rstd = rsqrtf(var * (1.0f / 64.0f) + p.eps);
#pragma unroll
      for (int ch = 0; ch < 4; ++ch) {
        uint32_t v[16];
        acc_ld<16>(ct, cp, trow, 16 * ch, v);
        if (live) {
          float* dst = p.C + row * p.ldc + 16 * ch;
#pragma unroll
          for (int c = 0; c < 16; c += 4) {
            float o[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int cc = 16 * ch + c + e;
              const float xv = fmaxf(__uint_as_float(v[c + e]) + (p.bias ? __ldg(p.bias + cc) : 0.f), 0.f);
              o[e] = (xv - mean) * rstd * __ldg(p.gamma + cc) + __ldg(p.beta + cc);
            }
            *reinterpret_cast<float4*>(dst + c) = make_float4(o[0], o[1], o[2], o[3]);
          }
        }
      }
    }
  } else {
    // softmax over the first ncols columns of the row (= softmax over dim 1 of S for the transposed product); the two warp halves
    // take alternate 16-column chunks and exchange their partial max / sum through shared memory
    const int nchunk = N / 16, r128 = q * 32 + lane;
    float mx = -INFINITY;
    for (int ch = half; ch < nchunk; ch += 2) {
      uint32_t v[16];
      acc_ld<16>(ct, cp, trow, 16 * ch, v);
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
        if (16 * ch + jj < p.ncols) mx = fmaxf(mx, __uint_as_float(v[jj]));
    }
    red[half * 128 + r128] = mx;
    __syncthreads();
    mx = fmaxf(red[r128], red[128 + r128]);
    __syncthreads();
    float sum = 0.f;
    for (int ch = half; ch < nchunk; ch += 2) {
      uint32_t v[16];
      acc_ld<16>(ct, cp, trow, 16 * ch, v);
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
        if (16 * ch + jj < p.ncols) sum += __expf(__uint_as_float(v[jj]) - mx);
    }
    red[half * 128 + r128] = sum;
    __syncthreads();
    const float inv = 1.0f / (red[r128] + red[128 + r128]);
    for (int ch = half; ch < nchunk; ch += 2) {
      uint32_t v[16];
      acc_ld<16>(ct, cp, trow, 16 * ch, v);
      if (live) {
        float* dst = p.C + row * p.ldc + 16 * ch;      // ldc % 4 == 0, C 16-byte aligned (checked on the host)
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          float o[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) o[e] = (16 * ch + 4 * jj + e < p.ncols) ? __expf(__uint_as_float(v[4 * jj + e]) - mx) * inv : 0.f;
          if (16 * ch + 4 * jj < p.ldc) *reinterpret_cast<float4*>(dst + 4 * jj) = make_float4(o[0], o[1], o[2], o[3]);
        }
      }
    }
  }
}

// packed [N][Kpad] hi | lo  ->  per k-block [hi tile | lo tile], each N x 128 B in the SWIZZLE_128B layout of the kernel's B stage
__global__ void k_gb_weight_image(const __half* __restrict__ hi, const __half* __restrict__ lo, int N, int nblk, unsigned char* __restrict__ img) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;     // one 16-byte chunk
  const long long per = (long long)N * 8;
  if (idx >= per * nblk * 2) return;
  const int kb = (int)(idx / (2 * per));
  const long long rem = idx - (long long)kb * 2 * per;
  const int half = (int)(rem / per);
  const int r = (int)(rem - half * per);
  const int n = r >> 3, c = r & 7;
  const __half* src = (half ? lo : hi) + (long long)n * nblk * 64 + kb * 64 + 8 * c;
  const uint4 v = *reinterpret_cast<const uint4*>(src);
  *reinterpret_cast<uint4*>(img + ((size_t)kb * 2 + half) * N * 128 + n * 128 + ((c ^ (n & 7)) << 4)) = v;
}

template <int EPI, int NCH>
int gb_launch_n(GbParams& p, cudaStream_t st) {
  const int smem = 2 * (2 * GB_A_BYTES + 2 * p.N * 128) + 48 + 256 * 4;
  if (smem > 232448) return set_error(STMP_EUNSUPPORTED, "blocked GEMM: N=%d needs %d B of shared memory", p.N, smem);
  STMP_CUDA_OK(cudaFuncSetAttribute(k_gemm_blocks<EPI, NCH>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const unsigned grid = EPI == EPI_SOFTMAX ? (unsigned)((p.M / p.Nn) * ((p.Nn + GB_BM - 1) / GB_BM)) : (unsigned)((p.M + GB_BM - 1) / GB_BM);
  k_gemm_blocks<EPI, NCH><<<grid, GB_NT, smem, st>>>(p);
  STMP_LAUNCH_OK("k_gemm_blocks");
  return STMP_OK;
}
template <int EPI>
int gb_launch(GbParams& p, cudaStream_t st) {
  // the accumulator registers are compiled in per instance: the smallest one that holds N
  if (EPI != EPI_SOFTMAX && p.N <= 64) return gb_launch_n<EPI, 4>(p, st);   // the block GEMMs of ASTGCN (N = 64), two CTAs per SM
  if (p.N <= 128) return gb_launch_n<EPI, 8>(p, st);
  return gb_launch_n<EPI, GB_MAXN / 16>(p, st);
}

int gb_dispatch(GbParams& p, int epi, cudaStream_t st) {
  switch (epi) {
    case EPI_BIAS: return gb_launch<EPI_BIAS>(p, st);
    case EPI_RELU: return gb_launch<EPI_RELU>(p, st);
    case EPI_RELU_LN: return gb_launch<EPI_RELU_LN>(p, st);
    case EPI_SOFTMAX: return gb_launch<EPI_SOFTMAX>(p, st);
  }
  return set_error(STMP_EINVAL, "blocked GEMM: unknown epilogue %d", epi);
}

}  // namespace
}  // namespace stmp

using namespace stmp;

extern "C" int stmp_gemm_blocks_f32(int64_t M, int64_t N, int64_t ncols, int64_t nblk, const float* const* blk_ptr, const int64_t* blk_ld,
                                    const int32_t* blk_width, const int32_t* blk_shift, int64_t seq, const void* packed, const void* image,
                                    const float* bias, int epilogue, const float* gamma, const float* beta, float eps, float* C, int64_t ldc, void* stream) {
  STMP_REQUIRE(blk_ptr && blk_ld && blk_width && blk_shift && packed, STMP_EINVAL, "stmp_gemm_blocks_f32: NULL pointer");
  STMP_REQUIRE(M >= 0 && nblk >= 1 && seq >= 1, STMP_EINVAL, "stmp_gemm_blocks_f32: bad sizes");
  if (nblk > GB_MAXBLK || N > 320 || N % 16 != 0 || N < 16 || ncols > N || ncols < 1 || M >= (1ll << 31) - 128)
    return set_error(STMP_EUNSUPPORTED, "blocked GEMM takes <= %d k-blocks, N <= 320, N %% 16 == 0 (nblk=%lld N=%lld)", GB_MAXBLK,
                     (long long)nblk, (long long)N);
  if (epilogue == EPI_RELU_LN && (N != 64 || ncols != 64 || !gamma || !beta || ldc % 4 != 0 || (reinterpret_cast<uintptr_t>(C) & 15)))
    return set_error(STMP_EUNSUPPORTED, "blocked GEMM: the LayerNorm epilogue needs N == 64, gamma/beta and 16-byte aligned rows");
  if (epilogue == EPI_SOFTMAX) return set_error(STMP_EINVAL, "blocked GEMM: the softmax epilogue belongs to stmp_spatial_attention_fwd");
  if (M == 0) return STMP_OK;
  STMP_REQUIRE(C != nullptr, STMP_EINVAL, "stmp_gemm_blocks_f32: NULL pointer");
  GbParams p = {};
  for (int i = 0; i < nblk; ++i) {
    STMP_REQUIRE(blk_ptr[i] != nullptr && blk_width[i] >= 1 && blk_width[i] <= 64, STMP_EINVAL, "stmp_gemm_blocks_f32: bad block %d", i);
    p.blk[i].ptr = blk_ptr[i]; p.blk[i].ld = blk_ld[i]; p.blk[i].width = blk_width[i]; p.blk[i].shift = blk_shift[i];
  }
  p.nblk = (int)nblk; p.M = (int)M; p.N = (int)N; p.seq = (int)seq; p.ncols = (int)ncols;
  p.w_hi = reinterpret_cast<const __half*>(packed); p.w_lo = p.w_hi + N * nblk * 64;
  p.w_img = reinterpret_cast<const unsigned char*>(image);
  p.bias = bias; p.C = C; p.ldc = ldc; p.gamma = gamma; p.beta = beta; p.eps = eps;
  return gb_dispatch(p, epilogue, (cudaStream_t)stream);
}

extern "C" int64_t stmp_gemm_blocks_image_bytes(int64_t N, int64_t nblk) { return nblk * 2 * N * 128; }

extern "C" int stmp_gemm_blocks_image(const void* packed, int64_t N, int64_t nblk, void* image, void* stream) {
  STMP_REQUIRE(packed && image && N > 0 && nblk > 0, STMP_EINVAL, "stmp_gemm_blocks_image: bad argument");
  const __half* hi = reinterpret_cast<const __half*>(packed);
  const long long total = (long long)N * 8 * nblk * 2;
  k_gb_weight_image<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(hi, hi + N * nblk * 64, (int)N, (int)nblk,
                                                                                      reinterpret_cast<unsigned char*>(image));
  STMP_LAUNCH_OK("k_gb_weight_image");
  return STMP_OK;
}

extern "C" int stmp_spatial_attention_fwd(int64_t B, int64_t n_nodes, int64_t n_steps, const float* lhs, const float* rhs, const float* bsT,
                                          const void* vsT_packed, const void* vsT_image, float* st_out, int64_t ld_out, void* stream) {
  STMP_REQUIRE(B >= 0 && n_nodes >= 1 && n_steps >= 1, STMP_EINVAL, "stmp_spatial_attention_fwd: bad sizes");
  const int64_t Npad = (n_nodes + 63) / 64 * 64;
  if (Npad > 320 || n_steps > 12 || ld_out < Npad || ld_out % 4 != 0 || (reinterpret_cast<uintptr_t>(st_out) & 15))
    return set_error(STMP_EUNSUPPORTED, "fused spatial attention takes <= 320 nodes, <= 12 timesteps and 16-byte aligned rows of >= %lld floats "
                                        "(nodes=%lld steps=%lld ld=%lld)", (long long)Npad, (long long)n_nodes, (long long)n_steps, (long long)ld_out);
  if (B == 0) return STMP_OK;
  STMP_REQUIRE(lhs && rhs && bsT && vsT_packed && st_out, STMP_EINVAL, "stmp_spatial_attention_fwd: NULL pointer");
  // at T == 12 the operand generator reads each 48-byte LHS row as three float4
  STMP_REQUIRE(n_steps != 12 || (reinterpret_cast<uintptr_t>(lhs) & 15) == 0, STMP_EINVAL, "stmp_spatial_attention_fwd: lhs must be 16-byte aligned");
  GbParams p = {};
  p.nblk = (int)(Npad / 64); p.M = (int)(B * n_nodes); p.N = (int)Npad; p.seq = 1; p.ncols = (int)n_nodes;
  p.w_hi = reinterpret_cast<const __half*>(vsT_packed); p.w_lo = p.w_hi + Npad * Npad;
  p.w_img = reinterpret_cast<const unsigned char*>(vsT_image);
  p.bias = nullptr; p.C = st_out; p.ldc = ld_out;
  p.spatt = 1; p.Nn = (int)n_nodes; p.Tn = (int)n_steps; p.lhs = lhs; p.rhs = rhs; p.bsT = bsT;
  return gb_dispatch(p, EPI_SOFTMAX, (cudaStream_t)stream);
}
