// graph_image.cuh -- the shared-memory image of a plan's operators that the fused wgmma graph-GRU kernel gathers from
// (built once per plan by plan.cu::k_build_graph_image, fetched by every CTA with ONE TMA bulk copy).
//
// A *task* = one (destination row, operator) pair: the weighted sum of the source rows of its CSR row.  The 16 warps of
// the kernel process tasks quarter-warp-wise (8 lanes x float4 = one 128-byte feature row per load), so four tasks run
// side by side in a warp ("warp-task").  The image holds
//
//   header   16 B     {n_warp_tasks, n_groups, valid, 0}
//   wstart   [16][4]  u16  first warp-task of warp w in segment s = 2 * (MMA row tile of the destination: rows <128 | >=128) + operator
//   wcount   [16][4]  u16  number of warp-tasks of warp w in segment s
//   wt       [n_warp_tasks][4] u32 task descriptors: row | op << 8 | n_groups << 9 | first_group << 16  (0xFFFFFFFF = none)
//   idx4     [n_groups + 1]  u32: four source rows of an edge group (pad entries point at the all-zero row 207), 8-bit row numbers
//   val4     [n_groups + 1]  float4: their four values (pad = 0)
//
// Edge order inside a task is the plan's CSR order (= the reference's scatter order).  Warp-tasks are dealt to warps by
// longest-processing-time-first over ALL segments, four equally long tasks per warp-task, so that (a) the four quarter-warps
// of a warp run equal trip counts and (b) all warps finish a gather round together (round-1 profile: 25 % of all warp time
// was spent waiting at barriers because quarter-warp 0 always drew the longest task of every 64).
#pragma once
#include <stdint.h>

namespace stmp {

constexpr int kImgMaxN = 207;        // row 207 of the gather buffer is the all-zero row pad entries point at
constexpr int kImgWarps = 16;
constexpr int kImgSegs = 4;
constexpr int kImgZeroRow = 207;
constexpr uint32_t kImgNoTask = 0xFFFFFFFFu;

struct GraphImageLayout {
  int off_wstart, off_wcount, off_wt, off_idx, off_val, bytes;
  int cap_wt, cap_groups;
};

__host__ __device__ inline int gi_align16(int v) { return (v + 15) & ~15; }

// capacity layout from (number of tasks, total nnz over the operators used): fixed offsets, computed identically by the
// builder (plan.cu), the kernel's shared-memory layout (dcrnn_seq_tc.cu) and the host (bytes to copy).
__host__ __device__ inline GraphImageLayout graph_image_layout(int n_tasks, int nnz) {
  GraphImageLayout L;
  L.cap_wt = (n_tasks + 3) / 4 + kImgSegs;              // at most one partial warp-task per segment
  L.cap_groups = (nnz + 3 * n_tasks) / 4 + 2;           // every task pads to a multiple of 4 edges; +1 prefetch slot
  int off = 16;
  L.off_wstart = off; off += kImgWarps * kImgSegs * 2;
  L.off_wcount = off; off += kImgWarps * kImgSegs * 2;
  off = gi_align16(off);
  L.off_wt = off; off += gi_align16(L.cap_wt * 16);
  L.off_idx = off; off += gi_align16(L.cap_groups * 4);
  L.off_val = off; off += L.cap_groups * 16;
  L.bytes = gi_align16(off);
  return L;
}

// shared memory the wgmma kernel leaves for the image (dcrnn_seq_tc.cu); a plan keeps an image only if L.bytes fits it
int tc_graph_image_budget();

}  // namespace stmp
