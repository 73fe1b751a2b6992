// row_image.cuh -- the shared-memory image of a plan's operators that the one-CTA wgmma graph-GRU kernel gathers from straight into
// wgmma register fragments (built once per plan on the host by plan.cu::build_row_image, fetched by every CTA with ONE TMA bulk copy).
//
// The kernel's 16 warps own the 256 MMA rows ("positions") of the two row tiles: position = 16 warp + 8 slot + quad, where quad =
// lane / 4 and slot = 0 / 1 are the two rows (r, r + 8) of a lane's m64nNk16 fragment.  The builder maps the graph's nodes onto the
// positions: nodes sorted by descending group count (a group = 4 CSR entries) are cut into 32 *bins* of 8 (one row of every quad of
// one (warp, slot)), and the bins are dealt longest-first to the least loaded warp with a free slot.  So the quads of a warp walk
// rows of near-equal length and the warps carry equal gather work over both operators.  A bin's list runs as long as its longest row
// per operator, so the plan sorts by operator 0's group count, then operator 1's (ROW_ORDER_BY_OPERATOR): rows of one bin then share
// both counts far more often than when sorted by their sum (ROW_ORDER_BY_TOTAL, kept for stmp_row_image_build), which mixes a
// (3, 2) row with a (2, 3) row into a bin that runs 3 + 3.
//
//   header  16 B     {n_groups, zero_pos, N, n_ops}
//   perm    [256]    i16  node at position (-1: empty)
//   ipos    [256]    u8   position of node
//   gstart  [16][2][2] u16  first group row of (warp, operator, slot)
//   gcount  [16][2][2] u16  its number of group rows (the longest quad's group count)
//   idx     [n_groups + 1][8] u32     per group row and quad: four 8-bit source positions (pad entries: zero_pos)
//   val     [n_groups + 1][8] float4  their four values (pad: 0)
//
// A row's entries keep the plan's CSR order (= the reference's scatter order).  Position zero_pos is empty: its rows of the kernel's
// gather buffers stay zero.  The last group row is a spare the gather loop prefetches past a list's end.
#pragma once
#include <stdint.h>

namespace stmp {

constexpr int kRiPos = 256;
constexpr int kRiMaxN = 255;          // one position must stay empty (the zero row)
constexpr int kRiWarps = 16;
constexpr int kRiOffPerm = 16;
constexpr int kRiOffIpos = kRiOffPerm + 2 * kRiPos;
constexpr int kRiOffGstart = kRiOffIpos + kRiPos;
constexpr int kRiOffGcount = kRiOffGstart + kRiWarps * 4 * 2;
constexpr int kRiOffIdx = kRiOffGcount + kRiWarps * 4 * 2;   // 1040: 16-byte aligned
static_assert(kRiOffIdx % 16 == 0, "row image group arrays must be 16-byte aligned");

struct RowImageLayout {
  int n_groups, off_val, bytes;
};

__host__ __device__ inline RowImageLayout row_image_layout(int n_groups) {
  RowImageLayout L;
  L.n_groups = n_groups;
  L.off_val = kRiOffIdx + (n_groups + 1) * 8 * 4;
  L.bytes = L.off_val + (n_groups + 1) * 8 * 16;
  return L;
}

// (warp, operator, slot) -> index into gstart / gcount
__host__ __device__ inline int ri_list(int warp, int op, int slot) { return (warp * 2 + op) * 2 + slot; }

enum RowOrder { ROW_ORDER_BY_TOTAL = 0, ROW_ORDER_BY_OPERATOR = 1 };

// Builds the image of n_ops (1, 2) operators given as host CSR arrays (rowptr [N+1], col / val [nnz]) into dst when capacity
// suffices, with the nodes sorted as `order` says (ties: node id).  Returns its size in bytes, or 0 for a graph the format cannot hold
// (N outside 1..255, a column outside [0, N)).
int64_t build_row_image(int N, int n_ops, const int* const rowptr[2], const int* const col[2], const float* const val[2], RowOrder order,
                        void* dst, int64_t capacity);

// shared memory the one-CTA kernel leaves for the image (dcrnn_seq_tc.cu); a plan keeps an image only if it fits
int tc_row_image_budget();

}  // namespace stmp
