// graph.h -- internal definition of the opaque rgcn_graph handle (host structure + device mirrors).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/rgcn_b200.h"

// A warp work item: messages [beg,end) of ONE row (destination row, source row or weight id).
// split = -1 when the row is covered by this single item, otherwise the index of the row in the
// split-row list (rows with more than `item_max` messages are cut into several items whose partial
// sums are combined with vector reductions in L2; the last arriver applies the epilogue).
struct WorkItem {
  int32_t beg, end, row, split;
};

struct CsrSide {
  // host
  std::vector<int32_t> rowptr;  // [rows+1]
  std::vector<int32_t> nbr;     // [M] the "other end" (gather index)
  std::vector<int32_t> relw;    // [M]
  std::vector<float> norm;      // [M]
  std::vector<int32_t> mid;     // [M] original message id
  std::vector<WorkItem> items;
  std::vector<int32_t> split_nitems;  // per split row: how many items cover it
  std::vector<int32_t> split_rows;    // per split row: the row id
  // device mirrors
  int32_t* d_rowptr = nullptr;
  int32_t* d_nbr = nullptr;
  int32_t* d_relw = nullptr;
  float* d_norm = nullptr;
  int32_t* d_mid = nullptr;  // only when keep_mid
  WorkItem* d_items = nullptr;
  int32_t* d_split_nitems = nullptr;
  int32_t* d_split_rows = nullptr;
  int64_t n_items = 0, n_split = 0;  // valid for host- and device-built graphs
};

// Weight-id major view: messages sorted by (supertile(row), weight id, row) where `row` is the row
// the message ACCUMULATES into (destination for the forward / dW pass, source for the dH pass) and
// `nbr` the row it gathers.  A supertile is a contiguous range of `supertile_rows` rows: keeping the
// accumulation target of consecutive work items inside one L2-sized window lets the vector
// reductions (red.global.add.v4.f32) resolve in L2 instead of HBM read-modify-write.
struct RelSide {
  std::vector<int32_t> ptr;  // [n_super * n_relw + 1]
  std::vector<int32_t> row, nbr, mid;
  std::vector<float> norm;
  std::vector<WorkItem> items;  // row = weight id, split = supertile index
  int32_t n_super = 1;
  int32_t* d_ptr = nullptr;
  int32_t* d_row = nullptr;
  int32_t* d_nbr = nullptr;
  float* d_norm = nullptr;
  int32_t* d_mid = nullptr;  // only when keep_mid
  WorkItem* d_items = nullptr;
  int64_t n_items = 0;
};

struct rgcn_graph {
  int64_t M = 0;
  int32_t V_dst = 0, V_src = 0, n_relw = 0;
  int device = -1;
  int item_max = 128;
  int64_t n_groups = 0;       // number of (dst, relw) runs in destination-major order
  int64_t device_bytes = 0;
  std::vector<float> msg_norm;  // [M] original order
  CsrSide by_dst;               // rows = destinations, nbr = source
  CsrSide by_src;               // rows = sources,      nbr = destination
  RelSide by_rel;               // weight-id major, row = dst, nbr = src  (forward, dW)
  RelSide by_rel_src;           // weight-id major, row = src, nbr = dst  (backward w.r.t. H)
  int supertile_rows = 8192;
  bool supertile_fixed = false;  // $RGCN_SUPERTILE_ROWS given: every view uses exactly supertile_rows
  bool built_on_device = false;  // structures were built by graph_device.cu (host vectors empty)
  bool keep_mid = true;          // keep message-id permutations / original-order norm for export
  bool has_csr = true;           // by_dst / by_src built (deterministic block mode, basis layers)
  bool has_rel = true;           // by_rel / by_rel_src built (weight-id-major block kernels)
  float* d_msg_norm = nullptr;
};

// Rows per supertile of ONE weight-id-major view.  The default (8192 rows = a 16 MB accumulation window at d = 512)
// suits views with >= ~48 messages per (supertile, weight id) work item.  A sparse view -- the halo-source view of a
// node shard at 8 GPUs: 22 M messages over 8 M halo rows x 2000 weight ids = 11 per item -- spends its time loading
// the item's 16 KB of block weights; there the supertiles grow (x2 steps, at most 16384 rows = a 32 MB window, which
// still fits the 50 MB L2 next to the evict-first gather stream) until the items are long enough.  Not measured on H100.  Host and device builders
// share this rule (bit-identical views).
inline int view_supertile_rows(const rgcn_graph* g, int32_t n_rows, int64_t M) {
  int rows = g->supertile_rows;
  if (g->supertile_fixed || rows <= 0) return rows;
  while (rows < 16384) {
    const int64_t n_super = ((int64_t)n_rows + rows - 1) / rows;
    const int64_t items = (n_super > 0 ? n_super : 1) * (int64_t)(g->n_relw > 0 ? g->n_relw : 1);
    if (M >= 48 * items) break;   // >= 48 messages per (supertile, weight id) on average
    rows *= 2;
  }
  return rows;
}

// graph_device.cu
int rgcn_build_on_device(rgcn_graph* g, const int32_t* d_dst, const int32_t* d_src,
                         const int32_t* d_relw, const float* d_norm, cudaStream_t st);
int rgcn_build_on_device_checked(rgcn_graph* g, const int32_t* d_dst, const int32_t* d_src,
                                 const int32_t* d_relw, const float* d_norm, const int* d_bad,
                                 cudaStream_t st, float* d_run_norm);
int rgcn_build_from_triples_device(rgcn_graph* g, const int32_t* d_triples, int64_t E, int32_t V,
                                   int32_t R, int norm_mode, const float* d_norm_f,
                                   const float* d_norm_b, cudaStream_t st);
int rgcn_check_messages_device(const int32_t* d_dst, const int32_t* d_src, const int32_t* d_relw,
                               int64_t M, int32_t V_dst, int32_t V_src, int32_t n_relw,
                               cudaStream_t st);

extern int g_graph_views;  // graph.cu
void rgcn_set_error(const std::string& s);
int rgcn_check_cuda(cudaError_t e, const char* what);
