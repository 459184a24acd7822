// graph_device.cu -- graph preparation ON THE GPU (the default when a device is given).
//
// Same result, bit for bit, as the host builder in graph.cu (tests compare the exported arrays):
//   messages -> per-direction 1/in-degree norm (or, RGCN_NORM_RELATION, 1/run length taken from the first
//   destination-keyed sort) -> four stable sorts (CUB LSD radix sort on a packed
//   64-bit (major, minor) key with the message id as payload; ties keep message-id order exactly
//   like the host counting sorts) -> CSR pointers (histogram + exclusive scan) -> warp work lists.
// The reference does this implicitly inside TF (extras/graph_representations.py:21-27, :84-93,
// :124-133) on every session.run; here it costs a handful of small kernels per fed edge list.
#include <cub/cub.cuh>

#include <algorithm>

#include "graph.h"
#include "kernels.cuh"

namespace {

#define DCK(x)                                       \
  do {                                               \
    int rc__ = rgcn_check_cuda((x), #x);             \
    if (rc__) return rc__;                           \
  } while (0)

int bits_for(uint64_t n) {  // bits needed to represent values in [0, n)
  int b = 1;
  while (b < 64 && (1ull << b) < n) ++b;
  return b;
}

__global__ void k_tri2msg(const int32_t* __restrict__ tri, int64_t E, int32_t R,
                          int32_t* __restrict__ dst, int32_t* __restrict__ src,
                          int32_t* __restrict__ relw, int32_t* __restrict__ cnt_f,
                          int32_t* __restrict__ cnt_b, int32_t V, int* __restrict__ bad) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < E;
       k += (int64_t)gridDim.x * blockDim.x) {
    const int32_t s = tri[3 * k], r = tri[3 * k + 1], o = tri[3 * k + 2];
    if (s < 0 || s >= V || o < 0 || o >= V || r < 0 || r >= R) {
      // flag it (checked by the host at the single synchronisation) and write memory-safe values so
      // the kernels already queued behind this one cannot index out of range
      atomicExch(bad, 1);
      dst[k] = src[k] = relw[k] = 0;
      dst[E + k] = src[E + k] = 0;
      relw[E + k] = R;
      continue;
    }
    dst[k] = o;
    src[k] = s;
    relw[k] = r;
    dst[E + k] = s;
    src[E + k] = o;
    relw[E + k] = r + R;
    atomicAdd(cnt_f + o, 1);
    atomicAdd(cnt_b + s, 1);
  }
}

__global__ void k_norm_canonical(const int32_t* __restrict__ dst, int64_t E,
                                 const int32_t* __restrict__ cnt_f,
                                 const int32_t* __restrict__ cnt_b, float* __restrict__ norm) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < E;
       k += (int64_t)gridDim.x * blockDim.x) {
    norm[k] = 1.0f / (float)cnt_f[dst[k]];
    norm[E + k] = 1.0f / (float)cnt_b[dst[E + k]];
  }
}

__global__ void k_fill(float* p, int64_t n, float v) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    p[i] = v;
}

__global__ void k_check_messages(const int32_t* dst, const int32_t* src, const int32_t* relw,
                                 int64_t M, int32_t V_dst, int32_t V_src, int32_t n_relw, int* bad) {
  for (int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; m < M;
       m += (int64_t)gridDim.x * blockDim.x)
    if (dst[m] < 0 || dst[m] >= V_dst || src[m] < 0 || src[m] >= V_src || relw[m] < 0 ||
        relw[m] >= n_relw)
      atomicExch(bad, 1);
}

// key = major * n_minor + minor ; value = message id ; also histogram of the major key
// mode 0: major = row,                       minor = relw            (CSR views)
// mode 1: major = (row / st_rows) * n_relw + relw, minor = row      (weight-id major views)
__global__ void k_make_keys(const int32_t* __restrict__ row, const int32_t* __restrict__ relw,
                            int64_t M, int mode, int32_t n_relw, int32_t st_rows, uint64_t n_minor,
                            uint64_t* __restrict__ keys, int32_t* __restrict__ vals,
                            int32_t* __restrict__ major_cnt) {
  for (int64_t m = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; m < M;
       m += (int64_t)gridDim.x * blockDim.x) {
    uint64_t major, minor;
    if (mode == 0) {
      major = (uint64_t)row[m];
      minor = (uint64_t)relw[m];
    } else {
      major = (uint64_t)(row[m] / st_rows) * n_relw + relw[m];
      minor = (uint64_t)row[m];
    }
    keys[m] = major * n_minor + minor;
    vals[m] = (int32_t)m;
    atomicAdd(major_cnt + major, 1);
  }
}

__global__ void k_gather3(const int32_t* __restrict__ perm, int64_t M, const int32_t* __restrict__ a,
                          const int32_t* __restrict__ b, const float* __restrict__ c,
                          int32_t* __restrict__ oa, int32_t* __restrict__ ob, float* __restrict__ oc) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t m = perm[i];
    oa[i] = a[m];
    ob[i] = b[m];
    oc[i] = c[m];
  }
}

// per-row item counts for the CSR views (same arithmetic as build_items() in graph.cu)
__global__ void k_csr_item_counts(const int32_t* __restrict__ rowptr, int32_t rows, int item_max,
                                  int32_t* __restrict__ nitems, int32_t* __restrict__ issplit) {
  for (int32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    const int32_t deg = rowptr[r + 1] - rowptr[r];
    int32_t n = 1, sp = 0;
    if (deg > item_max) {
      const int32_t n0 = (deg + item_max - 1) / item_max;
      const int32_t chunk = (deg + n0 - 1) / n0;
      n = (deg + chunk - 1) / chunk;
      sp = 1;
    }
    nitems[r] = n;
    issplit[r] = sp;
  }
}

__global__ void k_csr_fill_items(const int32_t* __restrict__ rowptr, int32_t rows, int item_max,
                                 const int32_t* __restrict__ item_off,
                                 const int32_t* __restrict__ split_off, WorkItem* __restrict__ items,
                                 int32_t* __restrict__ split_nitems, int32_t* __restrict__ split_rows) {
  for (int32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    const int32_t beg = rowptr[r], end = rowptr[r + 1], deg = end - beg;
    const int32_t o = item_off[r];
    if (deg <= item_max) {
      items[o] = WorkItem{beg, end, r, -1};
    } else {
      const int32_t n0 = (deg + item_max - 1) / item_max;
      const int32_t chunk = (deg + n0 - 1) / n0;
      const int32_t sidx = split_off[r];
      int32_t made = 0;
      for (int32_t b = beg; b < end; b += chunk, ++made)
        items[o + made] = WorkItem{b, min(end, b + chunk), r, sidx};
      split_nitems[sidx] = made;
      split_rows[sidx] = r;
    }
  }
}

__global__ void k_rel_item_counts(const int32_t* __restrict__ ptr, int32_t nkeys, int item_max,
                                  int32_t* __restrict__ nitems) {
  for (int32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < nkeys; k += gridDim.x * blockDim.x)
    nitems[k] = (ptr[k + 1] - ptr[k] + item_max - 1) / item_max;
}

__global__ void k_rel_fill_items(const int32_t* __restrict__ ptr, int32_t nkeys, int item_max,
                                 int32_t n_relw, const int32_t* __restrict__ item_off,
                                 WorkItem* __restrict__ items) {
  for (int32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < nkeys; k += gridDim.x * blockDim.x) {
    const int32_t beg = ptr[k], end = ptr[k + 1];
    int32_t o = item_off[k];
    for (int32_t b = beg; b < end; b += item_max, ++o)
      items[o] = WorkItem{b, min(end, b + item_max), k % n_relw, k / n_relw};
  }
}

__global__ void k_count_runs(const uint64_t* __restrict__ keys, int64_t M,
                             unsigned long long* __restrict__ out) {
  unsigned long long local = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M;
       i += (int64_t)gridDim.x * blockDim.x)
    local += (i == 0 || keys[i] != keys[i - 1]) ? 1ull : 0ull;
  for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
  if ((threadIdx.x & 31) == 0 && local) atomicAdd(out, local);
}

// RGCN_NORM_RELATION: a (dst, weight id) group is one run of equal keys in the sorted keys of a destination-keyed view
// (by_dst: dst * n_relw + relw; by_rel: ((dst / st_rows) * n_relw + relw) * V + dst).  Each sorted position finds
// the ends of its run by a galloping search from itself (a run of L messages costs O(log L) probes per message,
// neighbouring threads probe the same lines) and scatters 1/L to its message through the sort permutation.  No
// temporaries; the result is an integer count converted exactly like the host builder's.
__device__ __forceinline__ int64_t run_edge(const uint64_t* __restrict__ keys, int64_t M, int64_t i, int64_t dir) {
  const uint64_t k = keys[i];
  int64_t in = i, out = i, step = 1;  // keys[in] == k; `out` becomes the first probe past the run (or -1 / M)
  for (;;) {
    out = in + dir * step;
    if (out < 0 || out >= M || keys[out] != k) break;
    in = out;
    step <<= 1;
  }
  if (out < 0) out = -1;
  if (out > M) out = M;
  while (out - in > 1 || in - out > 1) {
    const int64_t mid = in + (out - in) / 2;
    if (keys[mid] == k) in = mid; else out = mid;
  }
  return in;  // last position of the run in direction `dir`
}

__global__ void k_norm_relation(const uint64_t* __restrict__ keys, const int32_t* __restrict__ perm, int64_t M,
                                float* __restrict__ norm) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < M;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t len = run_edge(keys, M, i, 1) - run_edge(keys, M, i, -1) + 1;
    norm[perm[i]] = 1.0f / (float)len;
  }
}

int grid_for(int64_t n) {
  int64_t b = (n + 255) / 256;
  if (b > 132 * 8) b = 132 * 8;
  if (b < 1) b = 1;
  return (int)b;
}

template <typename T>
int dalloc(T** p, int64_t count, cudaStream_t st, int64_t* bytes = nullptr) {
  size_t n = (size_t)std::max<int64_t>(count, 1) * sizeof(T);
  if (bytes) *bytes += (int64_t)n;
  return rgcn_check_cuda(cudaMallocAsync((void**)p, n, st), "cudaMallocAsync(graph)");
}

struct Scratch {  // temporaries of one view build, freed (stream-ordered) at the end
  cudaStream_t st;
  std::vector<void*> ptrs;
  explicit Scratch(cudaStream_t s) : st(s) {}
  template <typename T>
  int get(T** p, int64_t count) {
    int rc = dalloc(p, count, st);
    if (!rc) ptrs.push_back(*p);
    return rc;
  }
  ~Scratch() {
    for (void* p : ptrs) cudaFreeAsync(p, st);
  }
};

// Sort message ids by the packed key; returns perm (device), sorted keys (device) and the exclusive
// scan of the major-key histogram (ptr, n_major + 1 entries).
int sort_view(Scratch& sc, const int32_t* row, const int32_t* relw, int64_t M, int mode,
              int32_t n_relw, int32_t st_rows, uint64_t n_major, uint64_t n_minor, int32_t** perm_out,
              uint64_t** keys_out, int32_t* ptr_out /* persistent, n_major+1 */, cudaStream_t st) {
  uint64_t *keys_a, *keys_b;
  int32_t *vals_a, *vals_b, *cnt;
  int rc;
  if ((rc = sc.get(&keys_a, M))) return rc;
  if ((rc = sc.get(&keys_b, M))) return rc;
  if ((rc = sc.get(&vals_a, M))) return rc;
  if ((rc = sc.get(&vals_b, M))) return rc;
  if ((rc = sc.get(&cnt, (int64_t)n_major + 1))) return rc;
  DCK(cudaMemsetAsync(cnt, 0, (n_major + 1) * sizeof(int32_t), st));
  if (M > 0) {
    k_make_keys<<<grid_for(M), 256, 0, st>>>(row, relw, M, mode, n_relw, st_rows, n_minor, keys_a,
                                             vals_a, cnt);
    ++g_rgcn_launches;
    const int end_bit = bits_for(n_major * n_minor);
    size_t tb = 0;
    DCK(cub::DeviceRadixSort::SortPairs(nullptr, tb, keys_a, keys_b, vals_a, vals_b, (int)M, 0,
                                        end_bit, st));
    void* tmp;
    if ((rc = sc.get((char**)&tmp, (int64_t)tb))) return rc;
    DCK(cub::DeviceRadixSort::SortPairs(tmp, tb, keys_a, keys_b, vals_a, vals_b, (int)M, 0, end_bit,
                                        st));
  }
  {
    size_t tb = 0;
    DCK(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt, ptr_out, (int)(n_major + 1), st));
    void* tmp;
    if ((rc = sc.get((char**)&tmp, (int64_t)tb))) return rc;
    DCK(cub::DeviceScan::ExclusiveSum(tmp, tb, cnt, ptr_out, (int)(n_major + 1), st));
  }
  *perm_out = vals_b;
  *keys_out = keys_b;
  return RGCN_OK;
}

int scan_i32(Scratch& sc, const int32_t* in, int32_t* out, int64_t n, cudaStream_t st) {
  size_t tb = 0;
  DCK(cub::DeviceScan::ExclusiveSum(nullptr, tb, in, out, (int)n, st));
  void* tmp;
  int rc = sc.get((char**)&tmp, (int64_t)tb);
  if (rc) return rc;
  DCK(cub::DeviceScan::ExclusiveSum(tmp, tb, in, out, (int)n, st));
  return RGCN_OK;
}

// Each view is built in two phases so the whole preparation needs ONE host synchronisation:
//   phase A (all asynchronous): sort, gather, CSR pointer, per-row item counts + exclusive scans, the
//                               totals copied into a pinned host slot;
//   -- one cudaStreamSynchronize for all four views --
//   phase B: allocate the work-item arrays (sizes now known on the host) and fill them.
struct ViewTmp {
  Scratch sc;  // survives until phase B: only the item / split offsets (4 B per row or key)
  int32_t* item_off = nullptr;
  int32_t* split_off = nullptr;
  int32_t n_keys = 0;
  explicit ViewTmp(cudaStream_t st) : sc(st) {}
};
// The sort temporaries (two 64-bit key arrays, two id arrays, the radix-sort workspace: 28 B per message) live
// in a phase-local Scratch and return to the stream-ordered pool before the next view is built, so a
// 200 M-message graph peaks at one view's temporaries instead of four.

// run_norm (RGCN_NORM_RELATION, destination-keyed view built first): the message-order `norm` buffer, filled here from
// the sorted keys before this view -- and every later one -- gathers it
int csr_phase_a(rgcn_graph* g, CsrSide& side, ViewTmp& t, const int32_t* row, int32_t n_rows,
                const int32_t* nbr, const int32_t* relw, const float* norm, int64_t M,
                bool count_runs, unsigned long long* d_runs, int32_t* h_totals /* pinned [2] */,
                float* run_norm, cudaStream_t st, int64_t& bytes) {
  Scratch sc(st);
  int rc;
  if ((rc = dalloc(&side.d_rowptr, (int64_t)n_rows + 1, st, &bytes))) return rc;
  int32_t* perm;
  uint64_t* keys;
  if ((rc = sort_view(sc, row, relw, M, 0, g->n_relw, 1, (uint64_t)std::max(n_rows, 1),
                      (uint64_t)g->n_relw, &perm, &keys, side.d_rowptr, st)))
    return rc;
  if ((rc = dalloc(&side.d_nbr, M, st, &bytes))) return rc;
  if ((rc = dalloc(&side.d_relw, M, st, &bytes))) return rc;
  if ((rc = dalloc(&side.d_norm, M, st, &bytes))) return rc;
  if (M > 0) {
    if (run_norm) {
      k_norm_relation<<<grid_for(M), 256, 0, st>>>(keys, perm, M, run_norm);
      ++g_rgcn_launches;
    }
    k_gather3<<<grid_for(M), 256, 0, st>>>(perm, M, nbr, relw, norm, side.d_nbr, side.d_relw,
                                           side.d_norm);
    ++g_rgcn_launches;
    if (count_runs) {
      k_count_runs<<<grid_for(M), 256, 0, st>>>(keys, M, d_runs);
      ++g_rgcn_launches;
    }
  }
  if (g->keep_mid) {
    if ((rc = dalloc(&side.d_mid, M, st, &bytes))) return rc;
    DCK(cudaMemcpyAsync(side.d_mid, perm, (size_t)M * 4, cudaMemcpyDeviceToDevice, st));
  }
  int32_t *nitems, *issplit;
  if ((rc = sc.get(&nitems, (int64_t)n_rows + 1))) return rc;
  if ((rc = sc.get(&issplit, (int64_t)n_rows + 1))) return rc;
  if ((rc = t.sc.get(&t.item_off, (int64_t)n_rows + 1))) return rc;
  if ((rc = t.sc.get(&t.split_off, (int64_t)n_rows + 1))) return rc;
  DCK(cudaMemsetAsync(nitems, 0, ((size_t)n_rows + 1) * 4, st));
  DCK(cudaMemsetAsync(issplit, 0, ((size_t)n_rows + 1) * 4, st));
  if (n_rows > 0) {
    k_csr_item_counts<<<grid_for(n_rows), 256, 0, st>>>(side.d_rowptr, n_rows, g->item_max, nitems,
                                                         issplit);
    ++g_rgcn_launches;
  }
  if ((rc = scan_i32(sc, nitems, t.item_off, (int64_t)n_rows + 1, st))) return rc;
  if ((rc = scan_i32(sc, issplit, t.split_off, (int64_t)n_rows + 1, st))) return rc;
  DCK(cudaMemcpyAsync(&h_totals[0], t.item_off + n_rows, 4, cudaMemcpyDeviceToHost, st));
  DCK(cudaMemcpyAsync(&h_totals[1], t.split_off + n_rows, 4, cudaMemcpyDeviceToHost, st));
  return RGCN_OK;
}

int csr_phase_b(rgcn_graph* g, CsrSide& side, ViewTmp& t, int32_t n_rows, const int32_t* h_totals,
                cudaStream_t st, int64_t& bytes) {
  int rc;
  side.n_items = h_totals[0];
  side.n_split = h_totals[1];
  if ((rc = dalloc(&side.d_items, side.n_items, st, &bytes))) return rc;
  if ((rc = dalloc(&side.d_split_nitems, side.n_split, st, &bytes))) return rc;
  if ((rc = dalloc(&side.d_split_rows, side.n_split, st, &bytes))) return rc;
  if (n_rows > 0) {
    k_csr_fill_items<<<grid_for(n_rows), 256, 0, st>>>(side.d_rowptr, n_rows, g->item_max, t.item_off,
                                                        t.split_off, side.d_items, side.d_split_nitems,
                                                        side.d_split_rows);
    ++g_rgcn_launches;
  }
  return rgcn_check_cuda(cudaGetLastError(), "graph prep (csr view)");
}

int rel_phase_a(rgcn_graph* g, RelSide& side, ViewTmp& t, const int32_t* row, int32_t n_rows,
                const int32_t* nbr, const int32_t* relw, const float* norm, int64_t M,
                int32_t* h_total /* pinned [1] */, float* run_norm /* as in csr_phase_a */, cudaStream_t st,
                int64_t& bytes) {
  Scratch sc(st);
  int rc;
  const int st_rows = view_supertile_rows(g, n_rows, M);
  const int32_t n_super = std::max(1, (n_rows + st_rows - 1) / st_rows);
  side.n_super = n_super;
  const int64_t nkeys = (int64_t)n_super * g->n_relw;
  t.n_keys = (int32_t)nkeys;
  if ((rc = dalloc(&side.d_ptr, nkeys + 1, st, &bytes))) return rc;
  int32_t* perm;
  uint64_t* keys;
  if ((rc = sort_view(sc, row, relw, M, 1, g->n_relw, st_rows, (uint64_t)nkeys,
                      (uint64_t)std::max(n_rows, 1), &perm, &keys, side.d_ptr, st)))
    return rc;
  if ((rc = dalloc(&side.d_row, M, st, &bytes))) return rc;
  if ((rc = dalloc(&side.d_nbr, M, st, &bytes))) return rc;
  if ((rc = dalloc(&side.d_norm, M, st, &bytes))) return rc;
  if (M > 0) {
    if (run_norm) {
      k_norm_relation<<<grid_for(M), 256, 0, st>>>(keys, perm, M, run_norm);
      ++g_rgcn_launches;
    }
    k_gather3<<<grid_for(M), 256, 0, st>>>(perm, M, row, nbr, norm, side.d_row, side.d_nbr,
                                           side.d_norm);
    ++g_rgcn_launches;
  }
  if (g->keep_mid) {
    if ((rc = dalloc(&side.d_mid, M, st, &bytes))) return rc;
    DCK(cudaMemcpyAsync(side.d_mid, perm, (size_t)M * 4, cudaMemcpyDeviceToDevice, st));
  }
  int32_t* nitems;
  if ((rc = sc.get(&nitems, nkeys + 1))) return rc;
  if ((rc = t.sc.get(&t.item_off, nkeys + 1))) return rc;
  DCK(cudaMemsetAsync(nitems, 0, ((size_t)nkeys + 1) * 4, st));
  k_rel_item_counts<<<grid_for(nkeys), 256, 0, st>>>(side.d_ptr, (int32_t)nkeys, g->item_max, nitems);
  ++g_rgcn_launches;
  if ((rc = scan_i32(sc, nitems, t.item_off, nkeys + 1, st))) return rc;
  DCK(cudaMemcpyAsync(h_total, t.item_off + nkeys, 4, cudaMemcpyDeviceToHost, st));
  return RGCN_OK;
}

int rel_phase_b(rgcn_graph* g, RelSide& side, ViewTmp& t, const int32_t* h_total, cudaStream_t st,
                int64_t& bytes) {
  int rc;
  side.n_items = h_total[0];
  if ((rc = dalloc(&side.d_items, side.n_items, st, &bytes))) return rc;
  k_rel_fill_items<<<grid_for(t.n_keys), 256, 0, st>>>(side.d_ptr, t.n_keys, g->item_max, g->n_relw,
                                                        t.item_off, side.d_items);
  ++g_rgcn_launches;
  return rgcn_check_cuda(cudaGetLastError(), "graph prep (rel view)");
}

// pinned host slots for the few integers the host needs back (one set per thread)
struct HostSlots {
  int32_t* p = nullptr;  // [0..1] by_dst, [2..3] by_src, [4] by_rel, [5] by_rel_src, [6] bad flag
  unsigned long long* runs = nullptr;
  HostSlots() {
    cudaHostAlloc((void**)&p, 8 * sizeof(int32_t), cudaHostAllocDefault);
    cudaHostAlloc((void**)&runs, sizeof(unsigned long long), cudaHostAllocDefault);
  }
};

void tune_mempool_once(int device) {
  // keep freed blocks in the stream-ordered pool instead of returning them to the OS at every
  // synchronisation (the default release threshold is 0: every graph build would re-map memory)
  static bool done[64] = {false};
  if (device < 0 || device >= 64 || done[device]) return;
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    uint64_t thr = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  done[device] = true;
}

}  // namespace

// Builds every device-side structure of `g` from DEVICE message arrays (length M).
// d_bad (optional): device flag set by the caller's validation kernel; checked at the single sync.
// d_run_norm (optional, RGCN_NORM_RELATION): the buffer d_norm points to, not yet written; the first view built (by_dst,
// or by_rel when the CSR views are off -- both destination-keyed) fills it with 1 / (length of the (dst, weight id)
// run) before anything reads it.
int rgcn_build_on_device_checked(rgcn_graph* g, const int32_t* d_dst, const int32_t* d_src,
                                 const int32_t* d_relw, const float* d_norm, const int* d_bad,
                                 cudaStream_t st, float* d_run_norm) {
  static thread_local HostSlots hs;
  if (!hs.p || !hs.runs) {
    rgcn_set_error("cudaHostAlloc failed in graph prep");
    return RGCN_ERR_NOMEM;
  }
  tune_mempool_once(g->device);
  int64_t bytes = 0;
  const int64_t M = g->M;
  int rc;
  unsigned long long* d_runs;
  if ((rc = dalloc(&d_runs, 1, st))) return rc;
  DCK(cudaMemsetAsync(d_runs, 0, sizeof(unsigned long long), st));
  if (g->keep_mid) {
    if ((rc = dalloc(&g->d_msg_norm, M, st, &bytes))) return rc;
  }
  ViewTmp t0(st), t1(st), t2(st), t3(st);
  for (int i = 0; i < 8; ++i) hs.p[i] = 0;
  *hs.runs = 0;
  rc = RGCN_OK;
  if (g->has_csr) {
    rc = csr_phase_a(g, g->by_dst, t0, d_dst, g->V_dst, d_src, d_relw, d_norm, M, true, d_runs, hs.p + 0, d_run_norm,
                     st, bytes);
    d_run_norm = nullptr;
    if (!rc) rc = csr_phase_a(g, g->by_src, t1, d_src, g->V_src, d_dst, d_relw, d_norm, M, false, nullptr, hs.p + 2,
                              nullptr, st, bytes);
  }
  if (!rc && g->has_rel) {
    rc = rel_phase_a(g, g->by_rel, t2, d_dst, g->V_dst, d_src, d_relw, d_norm, M, hs.p + 4, d_run_norm, st, bytes);
    if (!rc) rc = rel_phase_a(g, g->by_rel_src, t3, d_src, g->V_src, d_dst, d_relw, d_norm, M, hs.p + 5, nullptr, st,
                              bytes);
  }
  if (!rc && g->keep_mid && M > 0)
    rc = rgcn_check_cuda(cudaMemcpyAsync(g->d_msg_norm, d_norm, (size_t)M * 4, cudaMemcpyDeviceToDevice, st),
                         "copy msg norm");
  if (!rc) rc = rgcn_check_cuda(cudaMemcpyAsync(hs.runs, d_runs, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st), "copy runs");
  if (!rc && d_bad) rc = rgcn_check_cuda(cudaMemcpyAsync(hs.p + 6, d_bad, 4, cudaMemcpyDeviceToHost, st), "copy flag");
  if (!rc) rc = rgcn_check_cuda(cudaStreamSynchronize(st), "sync(graph prep)");
  cudaFreeAsync(d_runs, st);
  if (!rc && hs.p[6]) {
    rgcn_set_error("rgcn_graph_create: index out of range");
    rc = RGCN_ERR_INVALID;
  }
  if (!rc && g->has_csr) {
    rc = csr_phase_b(g, g->by_dst, t0, g->V_dst, hs.p + 0, st, bytes);
    if (!rc) rc = csr_phase_b(g, g->by_src, t1, g->V_src, hs.p + 2, st, bytes);
  }
  if (!rc && g->has_rel) {
    rc = rel_phase_b(g, g->by_rel, t2, hs.p + 4, st, bytes);
    if (!rc) rc = rel_phase_b(g, g->by_rel_src, t3, hs.p + 5, st, bytes);
  }
  g->n_groups = (int64_t)*hs.runs;
  g->device_bytes = bytes;
  g->built_on_device = true;
  if (!rc && M >= (int64_t)(32 << 20)) {
    // a very large build leaves gigabytes of freed temporaries cached in the stream-ordered pool (release
    // threshold = max): hand them back to the driver so the caller's own allocator can use the memory
    rc = rgcn_check_cuda(cudaStreamSynchronize(st), "sync(graph prep end)");
    cudaMemPool_t pool;
    if (!rc && cudaDeviceGetDefaultMemPool(&pool, g->device) == cudaSuccess) cudaMemPoolTrimTo(pool, 0);
  }
  return rc;
}

int rgcn_build_on_device(rgcn_graph* g, const int32_t* d_dst, const int32_t* d_src,
                         const int32_t* d_relw, const float* d_norm, cudaStream_t st) {
  return rgcn_build_on_device_checked(g, d_dst, d_src, d_relw, d_norm, nullptr, st, nullptr);
}

// triples (DEVICE, int32 [E,3]) -> messages + norm -> rgcn_build_on_device
int rgcn_build_from_triples_device(rgcn_graph* g, const int32_t* d_triples, int64_t E, int32_t V,
                                   int32_t R, int norm_mode, const float* d_norm_f,
                                   const float* d_norm_b, cudaStream_t st) {
  Scratch sc(st);
  const int64_t M = 2 * E;
  int32_t *dst, *src, *relw, *cnt_f, *cnt_b;
  float* norm;
  int* bad;
  int rc;
  if ((rc = sc.get(&dst, M))) return rc;
  if ((rc = sc.get(&src, M))) return rc;
  if ((rc = sc.get(&relw, M))) return rc;
  if ((rc = sc.get(&norm, M))) return rc;
  if ((rc = sc.get(&cnt_f, V))) return rc;
  if ((rc = sc.get(&cnt_b, V))) return rc;
  if ((rc = sc.get(&bad, 1))) return rc;
  DCK(cudaMemsetAsync(cnt_f, 0, (size_t)std::max(V, 1) * 4, st));
  DCK(cudaMemsetAsync(cnt_b, 0, (size_t)std::max(V, 1) * 4, st));
  DCK(cudaMemsetAsync(bad, 0, 4, st));
  if (E > 0) {
    k_tri2msg<<<grid_for(E), 256, 0, st>>>(d_triples, E, R, dst, src, relw, cnt_f, cnt_b, V, bad);
    ++g_rgcn_launches;
    if (norm_mode == RGCN_NORM_CANONICAL) {
      k_norm_canonical<<<grid_for(E), 256, 0, st>>>(dst, E, cnt_f, cnt_b, norm);
      ++g_rgcn_launches;
    } else if (norm_mode == RGCN_NORM_EXPLICIT) {
      DCK(cudaMemcpyAsync(norm, d_norm_f, (size_t)E * 4, cudaMemcpyDeviceToDevice, st));
      DCK(cudaMemcpyAsync(norm + E, d_norm_b, (size_t)E * 4, cudaMemcpyDeviceToDevice, st));
      ++g_rgcn_launches;
    } else if (norm_mode == RGCN_NORM_NONE) {
      k_fill<<<grid_for(M), 256, 0, st>>>(norm, M, 1.0f);
      ++g_rgcn_launches;
    }  // RGCN_NORM_RELATION: written by the first view build (k_norm_relation)
  }
  return rgcn_build_on_device_checked(g, dst, src, relw, norm, bad, st,
                                      norm_mode == RGCN_NORM_RELATION ? norm : nullptr);
}

int rgcn_check_messages_device(const int32_t* d_dst, const int32_t* d_src, const int32_t* d_relw,
                               int64_t M, int32_t V_dst, int32_t V_src, int32_t n_relw,
                               cudaStream_t st) {
  if (M == 0) return RGCN_OK;
  int* bad;
  int rc = dalloc(&bad, 1, st);
  if (rc) return rc;
  DCK(cudaMemsetAsync(bad, 0, 4, st));
  k_check_messages<<<grid_for(M), 256, 0, st>>>(d_dst, d_src, d_relw, M, V_dst, V_src, n_relw, bad);
  ++g_rgcn_launches;
  int h_bad = 0;
  DCK(cudaMemcpyAsync(&h_bad, bad, 4, cudaMemcpyDeviceToHost, st));
  DCK(cudaStreamSynchronize(st));
  cudaFreeAsync(bad, st);
  if (h_bad) {
    rgcn_set_error("rgcn_graph_create_messages: index out of range");
    return RGCN_ERR_INVALID;
  }
  return RGCN_OK;
}
