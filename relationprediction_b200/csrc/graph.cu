// graph.cu -- graph preparation for the R-GCN hot path (host side, deterministic) + device upload.
//
// Replaces what the reference does implicitly inside its TF graph:
//   * MessageGraph.process (extras/graph_representations.py:21-27): split [E,3] triples into
//     sender / type / receiver index vectors; message id of triple k is k in both directions.
//   * forward_/backward_incidence_matrix('global') (:84-93, :124-133): per-direction row softmax of
//     an all-ones [V,E] incidence  ==  1 / (#messages of that direction into the row).
// Instead of a [V,E] COO matrix we build three sorted views of the 2E messages so that no kernel
// needs a global atomic per message:
//   by_dst : CSR over destinations, sorted by (dst, weight id)    -> forward aggregation
//   by_src : CSR over sources,      sorted by (src, weight id)    -> backward w.r.t. H
//   by_rel : weight-id major,       sorted by (weight id, dst)    -> backward w.r.t. block weights
// All sorts are stable counting sorts, so the result is a pure function of the input order.
#include "graph.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <chrono>
#include <cstdio>
#include <exception>
#include <new>
#include <thread>

static thread_local std::string g_last_error;

void rgcn_set_error(const std::string& s) { g_last_error = s; }

extern "C" const char* rgcn_last_error(void) { return g_last_error.c_str(); }

extern "C" int rgcn_version(void) { return 100; }

int rgcn_check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return RGCN_OK;
  rgcn_set_error(std::string(what) + ": " + cudaGetErrorString(e));
  return RGCN_ERR_CUDA;
}

// which sorted views new graphs get: bit 0 = the two CSR views, bit 1 = the two weight-id-major views
// (rgcn_set_option("graph_views", mask); GPU-prepared graphs only -- the host builder always builds all four)
int g_graph_views = 3;

namespace {

// Stable LSD counting sort of message ids by (major, minor).  Returns perm (sorted -> message id)
// and the CSR pointer over the major key.
void sort_two_keys(const int32_t* major, int32_t n_major, const int32_t* minor, int32_t n_minor,
                   int64_t M, std::vector<int32_t>& perm, std::vector<int32_t>& ptr) {
  std::vector<int32_t> tmp(M);
  {
    std::vector<int64_t> cnt((size_t)n_minor + 1, 0);
    for (int64_t m = 0; m < M; ++m) cnt[(size_t)minor[m] + 1]++;
    for (int32_t k = 0; k < n_minor; ++k) cnt[k + 1] += cnt[k];
    for (int64_t m = 0; m < M; ++m) tmp[cnt[minor[m]]++] = (int32_t)m;
  }
  perm.resize(M);
  ptr.assign((size_t)n_major + 1, 0);
  {
    std::vector<int64_t> cnt((size_t)n_major + 1, 0);
    for (int64_t m = 0; m < M; ++m) cnt[(size_t)major[m] + 1]++;
    for (int32_t k = 0; k < n_major; ++k) cnt[k + 1] += cnt[k];
    for (int32_t k = 0; k <= n_major; ++k) ptr[k] = (int32_t)cnt[k];
    for (int64_t i = 0; i < M; ++i) {
      int32_t m = tmp[i];
      perm[cnt[major[m]]++] = m;
    }
  }
}

void build_items(const std::vector<int32_t>& rowptr, int32_t rows, int item_max,
                 std::vector<WorkItem>& items, std::vector<int32_t>* split_nitems,
                 std::vector<int32_t>* split_rows, bool emit_empty) {
  items.clear();
  if (split_nitems) split_nitems->clear();
  if (split_rows) split_rows->clear();
  for (int32_t r = 0; r < rows; ++r) {
    int32_t beg = rowptr[r], end = rowptr[r + 1];
    int32_t deg = end - beg;
    if (deg == 0) {
      if (emit_empty) items.push_back({beg, end, r, -1});
      continue;
    }
    if (deg <= item_max || !split_nitems) {
      if (deg <= item_max) {
        items.push_back({beg, end, r, -1});
      } else {  // weight-id major list: chunks are independent (partials are reduced with atomics)
        for (int32_t b = beg; b < end; b += item_max)
          items.push_back({b, std::min(end, b + item_max), r, 0});
      }
      continue;
    }
    int32_t n = (deg + item_max - 1) / item_max;
    int32_t sidx = (int32_t)split_rows->size();
    split_rows->push_back(r);
    split_nitems->push_back(n);
    // equal-sized chunks (last one may be short)
    int32_t chunk = (deg + n - 1) / n;
    int32_t made = 0;
    for (int32_t b = beg; b < end; b += chunk, ++made)
      items.push_back({b, std::min(end, b + chunk), r, sidx});
    (*split_nitems)[sidx] = made;
  }
}

void fill_side(CsrSide& side, const std::vector<int32_t>& perm, const int32_t* other,
               const int32_t* relw, const float* norm) {
  int64_t M = (int64_t)perm.size();
  side.nbr.resize(M);
  side.relw.resize(M);
  side.norm.resize(M);
  side.mid = perm;
  for (int64_t i = 0; i < M; ++i) {
    int32_t m = perm[i];
    side.nbr[i] = other[m];
    side.relw[i] = relw[m];
    side.norm[i] = norm[m];
  }
}

void build_rel_side(RelSide& side, const int32_t* row, int32_t n_rows, const int32_t* nbr,
                    const int32_t* relw, const float* norm, int64_t M, int32_t n_relw,
                    int supertile_rows, int item_max) {
  const int32_t n_super = std::max(1, (n_rows + supertile_rows - 1) / supertile_rows);
  side.n_super = n_super;
  std::vector<int32_t> key(M);
  for (int64_t m = 0; m < M; ++m) key[m] = (row[m] / supertile_rows) * n_relw + relw[m];
  std::vector<int32_t> perm;
  sort_two_keys(key.data(), n_super * n_relw, row, std::max(n_rows, 1), M, perm, side.ptr);
  side.mid = perm;
  side.row.resize(M);
  side.nbr.resize(M);
  side.norm.resize(M);
  for (int64_t i = 0; i < M; ++i) {
    const int32_t m = perm[i];
    side.row[i] = row[m];
    side.nbr[i] = nbr[m];
    side.norm[i] = norm[m];
  }
  side.items.clear();
  for (int32_t k = 0; k < n_super * n_relw; ++k) {
    const int32_t beg = side.ptr[k], end = side.ptr[k + 1];
    for (int32_t b = beg; b < end; b += item_max)
      side.items.push_back({b, std::min(end, b + item_max), k % n_relw, k / n_relw});
  }
}

template <typename T>
int upload(T** dptr, const std::vector<T>& h, cudaStream_t st, int64_t& bytes) {
  size_t n = h.size() * sizeof(T);
  *dptr = nullptr;
  if (n == 0) n = sizeof(T);  // keep pointers non-null for empty graphs
  int rc = rgcn_check_cuda(cudaMalloc((void**)dptr, n), "cudaMalloc(graph)");
  if (rc) return rc;
  bytes += (int64_t)n;
  if (!h.empty())
    rc = rgcn_check_cuda(
        cudaMemcpyAsync(*dptr, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice, st),
        "cudaMemcpyAsync(graph)");
  return rc;
}

rgcn_graph* new_graph(int64_t M, int32_t V_dst, int32_t V_src, int32_t n_relw, int device) {
  rgcn_graph* g = new (std::nothrow) rgcn_graph();
  if (!g) return nullptr;
  g->M = M;
  g->V_dst = V_dst;
  g->V_src = V_src;
  g->n_relw = n_relw;
  g->device = device;
  if (const char* e = std::getenv("RGCN_ITEM_MAX")) {
    int v = std::atoi(e);
    if (v >= 8) g->item_max = v;
  }
  if (const char* e = std::getenv("RGCN_SUPERTILE_ROWS")) {
    int v = std::atoi(e);
    if (v >= 1) {
      g->supertile_rows = v;
      g->supertile_fixed = true;
    }
  }
  // message-id permutations are only needed by rgcn_graph_export: skip them on very large graphs
  g->keep_mid = M <= (int64_t)(16 << 20);
  if (const char* e = std::getenv("RGCN_KEEP_MID")) g->keep_mid = std::atoi(e) != 0;
  g->has_csr = (g_graph_views & 1) != 0;
  g->has_rel = (g_graph_views & 2) != 0;
  return g;
}

bool use_device_prep(int device) {
  if (device < 0) return false;
  const char* e = std::getenv("RGCN_PREP");
  return !(e && std::string(e) == "host");
}

int build(const int32_t* dst, const int32_t* src, const int32_t* relw, const float* norm, int64_t M,
          int32_t V_dst, int32_t V_src, int32_t n_relw, int device, void* stream,
          rgcn_graph_t** out) {
  if (!out) {
    rgcn_set_error("out is null");
    return RGCN_ERR_INVALID;
  }
  *out = nullptr;
  if (M < 0 || M > 0x7fffffffLL || V_dst < 0 || V_src < 0 || n_relw <= 0) {
    rgcn_set_error("rgcn_graph_create: bad sizes (need 0<=M<2^31, V_dst>=0, V_src>=0, n_relw>0)");
    return RGCN_ERR_INVALID;
  }
  rgcn_graph* g = new_graph(M, V_dst, V_src, n_relw, device);
  if (!g) return RGCN_ERR_NOMEM;
  if (use_device_prep(device)) {
    // GPU graph preparation (graph_device.cu): upload the raw message arrays, build there
    cudaStream_t st = (cudaStream_t)stream;
    int rc = rgcn_check_cuda(cudaSetDevice(device), "cudaSetDevice");
    int32_t *d_dst = nullptr, *d_src = nullptr, *d_relw = nullptr;
    float* d_norm = nullptr;
    const size_t nb = (size_t)std::max<int64_t>(M, 1) * 4;
    if (!rc) rc = rgcn_check_cuda(cudaMallocAsync((void**)&d_dst, nb, st), "cudaMallocAsync");
    if (!rc) rc = rgcn_check_cuda(cudaMallocAsync((void**)&d_src, nb, st), "cudaMallocAsync");
    if (!rc) rc = rgcn_check_cuda(cudaMallocAsync((void**)&d_relw, nb, st), "cudaMallocAsync");
    if (!rc) rc = rgcn_check_cuda(cudaMallocAsync((void**)&d_norm, nb, st), "cudaMallocAsync");
    if (!rc && M > 0) {
      rc = rgcn_check_cuda(cudaMemcpyAsync(d_dst, dst, (size_t)M * 4, cudaMemcpyHostToDevice, st), "H2D dst");
      if (!rc) rc = rgcn_check_cuda(cudaMemcpyAsync(d_src, src, (size_t)M * 4, cudaMemcpyHostToDevice, st), "H2D src");
      if (!rc) rc = rgcn_check_cuda(cudaMemcpyAsync(d_relw, relw, (size_t)M * 4, cudaMemcpyHostToDevice, st), "H2D relw");
      if (!rc) rc = rgcn_check_cuda(cudaMemcpyAsync(d_norm, norm, (size_t)M * 4, cudaMemcpyHostToDevice, st), "H2D norm");
    }
    if (!rc) rc = rgcn_check_messages_device(d_dst, d_src, d_relw, M, V_dst, V_src, n_relw, st);
    if (!rc) rc = rgcn_build_on_device(g, d_dst, d_src, d_relw, d_norm, st);
    cudaFreeAsync(d_dst, st);
    cudaFreeAsync(d_src, st);
    cudaFreeAsync(d_relw, st);
    cudaFreeAsync(d_norm, st);
    if (rc) {
      rgcn_graph_destroy(g);
      return rc;
    }
    *out = g;
    return RGCN_OK;
  }
  g->has_csr = g->has_rel = true;  // the host builder always produces all four views
  for (int64_t m = 0; m < M; ++m) {
    if (dst[m] < 0 || dst[m] >= V_dst || src[m] < 0 || src[m] >= V_src || relw[m] < 0 ||
        relw[m] >= n_relw) {
      delete g;
      rgcn_set_error("rgcn_graph_create: index out of range at message " + std::to_string(m));
      return RGCN_ERR_INVALID;
    }
  }
  try {
    g->msg_norm.assign(norm, norm + M);

    const bool timing = std::getenv("RGCN_PREP_TIMING") != nullptr;
    auto tnow = []() { return std::chrono::steady_clock::now(); };
    auto t_begin = tnow();
    // the four sorted views are independent: build them on four host threads
    std::exception_ptr err[4] = {nullptr, nullptr, nullptr, nullptr};
    auto guarded = [&](int slot, auto&& fn) {
      return std::thread([&err, slot, fn]() {
        try {
          fn();
        } catch (...) {
          err[slot] = std::current_exception();
        }
      });
    };
    std::thread t0 = guarded(0, [&]() {  // destination-major
      auto ta = tnow();
      std::vector<int32_t> perm;
      sort_two_keys(dst, V_dst, relw, n_relw, M, perm, g->by_dst.rowptr);
      fill_side(g->by_dst, perm, src, relw, norm);
      build_items(g->by_dst.rowptr, V_dst, g->item_max, g->by_dst.items, &g->by_dst.split_nitems,
                  &g->by_dst.split_rows, /*emit_empty=*/true);
      int64_t groups = 0;
      for (int32_t v = 0; v < V_dst; ++v) {
        int32_t prev = -1;
        for (int32_t i = g->by_dst.rowptr[v]; i < g->by_dst.rowptr[v + 1]; ++i) {
          if (g->by_dst.relw[i] != prev) {
            ++groups;
            prev = g->by_dst.relw[i];
          }
        }
      }
      g->n_groups = groups;
      if (timing) fprintf(stderr, "[rgcn prep] by_dst %.2f ms\n", std::chrono::duration<double, std::milli>(tnow() - ta).count());
    });
    std::thread t1 = guarded(1, [&]() {  // source-major
      std::vector<int32_t> perm;
      sort_two_keys(src, V_src, relw, n_relw, M, perm, g->by_src.rowptr);
      fill_side(g->by_src, perm, dst, relw, norm);
      build_items(g->by_src.rowptr, V_src, g->item_max, g->by_src.items, &g->by_src.split_nitems,
                  &g->by_src.split_rows, /*emit_empty=*/true);
    });
    // weight-id major views (see RelSide)
    std::thread t2 = guarded(2, [&]() {
      build_rel_side(g->by_rel, dst, V_dst, src, relw, norm, M, n_relw, view_supertile_rows(g, V_dst, M),
                     g->item_max);
    });
    std::thread t3 = guarded(3, [&]() {
      build_rel_side(g->by_rel_src, src, V_src, dst, relw, norm, M, n_relw, view_supertile_rows(g, V_src, M),
                     g->item_max);
    });
    t0.join();
    t1.join();
    t2.join();
    t3.join();
    for (auto& e : err)
      if (e) std::rethrow_exception(e);
    if (timing)
      fprintf(stderr, "[rgcn prep] views %.2f ms (M=%lld)\n",
              std::chrono::duration<double, std::milli>(tnow() - t_begin).count(), (long long)M);
  } catch (const std::bad_alloc&) {
    delete g;
    rgcn_set_error("host allocation failed in graph build");
    return RGCN_ERR_NOMEM;
  }

  g->by_dst.n_items = (int64_t)g->by_dst.items.size();
  g->by_dst.n_split = (int64_t)g->by_dst.split_rows.size();
  g->by_src.n_items = (int64_t)g->by_src.items.size();
  g->by_src.n_split = (int64_t)g->by_src.split_rows.size();
  g->by_rel.n_items = (int64_t)g->by_rel.items.size();
  g->by_rel_src.n_items = (int64_t)g->by_rel_src.items.size();
  if (device >= 0) {
    cudaStream_t st = (cudaStream_t)stream;
    int rc = rgcn_check_cuda(cudaSetDevice(device), "cudaSetDevice");
    int64_t bytes = 0;
    if (!rc) rc = upload(&g->by_dst.d_nbr, g->by_dst.nbr, st, bytes);
    if (!rc) rc = upload(&g->by_dst.d_relw, g->by_dst.relw, st, bytes);
    if (!rc) rc = upload(&g->by_dst.d_norm, g->by_dst.norm, st, bytes);
    if (!rc) rc = upload(&g->by_dst.d_items, g->by_dst.items, st, bytes);
    if (!rc) rc = upload(&g->by_dst.d_split_nitems, g->by_dst.split_nitems, st, bytes);
    if (!rc) rc = upload(&g->by_dst.d_split_rows, g->by_dst.split_rows, st, bytes);
    if (!rc) rc = upload(&g->by_src.d_nbr, g->by_src.nbr, st, bytes);
    if (!rc) rc = upload(&g->by_src.d_relw, g->by_src.relw, st, bytes);
    if (!rc) rc = upload(&g->by_src.d_norm, g->by_src.norm, st, bytes);
    if (!rc) rc = upload(&g->by_src.d_items, g->by_src.items, st, bytes);
    if (!rc) rc = upload(&g->by_src.d_split_nitems, g->by_src.split_nitems, st, bytes);
    if (!rc) rc = upload(&g->by_src.d_split_rows, g->by_src.split_rows, st, bytes);
    for (RelSide* rs : {&g->by_rel, &g->by_rel_src}) {
      if (!rc) rc = upload(&rs->d_row, rs->row, st, bytes);
      if (!rc) rc = upload(&rs->d_nbr, rs->nbr, st, bytes);
      if (!rc) rc = upload(&rs->d_norm, rs->norm, st, bytes);
      if (!rc) rc = upload(&rs->d_items, rs->items, st, bytes);
    }
    // the host vectors are pageable: make sure the copies are done before anyone frees/modifies them
    if (!rc) rc = rgcn_check_cuda(cudaStreamSynchronize(st), "cudaStreamSynchronize(graph upload)");
    g->device_bytes = bytes;
    if (rc) {
      rgcn_graph_destroy(g);
      return rc;
    }
  }
  *out = g;
  return RGCN_OK;
}

}  // namespace

extern "C" int rgcn_graph_create_messages(const int32_t* dst_host, const int32_t* src_host,
                                          const int32_t* relw_host, const float* norm_host,
                                          int64_t M, int32_t V_dst, int32_t V_src, int32_t n_relw,
                                          int device, void* stream, rgcn_graph_t** out) {
  if (M > 0 && (!dst_host || !src_host || !relw_host || !norm_host)) {
    rgcn_set_error("rgcn_graph_create_messages: null array");
    return RGCN_ERR_INVALID;
  }
  return build(dst_host, src_host, relw_host, norm_host, M, V_dst, V_src, n_relw, device, stream,
               out);
}

extern "C" int rgcn_graph_create(const int32_t* triples_host, int64_t E, int32_t V, int32_t R,
                                 int norm_mode, const float* norm_f_host, const float* norm_b_host,
                                 int device, void* stream, rgcn_graph_t** out) {
  if (E < 0 || V < 0 || R <= 0 || (E > 0 && !triples_host) || 2 * E > 0x7fffffffLL) {
    rgcn_set_error("rgcn_graph_create: bad sizes");
    return RGCN_ERR_INVALID;
  }
  if (norm_mode == RGCN_NORM_EXPLICIT && E > 0 && (!norm_f_host || !norm_b_host)) {
    rgcn_set_error("rgcn_graph_create: RGCN_NORM_EXPLICIT needs norm_f_host and norm_b_host");
    return RGCN_ERR_INVALID;
  }
  if (norm_mode < 0 || norm_mode > RGCN_NORM_RELATION) {
    rgcn_set_error("rgcn_graph_create: unknown norm_mode");
    return RGCN_ERR_INVALID;
  }
  int64_t M = 2 * E;
  if (use_device_prep(device)) {
    if (!out) {
      rgcn_set_error("out is null");
      return RGCN_ERR_INVALID;
    }
    *out = nullptr;
    rgcn_graph* g = new_graph(M, V, V, 2 * R, device);
    if (!g) return RGCN_ERR_NOMEM;
    cudaStream_t st = (cudaStream_t)stream;
    int rc = rgcn_check_cuda(cudaSetDevice(device), "cudaSetDevice");
    int32_t* d_tri = nullptr;
    float *d_nf = nullptr, *d_nb = nullptr;
    if (!rc) rc = rgcn_check_cuda(cudaMallocAsync((void**)&d_tri, (size_t)std::max<int64_t>(E, 1) * 12, st), "cudaMallocAsync");
    if (!rc && E > 0) rc = rgcn_check_cuda(cudaMemcpyAsync(d_tri, triples_host, (size_t)E * 12, cudaMemcpyHostToDevice, st), "H2D triples");
    if (!rc && norm_mode == RGCN_NORM_EXPLICIT && E > 0) {
      rc = rgcn_check_cuda(cudaMallocAsync((void**)&d_nf, (size_t)E * 4, st), "cudaMallocAsync");
      if (!rc) rc = rgcn_check_cuda(cudaMallocAsync((void**)&d_nb, (size_t)E * 4, st), "cudaMallocAsync");
      if (!rc) rc = rgcn_check_cuda(cudaMemcpyAsync(d_nf, norm_f_host, (size_t)E * 4, cudaMemcpyHostToDevice, st), "H2D norm_f");
      if (!rc) rc = rgcn_check_cuda(cudaMemcpyAsync(d_nb, norm_b_host, (size_t)E * 4, cudaMemcpyHostToDevice, st), "H2D norm_b");
    }
    if (!rc) rc = rgcn_build_from_triples_device(g, d_tri, E, V, R, norm_mode, d_nf, d_nb, st);
    cudaFreeAsync(d_tri, st);
    if (d_nf) cudaFreeAsync(d_nf, st);
    if (d_nb) cudaFreeAsync(d_nb, st);
    if (rc) {
      rgcn_graph_destroy(g);
      return rc;
    }
    *out = g;
    return RGCN_OK;
  }
  std::vector<int32_t> dst, src, relw;
  std::vector<float> norm;
  try {
    dst.resize(M);
    src.resize(M);
    relw.resize(M);
    norm.resize(M);
  } catch (const std::bad_alloc&) {
    return RGCN_ERR_NOMEM;
  }
  for (int64_t k = 0; k < E; ++k) {
    int32_t s = triples_host[3 * k + 0], r = triples_host[3 * k + 1], o = triples_host[3 * k + 2];
    if (s < 0 || s >= V || o < 0 || o >= V || r < 0 || r >= R) {
      rgcn_set_error("rgcn_graph_create: triple " + std::to_string(k) + " out of range");
      return RGCN_ERR_INVALID;
    }
    // forward message: sender = subject, receiver = object (graph_representations.py:23-24)
    dst[k] = o;
    src[k] = s;
    relw[k] = r;
    // backward message: sender = object, receiver = subject, separate weight table (W_backward)
    dst[E + k] = s;
    src[E + k] = o;
    relw[E + k] = r + R;
  }
  if (norm_mode == RGCN_NORM_CANONICAL) {
    // sparse_softmax over a row of ones == 1/row_count, per direction (graph_representations.py:84-93)
    std::vector<int32_t> cf((size_t)V, 0), cb((size_t)V, 0);
    for (int64_t k = 0; k < E; ++k) {
      cf[dst[k]]++;
      cb[dst[E + k]]++;
    }
    for (int64_t k = 0; k < E; ++k) {
      norm[k] = 1.0f / (float)cf[dst[k]];
      norm[E + k] = 1.0f / (float)cb[dst[E + k]];
    }
  } else if (norm_mode == RGCN_NORM_RELATION) {
    // 1 / (#messages in the message's (dst, weight id) group) -- the 'local' branch
    // (graph_representations.py:94-107, :134-147).  The groups are the runs of the by_dst order.
    std::vector<int32_t> perm, ptr;
    try {
      sort_two_keys(dst.data(), std::max(V, 1), relw.data(), 2 * R, M, perm, ptr);
    } catch (const std::bad_alloc&) {
      return RGCN_ERR_NOMEM;
    }
    for (int64_t i = 0; i < M;) {
      const int32_t d = dst[perm[i]], w = relw[perm[i]];
      int64_t j = i + 1;
      while (j < M && dst[perm[j]] == d && relw[perm[j]] == w) ++j;
      const float v = 1.0f / (float)(j - i);
      for (; i < j; ++i) norm[perm[i]] = v;
    }
  } else if (norm_mode == RGCN_NORM_EXPLICIT) {
    for (int64_t k = 0; k < E; ++k) {
      norm[k] = norm_f_host[k];
      norm[E + k] = norm_b_host[k];
    }
  } else {
    std::fill(norm.begin(), norm.end(), 1.0f);
  }
  return build(dst.data(), src.data(), relw.data(), norm.data(), M, V, V, 2 * R, device, stream,
               out);
}

// ------------------------------------------------------------------------------------------------
// Constructors over index arrays that already live on the device (the node-sharded path partitions the
// edge list on the GPU, bench.py generates it there): nothing visits the host, GPU preparation only.
// ------------------------------------------------------------------------------------------------
extern "C" int rgcn_graph_create_messages_device(const int32_t* dst_dev, const int32_t* src_dev,
                                                 const int32_t* relw_dev, const float* norm_dev, int64_t M,
                                                 int32_t V_dst, int32_t V_src, int32_t n_relw, int device,
                                                 void* stream, rgcn_graph_t** out) {
  if (!out) {
    rgcn_set_error("out is null");
    return RGCN_ERR_INVALID;
  }
  *out = nullptr;
  if (device < 0) {
    rgcn_set_error("rgcn_graph_create_messages_device: needs a device ordinal");
    return RGCN_ERR_NODEVICE;
  }
  if (M < 0 || M > 0x7fffffffLL || V_dst < 0 || V_src < 0 || n_relw <= 0 ||
      (M > 0 && (!dst_dev || !src_dev || !relw_dev || !norm_dev))) {
    rgcn_set_error("rgcn_graph_create_messages_device: bad sizes or null array");
    return RGCN_ERR_INVALID;
  }
  rgcn_graph* g = new_graph(M, V_dst, V_src, n_relw, device);
  if (!g) return RGCN_ERR_NOMEM;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = rgcn_check_cuda(cudaSetDevice(device), "cudaSetDevice");
  if (!rc) rc = rgcn_check_messages_device(dst_dev, src_dev, relw_dev, M, V_dst, V_src, n_relw, st);
  if (!rc) rc = rgcn_build_on_device(g, dst_dev, src_dev, relw_dev, norm_dev, st);
  if (rc) {
    rgcn_graph_destroy(g);
    return rc;
  }
  *out = g;
  return RGCN_OK;
}

extern "C" int rgcn_graph_create_device(const int32_t* triples_dev, int64_t E, int32_t V, int32_t R,
                                        int norm_mode, const float* norm_f_dev, const float* norm_b_dev,
                                        int device, void* stream, rgcn_graph_t** out) {
  if (!out) {
    rgcn_set_error("out is null");
    return RGCN_ERR_INVALID;
  }
  *out = nullptr;
  if (device < 0) {
    rgcn_set_error("rgcn_graph_create_device: needs a device ordinal");
    return RGCN_ERR_NODEVICE;
  }
  if (E < 0 || V < 0 || R <= 0 || (E > 0 && !triples_dev) || 2 * E > 0x7fffffffLL || norm_mode < 0 ||
      norm_mode > RGCN_NORM_RELATION || (norm_mode == RGCN_NORM_EXPLICIT && E > 0 && (!norm_f_dev || !norm_b_dev))) {
    rgcn_set_error("rgcn_graph_create_device: bad arguments");
    return RGCN_ERR_INVALID;
  }
  rgcn_graph* g = new_graph(2 * E, V, V, 2 * R, device);
  if (!g) return RGCN_ERR_NOMEM;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = rgcn_check_cuda(cudaSetDevice(device), "cudaSetDevice");
  if (!rc) rc = rgcn_build_from_triples_device(g, triples_dev, E, V, R, norm_mode, norm_f_dev, norm_b_dev, st);
  if (rc) {
    rgcn_graph_destroy(g);
    return rc;
  }
  *out = g;
  return RGCN_OK;
}

namespace {

template <typename FreeFn>
void free_device_arrays(rgcn_graph_t* g, FreeFn free_fn) {
  free_fn(g->by_dst.d_rowptr);
  free_fn(g->by_src.d_rowptr);
  free_fn(g->by_dst.d_mid);
  free_fn(g->by_src.d_mid);
  free_fn(g->d_msg_norm);
  free_fn(g->by_dst.d_nbr);
  free_fn(g->by_dst.d_relw);
  free_fn(g->by_dst.d_norm);
  free_fn(g->by_dst.d_items);
  free_fn(g->by_dst.d_split_nitems);
  free_fn(g->by_dst.d_split_rows);
  free_fn(g->by_src.d_nbr);
  free_fn(g->by_src.d_relw);
  free_fn(g->by_src.d_norm);
  free_fn(g->by_src.d_items);
  free_fn(g->by_src.d_split_nitems);
  free_fn(g->by_src.d_split_rows);
  for (RelSide* rs : {&g->by_rel, &g->by_rel_src}) {
    free_fn(rs->d_ptr);
    free_fn(rs->d_mid);
    free_fn(rs->d_row);
    free_fn(rs->d_nbr);
    free_fn(rs->d_norm);
    free_fn(rs->d_items);
  }
}

}  // namespace

extern "C" int rgcn_graph_destroy(rgcn_graph_t* g) {
  if (!g) return RGCN_OK;
  if (g->device >= 0) {
    cudaSetDevice(g->device);
    free_device_arrays(g, [](void* p) { cudaFree(p); });
  }
  delete g;
  return RGCN_OK;
}

// Stream-ordered variant (opt-in): a graph prepared on the GPU takes its arrays from the stream-ordered pool, so
// they can be returned with cudaFreeAsync on `stream` -- no device synchronisation.  The caller guarantees that
// every kernel that used the graph was launched on `stream` (or is ordered before it).  Host-prepared graphs
// (cudaMalloc) fall back to the synchronous path.
extern "C" int rgcn_graph_destroy_async(rgcn_graph_t* g, void* stream) {
  if (!g) return RGCN_OK;
  if (g->device < 0 || !g->built_on_device) return rgcn_graph_destroy(g);
  cudaSetDevice(g->device);
  cudaStream_t st = (cudaStream_t)stream;
  free_device_arrays(g, [st](void* p) {
    if (p) cudaFreeAsync(p, st);
  });
  delete g;
  return RGCN_OK;
}

extern "C" int rgcn_graph_info(const rgcn_graph_t* g, int64_t info[16]) {
  if (!g || !info) {
    rgcn_set_error("rgcn_graph_info: null");
    return RGCN_ERR_INVALID;
  }
  std::memset(info, 0, 16 * sizeof(int64_t));
  info[0] = g->M;
  info[1] = g->V_dst;
  info[2] = g->V_src;
  info[3] = g->n_relw;
  info[4] = g->by_dst.n_items;
  info[5] = g->by_src.n_items;
  info[6] = g->by_rel.n_items;
  info[7] = g->by_dst.n_split;
  info[8] = g->by_src.n_split;
  info[9] = g->n_groups;
  info[10] = g->device;
  info[11] = g->device_bytes;
  info[12] = g->item_max;
  info[13] = g->supertile_rows;
  info[14] = g->by_rel.n_super;
  info[15] = g->by_rel_src.n_items;
  return RGCN_OK;
}

namespace {
struct View {
  const void* p;
  int64_t n;
};
template <typename T>
View view(const std::vector<T>& v) {
  return {v.data(), (int64_t)(v.size() * sizeof(T))};
}
bool pick(const rgcn_graph_t* g, int which, View& v) {
  switch (which) {
    case RGCN_X_DST_ROWPTR: v = view(g->by_dst.rowptr); return true;
    case RGCN_X_DST_SRC: v = view(g->by_dst.nbr); return true;
    case RGCN_X_DST_RELW: v = view(g->by_dst.relw); return true;
    case RGCN_X_DST_NORM: v = view(g->by_dst.norm); return true;
    case RGCN_X_DST_MID: v = view(g->by_dst.mid); return true;
    case RGCN_X_SRC_ROWPTR: v = view(g->by_src.rowptr); return true;
    case RGCN_X_SRC_DST: v = view(g->by_src.nbr); return true;
    case RGCN_X_SRC_RELW: v = view(g->by_src.relw); return true;
    case RGCN_X_SRC_NORM: v = view(g->by_src.norm); return true;
    case RGCN_X_SRC_MID: v = view(g->by_src.mid); return true;
    case RGCN_X_REL_PTR: v = view(g->by_rel.ptr); return true;
    case RGCN_X_REL_DST: v = view(g->by_rel.row); return true;
    case RGCN_X_REL_SRC: v = view(g->by_rel.nbr); return true;
    case RGCN_X_REL_NORM: v = view(g->by_rel.norm); return true;
    case RGCN_X_REL_MID: v = view(g->by_rel.mid); return true;
    case RGCN_X_REL2_PTR: v = view(g->by_rel_src.ptr); return true;
    case RGCN_X_REL2_SRC: v = view(g->by_rel_src.row); return true;
    case RGCN_X_REL2_DST: v = view(g->by_rel_src.nbr); return true;
    case RGCN_X_REL2_NORM: v = view(g->by_rel_src.norm); return true;
    case RGCN_X_REL2_MID: v = view(g->by_rel_src.mid); return true;
    case RGCN_X_MSG_NORM: v = view(g->msg_norm); return true;
    default: return false;
  }
}
}  // namespace

namespace {
// device-built graphs keep no host copies: describe where each exported array lives on the device
bool pick_device(const rgcn_graph_t* g, int which, View& v) {
  const int64_t M4 = g->M * 4;
  const int64_t nk = (int64_t)g->by_rel.n_super * g->n_relw + 1;
  const int64_t nk2 = (int64_t)g->by_rel_src.n_super * g->n_relw + 1;
  switch (which) {
    case RGCN_X_DST_ROWPTR: v = {g->by_dst.d_rowptr, ((int64_t)g->V_dst + 1) * 4}; return true;
    case RGCN_X_DST_SRC: v = {g->by_dst.d_nbr, M4}; return true;
    case RGCN_X_DST_RELW: v = {g->by_dst.d_relw, M4}; return true;
    case RGCN_X_DST_NORM: v = {g->by_dst.d_norm, M4}; return true;
    case RGCN_X_DST_MID: v = {g->by_dst.d_mid, M4}; return g->keep_mid;
    case RGCN_X_SRC_ROWPTR: v = {g->by_src.d_rowptr, ((int64_t)g->V_src + 1) * 4}; return true;
    case RGCN_X_SRC_DST: v = {g->by_src.d_nbr, M4}; return true;
    case RGCN_X_SRC_RELW: v = {g->by_src.d_relw, M4}; return true;
    case RGCN_X_SRC_NORM: v = {g->by_src.d_norm, M4}; return true;
    case RGCN_X_SRC_MID: v = {g->by_src.d_mid, M4}; return g->keep_mid;
    case RGCN_X_REL_PTR: v = {g->by_rel.d_ptr, nk * 4}; return true;
    case RGCN_X_REL_DST: v = {g->by_rel.d_row, M4}; return true;
    case RGCN_X_REL_SRC: v = {g->by_rel.d_nbr, M4}; return true;
    case RGCN_X_REL_NORM: v = {g->by_rel.d_norm, M4}; return true;
    case RGCN_X_REL_MID: v = {g->by_rel.d_mid, M4}; return g->keep_mid;
    case RGCN_X_MSG_NORM: v = {g->d_msg_norm, M4}; return g->keep_mid;
    case RGCN_X_REL2_PTR: v = {g->by_rel_src.d_ptr, nk2 * 4}; return true;
    case RGCN_X_REL2_SRC: v = {g->by_rel_src.d_row, M4}; return true;
    case RGCN_X_REL2_DST: v = {g->by_rel_src.d_nbr, M4}; return true;
    case RGCN_X_REL2_NORM: v = {g->by_rel_src.d_norm, M4}; return true;
    case RGCN_X_REL2_MID: v = {g->by_rel_src.d_mid, M4}; return g->keep_mid;
    default: return false;
  }
}
}  // namespace

extern "C" int64_t rgcn_graph_export_bytes(const rgcn_graph_t* g, int which) {
  View v;
  if (g && g->built_on_device) {
    if (!pick_device(g, which, v)) {
      rgcn_set_error("rgcn_graph_export_bytes: bad selector (or message ids not kept for this graph)");
      return RGCN_ERR_INVALID;
    }
    return v.n;
  }
  if (!g || !pick(g, which, v)) {
    rgcn_set_error("rgcn_graph_export_bytes: bad handle or selector");
    return RGCN_ERR_INVALID;
  }
  return v.n;
}

extern "C" int rgcn_graph_export(const rgcn_graph_t* g, int which, void* dst_host, int64_t nbytes) {
  View v;
  if (g && dst_host && g->built_on_device) {
    if (!pick_device(g, which, v) || nbytes < v.n) {
      rgcn_set_error("rgcn_graph_export: bad selector or destination too small");
      return RGCN_ERR_INVALID;
    }
    cudaSetDevice(g->device);
    if (v.n == 0) return RGCN_OK;
    return rgcn_check_cuda(cudaMemcpy(dst_host, v.p, (size_t)v.n, cudaMemcpyDeviceToHost), "export D2H");
  }
  if (!g || !dst_host || !pick(g, which, v)) {
    rgcn_set_error("rgcn_graph_export: bad handle, selector or destination");
    return RGCN_ERR_INVALID;
  }
  if (nbytes < v.n) {
    rgcn_set_error("rgcn_graph_export: destination too small");
    return RGCN_ERR_INVALID;
  }
  if (v.n) std::memcpy(dst_host, v.p, (size_t)v.n);
  return RGCN_OK;
}
