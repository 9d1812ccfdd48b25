// pna_csr_build: edge list -> destination-sorted CSR + hub chunk plan.
//
// What torch_scatter does implicitly on every call (scatter by edge_index[1]; reference
// models/pytorch_geometric/pna.py:153,157) is done here ONCE per graph: a stable LSD radix sort of
// (dst, edge id) pairs over only ceil(log2 N) key bits, a binary-search row pointer, and a one-pass plan of the
// rows that are long enough to be split across warps.  Stability keeps the slots of a row in original edge order,
// which is the accumulation order of the reference's CPU scatter_add.
#include "common.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

namespace pna {

struct Counters {  // device-side, copied back once at the end of the build
  int n_hubs, n_chunks, max_degree, err, hot;
};

// ---- share of the gathers that go to frequent source rows (decides PNA_FLAG_GATHER_L1) ---------------------------------------
// n_sample evenly spaced CSR slots are counted into a small hash table; a sampled slot is "hot" when its source was seen at
// least 4 times, i.e. receives more than about E / (n_sample / 4) gathers.  An estimate: collisions and sampling noise move it
// by a percent, the graphs it has to tell apart differ by 0.9.
__device__ __forceinline__ unsigned hot_hash(int v, unsigned mask) { return ((unsigned)v * 2654435761u >> 7) & mask; }
__global__ void k_hot_count(const int* __restrict__ col, long long E, int n_sample, unsigned mask, int* __restrict__ table) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_sample) return;
  atomicAdd(table + hot_hash(__ldg(col + (long long)i * (E / n_sample)), mask), 1);
}
__global__ void k_hot_sum(const int* __restrict__ col, long long E, int n_sample, unsigned mask, const int* __restrict__ table,
                          Counters* ctr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int hot = 0;
  if (i < n_sample) hot = table[hot_hash(__ldg(col + (long long)i * (E / n_sample)), mask)] >= 4;
  const unsigned m = __ballot_sync(0xffffffffu, hot);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&ctr->hot, __popc(m));
}

__global__ void k_prepare_keys(const long long* __restrict__ src, const long long* __restrict__ dst, int E, long long N,
                               long long NS, int* __restrict__ keys, int* __restrict__ vals, Counters* ctr) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const long long d = dst[e], s = src[e];
  const bool bad = d < 0 || d >= N || s < 0 || s >= NS;
  if (bad) atomicOr(&ctr->err, 1);
  keys[e] = bad ? 0 : (int)d;
  vals[e] = e;
}

__global__ void k_fill_col(const long long* __restrict__ src, const int* __restrict__ perm, int E, long long N,
                           int* __restrict__ col) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= E) return;
  const long long s = src[perm[i]];
  col[i] = (s < 0 || s >= N) ? 0 : (int)s;
}

// rowptr[r] = number of sorted keys < r  (lower bound), r in [0, N]
__global__ void k_rowptr(const int* __restrict__ keys, int E, long long N, int* __restrict__ rowptr) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r > N) return;
  int lo = 0, hi = E;
  while (lo < hi) {
    const int mid = (int)(((long long)lo + hi) >> 1);
    if ((long long)keys[mid] < r) lo = mid + 1; else hi = mid;
  }
  rowptr[r] = lo;
}

__global__ void k_plan_hubs(const int* __restrict__ rowptr, long long N, int split, int chunk, int* __restrict__ hub_info,
                            int* __restrict__ chunk_items, long long cap_hubs, long long cap_chunks, Counters* ctr) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  int deg = 0;
  if (r < N) deg = rowptr[r + 1] - rowptr[r];
  // one atomicMax per warp
  int m = deg;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0 && m > 0) atomicMax(&ctr->max_degree, m);
  if (r >= N || deg < split) return;
  const int nch = (deg + chunk - 1) / chunk;
  const int h = atomicAdd(&ctr->n_hubs, 1);
  const int first = atomicAdd(&ctr->n_chunks, nch);
  if (h >= cap_hubs || (long long)first + nch > cap_chunks) { atomicOr(&ctr->err, 2); return; }
  hub_info[4 * h + 0] = (int)r;
  hub_info[4 * h + 1] = first;
  hub_info[4 * h + 2] = nch;
  hub_info[4 * h + 3] = deg;
  for (int j = 0; j < nch; ++j) {
    chunk_items[2 * (first + j) + 0] = h;
    chunk_items[2 * (first + j) + 1] = j;
  }
}

// A view has N real rows followed by (optionally) one pseudo-row per chunk of a split row: the chunk's slots are
// reduced by the same streaming kernel into fp32 partials instead of a finished output row.
struct ChunkRows {
  const int* hub_info;     // [4*h]: row, first chunk, n chunks, degree
  const int* chunk_items;  // [2*c]: hub, chunk-in-hub
  const int* n_chunks;     // device counter (number of valid chunk rows), NULL = no chunk rows in this view
  int chunk;               // slots per chunk
};

__device__ __forceinline__ int chunk_row_slots(const ChunkRows& cr, int c, int* first_slot_of_row, const int* rowptr) {
  const int h = cr.chunk_items[2 * c], j = cr.chunk_items[2 * c + 1];
  const int row = cr.hub_info[4 * h], deg = cr.hub_info[4 * h + 3];
  if (first_slot_of_row) *first_slot_of_row = rowptr[row] + j * cr.chunk;
  return min(cr.chunk, deg - j * cr.chunk);
}

// light view, step 1: deg (or -1 for split / masked-out rows) and the scan input max(deg, 0); scan_in[NV] = 0
__global__ void k_light_deg(const int* __restrict__ rowptr, long long N, long long NV, int split, const unsigned char* __restrict__ mask,
                            ChunkRows cr, int* __restrict__ light_deg, int* __restrict__ scan_in) {
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v > NV) return;
  if (v == NV) { scan_in[v] = 0; return; }
  const int M = cr.n_chunks ? *cr.n_chunks : 0;
  const ViewMap vm = {N, M};
  if (v >= vm.rows()) { light_deg[v] = -1; scan_in[v] = 0; return; }   // unused capacity
  const long long r = vm.to_row(v);
  int d;
  bool skip;
  if (r < N) {
    d = rowptr[r + 1] - rowptr[r];
    skip = d >= split || (mask && !mask[r]);
  } else {
    const int c = (int)(r - N);
    skip = false;
    d = chunk_row_slots(cr, c, nullptr, rowptr);
  }
  light_deg[v] = skip ? -1 : d;
  scan_in[v] = skip ? 0 : d;
}

// light view, step 2: one group of 8 lanes per view row copies the row's sources to their compacted position
__global__ void k_light_col(const int* __restrict__ rowptr, const int* __restrict__ light_rowptr, const int* __restrict__ light_deg,
                            const int* __restrict__ col, long long N, long long NV, ChunkRows cr, int* __restrict__ light_col) {
  const long long v = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  if (v >= NV) return;
  const int d = light_deg[v];
  if (d <= 0) return;
  const ViewMap vm = {N, cr.n_chunks ? *cr.n_chunks : 0};
  const long long r = vm.to_row(v);
  int first;
  if (r < N) first = rowptr[r];
  else chunk_row_slots(cr, (int)(r - N), &first, rowptr);
  const int* __restrict__ s = col + first;
  int* __restrict__ t = light_col + light_rowptr[v];
  for (int i = threadIdx.x & 7; i < d; i += 8) t[i] = s[i];
}

// equal-cost partition boundaries over the NV' = N + n_chunks valid view rows:
// part[i] = smallest row r with cost(r) >= i * cost(NV') / P, cost(r) = slots before r + 12 r
__global__ void k_partition(const int* __restrict__ light_rowptr, long long N, const int* __restrict__ n_chunks, int P,
                            int* __restrict__ part) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > P) return;
  const long long NV = N + (n_chunks ? *n_chunks : 0);
  if (i == P) { part[i] = (int)NV; return; }
  const long long total = (long long)light_rowptr[NV] + 12ll * NV;
  const long long target = (total * i) / P;
  long long lo = 0, hi = NV;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if ((long long)light_rowptr[mid] + 12ll * mid < target) lo = mid + 1; else hi = mid;
  }
  part[i] = (int)lo;
}

static int key_bits(long long N) {
  int b = 1;
  while (b < 31 && (1ll << b) < N) ++b;
  return b;
}

struct WsLayout {
  size_t keys_in, keys_out, vals_in, counters, cub_temp, cub_bytes, total;
};
// keys_in / vals_in are reused after the sort as the light-view scan input (needs N+1 ints), hence max(E, N+1).

static int ws_layout(long long N, long long E, WsLayout* L) {
  size_t cub_bytes = 0, scan_bytes = 0;
  const int n = (int)(E > 0 ? E : 1);
  PNA_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, (const int*)nullptr, (int*)nullptr, (const int*)nullptr,
                                                (int*)nullptr, n, 0, key_bits(N)));
  const long long scan_n = N + 2 * E + 4;   // view rows: N real + up to E/chunk + E/split + 2 chunk rows, + 1
  PNA_REQUIRE(scan_n < 0x7fffffffll, PNA_ERR_UNSUPPORTED, "pna_csr_build: graph too large for the int32 view scan");
  PNA_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const int*)nullptr, (int*)nullptr, (int)scan_n));
  if (scan_bytes > cub_bytes) cub_bytes = scan_bytes;
  size_t off = 0;
  const size_t eb = align_up((size_t)((long long)n > scan_n ? (long long)n : scan_n) * sizeof(int), 256);
  L->keys_in = off; off += eb;
  L->keys_out = off; off += eb;
  L->vals_in = off; off += eb;
  L->counters = off; off += 256;
  L->cub_temp = off; off += align_up(cub_bytes, 256);
  L->cub_bytes = cub_bytes;
  L->total = off;
  return PNA_OK;
}

// light view of the rows selected by `mask` (NULL = all rows below the split threshold) plus, when cr.n_chunks is set,
// one pseudo-row per chunk of the split rows; cap_view = N + chunk-row capacity; scan_in: cap_view+1 ints of scratch
static int light_view(const int* rowptr, const int* col, long long N, long long cap_view, int split, const unsigned char* mask,
                      ChunkRows cr, int n_part, int* light_rowptr, int* light_deg, int* light_col, int* part, int* scan_in,
                      void* cub_temp, size_t cub_bytes, cudaStream_t st) {
  const int TB = 256;
  k_light_deg<<<(unsigned)((cap_view + 1 + TB - 1) / TB), TB, 0, st>>>(rowptr, N, cap_view, split, mask, cr, light_deg, scan_in);
  PNA_CUDA_TRY(cudaGetLastError());
  PNA_CUDA_TRY(cub::DeviceScan::ExclusiveSum(cub_temp, cub_bytes, (const int*)scan_in, light_rowptr, (int)(cap_view + 1), st));
  if (cap_view > 0 && col != nullptr) {
    k_light_col<<<(unsigned)((cap_view * 8 + TB - 1) / TB), TB, 0, st>>>(rowptr, light_rowptr, light_deg, col, N, cap_view, cr, light_col);
    PNA_CUDA_TRY(cudaGetLastError());
  }
  k_partition<<<(unsigned)((n_part + 1 + TB - 1) / TB), TB, 0, st>>>(light_rowptr, N, cr.n_chunks, n_part, part);
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}

// ---- padded build (pna_csr_build_padded): fixed capacities, nothing read back -------------------------------------------------
// status[0] error bits, [1] real edges, [2] max in-degree, [3] reserved
__global__ void k_prepare_keys_padded(const long long* __restrict__ src, const long long* __restrict__ dst, int E, long long N,
                                      long long NS, int* __restrict__ keys, int* __restrict__ vals, int* __restrict__ status) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const long long d = dst[e], s = src[e];
  const bool pad = d == -1;
  const bool bad = !pad && (d < 0 || d >= N || s < 0 || s >= NS);
  if (bad) atomicOr(status, 1);
  keys[e] = (pad || bad) ? (int)N : (int)d;     // padding and dropped edges sort behind every row
  vals[e] = e;
}

// padding slots rowptr[N]..E-1 get col 0; max in-degree and the real-edge count go to the status word
__global__ void k_padded_finish(const int* __restrict__ rowptr, long long N, int E, int* __restrict__ col, int* __restrict__ status) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int real = rowptr[N];
  if (i < E && i >= real) col[i] = 0;
  int deg = 0;
  if (i < N) deg = rowptr[i + 1] - rowptr[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) deg = max(deg, __shfl_xor_sync(0xffffffffu, deg, o));
  if ((threadIdx.x & 31) == 0 && deg > 0) atomicMax(status + 2, deg);
  if (i == 0) status[1] = real;
}

// per slot: the slot-transposed build's destination key (col, or -1 = padding) and the row that owns the slot (0 = padding)
__global__ void k_slot_rows(const int* __restrict__ rowptr, const int* __restrict__ col, long long N, int E,
                            long long* __restrict__ transpose_dst, long long* __restrict__ dst_of_slot) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= E) return;
  if (s >= rowptr[N]) { transpose_dst[s] = -1; dst_of_slot[s] = 0; return; }
  long long lo = 0, hi = N;     // the last row r with rowptr[r] <= s
  while (lo < hi) {
    const long long mid = (lo + hi + 1) >> 1;
    if (rowptr[mid] <= s) lo = mid; else hi = mid - 1;
  }
  transpose_dst[s] = col[s];
  dst_of_slot[s] = lo;
}

// Building per-graph state reads counters back (pna_csr_build) and belongs before a CUDA graph capture, not in it: on a
// capturing stream both builders return PNA_ERR_CAPTURING before anything is enqueued, so the capture stays intact.
static int refuse_capture(cudaStream_t st, const char* who) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  PNA_CUDA_TRY(cudaStreamIsCapturing(st, &cs));
  PNA_REQUIRE(cs == cudaStreamCaptureStatusNone, PNA_ERR_CAPTURING,
              "%s: the stream is capturing a CUDA graph; build the graph's CSR and views before the capture", who);
  return PNA_OK;
}

}  // namespace pna

using namespace pna;

extern "C" int pna_csr_light_view(const int32_t* rowptr, const int32_t* col, int64_t n_nodes, int32_t split_threshold,
                                  const uint8_t* row_mask, int32_t n_part, int32_t* light_rowptr, int32_t* light_deg,
                                  int32_t* light_col, int32_t* part, void* workspace, size_t workspace_bytes, pna_stream_t stream) {
  PNA_REQUIRE(n_nodes >= 0 && n_nodes < 0x7fffffffll && split_threshold >= 2 && n_part >= 1, PNA_ERR_BAD_ARG,
              "pna_csr_light_view: bad sizes");
  PNA_REQUIRE(rowptr && light_rowptr && light_deg && part, PNA_ERR_BAD_ARG, "pna_csr_light_view: null pointer");
  size_t scan_bytes = 0;
  PNA_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const int*)nullptr, (int*)nullptr, (int)(n_nodes + 1)));
  const size_t scan_in_bytes = align_up((size_t)(n_nodes + 1) * sizeof(int), 256);
  const size_t need = scan_in_bytes + align_up(scan_bytes, 256);
  PNA_REQUIRE(workspace != nullptr && workspace_bytes >= need, PNA_ERR_WORKSPACE, "pna_csr_light_view: workspace %zu bytes < required %zu", workspace_bytes, need);
  const int rc = refuse_capture(static_cast<cudaStream_t>(stream), "pna_csr_light_view");
  if (rc != PNA_OK) return rc;
  char* ws = static_cast<char*>(workspace);
  ChunkRows none = {nullptr, nullptr, nullptr, 1};
  return light_view(rowptr, col, n_nodes, n_nodes, split_threshold, row_mask, none, n_part, light_rowptr, light_deg, light_col, part,
                    reinterpret_cast<int*>(ws), ws + scan_in_bytes, scan_bytes, static_cast<cudaStream_t>(stream));
}

extern "C" int pna_csr_light_view_workspace_bytes(int64_t n_nodes, size_t* bytes) {
  PNA_REQUIRE(bytes != nullptr && n_nodes >= 0 && n_nodes < 0x7fffffffll, PNA_ERR_BAD_ARG, "pna_csr_light_view_workspace_bytes: bad argument");
  size_t scan_bytes = 0;
  PNA_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const int*)nullptr, (int*)nullptr, (int)(n_nodes + 1)));
  *bytes = align_up((size_t)(n_nodes + 1) * sizeof(int), 256) + align_up(scan_bytes, 256);
  return PNA_OK;
}

extern "C" int pna_csr_workspace_bytes(int64_t n_nodes, int64_t n_edges, size_t* bytes) {
  PNA_REQUIRE(bytes != nullptr, PNA_ERR_BAD_ARG, "pna_csr_workspace_bytes: null out pointer");
  PNA_REQUIRE(n_nodes >= 0 && n_edges >= 0, PNA_ERR_BAD_ARG, "pna_csr_workspace_bytes: negative size");
  PNA_REQUIRE(n_nodes < 0x7fffffffll && n_edges < 0x7fffffffll, PNA_ERR_UNSUPPORTED,
              "pna_csr_workspace_bytes: n_nodes/n_edges must be < 2^31 (int32 CSR)");
  WsLayout L;
  const int rc = ws_layout(n_nodes, n_edges, &L);
  if (rc != PNA_OK) return rc;
  *bytes = L.total;
  return PNA_OK;
}

extern "C" int pna_csr_build(const int64_t* src, const int64_t* dst, pna_csr_t* csr, void* workspace, size_t workspace_bytes,
                             pna_stream_t stream) {
  PNA_REQUIRE(csr != nullptr, PNA_ERR_BAD_ARG, "pna_csr_build: null csr");
  const long long N = csr->n_nodes, E = csr->n_edges;
  const long long NS = csr->n_src_nodes > 0 ? csr->n_src_nodes : N;   // bipartite: sources may include halo rows
  PNA_REQUIRE(N >= 0 && E >= 0, PNA_ERR_BAD_ARG, "pna_csr_build: negative size");
  PNA_REQUIRE(N < 0x7fffffffll && E < 0x7fffffffll && NS < 0x7fffffffll, PNA_ERR_UNSUPPORTED,
              "pna_csr_build: n_nodes/n_src_nodes/n_edges must be < 2^31");
  PNA_REQUIRE(csr->split_threshold >= 2 && csr->chunk_edges >= 1 && csr->chunk_edges <= csr->split_threshold, PNA_ERR_BAD_ARG,
              "pna_csr_build: need split_threshold >= 2 and 1 <= chunk_edges <= split_threshold");
  PNA_REQUIRE(csr->rowptr != nullptr, PNA_ERR_BAD_ARG, "pna_csr_build: null rowptr");
  PNA_REQUIRE(E == 0 || (src && dst && csr->col && csr->perm), PNA_ERR_BAD_ARG, "pna_csr_build: null src/dst/col/perm");
  PNA_REQUIRE(csr->cap_hubs >= E / csr->split_threshold + 1, PNA_ERR_WORKSPACE, "pna_csr_build: cap_hubs too small");
  PNA_REQUIRE(csr->cap_chunks >= E / csr->chunk_edges + csr->cap_hubs + 1, PNA_ERR_WORKSPACE, "pna_csr_build: cap_chunks too small");
  PNA_REQUIRE(csr->hub_info && csr->chunk_items, PNA_ERR_BAD_ARG, "pna_csr_build: null hub_info/chunk_items");
  // the view scan runs over n_nodes + cap_chunks + 1 entries of workspace sized for n_nodes + 2 * n_edges + 4 (ws_layout)
  PNA_REQUIRE(csr->light_rowptr == nullptr || csr->cap_chunks <= 2 * E + 3, PNA_ERR_BAD_ARG,
              "pna_csr_build: cap_chunks %lld exceeds 2 * n_edges + 3 (the light view could not be scanned in the workspace)",
              (long long)csr->cap_chunks);
  WsLayout L;
  int rc = ws_layout(N, E, &L);
  if (rc != PNA_OK) return rc;
  PNA_REQUIRE(workspace != nullptr && workspace_bytes >= L.total, PNA_ERR_WORKSPACE,
              "pna_csr_build: workspace %zu bytes < required %zu", workspace_bytes, L.total);
  PNA_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255u) == 0, PNA_ERR_BAD_ARG, "pna_csr_build: workspace must be 256-byte aligned");
  rc = refuse_capture(static_cast<cudaStream_t>(stream), "pna_csr_build");     // after the argument checks, before any work
  if (rc != PNA_OK) return rc;

  cudaStream_t st = static_cast<cudaStream_t>(stream);
  char* ws = static_cast<char*>(workspace);
  int* keys_in = reinterpret_cast<int*>(ws + L.keys_in);
  int* keys_out = reinterpret_cast<int*>(ws + L.keys_out);
  int* vals_in = reinterpret_cast<int*>(ws + L.vals_in);
  Counters* ctr = reinterpret_cast<Counters*>(ws + L.counters);
  PNA_CUDA_TRY(cudaMemsetAsync(ctr, 0, sizeof(Counters), st));

  const int TB = 256;
  if (E > 0) {
    const int nE = (int)E;
    const unsigned gE = (unsigned)((E + TB - 1) / TB);
    k_prepare_keys<<<gE, TB, 0, st>>>(reinterpret_cast<const long long*>(src), reinterpret_cast<const long long*>(dst), nE, N, NS,
                                      keys_in, vals_in, ctr);
    PNA_CUDA_TRY(cudaGetLastError());
    size_t cub_bytes = L.cub_bytes;
    PNA_CUDA_TRY(cub::DeviceRadixSort::SortPairs(ws + L.cub_temp, cub_bytes, (const int*)keys_in, keys_out, (const int*)vals_in,
                                                  csr->perm, nE, 0, key_bits(N), st));
    k_fill_col<<<gE, TB, 0, st>>>(reinterpret_cast<const long long*>(src), csr->perm, nE, NS, csr->col);
    PNA_CUDA_TRY(cudaGetLastError());
  }
  {
    const unsigned gN = (unsigned)((N + 1 + TB - 1) / TB);
    k_rowptr<<<gN, TB, 0, st>>>(keys_out, (int)E, N, csr->rowptr);
    PNA_CUDA_TRY(cudaGetLastError());
    if (N > 0) {
      const unsigned gP = (unsigned)((N + TB - 1) / TB);
      k_plan_hubs<<<gP, TB, 0, st>>>(csr->rowptr, N, csr->split_threshold, csr->chunk_edges, csr->hub_info, csr->chunk_items,
                                     csr->cap_hubs, csr->cap_chunks, ctr);
      PNA_CUDA_TRY(cudaGetLastError());
    }
  }
  // hot-source estimate: keys_out is free once the row pointer exists; the table is the largest power of two it can hold
  int n_sample = 0;
  if (E >= 4096) {
    n_sample = E < 65536 ? (int)E : 65536;
    unsigned tsize = 131072;
    while ((size_t)tsize * sizeof(int) > (size_t)E * sizeof(int)) tsize >>= 1;    // keys_out holds >= E ints
    PNA_CUDA_TRY(cudaMemsetAsync(keys_out, 0, (size_t)tsize * sizeof(int), st));
    k_hot_count<<<(unsigned)((n_sample + TB - 1) / TB), TB, 0, st>>>(csr->col, E, n_sample, tsize - 1, keys_out);
    k_hot_sum<<<(unsigned)((n_sample + TB - 1) / TB), TB, 0, st>>>(csr->col, E, n_sample, tsize - 1, keys_out, ctr);
    PNA_CUDA_TRY(cudaGetLastError());
  }
  int n_light = 0;
  if (csr->light_rowptr) {   // light view (optional: all four arrays or none)
    PNA_REQUIRE(csr->light_deg && csr->part && (E == 0 || csr->light_col) && csr->n_part >= 1, PNA_ERR_BAD_ARG,
                "pna_csr_build: light view needs light_rowptr, light_deg, light_col, part and n_part >= 1");
    // the view carries one pseudo-row per chunk of the split rows (capacity cap_chunks; n_chunks of them are valid)
    const long long cap_view = N + csr->cap_chunks;
    ChunkRows cr = {csr->hub_info, csr->chunk_items, &ctr->n_chunks, csr->chunk_edges};
    rc = light_view(csr->rowptr, csr->col, N, cap_view, csr->split_threshold, nullptr, cr, csr->n_part, csr->light_rowptr,
                    csr->light_deg, csr->light_col, csr->part, keys_in, ws + L.cub_temp, L.cub_bytes, st);
    if (rc != PNA_OK) return rc;
    PNA_CUDA_TRY(cudaMemcpyAsync(&n_light, csr->light_rowptr + cap_view, sizeof(int), cudaMemcpyDeviceToHost, st));
  }
  Counters host;
  PNA_CUDA_TRY(cudaMemcpyAsync(&host, ctr, sizeof(Counters), cudaMemcpyDeviceToHost, st));
  PNA_CUDA_TRY(cudaStreamSynchronize(st));
  PNA_REQUIRE(!(host.err & 1), PNA_ERR_INDEX, "pna_csr_build: edge endpoint outside dst [0, %lld) / src [0, %lld)", N, NS);
  PNA_REQUIRE(!(host.err & 2), PNA_ERR_WORKSPACE, "pna_csr_build: hub/chunk capacity exceeded");
  csr->n_hubs = host.n_hubs;
  csr->n_chunks = host.n_chunks;
  csr->max_degree = host.max_degree;
  csr->n_light_edges = n_light;
  csr->hot_source_fraction = n_sample ? (float)host.hot / (float)n_sample : 0.0f;
  return PNA_OK;
}

extern "C" int pna_csr_padded_workspace_bytes(int64_t n_nodes, int64_t n_edges, size_t* bytes) {
  PNA_REQUIRE(bytes != nullptr, PNA_ERR_BAD_ARG, "pna_csr_padded_workspace_bytes: null out pointer");
  PNA_REQUIRE(n_nodes >= 0 && n_edges >= 0, PNA_ERR_BAD_ARG, "pna_csr_padded_workspace_bytes: negative size");
  PNA_REQUIRE(n_nodes < 0x7ffffffell && n_edges < 0x7fffffffll, PNA_ERR_UNSUPPORTED,
              "pna_csr_padded_workspace_bytes: n_nodes + 1 and n_edges must be < 2^31");
  WsLayout L;
  const int rc = ws_layout(n_nodes + 1, n_edges, &L);     // keys 0..N: the padding sorts under the sentinel N
  if (rc != PNA_OK) return rc;
  *bytes = L.total;
  return PNA_OK;
}

extern "C" int pna_csr_build_padded(const int64_t* src, const int64_t* dst, pna_csr_t* csr, int32_t* status, void* workspace,
                                    size_t workspace_bytes, pna_stream_t stream) {
  PNA_REQUIRE(csr != nullptr && status != nullptr, PNA_ERR_BAD_ARG, "pna_csr_build_padded: null csr/status");
  const long long N = csr->n_nodes, E = csr->n_edges;
  const long long NS = csr->n_src_nodes > 0 ? csr->n_src_nodes : N;
  PNA_REQUIRE(N >= 0 && E >= 0, PNA_ERR_BAD_ARG, "pna_csr_build_padded: negative size");
  PNA_REQUIRE(N < 0x7ffffffell && E < 0x7fffffffll && NS < 0x7fffffffll, PNA_ERR_UNSUPPORTED,
              "pna_csr_build_padded: n_nodes + 1, n_src_nodes and n_edges must be < 2^31");
  PNA_REQUIRE(csr->split_threshold >= 2 && (long long)csr->split_threshold > E, PNA_ERR_BAD_ARG,
              "pna_csr_build_padded: split_threshold %d must exceed n_edges %lld (a padded CSR has no split rows)",
              (int)csr->split_threshold, E);
  PNA_REQUIRE(csr->rowptr != nullptr, PNA_ERR_BAD_ARG, "pna_csr_build_padded: null rowptr");
  PNA_REQUIRE(E == 0 || (src && dst && csr->col && csr->perm), PNA_ERR_BAD_ARG, "pna_csr_build_padded: null src/dst/col/perm");
  PNA_REQUIRE(csr->light_rowptr == nullptr || (csr->light_deg && csr->part && (E == 0 || csr->light_col) && csr->n_part >= 1),
              PNA_ERR_BAD_ARG, "pna_csr_build_padded: light view needs light_rowptr, light_deg, light_col, part and n_part >= 1");
  WsLayout L;
  int rc = ws_layout(N + 1, E, &L);
  if (rc != PNA_OK) return rc;
  PNA_REQUIRE(workspace != nullptr && workspace_bytes >= L.total, PNA_ERR_WORKSPACE,
              "pna_csr_build_padded: workspace %zu bytes < required %zu", workspace_bytes, L.total);
  PNA_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 255u) == 0, PNA_ERR_BAD_ARG,
              "pna_csr_build_padded: workspace must be 256-byte aligned");

  cudaStream_t st = static_cast<cudaStream_t>(stream);
  char* ws = static_cast<char*>(workspace);
  int* keys_in = reinterpret_cast<int*>(ws + L.keys_in);
  int* keys_out = reinterpret_cast<int*>(ws + L.keys_out);
  int* vals_in = reinterpret_cast<int*>(ws + L.vals_in);
  PNA_CUDA_TRY(cudaMemsetAsync(status, 0, 4 * sizeof(int32_t), st));
  const int TB = 256;
  if (E > 0) {
    const int nE = (int)E;
    const unsigned gE = (unsigned)((E + TB - 1) / TB);
    k_prepare_keys_padded<<<gE, TB, 0, st>>>(reinterpret_cast<const long long*>(src), reinterpret_cast<const long long*>(dst), nE,
                                             N, NS, keys_in, vals_in, status);
    PNA_CUDA_TRY(cudaGetLastError());
    size_t cub_bytes = L.cub_bytes;
    PNA_CUDA_TRY(cub::DeviceRadixSort::SortPairs(ws + L.cub_temp, cub_bytes, (const int*)keys_in, keys_out, (const int*)vals_in,
                                                  csr->perm, nE, 0, key_bits(N + 1), st));
    k_fill_col<<<gE, TB, 0, st>>>(reinterpret_cast<const long long*>(src), csr->perm, nE, NS, csr->col);
    PNA_CUDA_TRY(cudaGetLastError());
  }
  k_rowptr<<<(unsigned)((N + 1 + TB - 1) / TB), TB, 0, st>>>(keys_out, (int)E, N, csr->rowptr);
  PNA_CUDA_TRY(cudaGetLastError());
  const long long n_fin = N > E ? N : E;
  k_padded_finish<<<(unsigned)((n_fin + TB) / TB), TB, 0, st>>>(csr->rowptr, N, (int)E, csr->col, status);
  PNA_CUDA_TRY(cudaGetLastError());
  if (csr->light_rowptr) {
    ChunkRows none = {nullptr, nullptr, nullptr, 1};
    rc = light_view(csr->rowptr, csr->col, N, N, csr->split_threshold, nullptr, none, csr->n_part, csr->light_rowptr,
                    csr->light_deg, csr->light_col, csr->part, keys_in, ws + L.cub_temp, L.cub_bytes, st);
    if (rc != PNA_OK) return rc;
  }
  csr->n_hubs = 0;
  csr->n_chunks = 0;
  csr->max_degree = 0;        // on the device: status[2]
  csr->n_light_edges = 0;     // on the device: status[1] (= light_rowptr[n_nodes])
  csr->hot_source_fraction = 0.0f;
  return PNA_OK;
}

extern "C" int pna_csr_slot_rows(const int32_t* rowptr, const int32_t* col, int64_t n_rows, int64_t n_slots, int64_t* transpose_dst,
                                 int64_t* dst_of_slot, pna_stream_t stream) {
  PNA_REQUIRE(n_rows >= 0 && n_slots >= 0 && n_rows < 0x7fffffffll && n_slots < 0x7fffffffll, PNA_ERR_BAD_ARG,
              "pna_csr_slot_rows: bad sizes");
  if (n_slots == 0) return PNA_OK;
  PNA_REQUIRE(rowptr && col && transpose_dst && dst_of_slot, PNA_ERR_BAD_ARG, "pna_csr_slot_rows: null pointer");
  const int TB = 256;
  k_slot_rows<<<(unsigned)((n_slots + TB - 1) / TB), TB, 0, static_cast<cudaStream_t>(stream)>>>(
      rowptr, col, n_rows, (int)n_slots, reinterpret_cast<long long*>(transpose_dst), reinterpret_cast<long long*>(dst_of_slot));
  PNA_CUDA_TRY(cudaGetLastError());
  return PNA_OK;
}
