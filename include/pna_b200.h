/*
 * pna_b200.h -- C ABI of libpna_sm90.so, the H100 (sm_90a) PNA aggregation path.
 *
 * This is the drop-in boundary for ONE hot path of lukecavabarrett/pna: the
 * neighbourhood aggregation of the PNA layer (gather of source features, the
 * simultaneous mean/max/min/std(/sum/var) aggregators, the degree scalers, the
 * concatenated [N, S*A*F] result).  Plain pointers and sizes only; every buffer
 * is owned by the caller (PyTorch in this repo); all pointers are DEVICE pointers
 * unless stated otherwise; every call enqueues on the caller's stream.
 *
 * Reference interfaces replaced (paths relative to the reference checkout):
 *   models/pytorch_geometric/pna.py:152-159, :242-249   PNAConv(.Simple).aggregate
 *   models/pytorch_geometric/aggregators.py:9-32        scatter sum/mean/min/max/var/std
 *   models/pytorch_geometric/scalers.py:8-29            identity/amplification/attenuation/linear/inverse_linear
 *   models/dgl/pna_layer.py:45-50, :189-194             PNATower.reduce_func / PNASimpleLayer.reduce_func
 *   models/dgl/aggregators.py:6-26, models/dgl/scalers.py:8-19
 *   torch_geometric MessagePassing.propagate gather of x_j (pna.py:129, :236)
 *
 * Return value of every int function: 0 = ok, negative = pna_status.
 * pna_last_error() gives a thread-local human-readable message for the last failure.
 */
#ifndef PNA_B200_H
#define PNA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PNA_ABI_VERSION 8

typedef void* pna_stream_t; /* a cudaStream_t / CUstream, passed opaquely */

enum pna_status {
  PNA_OK = 0,
  PNA_ERR_BAD_ARG = -1,     /* null pointer, negative size, inconsistent descriptor */
  PNA_ERR_UNSUPPORTED = -2, /* dtype / size outside what the kernels take (e.g. E >= 2^31) */
  PNA_ERR_CUDA = -3,        /* a CUDA runtime call failed; message carries cudaGetErrorString */
  PNA_ERR_INDEX = -4,       /* an edge endpoint outside [0, n_nodes) was found while building the CSR */
  PNA_ERR_WORKSPACE = -5,   /* caller-provided workspace / capacity too small */
  PNA_ERR_CAPTURING = -6    /* the stream is capturing a CUDA graph and the call would synchronise or read back; nothing
                               was enqueued (pna_csr_build, pna_csr_light_view: build per-graph state before the capture) */
};

enum pna_dtype { PNA_F32 = 0, PNA_BF16 = 1 };

/* Aggregator codes (order of appearance in the layer's ctor list fixes the column layout,
 * pna.py:70,153-154).  Packed 4 bits each, first aggregator in the low nibble. */
enum pna_aggr { PNA_AGGR_SUM = 0, PNA_AGGR_MEAN = 1, PNA_AGGR_MIN = 2, PNA_AGGR_MAX = 3, PNA_AGGR_VAR = 4, PNA_AGGR_STD = 5,
                /* central moments of order 3, 4, 5 (models/pytorch/pna/aggregators.py:122-146):
                     mu = sum / d,  M_k = (sum over slots of (m - mu)^k) / d,  r_k = sign(M_k) (|M_k| + 1e-5)^(1/k),  d == 0: 0.
                   Taken by pna_aggregate_fwd, pna_aggregate_bwd and pna_aggregate_bwd_slots; pna_aggregate_bwd_coef and
                   descriptors with peer_gathered or row_ids return PNA_ERR_UNSUPPORTED for them.  Rows at/above the split
                   threshold are merged in fixed chunk order (no atomics).  Rounding order: pna_b200/csrc/pna_aggregate_moments.cuh */
                PNA_AGGR_MOMENT3 = 6, PNA_AGGR_MOMENT4 = 7, PNA_AGGR_MOMENT5 = 8,
                /* weighted sums y = sum over slots of w_s m_s (models/pytorch/pna/aggregators.py:87-119), d == 0: 0:
                     softmax:          w_s = exp(m_s - M) / Z,  M = max m,  Z = sum exp(m_t - M)
                     softmin:          w_s = exp(M' - m_s) / Z', M' = min m (the reference's -softmax(-m))
                     normalised_mean:  w_s = D_i^(-1/2) D_j^(-1/2), j = col[s] (or degree_col[s] when given),
                                       D_k = rowptr[k+1] - rowptr[k] of the SAME CSR (0 weight where D_j == 0 or
                                       j >= n_rows); needs col != NULL or degree_col != NULL.
                   Taken by pna_aggregate_fwd, pna_aggregate_bwd and pna_aggregate_bwd_slots; pna_aggregate_bwd_coef and
                   descriptors with peer_gathered or row_ids return PNA_ERR_UNSUPPORTED for them, as for the moments.
                   Split rows are merged in fixed chunk order (no atomics).  Rounding order:
                   pna_b200/csrc/pna_aggregate_weighted.cuh */
                PNA_AGGR_SOFTMAX = 9, PNA_AGGR_SOFTMIN = 10, PNA_AGGR_NORMALISED_MEAN = 11,
                PNA_AGGR_SKIP = 15 /* keep the column slot but do not write it: lets two calls with different edge
                                       sets / messages fill one output row (dense reference layer, where max/min and
                                       mean/std see different messages: models/pytorch/pna/aggregators.py:30-51) */ };
/* Scaler codes (scalers.py:32-38), packed the same way. */
enum pna_scaler { PNA_SCALE_IDENTITY = 0, PNA_SCALE_AMPLIFICATION = 1, PNA_SCALE_ATTENUATION = 2, PNA_SCALE_LINEAR = 3, PNA_SCALE_INVERSE_LINEAR = 4 };

#define PNA_MAX_AGGR 6
#define PNA_MAX_SCALERS 5

enum pna_flags {
  PNA_FLAG_ZERO_ISOLATED = 1u, /* DGL semantics: a node with no in-edge is never reduced, all its S*A*F columns are 0
                                  (models/dgl/pna_layer.py:64 update_all).  Default (PyG/torch_scatter semantics):
                                  mean=min=max=0, std=sqrt(1e-5), then scaled. */
  PNA_FLAG_SKIP_LIGHT = 2u,    /* do not process rows below the split threshold (used to overlap halo exchange) */
  PNA_FLAG_SKIP_HUBS = 4u,     /* do not process rows at/above the split threshold */
  PNA_FLAG_GATHER_L1 = 16u,    /* hint: a few source rows receive a large share of all gathers (power-law graphs).  The
                                  gathered rows are then also kept in the SMs' L1, so a hot row is not served by the few L2
                                  slices that hold its lines.  Without hot sources the hint costs a few percent.  Honoured by
                                  the streamed kernel for the reference configs' aggregator / scaler lists. */
  PNA_FLAG_RELU_VAR = 8u       /* the "var" aggregator is clamped at 0 (models/dgl/aggregators.py:22-26 and
                                  models/pytorch/pna/aggregators.py:63-76 apply torch.relu; the PyG flavour,
                                  models/pytorch_geometric/aggregators.py:25-28, does not); its gradient is masked where
                                  the raw variance is <= 0 */
};

enum pna_query_what {
  PNA_QUERY_ABI_VERSION = 0,
  PNA_QUERY_SM_ARCH = 1,          /*  90 : compiled for sm_90a only */
  PNA_QUERY_DEFAULT_SPLIT = 2,    /* default in-degree at which a row is split across warps */
  PNA_QUERY_DEFAULT_CHUNK = 3,    /* default edges per chunk of a split row */
  PNA_QUERY_DEVICE_SM_COUNT = 4,  /* multiProcessorCount of the current device (needs a GPU) */
  PNA_QUERY_MAX_FEATURES = 5,     /* largest n_feat accepted by pna_aggregate_fwd */
  PNA_QUERY_SIZEOF_CSR = 6,       /* sizeof(pna_csr_t): lets an FFI binding verify its struct layout */
  PNA_QUERY_SIZEOF_AGG = 7        /* sizeof(pna_agg_t) */
};

/* ---- destination-sorted CSR ("sorts/segments edges by destination in CSR", north_star) ------------------
 * Replaces what torch_scatter does implicitly on every call (scatter by edge_index[1], pna.py:153,157).
 * Edges are ordered by destination, ties kept in original edge order (stable), duplicates and self loops kept:
 *   rowptr[i]..rowptr[i+1]  = CSR slots of the in-edges of node i;  in-degree = difference
 *   col[s]                  = source node of slot s
 *   perm[s]                 = original edge id of slot s (to bring per-edge tensors into CSR order)
 * Rows with in-degree >= split_threshold ("hubs") are additionally listed with a chunking of their slots so the
 * aggregation can spread them over many warps:
 *   hub_info[4*h+0..3]      = row, first chunk id, number of chunks, in-degree
 *   chunk_items[2*c+0..1]   = hub index h, chunk index within the hub
 */
typedef struct pna_csr {
  int64_t n_nodes;          /* in */
  int64_t n_edges;          /* in */
  int32_t split_threshold;  /* in: >= 2 */
  int32_t chunk_edges;      /* in: 1..split_threshold */
  int32_t* rowptr;          /* out [n_nodes+1] */
  int32_t* col;             /* out [n_edges] */
  int32_t* perm;            /* out [n_edges] */
  int32_t* hub_info;        /* out [4*cap_hubs] */
  int32_t* chunk_items;     /* out [2*cap_chunks] */
  int64_t cap_hubs;         /* in: >= n_edges/split_threshold + 1 */
  int64_t cap_chunks;       /* in: >= n_edges/chunk_edges + cap_hubs + 1 (and <= 2*n_edges + 3 when the light view is requested) */
  int64_t n_hubs;           /* out (host) */
  int64_t n_chunks;         /* out (host) */
  int32_t max_degree;       /* out (host) */
  int32_t n_part;           /* in: number of equal-cost row partitions to produce (>= 1) */
  /* "light view": the slots of the rows BELOW the split threshold, compacted so that any contiguous range of rows
   * is a contiguous range of slots -- what lets the streaming kernel treat a warp's rows as one slot stream.
   * Optional: pass light_rowptr == NULL to skip it. */
  /* The view built here has n_nodes + cap_chunks rows: after the real rows comes one PSEUDO-ROW per chunk of the
   * split rows (n_chunks valid), whose slots the same kernel reduces into hub_partials -- so all gathers of a layer
   * call run in one balanced launch. */
  int32_t* light_rowptr;    /* out [n_nodes+cap_chunks+1]: prefix sum of the view rows' slot counts (split rows: 0) */
  int32_t* light_deg;       /* out [n_nodes+cap_chunks]: slot count of each view row, -1 = skip (split row, unused chunk row) */
  int32_t* light_col;       /* out [n_edges]: source node of each view slot (first n_light_edges entries valid) */
  int32_t* part;            /* out [n_part+1]: view-row boundaries of partitions of equal cost (slots + 12 * rows) */
  int64_t n_light_edges;    /* out (host): slots in the view (= n_edges when chunk rows are included) */
  int64_t n_src_nodes;      /* in: sources are validated against [0, n_src_nodes); 0 = n_nodes.  > n_nodes for the
                               destination-partitioned multi-GPU path, where sources index [local rows ; halo rows] */
  float hot_source_fraction; /* out (host): estimated share of the gathers that go to frequent source rows (sampled: sources
                                seen >= 4 times among 65 536 evenly spaced slots).  ~0 for citation / molecule / kNN graphs,
                                ~0.9 for Zipf-distributed sources; above ~0.25 pass PNA_FLAG_GATHER_L1 to the aggregation */
  int32_t reserved;
} pna_csr_t;

/* Bytes of device scratch pna_csr_build needs for (n_nodes, n_edges) on the current device. */
int pna_csr_workspace_bytes(int64_t n_nodes, int64_t n_edges, size_t* bytes);

/* src[e] -> dst[e], e in [0, n_edges): int64 device arrays (edge_index[0], edge_index[1] of PyG;
 * g.edges() of DGL).  Synchronises the stream once at the end to return the host-side counts and to report
 * out-of-range endpoints (PNA_ERR_INDEX).  Call once per graph, not per layer.  On a stream that is capturing a CUDA graph
 * it returns PNA_ERR_CAPTURING before it enqueues anything. */
int pna_csr_build(const int64_t* src, const int64_t* dst, pna_csr_t* csr, void* workspace, size_t workspace_bytes,
                  pna_stream_t stream);

/* Light view restricted to the rows with row_mask[r] != 0 (NULL = all rows below the split threshold); rows outside
 * the mask get light_deg = -1 and no slots, so the streaming kernel skips them without a row list.  Used to run the
 * rows whose sources are all local while the halo all-to-all is in flight, then the rest.  workspace: at least
 * pna_csr_light_view_workspace_bytes(n_nodes) bytes of device scratch.  Per-graph state like the CSR: on a stream that is
 * capturing a CUDA graph it returns PNA_ERR_CAPTURING before it enqueues anything. */
int pna_csr_light_view(const int32_t* rowptr, const int32_t* col, int64_t n_nodes, int32_t split_threshold, const uint8_t* row_mask,
                       int32_t n_part, int32_t* light_rowptr, int32_t* light_deg, int32_t* light_col, int32_t* part,
                       void* workspace, size_t workspace_bytes, pna_stream_t stream);
int pna_csr_light_view_workspace_bytes(int64_t n_nodes, size_t* bytes);

/* Bytes of device scratch pna_csr_build_padded needs for the capacities (n_nodes, n_edges). */
int pna_csr_padded_workspace_bytes(int64_t n_nodes, int64_t n_edges, size_t* bytes);

/* CSR of a padded edge list into fixed capacities, with nothing read back: legal on a stream that is capturing a CUDA
 * graph (kernel launches, CUB sort / scan in the workspace and cudaMemsetAsync only; no synchronisation).
 *   src / dst: int64 device arrays of csr->n_edges = E entries (the edge capacity); csr->n_nodes = N is the row capacity.
 *   An edge with dst == -1 is padding.  Any other endpoint outside dst [0, N) / src [0, n_src) sets bit 0 of status[0]
 *   and the edge is dropped like padding (never read past the check).
 *   Output: the row CSR of the real edges, by the stable radix sort of pna_csr_build keyed on dst (padding keyed to the
 *   sentinel N).  rowptr[N] = number of real edges; slots rowptr[N] .. E-1 are padding with col = 0 and perm = their
 *   original edge id.  The light view (optional, as for pna_csr_build) covers the N rows with its part partition.
 *   split_threshold must exceed n_edges (else PNA_ERR_BAD_ARG): no row is split, every row is reduced by the light-row
 *   kernels in slot order.  n_hubs = n_chunks = max_degree = n_light_edges = 0 and hot_source_fraction = 0 on return; cap_hubs,
 *   cap_chunks, hub_info and chunk_items are not read.
 *   status: int32[4] on the device, written by the stream: error bits, real edges, max in-degree, reserved.
 *   workspace: pna_csr_padded_workspace_bytes(N, E) bytes, 256-byte aligned. */
int pna_csr_build_padded(const int64_t* src, const int64_t* dst, pna_csr_t* csr, int32_t* status, void* workspace,
                         size_t workspace_bytes, pna_stream_t stream);

/* Per-slot arrays of a (padded) CSR with n_rows rows and n_slots slots, one kernel: for a real slot s < rowptr[n_rows],
 * transpose_dst[s] = col[s] (the destination key of the slot-transposed build) and dst_of_slot[s] = the row owning s; for a
 * padding slot -1 and 0.  int64 device arrays of n_slots entries.  Capture-legal. */
int pna_csr_slot_rows(const int32_t* rowptr, const int32_t* col, int64_t n_rows, int64_t n_slots, int64_t* transpose_dst,
                      int64_t* dst_of_slot, pna_stream_t stream);

/* ---- the aggregation ("single hand-written sm_90a CUDA kernel", north_star) ------------------------------
 * For every destination row i (PyG semantics; In(i) = slots rowptr[i]..rowptr[i+1], d = |In(i)|):
 *   m_s   = gathered[col[s]] (+ row_bias[i] when given)          s in In(i)           pna.py:137-150 / :239-240
 *   sum   = fp32 sum of m_s in slot order;  mean = sum / max(d,1)                      aggregators.py:9-14
 *   min/max over m_s, 0 when d == 0                                                     aggregators.py:17-22
 *   var   = (sum of m_s*m_s)/max(d,1) - mean*mean ; std = sqrt(max(var,0) + 1e-5)       aggregators.py:25-32
 *   amplification = log(d+1)/avg_log ; attenuation = d ? avg_log/log(d+1) : 1           scalers.py:12-19
 *   linear = d/avg_lin ; inverse_linear = d ? avg_lin/d : 1                             scalers.py:22-29
 *   out[i, tower t, ((s*A + a)*Ft + f)] = scaler_s * aggr_a                            pna.py:154-159 (scaler-major)
 * With n_towers = T the n_feat columns are T blocks of Ft = n_feat/T, and the output row is T blocks of
 * (has_self + S*A)*Ft columns, i.e. the [N, T, (1+)S*A*Ft] tensor of pna.py:129-131 flattened; when self_feat is
 * given, block t starts with self_feat[i, t*self_tower_stride : +Ft] (the torch.cat([x, out]) of pna.py:131).
 * All accumulation, degree, log and scaling in fp32 for both dtypes; bf16 is converted on load / store.
 */
typedef struct pna_agg {
  const void* gathered;      /* [n_src, n_feat] rows to gather (x for PNAConvSimple, V = x W_j^T + b for PNAConv) */
  int64_t ld_gathered;       /* row pitch in elements */
  const int32_t* rowptr;     /* [n_rows+1] */
  const int32_t* col;        /* [n_edges]; NULL = identity (gathered[] holds per-edge messages already in CSR order) */
  const void* row_bias;      /* nullable [n_rows, n_feat]: destination-side term added to every gathered row */
  int64_t ld_row_bias;
  const void* self_feat;     /* nullable: prepend self features to every tower block of the output row */
  int64_t ld_self;
  int64_t self_tower_stride; /* Ft when the input is divided between towers, 0 when it is repeated (pna.py:123-126) */
  void* out;                 /* [n_rows, ld_out] */
  int64_t ld_out;            /* >= n_towers * (has_self + S*A) * Ft */
  int64_t n_rows;
  int32_t n_feat;            /* total gathered width = n_towers * Ft */
  int32_t n_towers;
  int32_t dtype;             /* pna_dtype of gathered / row_bias / self_feat / out */
  int32_t n_aggr;
  uint32_t aggr_codes;
  int32_t n_scalers;
  uint32_t scaler_codes;
  float avg_log;             /* avg_deg['log'] of the layer ctor (pna.py:84) */
  float avg_lin;             /* avg_deg['lin'] (pna.py:83); only read by linear / inverse_linear */
  uint32_t flags;            /* pna_flags */
  int32_t split_threshold;   /* must equal the value the CSR was built with */
  int32_t chunk_edges;
  const int32_t* hub_info;   /* from pna_csr_t; may be NULL when n_hubs == 0 */
  const int32_t* chunk_items;
  int64_t n_hubs;
  int64_t n_chunks;
  float* hub_partials;       /* fp32 scratch [n_chunks * 4 * n_feat] (pna_aggregate_bwd: [(n_chunks + n_hubs) * 6 * n_feat]);
                                may be NULL when n_hubs == 0 */
  const int32_t* row_ids;    /* nullable [n_row_ids]: process only these light rows (halo overlap); hubs unaffected.
                                With a light view, view row i is output row row_ids[i]. */
  int64_t n_row_ids;
  /* optional light view of the rows (pna_csr_t light_* / part; NULL = not available -> tile kernels on rowptr/col).
   * Without row_ids it has n_rows rows; with row_ids it has n_row_ids rows. */
  const int32_t* light_rowptr;
  const int32_t* light_deg;
  const int32_t* light_col;
  const int32_t* part;
  int32_t n_part;
  /* view rows beyond n_rows are chunk pseudo-rows (row n_rows + c reduces chunk c into hub_partials); 0 or n_rows = none */
  int64_t n_view_rows;
  /* destination-partitioned multi-GPU graph, gather fused with the exchange: peer_gathered[r] (DEVICE array of
   * n_ranks device pointers) is rank r's `gathered` buffer mapped into this process (CUDA IPC / symmetric memory over
   * NVLink); a col entry c then means row (c & ((1 << peer_shift) - 1)) of rank (c >> peer_shift).  NULL: single GPU,
   * col indexes `gathered` directly.  All ranks use the same ld_gathered. */
  const void* const* peer_gathered;
  int32_t peer_shift;
  int32_t max_degree;        /* pna_csr_t.max_degree, or 0 = unknown.  A row with more than 64 * 8 chunks (power-law graphs:
                              * millions of in-edges) has its chunk partials merged by a radix tree of small launches over the
                              * chunk array instead of by one CTA walking them -- same fixed order on every call */
  /* optional int32 [9 * n_hubs] completion counters, ZERO before the first call (the library leaves them zero): when
   * given together with a view that contains the chunk pseudo-rows, the warp that stores the last partial of a split row
   * also merges and finalizes it (same merge order as the separate finalize kernel), so a layer call is ONE launch with
   * no serial tail.  NULL: split rows are finalized by a second small kernel.  Not to be shared by concurrent calls. */
  int32_t* hub_done;
  /* optional int32 [n_rows]: the degree the SCALERS see, when it is not the in-degree of the CSR row.  The dense reference
   * layer aggregates over adj + I with self_loop=True but scales with D = adj.sum(-1) of the loop-free adjacency
   * (models/pytorch/pna/scalers.py:13,21,28,35), and its max/min reduce over the other adjacency axis while still being
   * scaled with the row degree.  NULL: scalers use rowptr[i+1] - rowptr[i] (PyG / DGL). */
  const int32_t* scaler_degree;
  /* optional: ONE int32 of device scratch (the library zeroes it on the stream before the launch).  When given, the streamed
   * kernel deals out only the first 70 % of the row partitions statically and hands out the rest one at a time through
   * this counter, so warps that finish their static range early take over work from slow ones.  Not to be shared by
   * concurrent calls.  NULL: fully static assignment. */
  int32_t* work_counter;
  /* optional int32 [n_edges]: for normalised_mean, the node whose row degree (rowptr[k+1] - rowptr[k] of this CSR) weighs
   * each slot, in place of col[slot].  It lets normalised_mean run on messages already in CSR order (col == NULL): the
   * dense layer with pretrans_layers >= 2 passes the row CSR's own col here.  Read by no other aggregator.  NULL: the
   * slot's col entry (and normalised_mean needs col). */
  const int32_t* degree_col;
} pna_agg_t;

int pna_aggregate_fwd(const pna_agg_t* desc, pna_stream_t stream);

/* Backward of pna_aggregate_fwd w.r.t. the gathered rows (SURVEY section 8(f)-1; needed by every training loop,
 * multitask_benchmark/util/train.py:148).  grad_out has the layout of out (self block, if any, is skipped);
 * grad_gathered [n_src, n_feat] fp32 must be zero-initialised by the caller, contributions are accumulated with
 * atomics; grad_row_bias (nullable) [n_rows, n_feat] fp32 is written.  min/max route to the first slot attaining
 * the extremum (torch_scatter arg semantics). */
int pna_aggregate_bwd(const pna_agg_t* desc, const void* grad_out, int64_t ld_grad_out, float* grad_gathered,
                      int64_t ld_grad_gathered, float* grad_row_bias, int64_t ld_grad_row_bias, pna_stream_t stream);

/* The same gradient without one atomic per (edge, feature), for gathered rows (desc->col != NULL) -- three calls:
 *  1. pna_aggregate_bwd_coef: per destination row i the gradient of a message is  c0_i + c1_i * m + routed min / max terms;
 *     writes coef[i] = [c0_i + c1_i * row_bias[i]  (n_feat floats at column 0) | c1_i (n_feat floats at column c1_column)]
 *     for every row with in-edges (other rows are left untouched and are never read in step 2), adds the min / max
 *     gradients to grad_gathered[col[arg slot]] -- one scalar atomic per (row, feature); grad_gathered zero-initialised by
 *     the caller as above -- and writes grad_row_bias (nullable).  c1_column >= n_feat, ld_coef >= c1_column + n_feat;
 *     16-byte aligned choices (c1_column % 4 == 0, ld_coef % 4 == 0) get vector stores.  desc->hub_partials as for
 *     pna_aggregate_bwd.
 *  2. the caller sums the coefficient rows over the out-edges of every source row: pna_aggregate_fwd on the CSR of the
 *     TRANSPOSED graph (pna_csr_build with source and destination swapped: n_nodes = n_src) with gathered = coef,
 *     n_feat = ld_coef, one aggregator PNA_AGGR_SUM, one scaler PNA_SCALE_IDENTITY -> sums [n_src, ld_coef].
 *  3. pna_aggregate_bwd_combine: grad_gathered[j, f] += sums[j, f] + gathered[j, f] * sums[j, c1_column + f].
 * Same results up to fp32 summation order (reference: autograd of aggregators.py:9-32; tests/test_bwd_two_phase_math.py
 * restates the algebra). */
int pna_aggregate_bwd_coef(const pna_agg_t* desc, const void* grad_out, int64_t ld_grad_out, float* coef, int64_t ld_coef,
                           int32_t c1_column, float* grad_gathered, int64_t ld_grad_gathered, float* grad_row_bias,
                           int64_t ld_grad_row_bias, pna_stream_t stream);
int pna_aggregate_bwd_combine(const float* coef_sums, int64_t ld_sums, int32_t c1_column, const void* gathered,
                              int64_t ld_gathered, int32_t dtype, float* grad_gathered, int64_t ld_grad_gathered, int64_t n_src,
                              int32_t n_feat, pna_stream_t stream);

/* The same gradient with no floating-point atomics: a fixed function of the inputs and the graph (bit-reproducible).
 * Per call one feature slab [f_begin, f_begin + f_count): f_begin a multiple of 4 (PNA_F32) / 8 (PNA_BF16), f_count too
 * unless the slab ends at n_feat; otherwise PNA_ERR_BAD_ARG.  Two steps per slab:
 *  1. pna_aggregate_bwd_slots: STORES the gradient of every message into grad_slots [E, f_count] fp32 (row = CSR slot,
 *     column = feature - f_begin; ld_grad_slots >= f_count, 16-byte aligned rows get vector stores) -- the value the atomic
 *     path adds into grad_gathered[col[slot]], bit for bit -- and writes columns [f_begin, f_begin + f_count) of
 *     grad_row_bias (nullable, [n_rows, n_feat] fp32, addressed like pna_aggregate_bwd's), split rows as the chunks' slot-order
 *     sums added in chunk order.  With desc->col == NULL (messages in CSR order) grad_slots IS the gradient of the messages.
 *     desc->hub_partials as for pna_aggregate_bwd.  Peer-memory descriptors: PNA_ERR_UNSUPPORTED (they take
 *     pna_aggregate_bwd_peer_slots below).
 *  2. (desc->col != NULL) the caller sums grad_slots over the out-edges of every source row: pna_aggregate_fwd on the
 *     slot-transposed CSR (pna_csr_build with src = slot id 0..E-1, dst = col, n_nodes = n_src: rows are source rows, slots
 *     are forward slot ids in ascending order) with gathered = grad_slots, one aggregator PNA_AGGR_SUM, one scaler
 *     PNA_SCALE_IDENTITY, out = the grad_gathered column slab.  The forward sums every row in a fixed order. */
int pna_aggregate_bwd_slots(const pna_agg_t* desc, const void* grad_out, int64_t ld_grad_out, int32_t f_begin, int32_t f_count,
                            float* grad_slots, int64_t ld_grad_slots, float* grad_row_bias, int64_t ld_grad_row_bias,
                            pna_stream_t stream);

/* ---- slot weights: a weighted adjacency (the dense reference's real-valued adj; GCN-normalised or attention weights) ----
 * The three calls below are pna_aggregate_fwd / pna_aggregate_bwd / pna_aggregate_bwd_slots with two more inputs (both
 * optional; with both NULL each is exactly the call it extends):
 *   slot_weight      fp32 [n_edges] in CSR slot order: a real weight w_s per slot.
 *   scaler_degree_f  fp32 [n_rows]: a real-valued degree D_i for the scalers (amplification log(D+1)/avg_log, attenuation
 *                    D ? avg_log/log(D+1) : 1, linear D/avg_lin, inverse_linear D ? avg_lin/D : 1); takes precedence over
 *                    desc->scaler_degree.  With slot_weight NULL every weight is 1.
 * For row i with slots s, W_i = fp32 sum of w_s in slot order (split rows: over all their slots in slot order too), every
 * product rounded:
 *   sum  = fp32 sum of fl(m_s * w_s) in slot order (split rows: chunk sums added in chunk order)
 *   mean = sum / W_i (correctly rounded);  var = fl(Q / W_i) - fl(mean * mean),  Q = sum of fl(fl(m_s * m_s) * w_s)
 *   std  = sqrt(max(var, 0) + 1e-5);  var is clamped at 0 with PNA_FLAG_RELU_VAR, as without weights
 *   min / max over the slots with w_s > 0 of the UNWEIGHTED m_s (the dense reference's adj > 0 mask), 0 when there is none
 * A row without slots gives what it gives without weights; a row whose weights sum to exactly 0 gets the IEEE quotient.
 * Gradient of slot s: fl(w_s * fl(c0 + c1 * m_s)) + the routed min / max terms, c0 and c1 the unweighted coefficients with
 * the degree replaced by W_i (so all-ones weights give the unweighted bits on rows below the split threshold).  No gradient
 * with respect to the weights.  Aggregators: sum / mean / min / max / var / std (and PNA_AGGR_SKIP); any other aggregator,
 * peer_gathered and row_ids return PNA_ERR_UNSUPPORTED before anything is enqueued.  The weighted calls have no coefficient
 * or peer-memory form.  Every other argument, check and scratch contract is the extended call's.  Rounding order:
 * pna_b200/csrc/pna_aggregate_adj_weight.cuh */
int pna_aggregate_fwd_weighted(const pna_agg_t* desc, const float* slot_weight, const float* scaler_degree_f,
                               pna_stream_t stream);
int pna_aggregate_bwd_weighted(const pna_agg_t* desc, const float* slot_weight, const float* scaler_degree_f,
                               const void* grad_out, int64_t ld_grad_out, float* grad_gathered, int64_t ld_grad_gathered,
                               float* grad_row_bias, int64_t ld_grad_row_bias, pna_stream_t stream);
int pna_aggregate_bwd_slots_weighted(const pna_agg_t* desc, const float* slot_weight, const float* scaler_degree_f,
                                     const void* grad_out, int64_t ld_grad_out, int32_t f_begin, int32_t f_count,
                                     float* grad_slots, int64_t ld_grad_slots, float* grad_row_bias, int64_t ld_grad_row_bias,
                                     pna_stream_t stream);

/* Step 1 of pna_aggregate_bwd_slots for a peer-memory graph (desc->peer_gathered != NULL, required: PNA_ERR_BAD_ARG
 * otherwise): the source row of slot s is row (col[s] & mask) of rank (col[s] >> peer_shift), read over NVLink as
 * pna_aggregate_fwd reads it.  Same arguments, slab rules and results: grad_slots row s and grad_row_bias are the bits
 * pna_aggregate_bwd_slots stores for the same slot of the unpartitioned graph; no floating-point atomics.  What the peer
 * forward refuses is refused here: moment, softmax / softmin / normalised_mean aggregators and row_ids
 * (PNA_ERR_UNSUPPORTED), and col == NULL (PNA_ERR_UNSUPPORTED).  Every rank's gathered rows must stay unchanged until all
 * ranks' calls that read them have completed.  Step 2 is the owners': each adds the slots that name its rows into its
 * own gradient (pna_halo_grad_pull over the ranks' grad_slots buffers, slots in ascending (rank, slot) order). */
int pna_aggregate_bwd_peer_slots(const pna_agg_t* desc, const void* grad_out, int64_t ld_grad_out, int32_t f_begin,
                                 int32_t f_count, float* grad_slots, int64_t ld_grad_slots, float* grad_row_bias,
                                 int64_t ld_grad_row_bias, pna_stream_t stream);

/* ---- the per-edge pretrans MLP of the dense layer with pretrans_layers = L >= 2 (models/layers.py:200-229) ------------
 * For every slot s of a destination-sorted CSR (row i, source j = col[s]) and tower t (all fp32, row-major, contiguous,
 * TF = n_towers * width):
 *   z_1 = relu(a[i, t] + b[j, t] + bias1[t]),  z_k = relu(W_k[t] z_(k-1) + b_k[t]) (k = 2..L-1),
 *   messages[s, t] = W_L[t] z_(L-1) + b_L[t]                                                   [n_edges, TF]
 * a [n_rows, TF] is the destination half of the first layer's product, b [n_src, TF] the source half, bias1 [TF];
 * weight [(L-1), n_towers, width, width] (nn.Linear's [out, in]) and bias [(L-1), n_towers, width] hold layers 2..L.
 * activations (nullable) [(L-1), n_edges, TF] receives z_1 .. z_(L-1) for the backward.
 * pna_edge_mlp_bwd: grad_pre [(L-1), n_edges, TF] receives G_1 .. G_(L-1), the gradients of the pre-activations of layers
 * 1 .. L-1 (G_L is grad_messages):  G_(k-1) = (W_k[t]^T G_k) * [z_(k-1) > 0].  Weight / bias gradients and the
 * gradients of a and b are the caller's (G_k^T z_(k-1), sums of G_k; sums of G_1 over rows and over sources).
 * One thread per (slot, tower), no atomics: every value is a fixed function of its inputs.  n_layers < 2, width < 1,
 * n_towers < 1 or a null pointer (with n_edges > 0): PNA_ERR_BAD_ARG; width > PNA_EDGE_MLP_MAX_WIDTH:
 * PNA_ERR_UNSUPPORTED.  Rounding order: pna_b200/csrc/pna_edge_mlp.cu */
#define PNA_EDGE_MLP_MAX_WIDTH 64
int pna_edge_mlp_fwd(const int32_t* rowptr, const int32_t* col, int64_t n_rows, int64_t n_edges, const float* a, const float* b,
                     const float* bias1, const float* weight, const float* bias, int32_t n_layers, int32_t n_towers,
                     int32_t width, float* messages, float* activations, pna_stream_t stream);
int pna_edge_mlp_bwd(const float* grad_messages, const float* activations, const float* weight, int64_t n_edges,
                     int32_t n_layers, int32_t n_towers, int32_t width, float* grad_pre, pna_stream_t stream);

/* ---- per-edge messages of the PyG PNAConv and the DGL PNALayer: the same MLP with an edge term, any L >= 1 ------------
 * As pna_edge_mlp_fwd, with two changes (rounding order: pna_b200/csrc/pna_edge_mlp.cu):
 *   u1 = fl(fl(fl(a[i, t] + b[j, t]) + bias1[t]) + edge_term[s, t])      edge_term (nullable) [n_edges, TF], slot order;
 *                                                                         NULL: exactly pna_edge_mlp_fwd's u1
 *   messages [n_edges, n_towers * msg_pitch]: messages[s, t*msg_pitch + o] = u_L,o for o < width and exact zeros for
 *   width <= o < msg_pitch, so the aggregation reads it at width msg_pitch with n_towers towers.
 * n_layers == 1: the message is u1 itself (no ReLU; weight, bias and activations are not read) and any width is taken.
 * n_layers >= 2: width <= PNA_EDGE_MLP_MAX_WIDTH; activations (nullable) as pna_edge_mlp_fwd, at pitch width.
 * pna_edge_msg_bwd (n_layers >= 2): pna_edge_mlp_bwd with grad_messages read at pitch msg_pitch; grad_pre at pitch width.
 * n_layers < 1 (< 2 for the backward), msg_pitch < width, width < 1, n_towers < 1 or a null required pointer (with
 * n_edges > 0): PNA_ERR_BAD_ARG; n_layers >= 2 with width > PNA_EDGE_MLP_MAX_WIDTH: PNA_ERR_UNSUPPORTED. */
int pna_edge_msg_fwd(const int32_t* rowptr, const int32_t* col, int64_t n_rows, int64_t n_edges, const float* a, const float* b,
                     const float* bias1, const float* edge_term, const float* weight, const float* bias, int32_t n_layers,
                     int32_t n_towers, int32_t width, int32_t msg_pitch, float* messages, float* activations,
                     pna_stream_t stream);
int pna_edge_msg_bwd(const float* grad_messages, int32_t msg_pitch, const float* activations, const float* weight,
                     int64_t n_edges, int32_t n_layers, int32_t n_towers, int32_t width, float* grad_pre, pna_stream_t stream);

/* The same two calls with bf16 storage (the layers under bf16 autocast).  a, b, edge_term, messages, activations and
 * grad_messages are bf16 (const void* / void*: 2-byte elements, same layouts and pitches); bias1, weight, bias and grad_pre
 * stay fp32.  A load widens to fp32 exactly and the arithmetic is the fp32 calls', so bit for bit
 *     messages_bf16 = RN_bf16(pna_edge_msg_fwd(a, b, edge_term widened)),   activations likewise,
 *     grad_pre      = pna_edge_msg_bwd(grad_messages widened, activations widened)   (ReLU mask: stored z > 0).
 * Same arguments, checks and status codes as the fp32 calls.  (Appended in ABI version 8.) */
int pna_edge_msg_fwd_bf16(const int32_t* rowptr, const int32_t* col, int64_t n_rows, int64_t n_edges, const void* a, const void* b,
                          const float* bias1, const void* edge_term, const float* weight, const float* bias, int32_t n_layers,
                          int32_t n_towers, int32_t width, int32_t msg_pitch, void* messages, void* activations,
                          pna_stream_t stream);
int pna_edge_msg_bwd_bf16(const void* grad_messages, int32_t msg_pitch, const void* activations, const float* weight,
                          int64_t n_edges, int32_t n_layers, int32_t n_towers, int32_t width, float* grad_pre, pna_stream_t stream);

/* ---- halo rows for the destination-partitioned multi-GPU path (north_star: "single NCCL all-to-all for halo
 * source features per layer"): dst[i, :] = src[idx[i], :], n_feat elements per row.  Used to pack the send buffer. */
int pna_gather_rows(const void* src, int64_t ld_src, const int32_t* idx, int64_t n_idx, void* dst, int64_t ld_dst,
                    int32_t n_feat, int32_t dtype, pna_stream_t stream);

/* ---- the same exchange as ONE kernel of peer loads (no pack, no collective, no unpack) -------------------------------
 * Every rank's feature rows live in a buffer that is mapped into every process (symmetric memory / CUDA IPC over NVLink).
 * peer_rows: DEVICE array of n_ranks base pointers of those buffers (row pitch ld_rows elements on every rank);
 * enc[i] = owner << peer_shift | row-on-owner names the i-th de-duplicated remote source row this rank needs;
 * dst[i, :] (pitch ld_dst; normally the tail of the rank's [local ; halo] buffer) receives it.  One remote row crosses
 * NVLink once per layer however many local destinations gather it afterwards. */
int pna_halo_pull(const void* const* peer_rows, int64_t ld_rows, const int32_t* enc, int32_t peer_shift, int64_t n_idx, void* dst,
                  int64_t ld_dst, int32_t n_feat, int32_t dtype, pna_stream_t stream);

/* The transpose of pna_halo_pull, for the backward: return the gradients of halo copies to the rows' owner.
 * peer_rows: DEVICE array of n_ranks pointers, each to the start of that rank's fp32 halo-gradient rows (row pitch ld_rows
 * elements on every rank), so the row index of a slot is a position in that rank's halo.  For i in [0, n_rows):
 *     grad[rows[i], :] += sum over s in [rowptr[i], rowptr[i+1]) of  peer_rows[enc[s] >> enc_shift][enc[s] & mask, :]
 * summed in slot order in fp32, one rounding per add, starting from the current grad row (pitch ld_grad).  rows must not
 * repeat: each row is owned by one warp and there are no atomics, so with slots in a fixed order (ascending peer rank, as
 * pna_b200/dist.py plans them) the result is bit-reproducible.  enc_shift in 1..30; n_rows == 0 launches nothing. */
int pna_halo_grad_pull(const void* const* peer_rows, int64_t ld_rows, const int32_t* rows, const int32_t* rowptr, const int32_t* enc,
                       int32_t enc_shift, int64_t n_rows, float* grad, int64_t ld_grad, int32_t n_feat, pna_stream_t stream);

/* Device-side barrier between the ranks of one box, enqueued on `stream`: peer_flags is a DEVICE array of n_ranks pointers to
 * each rank's uint64 flags[n_ranks] (zero-initialised once, mapped into every process like the feature rows).  Rank r
 * stores `epoch` into flags[r] of every peer and waits until its own flags all reach `epoch`; epochs must increase by
 * one per call on every rank.  Orders "every rank has written its feature rows" before the pulls / peer gathers of the
 * next kernel.  If a peer does not arrive within timeout_ns (0 = 2 s) the kernel gives up and sets *status = 1 (DEVICE int,
 * nullable) instead of hanging the GPU. */
int pna_peer_barrier(const void* const* peer_flags, int32_t rank, int32_t world, uint64_t epoch, uint64_t timeout_ns,
                     int32_t* status, pna_stream_t stream);

/* ---- first dense linear of the post-aggregation MLP on the tensor cores (north_star: "the post-MLP uses tensor
 * cores only for its dense linear"; reference pna.py:222-227 post_nn[0], models/dgl/pna_layer.py:31 posttrans) -----
 * y[n_rows, n_out] = a[n_rows, n_in] . weight[n_out, n_in]^T + bias, fp32 in / fp32 out, fp32-accurate: every operand
 * is split hi + lo and three wgmma tf32 products (hi.hi + hi.lo + lo.hi) accumulate in registers, because plain
 * TF32 (10-bit mantissa) cannot meet the 1e-5 parity bar.  n_in % 32 == 0, n_out in {64, 128, 256}; other shapes
 * return PNA_ERR_UNSUPPORTED and the caller keeps its library GEMM.  workspace: 2 * n_in * n_out floats (split weight). */
int pna_linear_workspace_bytes(int32_t n_in, int32_t n_out, size_t* bytes);
int pna_linear_fwd(const float* a, int64_t lda, const float* weight, const float* bias, float* y, int64_t ldy, int64_t n_rows,
                   int32_t n_in, int32_t n_out, void* workspace, size_t workspace_bytes, pna_stream_t stream);

/* ---- the same linear fed by the COMPACT aggregate (SURVEY section 8(f)-2: the [N, S*A*F] tensor is never written) --
 * The reference's post-MLP input is cat over the scalers s of  scale_s(deg_i) * agg_i  (pna.py:247-249,
 * scalers.py:8-29): S scaled copies of one [N, A*F] tensor.  With a = that tensor for the identity scaler alone
 * (pna_aggregate_fwd with n_scalers = 1, scaler_codes = PNA_SCALE_IDENTITY) and row_scale[i, s] = the factor of scaler s
 * for row i (pna_row_scales),
 *     y[i, :] = sum_s sum_k  fl(row_scale[i, s] * a[i, k]) * weight[:, s * n_a + k]  + bias,      n_a = n_in / n_scalers
 * which is the reference's  post_nn[0](cat_s(...))  with every product rounded as the reference rounds it; the scaled
 * copies exist only in registers.  weight keeps the reference's layout [n_out, n_in = S*A*F] (scaler-major columns).
 * n_a % 32 == 0, n_out in {64, 128, 256}; workspace as for pna_linear_fwd. */
int pna_linear_scaled_fwd(const float* a, int64_t lda, const float* row_scale, int32_t n_scalers, const float* weight,
                          const float* bias, float* y, int64_t ldy, int64_t n_rows, int32_t n_in, int32_t n_out, void* workspace,
                          size_t workspace_bytes, pna_stream_t stream);

/* ---- backward of pna_linear_fwd / pna_linear_scaled_fwd on the tensor cores, at the same fp32 accuracy (3xTF32) -----
 * Both calls are deterministic: no atomics, every sum in a fixed order, so the result is a fixed function of the inputs
 * (what torch.use_deterministic_algorithms promises).  n_scalers == 1 with row_scale NULL is the plain linear; otherwise
 * row_scale is the [n_rows, n_scalers] contiguous factor array of pna_linear_scaled_fwd and n_a = n_in / n_scalers.  Shapes
 * as the forward's: n_a % 32 == 0 and n_out in {64, 128, 256} (else PNA_ERR_UNSUPPORTED); n_scalers outside 1..5, null
 * pointers, or row_scale NULL with n_scalers > 1: PNA_ERR_BAD_ARG.  grad_y, a, grad_a, grad_weight and workspace 16-byte
 * aligned, row pitches (in elements) multiples of 4.  n_rows == 0 returns PNA_OK and launches nothing.
 *
 * Data gradient, grad_a [n_rows, n_a] (pitch ld_grad_a) written:
 *     grad_a[i, k] = sum_s sum_o  fl(row_scale[i, s] * grad_y[i, o]) * weight[o, s * n_a + k]
 * (plain: sum_o grad_y[i, o] * weight[o, k]).  The forward kernel run on grad_y with the transposed (and, with scalers,
 * re-blocked) weight; the scaled copies of grad_y exist only in registers.
 * Weight gradient, grad_weight [n_out, n_in] contiguous written (not accumulated):
 *     grad_weight[o, s * n_a + k] = sum_i  grad_y[i, o] * fl(row_scale[i, s] * a[i, k])
 * where fl(c * a) is the operand the forward's loaders formed, so this is the exact gradient of what the forward multiplied.
 * The rows are split across CTAs by a rule that depends on the shape alone; each CTA folds its tensor-core accumulators
 * into an fp32 partial every 64 rows and a second kernel adds the partials in ascending split order.  grad_a folds the
 * same way every 128 products.
 * workspace: pna_linear_bwd_workspace_bytes(n_rows, n_in, n_out, n_scalers) bytes, enough for either call (the weight
 * images of the data gradient, the partials of the weight gradient); calls on one stream may share it. */
int pna_linear_bwd_workspace_bytes(int64_t n_rows, int32_t n_in, int32_t n_out, int32_t n_scalers, size_t* bytes);
int pna_linear_bwd_data(const float* grad_y, int64_t ld_grad_y, const float* row_scale, int32_t n_scalers, const float* weight,
                        float* grad_a, int64_t ld_grad_a, int64_t n_rows, int32_t n_in, int32_t n_out, void* workspace,
                        size_t workspace_bytes, pna_stream_t stream);
int pna_linear_bwd_weight(const float* grad_y, int64_t ld_grad_y, const float* a, int64_t lda, const float* row_scale,
                          int32_t n_scalers, float* grad_weight, int64_t n_rows, int32_t n_in, int32_t n_out, void* workspace,
                          size_t workspace_bytes, pna_stream_t stream);

/* scales[i, s] = factor of scaler s (code (scaler_codes >> 4s) & 15) at in-degree rowptr[i+1] - rowptr[i]; bit-identical
 * to the factors pna_aggregate_fwd applies (one device function computes both). */
int pna_row_scales(const int32_t* rowptr, int64_t n_rows, int32_t n_scalers, uint32_t scaler_codes, float avg_log, float avg_lin,
                   float* scales, pna_stream_t stream);

/* ---- first post Linear of the tower layers (PNAConv, the DGL PNALayer) on the compact tower aggregate (3xTF32) ----------
 * a [n_rows, T * (1 + A) * F] (pitch lda) is what pna_aggregate_fwd writes with self_feat and the identity scaler alone:
 * per tower t the block [self_t | agg_t] of F + A * F columns.  weight [T, n_out, (1 + S * A) * F] contiguous is every
 * tower's first post Linear in the reference's column layout (self block, then scaler-major aggregate blocks), bias
 * [T, n_out] or NULL, row_scale the [n_rows, S] factors of pna_row_scales.  y [n_rows, T * n_out] (pitch ldy), tower-major:
 *     y[i, t * n_out + o] = b_t[o] + sum_k self_t[i, k] W_t[o, k] + sum_s sum_k fl(row_scale[i, s] * agg_t[i, k]) W_t[o, F + s A F + k]
 * Each tower reads only its own columns; the scaled copies exist only in registers.  Same split and fp32 accuracy as
 * pna_linear_fwd; the tensor-core chains are folded into an fp32 total every 128 products.
 * pna_linear_towers_bwd_data writes grad_a [n_rows, T * (1 + A) * F] (pitch ld_grad_a) from grad_y [n_rows, T * n_out]:
 *     self columns       grad_a[i, t, k]     = sum_o grad_y[i, t, o] W_t[o, k]
 *     aggregate columns  grad_a[i, t, F + k] = sum_s sum_o fl(row_scale[i, s] * grad_y[i, t, o]) W_t[o, F + s A F + k]
 * with the same folds.  Neither call uses atomics or a workspace; the results are a fixed function of the inputs.
 * n_towers <= 8, n_out <= 64, n_towers * n_out <= 256 and F % 4 == 0, else PNA_ERR_UNSUPPORTED; n_scalers outside 1..5,
 * n_aggr outside 1..6, a null pointer or a pitch shorter than the row: PNA_ERR_BAD_ARG.  No alignment is required.
 * n_rows == 0 returns PNA_OK and launches nothing.  (Appended in ABI version 8.) */
int pna_linear_towers_scaled_fwd(const float* a, int64_t lda, const float* row_scale, int32_t n_scalers, const float* weight,
                                 const float* bias, float* y, int64_t ldy, int64_t n_rows, int32_t n_towers, int32_t n_feat,
                                 int32_t n_aggr, int32_t n_out, pna_stream_t stream);
int pna_linear_towers_bwd_data(const float* grad_y, int64_t ld_grad_y, const float* row_scale, int32_t n_scalers, const float* weight,
                               float* grad_a, int64_t ld_grad_a, int64_t n_rows, int32_t n_towers, int32_t n_feat, int32_t n_aggr,
                               int32_t n_out, pna_stream_t stream);
/* pna_linear_towers_scaled_fwd with a bf16 compact aggregate `a` (const void*: 2-byte elements, pitch lda in elements);
 * row_scale, weight, bias and y stay fp32.  Each element of a is widened to fp32 (exact) as it is loaded; from there on
 * the arithmetic is the fp32 call's, so y equals pna_linear_towers_scaled_fwd(a widened) bit for bit.  Same checks and
 * status codes.  The data gradient needs no bf16 call: grad_y is fp32.  (Appended in ABI version 8.) */
int pna_linear_towers_scaled_fwd_bf16(const void* a, int64_t lda, const float* row_scale, int32_t n_scalers, const float* weight,
                                      const float* bias, float* y, int64_t ldy, int64_t n_rows, int32_t n_towers, int32_t n_feat,
                                      int32_t n_aggr, int32_t n_out, pna_stream_t stream);

/* ---- Set2Set graph readout (reference models/layers.py:53-98, the readout of S2SReadout) --------------------------------
 * x [n_graphs, n_nodes, n_feat = D] fp32 contiguous; the LSTM is nn.LSTM(2D, D, num_layers=1) with PyTorch's gate order
 * i, f, g, o: w_ih [4D, 2D], w_hh [4D, D], b_ih [4D], b_hh [4D], all contiguous.  With h, c, q* = 0 at the start, each of
 * the `steps` steps computes
 *     q, (h, c) = LSTM(q*, (h, c));   e_i = x_i . q;   alpha = softmax_i(e) (maximum subtracted);   r = sum_i alpha_i x_i;
 *     q* = [q, r]
 * and out [n_graphs, 2D] is q* after the last step.  One CTA per graph runs every step; no atomics, every sum in an order
 * fixed by the shape, so the results are a fixed function of the inputs.
 * saved (the forward writes it when non-NULL; the backward reads it): pna_set2set_saved_floats floats, one record of
 * 7D + n_nodes floats per step t and graph b, record index t * n_graphs + b:
 *     [ q*_t (2D) | c_t (D) | i_t f_t g_t o_t, the gate activations (4D) | alpha_t (n_nodes) ]
 * so the records' first 2D floats, at a pitch of 7D + n_nodes, are the matrix Q* [steps * n_graphs, 2D].
 * pna_set2set_bwd, from grad_out [n_graphs, 2D], writes grad_x [n_graphs, n_nodes, D] (NULL: not computed) and the
 * pre-activation gate gradients grad_gates [steps, n_graphs, 4D] (gate order i, f, g, o).  The weight gradients are then
 * GEMMs over the steps * n_graphs rows: dW_ih = dG[1:]^T Q*[:-1], dW_hh = dG[1:]^T Q*[:-1, :D] (steps shifted by one; the
 * input of step 0 is zero) and db_ih = db_hh = sum of dG over all rows.
 * Limits: 1 <= n_feat <= 128, n_nodes * n_feat <= 16384, n_graphs < 2^31, else PNA_ERR_UNSUPPORTED; a size <= 0 or a
 * null pointer: PNA_ERR_BAD_ARG.  No alignment is required.  The calls allocate nothing, read nothing back and do not
 * synchronise, so they may be enqueued on a stream that is capturing a CUDA graph.  (Appended in ABI version 8.) */
int pna_set2set_saved_floats(int64_t n_graphs, int32_t n_nodes, int32_t n_feat, int32_t steps, int64_t* n_floats);
int pna_set2set_fwd(const float* x, int64_t n_graphs, int32_t n_nodes, int32_t n_feat, int32_t steps, const float* w_ih,
                    const float* w_hh, const float* b_ih, const float* b_hh, float* out, float* saved, pna_stream_t stream);
int pna_set2set_bwd(const float* x, int64_t n_graphs, int32_t n_nodes, int32_t n_feat, int32_t steps, const float* w_ih,
                    const float* w_hh, const float* saved, const float* grad_out, float* grad_x, float* grad_gates,
                    pna_stream_t stream);

int pna_query(int what);
const char* pna_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* PNA_B200_H */
