// pna_aggregate_fwd: C-ABI entry point -- argument checks and dtype / alignment dispatch.
#include "pna_aggregate.cuh"

namespace pna {

template <typename T, int VEC>
int launch_typed(const KParams& p, cudaStream_t st);   // defined in pna_aggregate_{f32,bf16}_{vec,scalar}.cu

static bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15u) == 0; }

// The moment columns (pna_aggregate_moments.cuh), after the existing kernels have written every other column.
template <typename T>
static int launch_moments_fwd(const MParams& p, cudaStream_t st) {
  const unsigned gy = (unsigned)((p.F + 31) / 32);
  constexpr long long per_block = kMomThreads / 32;
  if (!(p.flags & PNA_FLAG_SKIP_LIGHT)) {
    const long long gx = (p.n_rows + per_block - 1) / per_block;
    PNA_REQUIRE(gx <= 0x7fffffffll, PNA_ERR_UNSUPPORTED, "pna_aggregate_fwd: too many rows");
    k_mom_rows<T><<<dim3((unsigned)gx, gy), kMomThreads, 0, st>>>(p);
    PNA_CUDA_TRY(cudaGetLastError());
  }
  if (!(p.flags & PNA_FLAG_SKIP_HUBS) && p.n_hubs > 0) {
    const unsigned gc = (unsigned)((p.n_chunks + per_block - 1) / per_block), gh = (unsigned)((p.n_hubs + per_block - 1) / per_block);
    k_mom_chunk_sum<T, 4><<<dim3(gc, gy), kMomThreads, 0, st>>>(p);
    PNA_CUDA_TRY(cudaGetLastError());
    k_mom_hub_mean<4><<<dim3(gh, gy), kMomThreads, 0, st>>>(p);
    PNA_CUDA_TRY(cudaGetLastError());
    k_mom_chunk_central<T, 4><<<dim3(gc, gy), kMomThreads, 0, st>>>(p);
    PNA_CUDA_TRY(cudaGetLastError());
    k_mom_hub_final<T><<<dim3(gh, gy), kMomThreads, 0, st>>>(p);
    PNA_CUDA_TRY(cudaGetLastError());
  }
  return PNA_OK;
}

// The columns of one weighted aggregator (pna_aggregate_weighted.cuh), after the existing kernels and the moments.
template <typename T>
static int launch_weighted_fwd(const MParams& p, unsigned code, cudaStream_t st) {
  const unsigned gy = (unsigned)((p.F + 31) / 32);
  constexpr long long per_block = kMomThreads / 32;
  if (!(p.flags & PNA_FLAG_SKIP_LIGHT)) {
    const long long gx = (p.n_rows + per_block - 1) / per_block;
    PNA_REQUIRE(gx <= 0x7fffffffll, PNA_ERR_UNSUPPORTED, "pna_aggregate_fwd: too many rows");
    k_wsum_rows<T><<<dim3((unsigned)gx, gy), kMomThreads, 0, st>>>(p, code);
    PNA_CUDA_TRY(cudaGetLastError());
  }
  if (!(p.flags & PNA_FLAG_SKIP_HUBS) && p.n_hubs > 0) {
    const unsigned gc = (unsigned)((p.n_chunks + per_block - 1) / per_block), gh = (unsigned)((p.n_hubs + per_block - 1) / per_block);
    if (code != PNA_AGGR_NORMALISED_MEAN) {
      k_wsum_chunk_max<T, 4><<<dim3(gc, gy), kMomThreads, 0, st>>>(p, code);
      PNA_CUDA_TRY(cudaGetLastError());
      k_wsum_hub_max<4><<<dim3(gh, gy), kMomThreads, 0, st>>>(p);
      PNA_CUDA_TRY(cudaGetLastError());
    }
    k_wsum_chunk_zs<T, 4><<<dim3(gc, gy), kMomThreads, 0, st>>>(p, code);
    PNA_CUDA_TRY(cudaGetLastError());
    k_wsum_hub_final<T><<<dim3(gh, gy), kMomThreads, 0, st>>>(p, code);
    PNA_CUDA_TRY(cudaGetLastError());
  }
  return PNA_OK;
}

// The add-on aggregators after the existing kernels: the moments, then each weighted aggregator in turn (stream order,
// so that each reuses hub_partials).
template <typename T>
static int launch_addons_fwd(const pna_agg_t* d, cudaStream_t st) {
  const MParams mp = moment_params(d);
  if (mp.orders) {
    const int rc = launch_moments_fwd<T>(mp, st);
    if (rc != PNA_OK) return rc;
  }
  const unsigned w = weighted_codes(d->aggr_codes, d->n_aggr);
  for (unsigned c = PNA_AGGR_SOFTMAX; c <= PNA_AGGR_NORMALISED_MEAN; ++c) {
    if (!((w >> (c - PNA_AGGR_SOFTMAX)) & 1u)) continue;
    const int rc = launch_weighted_fwd<T>(mp, c, st);
    if (rc != PNA_OK) return rc;
  }
  return PNA_OK;
}

// A weighted call (pna_aggregate_fwd_weighted): every column, in place of the existing kernels.
template <typename T>
static int launch_adj_weight_fwd(const AWParams& a, cudaStream_t st) {
  const MParams& p = a.m;
  const unsigned gy = (unsigned)((p.F + 31) / 32);
  constexpr long long per_block = kMomThreads / 32;
  if (!(p.flags & PNA_FLAG_SKIP_LIGHT)) {
    const long long gx = (p.n_rows + per_block - 1) / per_block;
    PNA_REQUIRE(gx <= 0x7fffffffll, PNA_ERR_UNSUPPORTED, "pna_aggregate_fwd: too many rows");
    k_aw_rows<T><<<dim3((unsigned)gx, gy), kMomThreads, 0, st>>>(a);
    PNA_CUDA_TRY(cudaGetLastError());
  }
  if (!(p.flags & PNA_FLAG_SKIP_HUBS) && p.n_hubs > 0) {
    const unsigned gc = (unsigned)((p.n_chunks + per_block - 1) / per_block), gh = (unsigned)((p.n_hubs + per_block - 1) / per_block);
    k_aw_chunk<T><<<dim3(gc, gy), kMomThreads, 0, st>>>(a);
    PNA_CUDA_TRY(cudaGetLastError());
    k_aw_hub_final<T><<<dim3(gh, gy), kMomThreads, 0, st>>>(a);
    PNA_CUDA_TRY(cudaGetLastError());
  }
  return PNA_OK;
}

}  // namespace pna

using namespace pna;

// sw / sdf: pna_aggregate_fwd_weighted's slot weights and real-valued scaler degree (both NULL: pna_aggregate_fwd)
static int fwd_entry(const pna_agg_t* d, const float* sw, const float* sdf, pna_stream_t stream) {
  PNA_REQUIRE(d != nullptr, PNA_ERR_BAD_ARG, "pna_aggregate_fwd: null descriptor");
  PNA_REQUIRE(d->n_rows >= 0 && d->n_feat > 0 && d->n_towers > 0, PNA_ERR_BAD_ARG,
              "pna_aggregate_fwd: bad sizes n_rows=%lld n_feat=%d n_towers=%d", (long long)d->n_rows, d->n_feat,
              d->n_towers);
  PNA_REQUIRE(d->n_feat % d->n_towers == 0, PNA_ERR_BAD_ARG, "pna_aggregate_fwd: n_feat %d not divisible by n_towers %d",
              d->n_feat, d->n_towers);
  PNA_REQUIRE(d->n_feat <= pna_query(PNA_QUERY_MAX_FEATURES), PNA_ERR_UNSUPPORTED, "pna_aggregate_fwd: n_feat %d too large",
              d->n_feat);
  PNA_REQUIRE(d->n_aggr >= 1 && d->n_aggr <= PNA_MAX_AGGR && d->n_scalers >= 1 && d->n_scalers <= PNA_MAX_SCALERS,
              PNA_ERR_BAD_ARG, "pna_aggregate_fwd: n_aggr=%d n_scalers=%d out of range", d->n_aggr, d->n_scalers);
  for (int a = 0; a < d->n_aggr; ++a)
    PNA_REQUIRE(((d->aggr_codes >> (4 * a)) & 15u) <= PNA_AGGR_NORMALISED_MEAN || ((d->aggr_codes >> (4 * a)) & 15u) == PNA_AGGR_SKIP,
                PNA_ERR_BAD_ARG, "pna_aggregate_fwd: bad aggregator code");
  const bool moments = moment_orders(d->aggr_codes, d->n_aggr) != 0;
  const unsigned weighted = weighted_codes(d->aggr_codes, d->n_aggr);
  const bool addons = moments || weighted;
  PNA_REQUIRE(!moments || (!d->peer_gathered && !d->row_ids), PNA_ERR_UNSUPPORTED,
              "pna_aggregate_fwd: moment aggregators are not available with peer_gathered or row_ids");
  PNA_REQUIRE(!weighted || (!d->peer_gathered && !d->row_ids), PNA_ERR_UNSUPPORTED,
              "pna_aggregate_fwd: softmax / softmin / normalised_mean are not available with peer_gathered or row_ids");
  for (int s = 0; s < d->n_scalers; ++s)
    PNA_REQUIRE(((d->scaler_codes >> (4 * s)) & 15u) <= PNA_SCALE_INVERSE_LINEAR, PNA_ERR_BAD_ARG,
                "pna_aggregate_fwd: bad scaler code");
  PNA_REQUIRE(d->dtype == PNA_F32 || d->dtype == PNA_BF16, PNA_ERR_UNSUPPORTED, "pna_aggregate_fwd: dtype %d", d->dtype);
  PNA_REQUIRE(!((weighted >> (PNA_AGGR_NORMALISED_MEAN - PNA_AGGR_SOFTMAX)) & 1u) || d->col || d->degree_col,
              PNA_ERR_UNSUPPORTED, "pna_aggregate_fwd: normalised_mean needs col or degree_col (the source of every slot)");
  const bool adj_weight = sw || sdf;
  if (adj_weight) {
    for (int a = 0; a < d->n_aggr; ++a)
      PNA_REQUIRE(adj_weight_code((d->aggr_codes >> (4 * a)) & 15u), PNA_ERR_UNSUPPORTED,
                  "pna_aggregate_fwd: slot_weight / scaler_degree_f take sum, mean, min, max, var and std only");
    PNA_REQUIRE(!d->peer_gathered && !d->row_ids, PNA_ERR_UNSUPPORTED,
                "pna_aggregate_fwd: slot_weight / scaler_degree_f are not available with peer_gathered or row_ids");
  }
  if (d->n_rows == 0) return PNA_OK;
  PNA_REQUIRE(d->gathered && d->rowptr && d->out, PNA_ERR_BAD_ARG, "pna_aggregate_fwd: null gathered/rowptr/out");
  PNA_REQUIRE(d->split_threshold >= 2 && d->chunk_edges >= 1, PNA_ERR_BAD_ARG, "pna_aggregate_fwd: bad split/chunk");
  if (d->n_hubs > 0 && !(d->flags & PNA_FLAG_SKIP_HUBS))
    PNA_REQUIRE(d->hub_info && d->chunk_items && d->hub_partials, PNA_ERR_BAD_ARG,
                "pna_aggregate_fwd: n_hubs=%lld but hub_info/chunk_items/hub_partials missing", (long long)d->n_hubs);
  if (adj_weight) {
    PNA_REQUIRE(d->ld_out >= (long long)d->n_towers * ((d->self_feat ? 1 : 0) + d->n_aggr * d->n_scalers) * (d->n_feat / d->n_towers),
                PNA_ERR_BAD_ARG, "pna_aggregate_fwd: ld_out smaller than the row width");
    const AWParams a = adj_weight_params(d, sw, sdf);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return d->dtype == PNA_F32 ? launch_adj_weight_fwd<float>(a, st) : launch_adj_weight_fwd<__nv_bfloat16>(a, st);
  }

  KParams p;
  p.x = d->gathered; p.ldx = d->ld_gathered;
  p.rowptr = d->rowptr; p.col = d->col;
  p.bias = d->row_bias; p.ldb = d->ld_row_bias;
  p.self = d->self_feat; p.lds = d->ld_self; p.self_tstride = d->self_tower_stride;
  p.out = d->out; p.ldo = d->ld_out;
  p.n_rows = d->n_rows;
  p.F = d->n_feat; p.T = d->n_towers; p.Ft = d->n_feat / d->n_towers;
  p.has_self = d->self_feat ? 1 : 0;
  p.nA = d->n_aggr; p.nS = d->n_scalers; p.scodes = d->scaler_codes;
  p.acodes = addons ? strip_addons(d->aggr_codes, d->n_aggr) : d->aggr_codes;   // the add-on kernels write those columns
  p.Wt = (p.has_self + p.nA * p.nS) * p.Ft;
  p.avg_log = d->avg_log; p.avg_lin = d->avg_lin;
  p.flags = d->flags; p.split = d->split_threshold; p.chunk = d->chunk_edges;
  p.hub_info = d->hub_info; p.chunk_items = d->chunk_items; p.n_hubs = d->n_hubs; p.n_chunks = d->n_chunks;
  p.partials = d->hub_partials;
  p.hub_done = d->hub_done;
  p.row_ids = d->row_ids; p.n_row_ids = d->row_ids ? d->n_row_ids : 0;
  // a view that contains chunk pseudo-rows cannot be used when the split rows are to be skipped
  const bool view = d->light_rowptr && d->light_deg && d->part && d->n_part >= 1 && (d->light_col || !d->col) &&
                    !(d->n_view_rows > d->n_rows && ((d->flags & PNA_FLAG_SKIP_HUBS) || d->row_ids));
  p.lrowptr = view ? d->light_rowptr : nullptr; p.ldeg = view ? d->light_deg : nullptr; p.lcol = d->light_col; p.part = d->part;
  p.n_part = d->n_part;
  // chunk pseudo-rows are only usable when the split rows are to be processed in this call
  p.n_view_rows = (view && d->n_view_rows > d->n_rows && !(d->flags & PNA_FLAG_SKIP_HUBS) && d->n_hubs > 0 && !d->row_ids)
                      ? d->n_view_rows : d->n_rows;
  PNA_REQUIRE(p.n_view_rows == d->n_rows || d->n_view_rows == d->n_rows + d->n_chunks, PNA_ERR_BAD_ARG,
              "pna_aggregate_fwd: n_view_rows must be n_rows + n_chunks");
  p.work_ctr = d->work_counter; p.n_static = 0;
  p.sdeg = d->scaler_degree;
  // more than 512 chunks in one row: merge the partials with the radix tree (k_hub_tree) before the finalize
  p.hub_merged = (d->max_degree > 0 && (long long)d->max_degree > 512ll * d->chunk_edges) ? 1 : 0;
  p.peer_x = reinterpret_cast<const void* const*>(d->peer_gathered); p.peer_shift = d->peer_shift;
  if (p.peer_x) PNA_REQUIRE(d->peer_shift >= 1 && d->peer_shift <= 30, PNA_ERR_BAD_ARG, "pna_aggregate_fwd: peer_shift out of range");
  PNA_REQUIRE(p.ldx < 0x3fffffffll && p.ldb < 0x7fffffffll && p.lds < 0x7fffffffll, PNA_ERR_UNSUPPORTED,
              "pna_aggregate_fwd: row pitch too large");     // ld_gathered in BYTES is a 32-bit kernel operand
  PNA_REQUIRE(p.ldo >= (long long)p.T * p.Wt, PNA_ERR_BAD_ARG, "pna_aggregate_fwd: ld_out %lld < row width %lld",
              (long long)p.ldo, (long long)p.T * p.Wt);

  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int esz = d->dtype == PNA_F32 ? 4 : 2;
  const int vec = 16 / esz;
  // 128-bit path needs every row start and every output segment 16-byte aligned.
  bool vec_ok = (p.Ft % vec == 0) && aligned16(p.x) && aligned16(p.out) && (p.ldx % vec == 0) && (p.ldo % vec == 0);
  if (p.bias) vec_ok = vec_ok && aligned16(p.bias) && (p.ldb % vec == 0);
  if (p.self) vec_ok = vec_ok && aligned16(p.self) && (p.lds % vec == 0) && (p.self_tstride % vec == 0);
  int rc;
  if (d->dtype == PNA_F32) {
    rc = vec_ok ? launch_typed<float, 4>(p, st) : launch_typed<float, 1>(p, st);
  } else {
    rc = vec_ok ? launch_typed<__nv_bfloat16, 8>(p, st) : launch_typed<__nv_bfloat16, 1>(p, st);
  }
  if (rc != PNA_OK || !addons) return rc;
  return d->dtype == PNA_F32 ? launch_addons_fwd<float>(d, st) : launch_addons_fwd<__nv_bfloat16>(d, st);
}

extern "C" int pna_aggregate_fwd(const pna_agg_t* d, pna_stream_t stream) { return fwd_entry(d, nullptr, nullptr, stream); }

extern "C" int pna_aggregate_fwd_weighted(const pna_agg_t* d, const float* slot_weight, const float* scaler_degree_f,
                                          pna_stream_t stream) {
  return fwd_entry(d, slot_weight, scaler_degree_f, stream);
}
