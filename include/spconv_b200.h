/*
 * spconv_b200.h -- C ABI of the H100-native (sm_90a) sparse-convolution hot path.
 *
 * This is the drop-in boundary: plain pointers, sizes and a cudaStream_t; no torch /
 * tv::Tensor types.  Every entry point replaces one pybind entry of the reference's
 * generated `core_cc` module (paths relative to the reference tree):
 *
 *   spx_subm_rulebook / spx_conv_rulebook_stage1+2 / spx_native_pairs
 *        <- SpconvOps.get_indice_pairs              spconv/csrc/sparse/all.py:2020-2218
 *        <- SpconvOps.get_indice_pairs_implicit_gemm spconv/csrc/sparse/all.py:1660-2016
 *           (kernels spconv/csrc/sparse/indices.py:292-939)
 *   spx_mask_argsort
 *        <- SpconvOps.sort_1d_by_key_allocator[_v2]  spconv/csrc/sparse/all.py:935-1134
 *   spx_rulebook_workspace_size
 *        <- SpconvOps.get_indice_gen_workspace_size  spconv/csrc/sparse/all.py:1582-1656
 *   spx_implicit_gemm_fwd
 *        <- ConvGemmOps.implicit_gemm                spconv/csrc/sparse/convops.py:2075-2243
 *   spx_implicit_gemm_dgrad / spx_implicit_gemm_wgrad
 *        <- ConvGemmOps.implicit_gemm_backward       spconv/csrc/sparse/convops.py:2247-2440
 *   spx_pairs_to_table (+ the three above)
 *        <- ConvGemmOps.indice_conv / indice_conv_backward
 *                                                    spconv/csrc/sparse/convops.py:1504-2071
 *   spx_bias_act_inplace
 *        <- InferenceOps.bias_add_act_inplace        spconv/csrc/sparse/inference.py:166-252
 *   spx_point2voxel_stage1 / _stage2
 *        <- SpconvOps.point2voxel_cuda               spconv/csrc/sparse/all.py:1349-1490
 *   spx_point2voxel_bounded
 *        <- no counterpart: MaskedPointToVoxel (a batch of clouds, voxel count kept on the device)
 *   spx_indice_pool_fwd / spx_indice_pool_bwd / spx_global_pool_rearrange
 *        <- SpconvOps.maxpool_forward / maxpool_backward / maxpool_implicit_gemm_forward /
 *           maxpool_implicit_gemm_backward / avgpool_implicit_gemm_forward / _backward /
 *           global_pool_rearrange                    spconv/csrc/sparse/all.py:664-905
 *           (kernels spconv/csrc/sparse/maxpool.py:41-341)
 *   spx_global_pool_fwd / spx_global_pool_bwd
 *        <- no kernel: the per-sample torch loop of SparseGlobalMaxPool / AvgPool, spconv/pytorch/pool.py:251-278
 *   spx_sparse_add_group / _fwd / _gather (+ spx_conv_rulebook_stage1+2 for the union)
 *        <- functional.sparse_add / sparse_add_hash_based spconv/pytorch/functional.py:441-544
 *   spx_sparse_add_union / spx_masked_sparse_add_plan / _heads (+ _group / _fwd / _gather)
 *        <- no counterpart: functional.masked_sparse_add / masked_remove_duplicate (padded operands, no read-back)
 *   spx_point_scatter_group / _fwd / _bwd (+ spx_sparse_add_gather for the sum's backward)
 *        <- no counterpart: PointVoxelScatter (per-voxel max / mean / sum of point features, no read-back)
 *   spx_point_interp_plan / _fwd / _bwd
 *        <- no counterpart: VoxelPointInterpolator (trilinear / nearest voxel -> point, torchsparse's voxel_to_point)
 *   spx_hash_clear / _insert / _query / _insert_exist / _rank
 *        <- HashTable (spconv/pytorch/hash.py)        spconv/csrc/hash/core.py
 *   spx_depthwise_fwd / _dgrad / _wgrad (+ _wgrad_workspace_size)
 *        <- no counterpart: the conv modules with groups = in_channels = out_channels (the reference refuses groups)
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in `_host`;
 *   - every function returns 0 on success, non-zero on failure; spx_last_error() gives the
 *     message of the last failure on the calling thread (reference: C++ exception text);
 *   - nothing allocates: outputs and scratch are caller-provided (the reference routes all
 *     allocations through ExternalAllocator callbacks, spconv/csrc/sparse/alloc.py:38-123);
 *   - all launches go to `stream`; no function synchronises the stream except
 *     spx_conv_rulebook_stage1, which must return the data-dependent output count
 *     (the reference syncs at the same point, spconv/csrc/sparse/indices.py:1454-1455).
 */
#ifndef SPCONV_B200_H_
#define SPCONV_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SPX_MAX_NDIM 4

/* element types of features / filters */
enum spx_dtype { SPX_F32 = 0, SPX_F16 = 1, SPX_BF16 = 2, SPX_I8 = 3, SPX_E4M3 = 4 };   /* E4M3: OCP fp8 e4m3fn */
/* tv::gemm::Activation as used by the reference epilogues */
enum spx_act { SPX_ACT_NONE = 0, SPX_ACT_RELU = 1, SPX_ACT_SIGMOID = 2, SPX_ACT_LEAKY_RELU = 3 };
/* how fp32 features are multiplied: exact fp32 FMA, or TF32 tensor cores
 * (reference: SPCONV_ALLOW_TF32, spconv/constants.py:117) */
enum spx_f32_mode { SPX_F32_EXACT = 0, SPX_F32_TF32 = 1 };

typedef void *spx_stream_t; /* cudaStream_t */

const char *spx_last_error(void);
int spx_version(void);
/* 0 if device `dev` is usable by this library (compute capability 10.x); fills sm count */
int spx_device_check(int dev, int *sm_count, int *cc_major, int *cc_minor);

/* ------------------------------------------------------------------ rulebook */

typedef struct {
    int ndim;                       /* 1..4 */
    int batch_size;
    int in_dims[SPX_MAX_NDIM];      /* input spatial shape */
    int out_dims[SPX_MAX_NDIM];     /* output spatial shape (== in_dims for SubM) */
    int ksize[SPX_MAX_NDIM];
    int stride[SPX_MAX_NDIM];
    int padding[SPX_MAX_NDIM];
    int dilation[SPX_MAX_NDIM];
    int transposed;                 /* regular conv only */
} spx_conv_geometry;

/* scratch bytes needed by the rulebook entry points for `num_in` inputs
 * (`max_out` = upper bound on outputs; ignored for SubM) */
size_t spx_rulebook_workspace_size(const spx_conv_geometry *g, int64_t num_in, int64_t max_out,
                                   int is_subm);
/* upper bound on active outputs of a regular conv (reference: get_handcrafted_max_act_out,
 * spconv/csrc/sparse/all.py:1559-1580) */
int64_t spx_conv_max_out(const spx_conv_geometry *g, int64_t num_in);

/*
 * SubM rulebook.  indices [N, ndim+1] int32 (b, d0, d1, ..).  Writes every element of
 *   pair_fwd [kv, N]   pair_fwd[k][o] = i  (-1 = none)
 *   pair_bwd [kv, N]   pair_bwd[k][i] = o  (may be NULL)
 *   mask     [N, words] uint32, bit k%32 of word k/32 set iff pair_fwd[k][o] != -1  (may be NULL)
 * `words` = ceil(kv/32).
 * Every rulebook entry point that takes `indices` (here and below, spx_sparse_add_union too) reads its rows as
 * 16-byte vectors and refuses (returns 2) an `indices` pointer that is not 16-byte aligned.
 */
int spx_subm_rulebook(const spx_conv_geometry *g, const int32_t *indices, int64_t N,
                      int32_t *pair_fwd, int32_t *pair_bwd, uint32_t *mask, void *workspace,
                      size_t workspace_bytes, spx_stream_t stream);

/*
 * Regular / transposed conv rulebook, two-phase because the output count M is
 * data-dependent.  Stage 1 hashes every (offset, input) hit, ranks the distinct outputs in
 * the reference CPU's first-touch order and returns M (host sync).  Stage 2 fills
 *   out_inds [M, ndim+1], pair_fwd [kv, M], pair_bwd [kv, N],
 *   mask_fwd [M, words], mask_bwd [N, words]   (masks may be NULL).
 * The same workspace must be passed, untouched, to both stages.
 */
int spx_conv_rulebook_stage1(const spx_conv_geometry *g, const int32_t *indices, int64_t N,
                             int64_t *num_out_host, void *workspace, size_t workspace_bytes,
                             spx_stream_t stream);
int spx_conv_rulebook_stage2(const spx_conv_geometry *g, const int32_t *indices, int64_t N,
                             int64_t M, int32_t *out_inds, int32_t *pair_fwd, int32_t *pair_bwd,
                             uint32_t *mask_fwd, uint32_t *mask_bwd, void *workspace,
                             size_t workspace_bytes, spx_stream_t stream);

/*
 * Fused host entry points: one call = the launches of spx_subm_rulebook + spx_mask_argsort +
 * spx_build_tile_table (resp. spx_conv_rulebook_stage2 + both argsorts + both tile tables), all
 * scratch carved from ONE workspace.  They exist because an eager Python caller pays ~10 us of
 * interpreter / ctypes / allocator time per separate call; results are identical.
 * `mask` is left sorted; tile_table / tile_mask (spx_tile_table_elems, tiles * words) are required.
 * argsort_bwd, table_bwd and tmask_bwd are all NULL (inference: no backward direction) or all given.
 * For a 3-D 3x3x3 SubM with 32-bit keys spx_subm_rulebook_all also keeps a row-major copy of
 * pair_fwd in its workspace (one 128-byte line per voxel), from which the tile table is built with
 * 4 sectors per row instead of one per (row, offset).
 * spx_conv_rulebook_stage2_all continues a spx_conv_rulebook_stage1 that was given a workspace of
 * spx_conv_rulebook_all_workspace_size bytes.
 */
size_t spx_subm_rulebook_all_workspace_size(const spx_conv_geometry *g, int64_t N);
int spx_subm_rulebook_all(const spx_conv_geometry *g, const int32_t *indices, int64_t N,
                          int32_t *pair_fwd, int32_t *pair_bwd, uint32_t *mask, int32_t *argsort,
                          int do_sort, int32_t *tile_table, uint32_t *tile_mask, void *workspace,
                          size_t workspace_bytes, spx_stream_t stream);
size_t spx_conv_rulebook_all_workspace_size(const spx_conv_geometry *g, int64_t N);
int spx_conv_rulebook_stage2_all(const spx_conv_geometry *g, const int32_t *indices, int64_t N,
                                 int64_t M, int32_t *out_inds, int32_t *pair_fwd, int32_t *pair_bwd,
                                 uint32_t *mask_fwd, uint32_t *mask_bwd, int32_t *argsort_fwd,
                                 int32_t *argsort_bwd, int do_sort, int32_t *table_fwd,
                                 uint32_t *tmask_fwd, int32_t *table_bwd, uint32_t *tmask_bwd,
                                 void *workspace, size_t workspace_bytes, spx_stream_t stream);

/*
 * Regular / transposed conv rulebook with the output count kept on the device: the bounded twin of
 * spx_conv_rulebook_stage1 + spx_conv_rulebook_stage2_all in ONE call with no host read-back, so the
 * launch sequence is fixed and CUDA-graph capturable.  The caller gives `bound`, an upper limit on the
 * number of outputs (the role of the reference's num_out_act_bound, spconv/csrc/sparse/all.py:1915);
 * every output-side tensor has exactly `bound` rows: out_inds [bound, ndim+1], pair_fwd [kv, bound],
 * mask_fwd [bound, words], argsort_fwd [bound], table_fwd / tmask_fwd for `bound` rows.  With M the true
 * count (M <= bound):
 *   - rows [0, M) of out_inds, pair_fwd, mask_fwd (before the sort) and all of pair_bwd / mask_bwd are
 *     bit-identical to the unbounded rulebook of the same input (same first-touch ranking);
 *   - rows [M, bound) are padding: out_inds = -1 in every column, pair_fwd = -1, mask 0; pair_bwd never
 *     refers to a padding row.  A padded out_inds fed to the next rulebook contributes nothing: rows
 *     whose batch index is outside [0, batch) are dropped by every insert / probe kernel;
 *   - *num_out = M;  *status |= 1 when more than `bound` outputs existed: those ranked >= bound were
 *     dropped and every pair that pointed at them is -1 (deterministic truncation, *num_out = bound);
 *     *status |= 2 when a hash probe chain overflowed (far more outputs than `bound`): then *num_out = 0
 *     and every pair is -1.  `status` is only ever ORed into: the caller zeroes it once.
 * The hash table is sized from `bound` (load <= 0.5 at M = bound).  1-D to 4-D, 32- and 64-bit keys,
 * 1 to 4 mask words.  argsort_bwd, table_bwd and tmask_bwd are all NULL (inference) or all given.
 */
size_t spx_conv_rulebook_bounded_workspace_size(const spx_conv_geometry *g, int64_t N, int64_t bound);
int spx_conv_rulebook_bounded_all(const spx_conv_geometry *g, const int32_t *indices, int64_t N,
                                  int64_t bound, int32_t *out_inds, int32_t *pair_fwd, int32_t *pair_bwd,
                                  uint32_t *mask_fwd, uint32_t *mask_bwd, int32_t *argsort_fwd,
                                  int32_t *argsort_bwd, int do_sort, int32_t *table_fwd,
                                  uint32_t *tmask_fwd, int32_t *table_bwd, uint32_t *tmask_bwd,
                                  int32_t *num_out, int32_t *status, void *workspace,
                                  size_t workspace_bytes, spx_stream_t stream);

/*
 * Rulebook onto GIVEN output coordinates: a convolution from the source rows `src_indices` [N, ndim+1] (grid in_dims)
 * onto the target rows `out_indices` [M, ndim+1] (grid out_dims), both in batch_size samples.  The geometry is
 * taken as given: a SubM layer passes stride 1 and padding (ksize/2) * dilation with out_dims = in_dims.
 *   - usable source row i: i < *num_valid (every row when num_valid is NULL), batch in [0, batch_size), every
 *     coordinate inside in_dims; among usable rows with equal coordinates the lowest row wins;
 *   - active target row o: the same against *out_num_valid and out_dims, and no lower active row has its
 *     coordinate (a later duplicate is inactive: pair_fwd -1, mask 0);
 *   - per axis, for target o and tap r: regular c = o * stride - pad + r * dil; transposed
 *     c = (o + pad - r * dil) / stride when the division is exact; valid iff 0 <= c < in_dims;
 *   - pair_fwd [kv, M]: pair_fwd[k][o] = the usable row at c, else -1; mask_fwd [M, words] its bits;
 *     pair_bwd [kv, N]: pair_bwd[k][i] = o for every such pair, else -1; mask_bwd [N, words] its bits.
 * Then both mask argsorts and both tile tables, as spx_conv_rulebook_stage2_all (argsort_bwd, table_bwd and
 * tmask_bwd all NULL for inference; pair_bwd and mask_bwd are always written).  M is the caller's, so there is no
 * host read-back: the launch sequence is fixed and CUDA-graph capturable.  Every output is bit-reproducible.
 * Kernel volume <= 128, 1-D to 4-D, padding >= 0, 64-bit keys once batch * prod(dims) of either grid reaches
 * 2^31 - 1.  Both index pointers must be 16-byte aligned.  Either side may be empty.
 */
size_t spx_cross_rulebook_all_workspace_size(const spx_conv_geometry *g, int64_t N, int64_t M);
int spx_cross_rulebook_all(const spx_conv_geometry *g, const int32_t *src_indices, int64_t N,
                           const int32_t *num_valid, const int32_t *out_indices, int64_t M,
                           const int32_t *out_num_valid, int32_t *pair_fwd, int32_t *pair_bwd,
                           uint32_t *mask_fwd, uint32_t *mask_bwd, int32_t *argsort_fwd, int32_t *argsort_bwd,
                           int do_sort, int32_t *table_fwd, uint32_t *tmask_fwd, int32_t *table_bwd,
                           uint32_t *tmask_bwd, void *workspace, size_t workspace_bytes, spx_stream_t stream);

/* Zero rows [*count, rows) of a row-major matrix with `row_bytes` (even) bytes per row; `count` is a
 * device int32 (the num_out of a bounded rulebook).  Used on gradients that arrive for padded tensors. */
int spx_zero_rows_from_count(void *ptr, int64_t rows, int64_t row_bytes, const int32_t *count,
                             spx_stream_t stream);

/*
 * Compact "Native" rulebook  pairs [2, kv, N] (-1 padded) + indice_pair_num [kv]  in the
 * reference CPU order (ascending input index per offset), derived from pair_bwd [kv, N] by a
 * stable scan.  For SubM only offsets < kv/2 are counted and their mirrors written, the centre
 * row is the identity (spconv/csrc/sparse/indices.py:1670-1703).
 */
int spx_native_pairs(const int32_t *pair_bwd, int64_t N, int kv, int is_subm, int32_t *pairs,
                     int32_t *indice_pair_num, void *workspace, size_t workspace_bytes,
                     spx_stream_t stream);
size_t spx_native_pairs_workspace_size(int64_t N, int kv);

/*
 * Inverse of spx_native_pairs for the ConvAlgo.Native operator path: scatter a compact
 * rulebook into dense tables  table_fwd [kv, n_out] / table_bwd [kv, n_in]  and row masks.
 * `inverse` swaps the roles of pairs[0] / pairs[1] (SparseInverseConv).  Any output may be NULL.
 */
int spx_pairs_to_table(const int32_t *pairs, const int32_t *indice_pair_num, int kv,
                       int64_t pair_stride, int64_t n_in, int64_t n_out, int is_subm, int inverse,
                       int32_t *table_fwd, int32_t *table_bwd, uint32_t *mask_fwd,
                       uint32_t *mask_bwd, spx_stream_t stream);

/*
 * argsort[N] <- stable ascending argsort of mask[N, words] (word 0 most significant) and mask
 * is left SORTED, as thrust::sort_by_key leaves it in the reference.  do_sort == 0: iota only.
 */
size_t spx_mask_argsort_workspace_size(int64_t N, int words);
int spx_mask_argsort(uint32_t *mask, int32_t *argsort, int64_t N, int words, int kv, int do_sort,
                     void *workspace, size_t workspace_bytes, spx_stream_t stream);

/* ------------------------------------------------------------------ conv arithmetic */

typedef struct {
    int dtype;                  /* spx_dtype of features, filters, outputs */
    int f32_mode;               /* spx_f32_mode, only read when dtype == SPX_F32 */
    int kv;                     /* kernel volume */
    int c_in, c_out;            /* C, K of the KRSC filter [K, kv, C] */
    int64_t n_in, n_out;        /* rows of the input / output feature matrices */
    const int32_t *pair;        /* [kv, rows] gather table of THIS pass (see each function) */
    int64_t pair_stride;        /* elements between consecutive offsets of `pair` */
    const uint32_t *mask;       /* [rows, words] in argsort order, or NULL = all offsets */
    const int32_t *argsort;     /* [rows] row visiting order, or NULL = identity */
    int reverse_offsets;        /* 1: offset k of `pair`/`mask` multiplies filter kv-1-k
                                   (SubM dgrad through the forward table; reference
                                   reverse_mask, spconv/csrc/sparse/convops.py:2412) */
    const int32_t *tile_table;  /* optional: spx_build_tile_table output for (pair, argsort);  */
    const uint32_t *tile_mask;  /* both or neither.  Required by the wgmma kernels: without     */
                                /* them the call runs on the generic FMA kernels.               */
} spx_gemm_desc;

/*
 * Tile-blocked gather table: the (pair, argsort, mask) triple re-laid so that one 128-row tile is
 * one contiguous block the kernels fetch with a single bulk async copy:
 *   table     [tiles][kv + 1][128] int32:  table[t][k][r] = pair[k][row(t*128 + r)]  (k < kv),
 *                                          table[t][kv][r] = row(t*128 + r)   (-1 past the end)
 *             with row(j) = argsort ? argsort[j] : j
 *   tile_mask [tiles][words] uint32: OR of mask[t*128 .. t*128+127] (mask in visiting order;
 *             NULL mask = all kv offsets) == the reference's mask_output_fwd with mask_width 128
 *             (spconv/csrc/sparse/convops.py:2180-2189)
 * tiles = ceil(rows / 128).  Built once per rulebook, shared by fwd / dgrad / wgrad of every
 * layer that shares the indice_key.
 *
 * The `table` buffer (spx_tile_table_elems int32 elements, 16-byte aligned) continues behind the
 * blocks with what the dynamically scheduled kernels need:
 *   records [tiles][8] int32: {tile, mask words[4], 0, 0, 0}, tiles in order of decreasing
 *             offset count (ties: ascending tile) -- fwd / dgrad CTAs draw tickets from an atomic
 *             counter and take tiles in this order (longest-processing-time-first scheduling);
 *   scratch [64] int32: 32 {ticket counter, finished-CTA counter} pairs.  Zero after the build; every
 *             launch takes the next pair (round-robin per process) and its last CTA zeroes it again,
 *             so up to 32 launches may be in flight on one table (other streams, graph branches).
 */
size_t spx_tile_table_elems(int64_t rows, int kv);
int spx_build_tile_table(const int32_t *pair, int64_t pair_stride, int kv, const int32_t *argsort,
                         const uint32_t *mask, int64_t rows, int32_t *table, uint32_t *tile_mask,
                         spx_stream_t stream);

/*
 * out[o, :] = act( sum_k x[pair[k][o], :] @ W[:, k, :]^T  + bias )      rows = n_out
 * filters: KRSC [c_out, kv, c_in].  bias (same dtype as features) may be NULL.
 * The tensor-core kernels also need features, filters and out 16-byte aligned; otherwise the call runs on the
 * FMA kernels (under SPX_FORCE_TC=1 it returns 3).  The same holds for out_bp, filters, din of the input
 * gradient, features and out_bp of the weight gradient, and features, filters, out of the int8 forward.
 */
int spx_implicit_gemm_fwd(const spx_gemm_desc *d, const void *features, const void *filters,
                          void *out, const void *bias, int act, float act_alpha,
                          spx_stream_t stream);

/*
 * din[i, :] = sum_k dout[pair[k][i], :] @ W[:, k', :]        rows = n_in, k' = k or kv-1-k
 * `pair` is the backward table [kv, n_in] (in -> out).
 */
int spx_implicit_gemm_dgrad(const spx_gemm_desc *d, const void *out_bp, const void *filters,
                            void *din, spx_stream_t stream);

/*
 * dW[:, k, :] = sum_o dout[o, :]^T  x[pair[k][o], :]          rows = n_out, pair = forward table
 * dfilters: KRSC, same dtype as features.  workspace holds fp32 partial sums.
 */
size_t spx_implicit_gemm_wgrad_workspace_size(const spx_gemm_desc *d);
int spx_implicit_gemm_wgrad(const spx_gemm_desc *d, const void *features, const void *out_bp,
                            void *dfilters, void *workspace, size_t workspace_bytes,
                            spx_stream_t stream);

/*
 * Grouped convolution, 1 < groups: group j maps input channels [j Cg, (j+1) Cg) to output channels [j Kg, (j+1) Kg)
 * (Cg = c_in / groups, Kg = c_out / groups) with filter rows [j Kg, (j+1) Kg) of the filter [c_out, kv, Cg], torch's
 * grouped convention on the KRSC filter.  The descriptor is the dense one: c_in / c_out are the totals, the row counts,
 * tables and tile tables those of the layer's rulebook.  Cg and Kg must be multiples of 16; groups == 1 is refused
 * (the dense entry points are the one path for it), and so is every other bad shape, before any launch.
 *
 * Each call runs one pass per group, in ascending j, on `stream`: the dense kernel instance for (Cg, Kg), with the
 * same schedule and fp32 summation order, reading gathered rows at the full row stride (C or K) from the group's
 * column offset and writing output rows the same way.  So for every group, out[:, j Kg:(j+1) Kg], din[:, j Cg:(j+1) Cg]
 * and dW[j Kg:(j+1) Kg] equal bit for bit what spx_implicit_gemm_fwd / _dgrad / _wgrad return on the contiguous
 * slices of that group.  Routes: fp16 / bf16 run on the tensor cores when the dense calls would at (Cg, Kg) (tile
 * tables given, 16-byte aligned operands); fp32, in both f32 modes, and every other shape run on the FMA kernels (an
 * fp32 call in SPX_F32_TF32 mode therefore equals the dense call in SPX_F32_EXACT mode).  Pointers must be aligned to
 * their element size.  SPX_FORCE_SIMT / SPX_FORCE_TC apply; spx_last_kernel_family reports the route.  A tensor-core
 * pass holds one of the tile table's scheduler slots while it runs.
 *
 * The weight gradient's passes reuse one workspace (spx_grouped_gemm_wgrad_workspace_size).  _push writes dfilters
 * locally, then pushes the whole gradient to the peer group (spx_peer_push); spx_peer_finish completes the exchange.
 */
typedef struct spx_grouped_gemm {
    const void *features;       /* fwd, wgrad: [n_in, c_in] */
    const void *filters;        /* fwd, dgrad: [c_out, kv, c_in / groups] */
    const void *out_bp;         /* dgrad, wgrad: [n_out, c_out] */
    const void *bias;           /* fwd: [c_out] or NULL, dtype of features */
    void *out;                  /* fwd: [n_out, c_out] */
    void *din;                  /* dgrad: [n_in, c_in]; `pair` is the backward table, as in spx_implicit_gemm_dgrad */
    void *dfilters;             /* wgrad: [c_out, kv, c_in / groups]; `pair` is the forward table */
    void *workspace;            /* wgrad */
    size_t workspace_bytes;
    int act;                    /* fwd: spx_act */
    float act_alpha;
} spx_grouped_gemm;
int spx_grouped_gemm_fwd(const spx_gemm_desc *d, int groups, const spx_grouped_gemm *a, spx_stream_t stream);
int spx_grouped_gemm_dgrad(const spx_gemm_desc *d, int groups, const spx_grouped_gemm *a, spx_stream_t stream);
size_t spx_grouped_gemm_wgrad_workspace_size(const spx_gemm_desc *d, int groups);
int spx_grouped_gemm_wgrad(const spx_gemm_desc *d, int groups, const spx_grouped_gemm *a, spx_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Data-parallel weight-gradient exchange over NVLink peer memory (SURVEY 8e).  The reference has no
 * distributed code: users wrap it in torch DDP, i.e. an NCCL all-reduce of dW after the backward
 * pass.  Here the SEND side is the tail of the weight-gradient kernel itself (csrc/peer.cu): the kernel
 * that reduces the split-K partials writes this rank's fp32 slice sums into its own exchange buffer and
 * its last CTA publishes the epoch to every rank (one system fence, `world` flag stores over NVLink).
 * The RECEIVE side (finish) reads every rank's slices through the peer mapping and sums them in rank
 * order, so all replicas end with bit-identical gradients after one rounding.  Put independent work (the
 * input gradient of the same layer) between push and finish and the NVLink latency is hidden.
 *
 * Set-up (once per process group; the host side passes the 64-byte handles around, e.g. with
 * torch.distributed.all_gather_object): every rank creates its buffer, opens the others', and fills
 * a spx_peer_group with the addresses AS MAPPED IN ITS OWN PROCESS (buffers[rank] = its own).
 * Contract: on each rank, push and finish of one group alternate in stream order (one exchange in
 * flight), and all ranks issue the same sequence of exchanges.
 */
#define SPX_MAX_PEERS 16
typedef struct spx_peer_group {
    int world, rank;
    int timeout_ms;                 /* a peer that does not arrive in time: NaN result + spx_peer_error (0 = 20 s) */
    int colocated;                  /* ranks of this group that share ONE device (tests); 0 or 1 = one rank per GPU */
    uint64_t capacity_bytes;        /* largest exchanged tensor, as fp32 (what spx_peer_buffer_create got) */
    void *buffers[SPX_MAX_PEERS];   /* exchange buffer of every rank */
} spx_peer_group;

size_t spx_peer_buffer_bytes(size_t capacity_bytes, int world);
int spx_peer_buffer_create(size_t capacity_bytes, int world, void **buffer, unsigned char handle[64]);
int spx_peer_buffer_open(const unsigned char handle[64], void **mapped);
int spx_peer_buffer_close(void *mapped);
int spx_peer_buffer_destroy(void *buffer);
/* sticky error word of this rank's buffer (1 = a peer timed out); synchronous copy */
int spx_peer_error(const spx_peer_group *pg, int *error);

/* Weight gradient of this rank (see spx_implicit_gemm_wgrad), published to the group in fp32 by the kernel
 * that reduces the split-K partials.  dfilters is NOT valid afterwards (scratch for shapes
 * the tensor-core kernel does not tile): spx_peer_finish(pg, dfilters, kv*C*K, dtype, scale) writes it. */
int spx_implicit_gemm_wgrad_push(const spx_gemm_desc *d, const void *features, const void *out_bp,
                                 void *dfilters, void *workspace, size_t workspace_bytes,
                                 const spx_peer_group *pg, spx_stream_t stream);
/* Grouped weight gradient (see spx_grouped_gemm_wgrad) written to a->dfilters, then pushed whole to the group;
 * spx_peer_finish(pg, dfilters, kv*C/groups*K, dtype, scale) completes it. */
int spx_grouped_gemm_wgrad_push(const spx_gemm_desc *d, int groups, const spx_grouped_gemm *a,
                                const spx_peer_group *pg, spx_stream_t stream);
/* the same exchange for an existing small tensor (bias gradients ...): push sends `data` (dtype SPX_F32 /
 * SPX_F16 / SPX_BF16), finish writes out = scale * sum over ranks (out may be data); allreduce = both */
int spx_peer_push(const spx_peer_group *pg, const void *data, int64_t count, int dtype, spx_stream_t stream);
int spx_peer_finish(const spx_peer_group *pg, void *out, int64_t count, int dtype, float scale, spx_stream_t stream);
int spx_peer_allreduce(const spx_peer_group *pg, void *data, int64_t count, int dtype, float scale,
                       spx_stream_t stream);
/* gather: every rank's `count` 32-bit words of src land, unchanged, in dst[r * count, (r + 1) * count) for r in
 * rank order, on every rank.  The same push and finish protocol (one exchange in flight); a timed-out peer
 * leaves dst NaN (0x7fc00000) and sets spx_peer_error. */
int spx_peer_allgather(const spx_peer_group *pg, const uint32_t *src, int64_t count, uint32_t *dst,
                       spx_stream_t stream);

/* x[r, j] = act(x[r, j] + bias[j])   in place; bias may be NULL */
int spx_bias_act_inplace(void *x, const void *bias, int64_t rows, int cols, int dtype, int act,
                         float act_alpha, spx_stream_t stream);

/* ------------------------------------------------------------------ point cloud -> voxels */

/*
 * Replaces SpconvOps.point2voxel_cuda / Point2Voxel (spconv/csrc/sparse/all.py:1349-1490,
 * spconv/csrc/sparse/pointops.py:120-490) with the deterministic semantics of the reference's CPU
 * implementation (Point2VoxelCPU, pointops.py:589-695): voxel id = rank of the voxel's first point
 * in input order; voxels beyond max_voxels are dropped; a voxel keeps its first
 * max_points_per_voxel points in input order.
 *   points [N, num_features] fp32 (device), the first ndim features are coordinates (x, y, z, ..);
 *   vsize / grid_size / coors_range are HOST arrays in the internal axis order that
 *   calc_meta_data produces (zyx != 0: axis j reads point feature ndim-1-j);  coors_range holds the
 *   ndim lower bounds first.
 * Stage 1 hashes and ranks the voxels and returns their number (host sync, as the reference's
 * sliced return tensors require): *num_voxels = min(total, max_voxels).  Stage 2 (same untouched
 * workspace) fills
 *   voxels [>= num_voxels, max_points, num_features] (unused slots are left as the caller set them,
 *          or receive the voxel mean when empty_mean != 0),  indices [>= num_voxels, ndim],
 *   num_per_voxel [>= num_voxels],  pc_voxel_id [N] int64 (-1 = no voxel).
 */
size_t spx_point2voxel_workspace_size(int64_t num_points, int ndim);
int spx_point2voxel_stage1(const float *points, int64_t N, int num_features, int ndim, int zyx,
                           const float *vsize_host, const int *grid_size_host,
                           const float *coors_range_host, int64_t max_voxels, int64_t *num_voxels_host,
                           int64_t *total_voxels_host, void *workspace, size_t workspace_bytes,
                           spx_stream_t stream);
int spx_point2voxel_stage2(const float *points, int64_t N, int num_features, int ndim, int zyx,
                           const float *vsize_host, const int *grid_size_host,
                           const float *coors_range_host, int64_t num_voxels, int64_t total_voxels,
                           int max_points_per_voxel, int empty_mean, float *voxels, int32_t *indices,
                           int32_t *num_per_voxel, int64_t *pc_voxel_id, void *workspace,
                           size_t workspace_bytes, spx_stream_t stream);

/*
 * A batch of clouds in one call, with the voxel count kept on the device (MaskedPointToVoxel): nothing is read
 * back, so the call captures into a CUDA graph.  Geometry, points and the per-sample semantics as above.
 *   point_offsets [batch_size + 1] device int32 (NULL: one sample of all N points, batch_size must be 1).  The
 *   offsets are normalised on the device: each is clamped to [0, N], then the prefix maximum is taken; sample b
 *   owns the points [off[b], off[b+1]), points outside every sample are padding and are never read.
 *   Per sample, the voxels are those of spx_point2voxel_stage1/2 with max_voxels run on the sample's points
 *   alone, bit for bit (order, cap, kept points, empty_mean fill).  Rows hold sample 0's kept voxels, then
 *   sample 1's, .. packed; M = *num_valid = min(sum of the kept counts, bound).  Every output element is written:
 *   voxels [bound, max_points, num_features] (unused slots: the voxel mean when empty_mean != 0, else 0),
 *   indices [bound, ndim + 1] (batch index, then the cell in the internal axis order), num_per_voxel [bound];
 *   rows [M, bound) hold indices -1, voxels 0, num_per_voxel 0.  pc_voxel_id [N] int64: the row of the point's
 *   voxel, -1 for padding points, points out of range and points of dropped voxels.  *status |= 1 when more
 *   than `bound` voxels were kept (the rows ranked >= bound are dropped); status is only ever ORed into.
 * Limits: batch_size in [1, SPX_P2V_MAX_BATCH], N and bound below 2^31 - 1, bound >= 1, batch_size x grid
 * volume below 2^62 (64-bit hash keys from 2^31 - 1 on).  workspace: spx_point2voxel_bounded_workspace_size
 * bytes (0 = invalid sizes).
 */
#define SPX_P2V_MAX_BATCH 65536
size_t spx_point2voxel_bounded_workspace_size(int64_t num_points, int batch_size, int64_t bound);
int spx_point2voxel_bounded(const float *points, int64_t N, int num_features, int ndim, int zyx,
                            const float *vsize_host, const int *grid_size_host, const float *coors_range_host,
                            const int32_t *point_offsets, int batch_size, int64_t max_voxels, int64_t bound,
                            int max_points_per_voxel, int empty_mean, float *voxels, int32_t *indices,
                            int32_t *num_per_voxel, int64_t *pc_voxel_id, int32_t *num_valid, int32_t *status,
                            void *workspace, size_t workspace_bytes, spx_stream_t stream);

/* ------------------------------------------------------------------ pooling on the rulebook */

/*
 * out[o, :] = reduce over the offsets k with pair_fwd[k][o] >= 0 of x[pair_fwd[k][o], :]
 *   mode 0  max, rows without any input get the dtype's lowest value
 *           (SparseMaxPool, ConvAlgo.MaskImplicitGemm: maxpool.py:76-117)
 *   mode 1  max with a floor of 0 (ConvAlgo.Native: the reference raises a zero-initialised buffer,
 *           spconv/pytorch/ops.py:1910-1936 + maxpool.py:41-73); the caller passes the dense table
 *           made by spx_pairs_to_table from the compact pairs
 *   mode 2  mean over the valid inputs; count_out [n_out] int32 (may be NULL) receives their number
 *           (SparseAvgPool: maxpool.py:211-259)
 * channels * element size must be a multiple of 16 bytes, and features / out 16-byte aligned (returns 2
 * otherwise; spx_indice_pool_bwd likewise for features, out_features, out_bp and din).  dtype: f32 / f16 /
 * bf16, int8 for max.
 */
int spx_indice_pool_fwd(int mode, const void *features, void *out, const int32_t *pair_fwd,
                        int64_t pair_stride, int kv, int64_t n_out, int channels, int dtype,
                        int32_t *count_out, spx_stream_t stream);
/*
 * Input gradient through pair_bwd [kv, n_in] (in -> out):
 *   modes 0, 1  din[i] = sum_k (x[i] == y[o_k]) ? dy[o_k] : 0        (maxpool.py:120-208)
 *   mode 2      din[i] = sum_k dy[o_k] * count_out[o_k]              (maxpool.py:262-300, as is)
 */
int spx_indice_pool_bwd(int mode, const void *features, const void *out_features, const void *out_bp,
                        void *din, const int32_t *pair_bwd, int64_t pair_stride, int kv, int64_t n_in,
                        int channels, int dtype, const int32_t *count_out, spx_stream_t stream);
/*
 * Rows of every sample in input order: out_indices [batch_size, n] (only the first counts[b]
 * entries of row b are written), counts [batch_size]; coords [n, row_ints] with the batch index
 * first.  Deterministic (the reference appends with atomics, maxpool.py:303-341; the CPU version
 * keeps input order, :599-620).
 */
int spx_global_pool_rearrange(const int32_t *coords, int64_t n, int row_ints, int batch_size,
                              int32_t *out_indices, int32_t *counts, spx_stream_t stream);
/*
 * Padding-aware global pooling (MaskedGlobalMaxPool / MaskedGlobalAvgPool): out [batch_size, channels] per
 * sample, with no host read-back.  M = *num_valid (device int32, clamped to [0, rows]; NULL = every row).
 * Row r counts for sample b when r < M and coords[r * row_ints] == b with 0 <= b < batch_size; rows [M, rows)
 * are never read (features nor coords), rows with another batch index are dropped.
 *   mode 0  max: out[b, c] = x[a, c] bit for bit, a = argmax[b, c] [batch_size, channels] the first row in
 *           ascending order that attains the maximum; a NaN counts as the maximum, -0 and +0 tie
 *   mode 1  mean: out[b, c] = (fp32 sum of the sample's rows) / count[b], rounded once; count [batch_size]
 * An empty sample gives out = 0, argmax = -1, count = 0.  The rows of a sample are reduced in a fixed order
 * that depends on them alone (chunks of rows merged in chunk order, no float atomics), so every result is
 * bit-reproducible and independent of `rows` (padding).
 * bwd: din [rows, channels], every element written once: mode 0 din[a, c] = dy[b, c] at a = argmax[b, c],
 *      mode 1 din[r, c] = dy[b, c] / count[b] in fp32, rounded once; 0 on padding and dropped rows.
 * dtype: f32 / f16 / bf16.  batch_size in [1, 2^20], channels in [1, 65536], rows < 2^31 - 1.
 * workspace (fwd only): spx_global_pool_workspace_size(rows, batch_size, channels) bytes.
 */
size_t spx_global_pool_workspace_size(int64_t rows, int batch_size, int channels);
int spx_global_pool_fwd(int mode, const void *features, const int32_t *coords, int64_t rows, int row_ints,
                        int batch_size, int channels, int dtype, const int32_t *num_valid, void *out, int32_t *argmax,
                        int32_t *count, void *workspace, size_t workspace_bytes, spx_stream_t stream);
int spx_global_pool_bwd(int mode, const void *dy, const int32_t *coords, int64_t rows, int row_ints, int batch_size,
                        int channels, int dtype, const int32_t *num_valid, const int32_t *argmax, const int32_t *count,
                        void *din, spx_stream_t stream);

/* ------------------------------------------------------------------ sum over different coordinates */

/*
 * Replaces spconv.pytorch.functional.sparse_add / sparse_add_hash_based (spconv/pytorch/functional.py:441-544).
 * The operands are concatenated in VISIT order (the caller's choice; sparse_add visits the largest operand
 * first); row g of the concatenation is row g - start[t] of operand t.  The union of their coordinates is
 * the regular-conv rulebook of a 1x..x1 stride-1 convolution over the concatenated coordinates: stage 1/2
 * give out_inds [M] and dst = pair_bwd[0] [rows] (output row of every visited row, -1 = out of range).
 *
 * group:  order [rows] = stable argsort of dst (rows with dst = -1 last), offsets [M + 1]: the visited rows of
 *         output o are order[offsets[o] .. offsets[o+1]) in ascending visit order.  dst must come from
 *         the union above (M = its output count).
 * fwd:    out [M, channels] = per output, the fp32 sum of its rows in visit order, rounded once.
 * gather: for every visited row g with grads[t] != NULL: grads[t][g - start[t]] = index[g] >= 0 ?
 *         src[index[g]] : 0 (bit copy), index [rows], src [src_rows, channels].
 * dtype: f32 / f16 / bf16.  Any channel count >= 1 (16-byte vectors when rows and pointers allow them).
 */
#define SPX_SPARSE_ADD_MAX_OPERANDS 64
typedef struct {
    int count;                                              /* 1 .. SPX_SPARSE_ADD_MAX_OPERANDS */
    int64_t rows[SPX_SPARSE_ADD_MAX_OPERANDS];              /* rows of every operand, in visit order */
    const void *features[SPX_SPARSE_ADD_MAX_OPERANDS];      /* [rows[t], channels], read by fwd */
    void *grads[SPX_SPARSE_ADD_MAX_OPERANDS];               /* [rows[t], channels], written by gather (NULL = skip) */
} spx_sparse_add_operands;

size_t spx_sparse_add_group_workspace_size(int64_t rows);
int spx_sparse_add_group(const int32_t *dst, int64_t rows, int64_t M, int32_t *order, int32_t *offsets,
                         void *workspace, size_t workspace_bytes, spx_stream_t stream);
int spx_sparse_add_fwd(const spx_sparse_add_operands *operands, const int32_t *order, const int32_t *offsets,
                       int64_t M, int channels, int dtype, void *out, spx_stream_t stream);
int spx_sparse_add_gather(const int32_t *index, const void *src, int64_t src_rows,
                          const spx_sparse_add_operands *operands, int channels, int dtype, spx_stream_t stream);

/*
 * The union with the output count kept on the device: the bounded rulebook (spx_conv_rulebook_bounded_all) of
 * the 1x..x1, stride-1, padding-0 convolution `g` (out_dims = in_dims) over indices [N, ndim+1], without masks,
 * mask sorts or tile tables.  out_inds [bound, ndim+1]: the distinct in-range coordinates in first-touch order,
 * rows [M, bound) -1; dst [N] = output row of every row (-1: out of range, or ranked >= bound); *num_out = M;
 * *status |= 1 when more than `bound` outputs existed (those ranked >= bound dropped), |= 2 on a probe-chain
 * overflow (then M = 0).  1 <= bound <= N, bound < 2^30.  32- and 64-bit keys.
 */
size_t spx_sparse_add_union_workspace_size(const spx_conv_geometry *g, int64_t N, int64_t bound);
int spx_sparse_add_union(const spx_conv_geometry *g, const int32_t *indices, int64_t N, int64_t bound,
                         int32_t *out_inds, int32_t *dst, int32_t *num_out, int32_t *status, void *workspace,
                         size_t workspace_bytes, spx_stream_t stream);

/*
 * Padded operands (functional.masked_sparse_add): the operand table and `indices` [rows, ndim+1] are in ARGUMENT
 * order (operands->rows only is read).  num_valid: host array of operands->count device int32 pointers (an entry,
 * or the array, NULL = every row valid); operand t's valid rows are [0, valid_t), valid_t = *num_valid[t] clamped
 * to [0, rows_t].  Rows at and beyond valid_t are never read.  The visit order is decided on the device from the
 * valid counts exactly as sparse_add decides it from the row counts (largest first, ties: the earliest, then the
 * others in argument order), so rows [0, M) of every output equal sparse_add of the valid rows bit for bit.
 *   plan:  out_inds [bound, ndim+1], *num_out, *status as spx_sparse_add_union; dst [rows] (argument order, -1
 *          on padding, out-of-range and dropped rows); order [rows] and offsets [bound + 1] as spx_sparse_add_group
 *          with argument-order row ids (segments in ascending visit order; offsets[o] = offsets[o+1] for o >= M).
 *          spx_sparse_add_fwd (M = bound, argument-order operands) then gives out [bound, C] with rows [M, bound)
 *          0, and spx_sparse_add_gather (index = dst) the gradients.  0 <= bound <= rows, bound >= 1 unless
 *          rows == 0 (then *num_out = 0 and offsets[0] = 0).
 *   heads: heads [bound] = order[offsets[o]] (the row that created output o) for o < *num_out, else -1;
 *          inverse [rows] = o at heads[o], -1 elsewhere (RemoveDuplicate's gather indices).
 */
size_t spx_masked_sparse_add_workspace_size(const spx_conv_geometry *g, int64_t rows, int64_t bound);
int spx_masked_sparse_add_plan(const spx_conv_geometry *g, const spx_sparse_add_operands *operands,
                               const int32_t *const *num_valid, const int32_t *indices, int64_t bound,
                               int32_t *out_inds, int32_t *dst, int32_t *order, int32_t *offsets, int32_t *num_out,
                               int32_t *status, void *workspace, size_t workspace_bytes, spx_stream_t stream);
int spx_masked_sparse_add_heads(const int32_t *order, const int32_t *offsets, const int32_t *num_out, int64_t bound,
                                int64_t rows, int32_t *heads, int32_t *inverse, spx_stream_t stream);

/* ------------------------------------------------------------------ point -> voxel reductions */

/*
 * Per-row reductions of point features x [num_points, channels] (PointVoxelScatter: the scatter of a dynamic
 * VFE), with no host read-back.  ids [num_points] (id_bytes 4: int32, 8: int64; e.g. the pc_voxel_id of
 * spx_point2voxel_bounded) give every point's output row; a point whose id is outside [0, rows) is dropped.
 *   group: row32 [num_points] = the id, or -1 for a dropped point; order [num_points] and offsets [rows + 1] as
 *          spx_sparse_add_group: the points of row r are order[offsets[r] .. offsets[r+1]) in ascending point
 *          index, dropped points last.  rows may exceed num_points; num_points == 0 gives rows + 1 zero offsets.
 *          workspace: spx_point_scatter_group_workspace_size(num_points) bytes.
 *   fwd:   out [rows, channels]; a row without points gives 0 and every element is written:
 *          mode 0 max:  out[r, c] = x[a, c] bit for bit, a = argmax[r, c] ([rows, channels] int32, -1 on an empty
 *                       row) the first point in ascending order that attains the maximum; a NaN counts as the
 *                       maximum, -0 and +0 tie;
 *          mode 1 mean: the fp32 sum of the row's points in ascending order divided by their count, rounded once;
 *          mode 2 sum:  the fp32 sum in ascending order, rounded once (the kernel of spx_sparse_add_fwd).
 *   bwd:   dx [num_points, channels], every element written once, 0 for a dropped point:
 *          mode 0 dx[p, c] = dy[r, c] where argmax[r, c] == p, else 0;  mode 1 dy[r, c] / count[r] in fp32,
 *          rounded once (count [rows] int32 = offsets[r+1] - offsets[r]);  mode 2 dy[r, c]
 *          (spx_sparse_add_gather with index = row32).
 * No float atomics: every result is bit-reproducible and independent of the dropped points, wherever they sit.
 * dtype: f32 / f16 / bf16, any channels >= 1 (16-byte vectors when the row size and pointers allow them).
 * num_points and rows below 2^31 - 1.
 */
size_t spx_point_scatter_group_workspace_size(int64_t num_points);
int spx_point_scatter_group(const void *ids, int id_bytes, int64_t num_points, int64_t rows, int32_t *row32,
                            int32_t *order, int32_t *offsets, void *workspace, size_t workspace_bytes,
                            spx_stream_t stream);
int spx_point_scatter_fwd(int mode, const void *x, int64_t num_points, int channels, int dtype, const int32_t *order,
                          const int32_t *offsets, int64_t rows, void *out, int32_t *argmax, spx_stream_t stream);
int spx_point_scatter_bwd(int mode, const void *dy, const int32_t *row32, int64_t num_points, int64_t rows,
                          int channels, int dtype, const int32_t *argmax, const int32_t *count, void *dx,
                          spx_stream_t stream);

/* ------------------------------------------------------------------ voxel -> point interpolation */

/*
 * Trilinear or nearest interpolation of the features of a sparse tensor at query points (VoxelPointInterpolator:
 * the voxel -> point step of point-voxel networks), with no host read-back.  The tensor is indices [rows, 1 + ndim]
 * (batch, then the coordinates), spatial_shape [ndim], batch_size and num_valid (a device int32, or NULL = every
 * row).  The arguments travel in one block, spx_point_interp (read on the host during the call), as those of
 * spx_masked_group_norm do; each entry reads the fields it names below, plus ndim and mode (which give K).  pos [num_points, ndim] fp32 are positions in the tensor's index space, in the axis
 * order of indices[:, 1:] (voxel v's feature sits at position v); batch_ids [num_points] int32.
 *   A row is usable when r < M (M = *num_valid clamped to [0, rows]) and 0 <= b < batch_size and every coordinate
 *   is in [0, shape_a).  Of rows with equal coordinates the lowest is used.  A point is dropped when its batch id
 *   is outside [0, batch_size) or a component of pos is not finite or lies outside [-1, shape_a) (checked on the
 *   float).
 *   mode 0 trilinear, corners K = 2^ndim: base_a = floor(pos_a), f_a = pos_a - base_a; corner j takes base_a + 1 on
 *          axis a when bit a of j is set, else base_a; its weight is the fp32 product, in ascending a, of f_a (bit
 *          set) or 1 - f_a, one rounding per operation (no FMA).
 *   mode 1 nearest, K = 1: the corner base_a + (f_a >= 0.5), weight 1.
 *   A corner is found when a usable row has its coordinates; a missing corner gets index -1 and weight 0.
 *   normalize != 0 divides the found weights by (S + 1e-8f), S their fp32 sum in ascending j (torchsparse's rule).
 *   plan: index [num_points, K] int32 and weight [num_points, K] fp32, then order [num_points * K] and offsets
 *         [rows + 1] as spx_sparse_add_group keyed by index: the entries e = p * K + j of row r are
 *         order[offsets[r] .. offsets[r+1]) in ascending e.  workspace:
 *         spx_point_interp_plan_workspace_size(args) bytes (ndim, spatial_shape, batch_size, rows, num_points,
 *         mode; 0 = invalid arguments).  Launches: one insert kernel
 *         (rows > 0) and one probe kernel (num_points > 0), then the grouping: 3 + 2 * ceil(bits / 9) kernels, bits
 *         the key width of rows (none when num_points = 0).
 *   fwd:  y [num_points, C]: y[p] = sum over the found corners in ascending j of weight[p, j] * x[index[p, j]], in
 *         fp32 from +0 (one rounding per multiply and per add), rounded once to dtype; 0 for a point without a found
 *         corner.  One launch.
 *   bwd:  dx [rows, C]: dx[r] = sum over the entries e of row r in ascending e of weight[e] * dy[e / K], in fp32,
 *         rounded once; every element written once, 0 for a row without entries.  One launch.
 * No float atomics: every result is bit-reproducible and independent of padding rows and dropped points.
 * dtype: f32 / f16 / bf16, any C >= 1 (16-byte vectors when the row size and pointers allow them, the same bits
 * either way).  rows, num_points and num_points * K below 2^31 - 1.  Keys are 64-bit once batch_size * volume
 * reaches 2^31 - 1.
 */
typedef struct spx_point_interp {
    int ndim, batch_size, mode, normalize, channels, dtype;   /* mode 0 trilinear, 1 nearest; K from ndim and mode */
    int spatial_shape[SPX_MAX_NDIM];
    int64_t rows, num_points;
    const int32_t *indices;     /* plan: [rows, 1 + ndim] */
    const int32_t *num_valid;   /* plan: 1 int32, or NULL */
    const float *pos;           /* plan: [num_points, ndim] */
    const int32_t *batch_ids;   /* plan: [num_points] */
    int32_t *index;             /* plan output, fwd input: [num_points, K] */
    float *weight;              /* plan output, fwd / bwd input: [num_points, K] */
    int32_t *order;             /* plan output, bwd input: [num_points * K] */
    int32_t *offsets;           /* plan output, bwd input: [rows + 1] */
    const void *x;              /* fwd: [rows, channels] */
    void *y;                    /* fwd: [num_points, channels] */
    const void *dy;             /* bwd: [num_points, channels] */
    void *dx;                   /* bwd: [rows, channels] */
} spx_point_interp;
size_t spx_point_interp_plan_workspace_size(const spx_point_interp *args);
int spx_point_interp_plan(const spx_point_interp *args, void *workspace, size_t workspace_bytes, spx_stream_t stream);
int spx_point_interp_fwd(const spx_point_interp *args, spx_stream_t stream);
int spx_point_interp_bwd(const spx_point_interp *args, spx_stream_t stream);

/* ------------------------------------------------------------------ depthwise convolution */

/*
 * Depthwise sparse convolution (groups = in_channels = out_channels = channels) on a dense rulebook table
 * T [kv, rows] int32 (row stride table_stride >= rows, -1 = no pair): pair_fwd / pair_bwd of the masked
 * implicit-GEMM rulebooks, or the tables of spx_pairs_to_table for ConvAlgo.Native.  weight is KRSC with one input
 * channel per group, [channels, kv], read as given.  Kernel offsets are visited in ascending k; every sum is fp32
 * from +0, rounded once to dtype; no float atomics, so every result is bit-reproducible.
 *   fwd:   out[o, c] = act(sum_k W[c, k] * x[T[k][o], c] + bias[c]) for o < n_out; bias may be NULL, act is
 *          SPX_ACT_NONE / RELU / SIGMOID / LEAKY_RELU (alpha = act_alpha).
 *   dgrad: din[i, c] = sum_k W[c, k] * dy[T[k'][i], c] for i < n_in, every row written once; k' = k (pair_bwd),
 *          or k' = kv - 1 - k with reverse_offsets != 0 (SubM: T is pair_fwd, whose mirrored offset gives pair_bwd).
 *   wgrad: dweight[c, k] = sum over o < n_out with T[k][o] >= 0 of dy[o, c] * x[T[k][o], c]: per chunk of 512 rows
 *          a fixed fold (ascending rows per lane, then a binary tree over lanes) into the workspace, then the
 *          chunks in ascending order.  Depends on the row indices alone: trailing rows without pairs or with
 *          dy = 0 leave it unchanged bit for bit.  n_out = 0 writes dweight = 0.
 *          workspace: spx_depthwise_wgrad_workspace_size(n_out, kv, channels) bytes (may be 0).
 * The gathered operand (features, out_bp; features in wgrad) is only read through table entries >= 0 and may be
 * NULL when it has no rows.
 * dtype: f32 / f16 / bf16.  kv in [1, 4096], channels in [1, 2^20], rows below 2^31 - 1.  Rows move as 16-byte
 * vectors when channels * element size is a multiple of 16 and the feature pointers are 16-byte aligned, else
 * one element per thread.
 */
int spx_depthwise_fwd(const void *features, const void *weight, const void *bias, void *out, const int32_t *table,
                      int64_t table_stride, int kv, int64_t n_out, int channels, int dtype, int act, float act_alpha,
                      spx_stream_t stream);
int spx_depthwise_dgrad(const void *out_bp, const void *weight, void *din, const int32_t *table, int64_t table_stride,
                        int kv, int64_t n_in, int channels, int dtype, int reverse_offsets, spx_stream_t stream);
size_t spx_depthwise_wgrad_workspace_size(int64_t n_out, int kv, int channels);
int spx_depthwise_wgrad(const void *features, const void *out_bp, void *dweight, const int32_t *table,
                        int64_t table_stride, int kv, int64_t n_out, int channels, int dtype, void *workspace,
                        size_t workspace_bytes, spx_stream_t stream);

/* ------------------------------------------------------------------ padding-aware BatchNorm */

/*
 * Training-mode BatchNorm1d over the valid rows of x [rows, channels] (MaskedBatchNorm1d).  M = *num_valid
 * (device int32, clamped to [0, rows]; NULL = every row).  Rows [M, rows) are never read; y and dx are 0 there.
 * dtype: f32 / f16 / bf16 features; param_dtype (weight, bias, running stats, dweight, dbias): f32 or dtype.
 * Statistics and every sum are fp32, reduced in fixed chunks of rows merged in chunk order, so all results
 * are bit-reproducible and independent of `rows` (padding).  Nothing is read back to the host.
 * fwd_train: y = (x - mean) * weight * invstd + bias with the batch mean and biased variance; save_mean /
 *            save_invstd [channels] fp32 receive them for the backward.  weight / bias may be NULL (1 / 0).
 *            running_mean / running_var (both or neither) are updated when M > 1:
 *            r = (1 - f) r + f s with s the mean / unbiased variance and f = momentum, or, when cumulative != 0,
 *            f = 1 / *num_batches_tracked (device int64, already incremented by the caller).
 *            M = 0: y = 0; M = 1: y = bias; running stats unchanged in both cases.
 * bwd:       dx = weight * invstd * (dy - sum(dy) / M - xhat * sum(dy * xhat) / M) on valid rows,
 *            dbias = sum(dy), dweight = sum(dy * xhat) over valid rows (either may be NULL).
 * workspace: the matching _workspace_size(rows, channels) bytes.
 */
size_t spx_masked_bn_fwd_train_workspace_size(int64_t rows, int channels);
int spx_masked_bn_fwd_train(const void *x, void *y, int64_t rows, int channels, int dtype, const int32_t *num_valid,
                            const void *weight, const void *bias, void *running_mean, void *running_var,
                            const int64_t *num_batches_tracked, int param_dtype, float momentum, int cumulative,
                            float eps, float *save_mean, float *save_invstd, void *workspace, size_t workspace_bytes,
                            spx_stream_t stream);
size_t spx_masked_bn_bwd_workspace_size(int64_t rows, int channels);
int spx_masked_bn_bwd(const void *x, const void *dy, void *dx, int64_t rows, int channels, int dtype,
                      const int32_t *num_valid, const void *weight, int param_dtype, const float *save_mean,
                      const float *save_invstd, void *dweight, void *dbias, void *workspace, size_t workspace_bytes,
                      spx_stream_t stream);

/*
 * Cross-rank training-mode BatchNorm (MaskedSyncBatchNorm1d): the statistics cover the valid rows of every rank.
 * A forward or backward is two calls on each rank around an exchange the caller runs (spx_peer_allgather or an
 * NCCL all-gather, both move the bits unchanged):
 *   *_local  reduces this rank's rows [0, M_r) as spx_masked_bn_* does and writes local = [M_r, A[C], B[C]] (fp32);
 *   exchange local of every rank into gathered = [world][2 C + 1] in rank order;
 *   *_merge  folds the gathered vectors in rank order, the same on every rank, then writes y / dx.
 * Forward:  A = sum of the rank's valid rows, B = their M2 about the rank's own mean.  The merge takes
 *           M = sum M_r (int64), mean = sum A_r / M, M2 = sum [B_r + M_r (A_r / M_r - mean)^2], and writes
 *           save_mean / save_invstd, y and the running stats exactly as spx_masked_bn_fwd_train does for M rows.
 * Backward: A = sum(dy), B = sum(dy * xhat) over the rank's rows with the global mean / invstd; dbias = A and
 *           dweight = B are the RANK-LOCAL sums (bwd_local writes them; average them like any other parameter
 *           gradient).  The merge sums A_r, B_r in rank order and writes dx with the global sums over M.
 * With one rank (gathered = local) every result equals spx_masked_bn_fwd_train / spx_masked_bn_bwd bit for bit.
 * A gathered count outside [0, 2^24] (NaN after a timed-out exchange) makes the statistics, the running stats and
 * y / dx NaN.  rows <= 2^24 per call.  One descriptor holds the operands of the layer call, so the local and the
 * merge call of one pass read the same ones; the workspace (spx_masked_sync_bn_workspace_size) is also shared
 * by the two calls of one pass.  Fields a call does not use may be anything.
 */
typedef struct spx_masked_sync_bn {
    int64_t rows;
    int channels, dtype, param_dtype;
    int world;                              /* vectors in `gathered` (merge calls), 1..SPX_MAX_PEERS */
    const int32_t *num_valid;               /* device int32, clamped to [0, rows]; NULL = every row */
    const void *x;                          /* [rows, channels] */
    void *y;                                /* fwd: [rows, channels] */
    const void *dy;                         /* bwd: [rows, channels] */
    void *dx;                               /* bwd: [rows, channels] */
    const void *weight, *bias;              /* [channels] param_dtype, or NULL (1 / 0) */
    void *running_mean, *running_var;       /* fwd: both or neither */
    const int64_t *num_batches_tracked;     /* fwd, cumulative != 0: device int64, already incremented */
    float momentum;
    int cumulative;
    float eps;
    float *save_mean, *save_invstd;         /* [channels] fp32: written by fwd_merge, read by the backward */
    void *dweight, *dbias;                  /* bwd: [channels] param_dtype or NULL */
    float *local;                           /* [2 channels + 1]: written by the local calls */
    const float *gathered;                  /* [world][2 channels + 1]: read by the merge calls */
} spx_masked_sync_bn;

size_t spx_masked_sync_bn_workspace_size(int64_t rows, int channels);
int spx_masked_sync_bn_fwd_local(const spx_masked_sync_bn *d, void *workspace, size_t workspace_bytes,
                                 spx_stream_t stream);
int spx_masked_sync_bn_fwd_merge(const spx_masked_sync_bn *d, void *workspace, size_t workspace_bytes,
                                 spx_stream_t stream);
int spx_masked_sync_bn_bwd_local(const spx_masked_sync_bn *d, void *workspace, size_t workspace_bytes,
                                 spx_stream_t stream);
int spx_masked_sync_bn_bwd_merge(const spx_masked_sync_bn *d, void *workspace, size_t workspace_bytes,
                                 spx_stream_t stream);

/* ------------------------------------------------------------------ padding-aware GroupNorm */

/*
 * Per-sample GroupNorm / InstanceNorm (MaskedGroupNorm) over x [rows, channels], with no host read-back.  One
 * descriptor holds the operands of a layer call; the forward and the backward of one call read the same one.
 * M = *num_valid (device int32, clamped to [0, rows]; NULL = every row).  Row r belongs to sample b when r < M and
 * coords[r * row_ints] == b with 0 <= b < batch_size; every other row is dropped: rows [M, rows) are never read
 * (features nor coords), and y and dx are 0 on dropped rows.  groups divides channels; group g holds channels
 * [g Cg, (g + 1) Cg), Cg = channels / groups, and sample b has n = count_b * Cg values in it.
 * fwd: mean [batch_size, groups] and the biased variance over those n values (fp32; an empty sample gives mean 0),
 *      invstd = rsqrt(var + eps) [batch_size, groups]; y = (x - mean) * (weight * invstd) + bias, in fp32, rounded
 *      once.  weight / bias may be NULL (1 / 0).  Also writes the grouping the backward reuses: order [rows] (the
 *      kept rows of sample b are order[offsets[b] .. offsets[b+1]) in ascending row order), offsets [batch_size + 1]
 *      and cstart [batch_size + 1] (the sample's first chunk of 512 rows; cstart[batch_size] = chunks).
 * bwd: with those outputs of the forward (nothing is sorted again): dbias = sum(dy), dweight = sum(dy * xhat) over
 *      every kept row (either may be NULL); dx = invstd * (weight dy - S1 / n - xhat * S2 / n) with
 *      S1 = sum over the group's channels of weight_c sum(dy), S2 = sum of weight_c sum(dy * xhat).  Every element of
 *      dx is written once.
 * Every sum is fp32 in an order fixed by the sample's kept rows (chunks of 512 rows merged in chunk order, the
 * channels of a group in ascending order, the samples in ascending order), with no float atomics, so every result
 * is bit-reproducible and independent of `rows` (padding) and of dropped rows.
 * dtype: f32 / f16 / bf16 features; param_dtype (weight, bias, dweight, dbias): f32 or dtype.  batch_size in
 * [1, 2^20], channels in [1, 65536], rows < 2^31 - 1, row_ints >= 1, eps > 0.  Rows move as 16-byte vectors when
 * channels * element size is a multiple of 16 and the feature pointers are 16-byte aligned, else element by element
 * with the same bits.
 * workspace (fwd and bwd): spx_masked_group_norm_workspace_size(rows, batch_size, channels) bytes.  Fields a
 * call does not use may be anything.
 */
typedef struct spx_masked_group_norm {
    int64_t rows;
    int row_ints, batch_size, channels, groups, dtype, param_dtype;
    float eps;                              /* fwd: > 0 */
    const int32_t *coords;                  /* [rows, row_ints], the batch index first */
    const int32_t *num_valid;               /* device int32, clamped to [0, rows]; NULL = every row */
    const void *x;                          /* [rows, channels] */
    void *y;                                /* fwd: [rows, channels] */
    const void *dy;                         /* bwd: [rows, channels] */
    void *dx;                               /* bwd: [rows, channels] */
    const void *weight, *bias;              /* [channels] param_dtype, or NULL (1 / 0) */
    void *dweight, *dbias;                  /* bwd: [channels] param_dtype, or NULL */
    float *mean, *invstd;                   /* [batch_size, groups] fp32: written by fwd, read by bwd */
    int32_t *order;                         /* [rows]: written by fwd, read by bwd */
    int32_t *offsets, *cstart;              /* [batch_size + 1]: written by fwd, read by bwd */
} spx_masked_group_norm;

size_t spx_masked_group_norm_workspace_size(int64_t rows, int batch_size, int channels);
int spx_masked_group_norm_fwd(const spx_masked_group_norm *d, void *workspace, size_t workspace_bytes,
                              spx_stream_t stream);
int spx_masked_group_norm_bwd(const spx_masked_group_norm *d, void *workspace, size_t workspace_bytes,
                              spx_stream_t stream);

/*
 * MaskedGroupNorm with per-sample modulation and an activation (AdaGN, as guided-diffusion's use_scale_shift_norm):
 * `norm` is the call above, unchanged, and for a kept row of sample b, channel c
 *   h = (x - mean) * (weight * invstd) + bias          (the apply above)
 *   z = h * (1 + scale[b][c]) + shift[b][c]            (one fmaf; z = h when scale and shift are both NULL)
 *   y = act(z)                                         (rounded once to dtype)
 * with relu(z) = z <= 0 ? 0 : z and silu(z) = z / (1 + exp(-z)).  Dropped rows stay 0 in y and dx and never touch
 * scale, shift, dscale or dshift.
 * bwd: dz = dy * act'(z), z recomputed from x as the forward computes it (relu' = z > 0,
 *      silu' = sigmoid(z) (1 + z (1 - sigmoid(z)))); the sums of `norm` are taken over dz, weight_c becomes
 *      weight_c (1 + scale[b][c]) in S1, S2 and dx, and
 *        dbias_c = sum_b (1 + scale[b][c]) sum(dz),  dweight_c = sum_b (1 + scale[b][c]) sum(dz * xhat),
 *        dshift[b][c] = sum(dz),  dscale[b][c] = weight_c sum(dz * xhat) + bias_c sum(dz)
 *      over the kept rows of sample b (0 for an empty sample), in the fixed orders of `norm`.  Same 4 launches.
 *      Unlike spx_masked_group_norm_bwd (which never reads it), this bwd reads norm.bias ([channels] param_dtype,
 *      or NULL = 0) when act != SPX_GN_ACT_NONE (to recompute z) or dscale is given; otherwise it may be anything.
 * scale, shift, dscale, dshift: fp32 [batch_size, channels], row-major, 4-byte aligned, read and written element by
 * element; any of them may be NULL (scale / shift 0, the gradient not written).  act is checked before any launch.
 * With scale = shift = NULL and SPX_GN_ACT_NONE the results are those of spx_masked_group_norm_fwd / _bwd bit for
 * bit.  workspace: spx_masked_group_norm_workspace_size, as above.
 */
enum spx_gn_act { SPX_GN_ACT_NONE = 0, SPX_GN_ACT_RELU = 1, SPX_GN_ACT_SILU = 2 };

typedef struct spx_masked_group_norm_mod {
    spx_masked_group_norm norm;
    const float *scale, *shift;             /* [batch_size, channels] fp32, or NULL (0) */
    int act;                                /* spx_gn_act */
    float *dscale, *dshift;                 /* bwd: [batch_size, channels] fp32, or NULL */
} spx_masked_group_norm_mod;

int spx_masked_group_norm_mod_fwd(const spx_masked_group_norm_mod *m, void *workspace, size_t workspace_bytes,
                                  spx_stream_t stream);
int spx_masked_group_norm_mod_bwd(const spx_masked_group_norm_mod *m, void *workspace, size_t workspace_bytes,
                                  spx_stream_t stream);

/* ------------------------------------------------------------------ hash table */

/*
 * Replaces the CUDA branch of spconv.pytorch.hash.HashTable (spconv/pytorch/hash.py, spconv/csrc/hash/core.py)
 * with the semantics of its CPU branch (tsl::robin_map) plus a defined order.  One table is:
 *   table_keys [max_size] (key_size bytes each), table_values [max_size] (value_size bytes, moved as raw bits),
 *   first [max_size] int32 (insertion ordinal of the stored key, INT32_MAX = empty slot),
 *   tag [max_size] (epoch << 32 | position of the last insert_exist write).
 * key_size and value_size are 4 or 8; 1 <= max_size <= 2^31 - 1 (slots = max_size exactly).  The largest
 * value of the signed key type marks an empty slot: that key is never stored and is never found.
 *
 * clear:        every slot empty, values 0, first INT32_MAX, tag 0.
 * insert:       keys [n], values [n] or NULL (value 0); key i gets ordinal ordinal_base + i.  The first
 *               insertion of a key wins; later duplicates and re-inserts leave its value unchanged.  Requires
 *               ordinal_base + n < max_size (the reference's capacity rule), so a probe always ends.
 * query:        values [n] (written for found keys only), is_empty [n] = 1 for a missing key.
 * insert_exist: found keys take the value of their LAST occurrence in the call; missing keys are not inserted
 *               (is_empty [n] = 1).  epoch in [1, 2^32 - 1] must grow from call to call of one table.
 * rank:         numbers the stored keys 0 .. count-1 in first-insertion order; ordinal_count = the sum of n
 *               over all inserts.  assign != 0: each stored value becomes its number (integer values);
 *               otherwise row r < out_rows of out_keys / out_values gets the key numbered r and its value.
 *               count [1] (key_size bytes, unsigned) = the number of stored keys, written on the device.
 * workspace:    spx_hash_workspace_size(n, 0) bytes for insert / insert_exist,
 *               spx_hash_workspace_size(0, ordinal_count) for rank.  Nothing reads back to the host.
 */
size_t spx_hash_workspace_size(int64_t num_keys, int64_t ordinal_count);
int spx_hash_clear(void *table_keys, void *table_values, int32_t *first, uint64_t *tag, int64_t max_size,
                   int key_size, int value_size, spx_stream_t stream);
int spx_hash_insert(void *table_keys, void *table_values, int32_t *first, int64_t max_size, int key_size,
                    int value_size, const void *keys, const void *values, int64_t n, int64_t ordinal_base,
                    void *workspace, size_t workspace_bytes, spx_stream_t stream);
int spx_hash_query(const void *table_keys, const void *table_values, int64_t max_size, int key_size, int value_size,
                   const void *keys, void *values, uint8_t *is_empty, int64_t n, spx_stream_t stream);
int spx_hash_insert_exist(const void *table_keys, void *table_values, uint64_t *tag, int64_t max_size, int key_size,
                          int value_size, const void *keys, const void *values, uint8_t *is_empty, int64_t n,
                          int64_t epoch, void *workspace, size_t workspace_bytes, spx_stream_t stream);
int spx_hash_rank(const void *table_keys, void *table_values, const int32_t *first, int64_t max_size, int key_size,
                  int value_size, int64_t ordinal_count, int assign, void *out_keys, void *out_values,
                  int64_t out_rows, void *count, void *workspace, size_t workspace_bytes, spx_stream_t stream);

/*
 * int8 inference forward (reference formula: test/test_all_algo.py:272-287,
 * spconv/pytorch/quantization/quantized/conv.py:368-377):
 *   acc_i32 = sum_k x_i8[pair[k][o]] @ W_i8[:, k, :]^T
 *   y = acc * scale[j] + bias[j] (+ add_i8[o, j] * add_scale);  act;  q = clip(rint(y), -128, 127)
 * out_dtype: SPX_I8 (quantised) or SPX_F32 / SPX_F16 (y stored directly).
 */
int spx_implicit_gemm_fwd_int8(const spx_gemm_desc *d, const int8_t *features,
                               const int8_t *filters, void *out, int out_dtype,
                               const float *scale, const float *bias, const int8_t *output_add,
                               float output_add_scale, int act, float act_alpha,
                               spx_stream_t stream);

/*
 * FP8 (e4m3) inference forward; the operands come in one argument block, spx_fp8_gemm.  d->dtype is SPX_E4M3;
 * features [n_in, C] and filters [K, kv, C] are e4m3 bytes (OCP e4m3fn: finite range +-448, one NaN pattern per
 * sign, no infinities).  Every scale is a device pointer, so no call reads anything back to the host:
 *   in_scale  fp32 [1]  the features' per-tensor scale            (x_real = x_e4m3 * in_scale)
 *   w_scale   fp32 [K]  the filter's per-output-channel scale     (W_real[k] = W_e4m3[k] * w_scale[k])
 *   bias      fp32 [K]  or NULL
 *   output_add          NULL, or the residual [n_out, K] in out_dtype
 *   add_scale fp32 [1]  the residual's scale: required for an SPX_E4M3 residual; NULL = 1 otherwise
 *   out_scale fp32 [1]  required for SPX_E4M3 output, ignored otherwise
 * The epilogue, the same in the tensor-core and the FMA kernels, is fp32 in registers, one IEEE operation per
 * step and no fused multiply-add, in this order:
 *   acc = sum over k, c of x[pair[k][o], c] * W[j, k, c]    fp32 (every product of two e4m3 values is exact)
 *   s_j = in_scale * w_scale[j]
 *   y   = acc * s_j;  y = y + bias[j];  y = y + add[o, j] * add_scale;  y = act(y)
 * out_dtype SPX_F32 stores y, SPX_F16 / SPX_BF16 y rounded once to nearest-even, SPX_E4M3
 * satfinite_rne(y / out_scale): ties to even, beyond +-448 (and +-Inf) saturates to +-448, NaN stays NaN.
 * C and K multiples of 32 up to 256 with 16-byte aligned operands run on the tensor cores (wgmma e4m3); every
 * other shape on the FMA kernel, which sums in fp32 throughout.  The tensor cores sum each kernel offset's
 * channels in the FP8 MMA, which keeps about 14 bits per 32-channel step, and add the offsets in fp32: a row's
 * error stays below (33 * ceil(C / 32) * 2^-13 + offsets * 2^-24) * sum |x| |W| before the epilogue.
 * SPX_FORCE_SIMT / SPX_FORCE_TC apply.
 */
typedef struct spx_fp8_gemm {
    const void *features;       /* e4m3 [n_in, C] */
    const void *filters;        /* e4m3 [K, kv, C] */
    const float *in_scale, *w_scale, *bias;
    const void *output_add;     /* NULL or [n_out, K] in out_dtype */
    const float *add_scale;
    void *out;                  /* [n_out, K] in out_dtype */
    int out_dtype;
    const float *out_scale;
    int act;                    /* spx_act */
    float act_alpha;
} spx_fp8_gemm;
int spx_implicit_gemm_fwd_fp8(const spx_gemm_desc *d, const spx_fp8_gemm *a, spx_stream_t stream);

/*
 * Quantise fp32 / fp16 / bf16 rows x [rows, channels] (spx_dtype dtype) to e4m3 rows out [rows, channels]:
 *   out = satfinite_rne(x / scale)        rows [0, M), M = *num_valid clamped to [0, rows] (NULL: M = rows)
 *   out = 0                               rows [M, rows), which are never read
 * scale_in != NULL: the given device scale (fp32 [1]) is used; scale_out, when not NULL, receives a copy.
 * scale_in == NULL: dynamic, scale = amax / 448 over rows [0, M) and all channels, NaN and +-Inf left out of
 *   the amax, 1 when that amax is 0; written to scale_out (required).
 * NaN stays NaN, +-Inf and values beyond +-448 * scale saturate.  No float atomics and no host read-back:
 * the output is bit-reproducible.  One launch with a given scale, two when dynamic.
 * workspace: spx_fp8_quantize_workspace_size(rows, channels) bytes (dynamic mode only; may be NULL otherwise).
 */
typedef struct spx_fp8_quant {
    const void *x;
    int dtype;
    int64_t rows;
    int channels;
    const int32_t *num_valid;   /* device [1] or NULL */
    const float *scale_in;      /* device [1], or NULL: dynamic */
    void *out;                  /* e4m3 [rows, channels] */
    float *scale_out;           /* device [1] */
} spx_fp8_quant;
size_t spx_fp8_quantize_workspace_size(int64_t rows, int channels);
int spx_fp8_quantize(const spx_fp8_quant *q, void *workspace, size_t workspace_bytes, spx_stream_t stream);

/* which kernel family served the last call of each kind on this thread: 0 none, 1 SIMT,
 * 2 wgmma tensor-core kernels.  Used by tests/bench to prove the tensor-core path ran. */
int spx_last_kernel_family(void);
/* number of kernel launches issued by this library (all host threads) since the last reset */
int64_t spx_launch_count(int reset);
/*
 * Test switches (never needed for correct operation; the reference's counterpart is the
 * SPCONV_DEBUG_* environment, spconv/constants.py:100-125).
 *   force_family: -1 keep, 0 automatic, 1 generic FMA kernels, 2 tensor-core kernels (error if the
 *                 shape does not tile) -- the start-up value comes from SPX_FORCE_SIMT / SPX_FORCE_TC,
 *                 read once when the library is loaded;
 *   tc_ctas:      ignored (kept for ABI compatibility: the tensor-core kernels run one CTA per SM);
 *   debug_bits:   any combination of 256 (fp32+TF32 input gradient on the FMA kernel instead of wgmma)
 *                 and 4096 (the same for the weight gradient); 0 clears both.  Any other bit is refused
 *                 (returns 2) and leaves every switch unchanged;
 *   trace_buf:    must be NULL (refused otherwise); trace_bytes is ignored.
 */
int spx_debug_configure(int force_family, int tc_ctas, int debug_bits, void *trace_buf,
                        size_t trace_bytes);

#ifdef __cplusplus
}
#endif
#endif /* SPCONV_B200_H_ */
