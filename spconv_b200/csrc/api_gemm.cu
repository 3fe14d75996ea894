// C-ABI entry points of the conv arithmetic: validation + dispatch between the tensor-core
// kernels (gemm_tc.cu) and the generic fp32-FMA kernels (gemm_simt.cu).
#include "gemm.cuh"
#include "peer.cuh"
#include <stdlib.h>

using namespace spx;

// SPX_FORCE_SIMT=1 pins the generic kernels (debug / A-B comparisons in tests); read once at load
static bool force_simt() { return runtime_cfg().force_simt != 0; }
static bool force_tc() { return runtime_cfg().force_tc != 0; }

static int check_desc(const spx_gemm_desc *d, const char *who) {
    SPX_REQUIRE(d != nullptr, "%s: descriptor is NULL", who);
    SPX_REQUIRE(d->kv >= 1 && d->kv <= 128, "%s: kernel volume %d not in [1,128]", who, d->kv);
    SPX_REQUIRE(d->c_in >= 1 && d->c_out >= 1, "%s: bad channel counts %d -> %d", who, d->c_in, d->c_out);
    SPX_REQUIRE(d->n_in >= 0 && d->n_out >= 0, "%s: negative row counts", who);
    SPX_REQUIRE(d->n_in < 2147483647ll && d->n_out < 2147483647ll, "%s: row counts must fit in int32", who);
    SPX_REQUIRE(d->pair != nullptr || (d->n_in == 0 || d->n_out == 0), "%s: pair table is NULL", who);
    SPX_REQUIRE((d->tile_table == nullptr) == (d->tile_mask == nullptr), "%s: tile_table and tile_mask go together", who);
    return 0;
}

static GatherGemmArgs make_args(const spx_gemm_desc *d, bool dgrad) {
    GatherGemmArgs a;
    memset(&a, 0, sizeof(a));
    a.dtype = d->dtype; a.f32_mode = d->f32_mode; a.kv = d->kv; a.c_in = d->c_in; a.c_out = d->c_out;
    a.transpose_w = dgrad ? 1 : 0;
    a.reverse = d->reverse_offsets;
    a.rows = dgrad ? d->n_in : d->n_out;
    a.x_rows = dgrad ? d->n_out : d->n_in;
    a.pair = d->pair; a.pair_stride = d->pair_stride;
    a.mask = d->mask; a.argsort = d->argsort;
    a.tile_table = d->tile_table; a.tile_mask = d->tile_mask;
    return a;
}

static int run_gather_gemm(const GatherGemmArgs &a, cudaStream_t stream) {
    if (a.rows == 0) return 0;
    bool exact_f32 = a.dtype == SPX_F32 && a.f32_mode == SPX_F32_EXACT;
    bool tc_ok = !force_simt() && !exact_f32 && tc_gather_gemm_supported(a);
    if (force_tc() && !tc_ok) {
        set_error("SPX_FORCE_TC=1 but the tensor-core path does not support this call (dtype %d, C %d, K %d)",
                  a.dtype, a.c_in, a.c_out);
        return 3;
    }
    if (tc_ok) { set_family(2); return tc_gather_gemm(a, stream); }
    set_family(1);
    return simt_gather_gemm(a, stream);
}

extern "C" int spx_implicit_gemm_fwd(const spx_gemm_desc *d, const void *features, const void *filters, void *out,
                                     const void *bias, int act, float act_alpha, spx_stream_t stream) {
    if (check_desc(d, "implicit_gemm_fwd")) return 2;
    SPX_REQUIRE(d->dtype == SPX_F32 || d->dtype == SPX_F16 || d->dtype == SPX_BF16,
                "implicit_gemm_fwd: dtype %d not supported (int8 has its own entry point)", d->dtype);
    if (d->n_out == 0) return 0;
    SPX_REQUIRE(features && filters && out, "implicit_gemm_fwd: NULL tensor");
    GatherGemmArgs a = make_args(d, false);
    a.x = features; a.w = filters; a.y = out; a.bias = bias; a.act = act; a.alpha = act_alpha;
    return run_gather_gemm(a, (cudaStream_t)stream);
}

extern "C" int spx_implicit_gemm_dgrad(const spx_gemm_desc *d, const void *out_bp, const void *filters, void *din,
                                       spx_stream_t stream) {
    if (check_desc(d, "implicit_gemm_dgrad")) return 2;
    SPX_REQUIRE(d->dtype == SPX_F32 || d->dtype == SPX_F16 || d->dtype == SPX_BF16,
                "implicit_gemm_dgrad: dtype %d not supported", d->dtype);
    if (d->n_in == 0) return 0;
    SPX_REQUIRE(out_bp && filters && din, "implicit_gemm_dgrad: NULL tensor");
    GatherGemmArgs a = make_args(d, true);
    a.x = out_bp; a.w = filters; a.y = din; a.bias = nullptr; a.act = SPX_ACT_NONE;
    return run_gather_gemm(a, (cudaStream_t)stream);
}

static WgradArgs make_wgrad(const spx_gemm_desc *d) {
    WgradArgs w;
    memset(&w, 0, sizeof(w));
    w.dtype = d->dtype; w.f32_mode = d->f32_mode; w.kv = d->kv; w.c_in = d->c_in; w.c_out = d->c_out;
    w.n_in = d->n_in; w.n_out = d->n_out;
    w.pair = d->pair; w.pair_stride = d->pair_stride; w.mask = d->mask; w.argsort = d->argsort;
    w.tile_table = d->tile_table; w.tile_mask = d->tile_mask;
    return w;
}

extern "C" size_t spx_implicit_gemm_wgrad_workspace_size(const spx_gemm_desc *d) {
    if (!d) return 0;
    WgradArgs w = make_wgrad(d);
    bool exact_f32 = d->dtype == SPX_F32 && d->f32_mode == SPX_F32_EXACT;
    if (!force_simt() && !exact_f32 && tc_wgrad_supported(w)) return tc_wgrad_workspace_size(w);
    return 256;
}

// pg == NULL: plain weight gradient.  pg != NULL: push this rank's fp32 gradient to the group; the caller runs the
// receive side (spx_peer_finish) after the work it wants to overlap.
static int wgrad_entry(const spx_gemm_desc *d, const void *features, const void *out_bp, void *dfilters, void *workspace,
                       size_t workspace_bytes, const spx_peer_group *pg, spx_stream_t stream);

extern "C" int spx_implicit_gemm_wgrad(const spx_gemm_desc *d, const void *features, const void *out_bp,
                                       void *dfilters, void *workspace, size_t workspace_bytes,
                                       spx_stream_t stream) {
    return wgrad_entry(d, features, out_bp, dfilters, workspace, workspace_bytes, nullptr, stream);
}

extern "C" int spx_implicit_gemm_wgrad_push(const spx_gemm_desc *d, const void *features, const void *out_bp,
                                            void *dfilters, void *workspace, size_t workspace_bytes,
                                            const spx_peer_group *pg, spx_stream_t stream) {
    SPX_REQUIRE(pg != nullptr, "implicit_gemm_wgrad_push: peer group is NULL");
    return wgrad_entry(d, features, out_bp, dfilters, workspace, workspace_bytes, pg, stream);
}

static int wgrad_entry(const spx_gemm_desc *d, const void *features, const void *out_bp, void *dfilters, void *workspace,
                       size_t workspace_bytes, const spx_peer_group *pg, spx_stream_t stream) {
    if (check_desc(d, "implicit_gemm_wgrad")) return 2;
    SPX_REQUIRE(d->dtype == SPX_F32 || d->dtype == SPX_F16 || d->dtype == SPX_BF16,
                "implicit_gemm_wgrad: dtype %d not supported", d->dtype);
    SPX_REQUIRE(dfilters != nullptr, "implicit_gemm_wgrad: dfilters is NULL");
    const int64_t dw_count = (int64_t)d->kv * d->c_in * d->c_out;
    if (d->n_out == 0 || d->n_in == 0) {       // an empty shard still takes part in the exchange
        SPX_CHECK_CUDA(cudaMemsetAsync(dfilters, 0, (size_t)dw_count * dtype_bytes(d->dtype), (cudaStream_t)stream));
        if (pg) return peer_push(nullptr, 0, 0, dfilters, dw_count, d->dtype, pg, (cudaStream_t)stream);
        return 0;
    }
    SPX_REQUIRE(features && out_bp, "implicit_gemm_wgrad: NULL tensor");
    WgradArgs w = make_wgrad(d);
    w.peers = pg;
    w.x = features; w.dout = out_bp; w.dw = dfilters; w.workspace = workspace; w.workspace_bytes = workspace_bytes;
    bool exact_f32 = d->dtype == SPX_F32 && d->f32_mode == SPX_F32_EXACT;
    bool tc_ok = !force_simt() && !exact_f32 && tc_wgrad_supported(w);
    if (force_tc() && !tc_ok) {
        set_error("SPX_FORCE_TC=1 but the tensor-core wgrad does not support this call (dtype %d, C %d, K %d)", d->dtype,
                  d->c_in, d->c_out);
        return 3;
    }
    if (tc_ok) {
        SPX_REQUIRE(workspace && workspace_bytes >= tc_wgrad_workspace_size(w),
                    "implicit_gemm_wgrad: workspace too small (%zu < %zu)", workspace_bytes, tc_wgrad_workspace_size(w));
        set_family(2);
        return tc_wgrad(w, (cudaStream_t)stream);     // with peers: partial sums pushed, dW not written yet
    }
    set_family(1);
    if (int rc = simt_wgrad(w, (cudaStream_t)stream)) return rc;
    if (pg) return peer_push(nullptr, 0, 0, dfilters, dw_count, d->dtype, pg, (cudaStream_t)stream);
    return 0;
}

extern "C" int spx_implicit_gemm_fwd_int8(const spx_gemm_desc *d, const int8_t *features, const int8_t *filters,
                                          void *out, int out_dtype, const float *scale, const float *bias,
                                          const int8_t *output_add, float output_add_scale, int act,
                                          float act_alpha, spx_stream_t stream) {
    if (check_desc(d, "implicit_gemm_fwd_int8")) return 2;
    SPX_REQUIRE(d->dtype == SPX_I8, "implicit_gemm_fwd_int8: descriptor dtype must be SPX_I8");
    SPX_REQUIRE(out_dtype == SPX_I8 || out_dtype == SPX_F32 || out_dtype == SPX_F16,
                "implicit_gemm_fwd_int8: out dtype %d not supported", out_dtype);
    if (d->n_out == 0) return 0;
    SPX_REQUIRE(features && filters && out && scale, "implicit_gemm_fwd_int8: NULL tensor");
    Int8Args q;
    memset(&q, 0, sizeof(q));
    q.g = make_args(d, false);
    q.g.x = features; q.g.w = filters; q.g.y = out; q.g.act = act; q.g.alpha = act_alpha;
    q.out_dtype = out_dtype; q.scale = scale; q.bias_f32 = bias; q.output_add = output_add;
    q.output_add_scale = output_add_scale;
    bool tc_ok = !force_simt() && tc_gather_gemm_int8_supported(q);
    if (force_tc() && !tc_ok) {
        set_error("SPX_FORCE_TC=1 but the tensor-core int8 path does not support C %d, K %d", d->c_in, d->c_out);
        return 3;
    }
    if (tc_ok) { set_family(2); return tc_gather_gemm_int8(q, (cudaStream_t)stream); }
    set_family(1);
    return simt_gather_gemm_int8(q, (cudaStream_t)stream);
}

extern "C" int spx_implicit_gemm_fwd_fp8(const spx_gemm_desc *d, const spx_fp8_gemm *a, spx_stream_t stream) {
    SPX_REQUIRE(a != nullptr, "implicit_gemm_fwd_fp8: argument block is NULL");
    const void *features = a->features, *filters = a->filters, *output_add = a->output_add;
    const float *in_scale = a->in_scale, *w_scale = a->w_scale, *bias = a->bias, *add_scale = a->add_scale;
    const float *out_scale = a->out_scale;
    void *out = a->out;
    const int out_dtype = a->out_dtype, act = a->act;
    const float act_alpha = a->act_alpha;
    if (check_desc(d, "implicit_gemm_fwd_fp8")) return 2;
    SPX_REQUIRE(d->dtype == SPX_E4M3, "implicit_gemm_fwd_fp8: descriptor dtype must be SPX_E4M3");
    SPX_REQUIRE(out_dtype == SPX_E4M3 || out_dtype == SPX_F32 || out_dtype == SPX_F16 || out_dtype == SPX_BF16,
                "implicit_gemm_fwd_fp8: out dtype %d not supported", out_dtype);
    SPX_REQUIRE(act >= SPX_ACT_NONE && act <= SPX_ACT_LEAKY_RELU, "implicit_gemm_fwd_fp8: unknown activation %d", act);
    if (d->n_out == 0) return 0;
    SPX_REQUIRE(features && filters && out && in_scale && w_scale, "implicit_gemm_fwd_fp8: NULL tensor");
    SPX_REQUIRE(out_dtype != SPX_E4M3 || out_scale, "implicit_gemm_fwd_fp8: e4m3 output needs out_scale");
    SPX_REQUIRE(out_dtype != SPX_E4M3 || !output_add || add_scale,
                "implicit_gemm_fwd_fp8: an e4m3 residual needs add_scale");
    Fp8Args q;
    memset(&q, 0, sizeof(q));
    q.g = make_args(d, false);
    q.g.x = features; q.g.w = filters; q.g.y = out; q.g.act = act; q.g.alpha = act_alpha;
    q.out_dtype = out_dtype; q.in_scale = in_scale; q.w_scale = w_scale; q.bias_f32 = bias;
    q.output_add = output_add; q.add_scale = add_scale; q.out_scale = out_scale;
    bool tc_ok = !force_simt() && tc_gather_gemm_fp8_supported(q);
    if (force_tc() && !tc_ok) {
        set_error("SPX_FORCE_TC=1 but the tensor-core fp8 path does not support C %d, K %d", d->c_in, d->c_out);
        return 3;
    }
    if (tc_ok) { set_family(2); return tc_gather_gemm_fp8(q, (cudaStream_t)stream); }
    set_family(1);
    return simt_gather_gemm_fp8(q, (cudaStream_t)stream);
}

// ------------------------------------------------------------------ grouped conv (1 < groups)
// One pass per group j, in ascending j, on the caller's stream.  Each pass is the dense (Cg -> Kg) GEMM of that
// group (Cg = c_in / groups, Kg = c_out / groups): the same kernel family and instance as the dense entry point would
// run on the group's contiguous slices, with the gathered and written rows read at the full row stride.  The route is
// chosen once, from group 0 (every group has the same shape, and its column offsets are multiples of 32 bytes, so it
// has the same alignment); every argument is checked before the first launch.

static int check_grouped(const spx_gemm_desc *d, int groups, const spx_grouped_gemm *a, const char *who) {
    if (check_desc(d, who)) return 2;
    SPX_REQUIRE(a != nullptr, "%s: argument block is NULL", who);
    SPX_REQUIRE(groups > 1, "%s: groups %d must be at least 2 (groups == 1 is the dense entry point)", who, groups);
    SPX_REQUIRE(d->dtype == SPX_F32 || d->dtype == SPX_F16 || d->dtype == SPX_BF16, "%s: dtype %d not supported", who,
                d->dtype);
    SPX_REQUIRE(d->c_in % groups == 0 && d->c_out % groups == 0, "%s: groups %d must divide C %d and K %d", who, groups,
                d->c_in, d->c_out);
    SPX_REQUIRE((d->c_in / groups) % 16 == 0 && (d->c_out / groups) % 16 == 0,
                "%s: group widths C/groups = %d and K/groups = %d must be multiples of 16", who, d->c_in / groups,
                d->c_out / groups);
    return 0;
}

// every tensor the FMA kernels read element by element must at least be aligned to its element
static int check_elem_aligned(const void *p, int dtype, const char *who, const char *what) {
    SPX_REQUIRE(((uintptr_t)p % (uintptr_t)dtype_bytes(dtype)) == 0, "%s: %s is not aligned to its element size", who,
                what);
    return 0;
}

static bool route_tc_16bit(int dtype, bool tc_supported) {
    return !force_simt() && (dtype == SPX_F16 || dtype == SPX_BF16) && tc_supported;
}

// the dense GEMM of group j: operands at the group's columns, filter rows and bias
static GatherGemmArgs group_args(const GatherGemmArgs &all, int groups, int j, size_t e) {
    GatherGemmArgs g = all;
    g.c_in = all.c_in / groups; g.c_out = all.c_out / groups;
    const int cx = g.cx(), cy = g.cy();
    g.x = (const uint8_t *)all.x + (size_t)j * cx * e;
    g.y = (uint8_t *)all.y + (size_t)j * cy * e;
    g.w = (const uint8_t *)all.w + (size_t)j * g.c_out * g.kv * g.c_in * e;
    g.bias = all.bias ? (const uint8_t *)all.bias + (size_t)j * g.c_out * e : nullptr;
    return g;
}

static int run_grouped_gemm(const GatherGemmArgs &all, int groups, const char *who, cudaStream_t stream) {
    if (all.rows == 0) return 0;
    const size_t e = (size_t)dtype_bytes(all.dtype);
    const GatherGemmArgs g0 = group_args(all, groups, 0, e);
    const bool tc_ok = route_tc_16bit(all.dtype, tc_gather_gemm_supported(g0));
    if (force_tc() && !tc_ok) {
        set_error("%s: SPX_FORCE_TC=1 but the tensor-core path does not support this call (dtype %d, C/g %d, K/g %d)",
                  who, all.dtype, g0.c_in, g0.c_out);
        return 3;
    }
    set_family(tc_ok ? 2 : 1);
    const int64_t ldx = all.cx(), ldy = all.cy();
    for (int j = 0; j < groups; ++j) {
        const GatherGemmArgs g = group_args(all, groups, j, e);
        if (int rc = tc_ok ? tc_gather_gemm(g, stream, ldx, ldy) : simt_gather_gemm(g, stream, ldx, ldy)) return rc;
    }
    return 0;
}

extern "C" int spx_grouped_gemm_fwd(const spx_gemm_desc *d, int groups, const spx_grouped_gemm *a, spx_stream_t stream) {
    const char *who = "grouped_gemm_fwd";
    if (check_grouped(d, groups, a, who)) return 2;
    SPX_REQUIRE(a->act >= SPX_ACT_NONE && a->act <= SPX_ACT_LEAKY_RELU, "%s: unknown activation %d", who, a->act);
    if (d->n_out == 0) return 0;
    SPX_REQUIRE(a->features && a->filters && a->out, "%s: NULL tensor", who);
    if (check_elem_aligned(a->features, d->dtype, who, "features") || check_elem_aligned(a->filters, d->dtype, who, "filters") ||
        check_elem_aligned(a->out, d->dtype, who, "out") || check_elem_aligned(a->bias, d->dtype, who, "bias"))
        return 2;
    GatherGemmArgs all = make_args(d, false);
    all.x = a->features; all.w = a->filters; all.y = a->out; all.bias = a->bias; all.act = a->act; all.alpha = a->act_alpha;
    return run_grouped_gemm(all, groups, who, (cudaStream_t)stream);
}

extern "C" int spx_grouped_gemm_dgrad(const spx_gemm_desc *d, int groups, const spx_grouped_gemm *a,
                                      spx_stream_t stream) {
    const char *who = "grouped_gemm_dgrad";
    if (check_grouped(d, groups, a, who)) return 2;
    if (d->n_in == 0) return 0;
    SPX_REQUIRE(a->out_bp && a->filters && a->din, "%s: NULL tensor", who);
    if (check_elem_aligned(a->out_bp, d->dtype, who, "out_bp") || check_elem_aligned(a->filters, d->dtype, who, "filters") ||
        check_elem_aligned(a->din, d->dtype, who, "din"))
        return 2;
    GatherGemmArgs all = make_args(d, true);
    all.x = a->out_bp; all.w = a->filters; all.y = a->din; all.bias = nullptr; all.act = SPX_ACT_NONE;
    return run_grouped_gemm(all, groups, who, (cudaStream_t)stream);
}

// the dense weight gradient of group j: x and dout at the group's columns, dW at its filter rows
static WgradArgs group_wgrad(const WgradArgs &all, int groups, int j, size_t e) {
    WgradArgs g = all;
    g.c_in = all.c_in / groups; g.c_out = all.c_out / groups;
    g.x = (const uint8_t *)all.x + (size_t)j * g.c_in * e;
    g.dout = (const uint8_t *)all.dout + (size_t)j * g.c_out * e;
    g.dw = (uint8_t *)all.dw + (size_t)j * g.c_out * g.kv * g.c_in * e;
    return g;
}

static bool grouped_wgrad_tc(const WgradArgs &g0) {
    return route_tc_16bit(g0.dtype, tc_wgrad_supported(g0));
}

extern "C" size_t spx_grouped_gemm_wgrad_workspace_size(const spx_gemm_desc *d, int groups) {
    if (!d || groups < 2 || d->c_in % groups || d->c_out % groups) return 0;
    WgradArgs all = make_wgrad(d);
    const WgradArgs g0 = group_wgrad(all, groups, 0, (size_t)dtype_bytes(d->dtype));
    // the passes run one after another and reuse one workspace
    return grouped_wgrad_tc(g0) ? tc_wgrad_workspace_size(g0) : 256;
}

static int grouped_wgrad_entry(const spx_gemm_desc *d, int groups, const spx_grouped_gemm *a, const spx_peer_group *pg,
                               spx_stream_t stream_) {
    const char *who = pg ? "grouped_gemm_wgrad_push" : "grouped_gemm_wgrad";
    cudaStream_t stream = (cudaStream_t)stream_;
    if (check_grouped(d, groups, a, who)) return 2;
    SPX_REQUIRE(a->dfilters != nullptr, "%s: dfilters is NULL", who);
    if (check_elem_aligned(a->dfilters, d->dtype, who, "dfilters")) return 2;
    const int64_t dw_count = (int64_t)d->kv * (d->c_in / groups) * d->c_out;
    if (d->n_out == 0 || d->n_in == 0) {       // an empty shard still takes part in the exchange
        SPX_CHECK_CUDA(cudaMemsetAsync(a->dfilters, 0, (size_t)dw_count * dtype_bytes(d->dtype), stream));
        if (pg) return peer_push(nullptr, 0, 0, a->dfilters, dw_count, d->dtype, pg, stream);
        return 0;
    }
    SPX_REQUIRE(a->features && a->out_bp, "%s: NULL tensor", who);
    if (check_elem_aligned(a->features, d->dtype, who, "features") || check_elem_aligned(a->out_bp, d->dtype, who, "out_bp"))
        return 2;
    WgradArgs all = make_wgrad(d);
    all.x = a->features; all.dout = a->out_bp; all.dw = a->dfilters;
    all.workspace = a->workspace; all.workspace_bytes = a->workspace_bytes;
    const size_t e = (size_t)dtype_bytes(d->dtype);
    const WgradArgs g0 = group_wgrad(all, groups, 0, e);
    const bool tc_ok = grouped_wgrad_tc(g0);
    if (force_tc() && !tc_ok) {
        set_error("%s: SPX_FORCE_TC=1 but the tensor-core wgrad does not support this call (dtype %d, C/g %d, K/g %d)",
                  who, d->dtype, g0.c_in, g0.c_out);
        return 3;
    }
    if (tc_ok)
        SPX_REQUIRE(a->workspace && a->workspace_bytes >= tc_wgrad_workspace_size(g0),
                    "%s: workspace too small (%zu < %zu)", who, a->workspace_bytes, tc_wgrad_workspace_size(g0));
    set_family(tc_ok ? 2 : 1);
    for (int j = 0; j < groups; ++j) {
        const WgradArgs g = group_wgrad(all, groups, j, e);
        if (int rc = tc_ok ? tc_wgrad(g, stream, d->c_in, d->c_out) : simt_wgrad(g, stream, d->c_in, d->c_out))
            return rc;
    }
    // data-parallel: dW is complete locally; push it whole, as the FMA and depthwise routes do
    if (pg) return peer_push(nullptr, 0, 0, a->dfilters, dw_count, d->dtype, pg, stream);
    return 0;
}

extern "C" int spx_grouped_gemm_wgrad(const spx_gemm_desc *d, int groups, const spx_grouped_gemm *a,
                                      spx_stream_t stream) {
    return grouped_wgrad_entry(d, groups, a, nullptr, stream);
}

extern "C" int spx_grouped_gemm_wgrad_push(const spx_gemm_desc *d, int groups, const spx_grouped_gemm *a,
                                           const spx_peer_group *pg, spx_stream_t stream) {
    SPX_REQUIRE(pg != nullptr, "grouped_gemm_wgrad_push: peer group is NULL");
    return grouped_wgrad_entry(d, groups, a, pg, stream);
}
