// Per-sample GroupNorm / InstanceNorm over the kept rows of a (possibly padded) feature matrix [rows, C]
// (MaskedGroupNorm, pytorch/modules.py).  M = *num_valid (NULL: every row); row r belongs to sample b when r < M and
// coords[r, 0] == b with 0 <= b < B.  Every other row is dropped: never read beyond coords[r, 0] (nor at all
// beyond M), and 0 in y and dx.  Group g of C / G = Cg channels; sample b and group g have n = count_b * Cg values.
//
// Forward:
//   group    : group_samples (global_pool.cu): keys -> sort_by_key -> offsets [B+1] and chunks of GP_CHUNK rows
//              numbered by cstart [B+1].  The rows of sample b are order[offsets[b] .. offsets[b+1]) in ascending
//              row order, whatever the padding;
//   stats    : one block per (chunk, channel slice), grid ceil(rows / GP_CHUNK) + B, blocks past the last chunk exit.
//              Row lane l folds sorted positions p0 + l, p0 + l + lanes, ... by Welford, then the lanes merge by
//              Chan's rule in a fixed binary tree into partials [chunk][C] (mean, M2);
//   finalize : per (b, c) 32 lanes merge the sample's chunks p, p + 32, ... in chunk order, then a fixed tree
//              (Chan) -> bc [B][C] (mean, M2);
//   group    : per (b, g) in ascending c: mean = sum(mean_bc) / Cg, M2 = sum(M2_bc + n_b (mean_bc - mean)^2);
//              mean [B, G], invstd = rsqrt(M2 / n + eps) [B, G], saved for the backward;
//   apply    : y = (x - mean_bg) * (gamma_c * invstd_bg) + beta_c, one thread per 16-byte vector (or element).
// Backward (order / offsets / cstart of the forward, nothing is sorted again):
//   reduce   : per (chunk, c) with the stats layout: sum(dy) and sum(dy * xhat) -> partials [chunk][C];
//   finalize : per (b, c) in chunk order -> bc [B][C];
//   coef     : per c over ascending b: dbeta = sum(dy), dgamma = sum(dy * xhat); per (b, g) over ascending c:
//              S1 = sum(gamma_c sum(dy)), S2 = sum(gamma_c sum(dy * xhat)) -> coef [B][G] = (S1 / n, S2 / n);
//   apply    : dx = invstd_bg * (gamma_c dy - S1 / n - xhat * S2 / n); every element of dx is written once.
// Modulated (spx_masked_group_norm_mod): the applies write act(fmaf(h, 1 + scale_bc, shift_bc)); the backward
// recomputes that z from x, folds dz = dy act'(z) in place of dy, and weighs gamma_c, dbeta and dgamma by
// (1 + scale_bc); coef also writes dshift = sum(dz), dscale = gamma sum(dz xhat) + beta sum(dz).  Same launches.
// The order of every sum depends only on the sample's kept rows, never on `rows`, the padding or the grid, and no
// float atomics are used, so every result is bit-reproducible and independent of padding and dropped rows.
#include "rows.cuh"
#include "segments.cuh"

namespace spx {

constexpr int GN_THREADS = 256;
constexpr int GN_FIN_CH = 8;         // finalize: channels per block
constexpr int GN_FIN_LANES = 32;     // finalize: partial lanes per channel
constexpr int GN_MAX_BATCH = 1 << 20;
constexpr int GN_MAX_CHANNELS = 1 << 16;

// sample of row r, or -1 for a padding or dropped row
__device__ __forceinline__ int gn_row_sample(const int32_t *coords, int64_t r, int row_ints, int batch_size,
                                             int64_t M) {
    if (r >= M) return -1;
    const int32_t b = __ldg(coords + r * row_ints);
    return b >= 0 && b < batch_size ? b : -1;
}

// ---------------------------------------------------------------- forward
template <typename T, int W, bool A>
__global__ void __launch_bounds__(GN_THREADS)
gn_stats_kernel(const T *__restrict__ x, const int32_t *__restrict__ order, const int32_t *__restrict__ offsets,
                const int32_t *__restrict__ cstart, int batch_size, int channels, int vecs, int tpr,
                float2 *__restrict__ partials) {
    __shared__ float s_mean[GN_THREADS * W], s_q[GN_THREADS * W], s_n[GN_THREADS];
    int b;
    int32_t p0, end;
    if (!sample_chunk(offsets, cstart, batch_size, b, p0, end)) return;
    const int lanes = GN_THREADS / tpr;
    const RowThread t = row_thread(vecs, tpr);
    float n = 0.f, mean[W], q[W];
#pragma unroll
    for (int j = 0; j < W; ++j) mean[j] = q[j] = 0.f;
    if (t.active) {
        const T *base = x + (int64_t)t.v * W;
        auto fold = [&](const float (&f)[W], float inv) {  // Welford, in ascending sorted position; inv = 1 / n
            n += 1.f;
#pragma unroll
            for (int j = 0; j < W; ++j) {
                const float d = f[j] - mean[j];
                mean[j] = fmaf(d, inv, mean[j]);
                q[j] = fmaf(d, f[j] - mean[j], q[j]);
            }
        };
        int32_t p = p0 + t.lane;
        for (; p + lanes < end; p += 2 * lanes) {          // two rows in flight, folded in order
            // the reciprocals first: their slow path is a call, and nothing of the rows is live across it
            const float inv0 = __frcp_rn(n + 1.f), inv1 = __frcp_rn(n + 2.f);
            int r[2];
            float f[2][W];
#pragma unroll
            for (int u = 0; u < 2; ++u) r[u] = __ldg(order + p + u * lanes);
#pragma unroll
            for (int u = 0; u < 2; ++u) row_load<T, W, A>(base + (int64_t)r[u] * channels, f[u]);
            fold(f[0], inv0);
            fold(f[1], inv1);
        }
        for (; p < end; p += lanes) {
            const float inv = __frcp_rn(n + 1.f);
            float f[W];
            row_load<T, W, A>(base + (int64_t)__ldg(order + p) * channels, f);
            fold(f, inv);
        }
    }
    welford_lane_tree<W>(s_mean, s_q, s_n, lanes, tpr, n, mean, q);
    if (t.lane == 0 && t.active) {
        float2 *dst = partials + (int64_t)blockIdx.x * channels + (int64_t)t.v * W;
#pragma unroll
        for (int j = 0; j < W; ++j) dst[j] = make_float2(mean[j], q[j]);
    }
}

// grid (B, ceil(C / GN_FIN_CH)); lane pl of channel cl merges chunks cstart[b] + pl, + 32, ... in order, then a
// fixed tree over the lanes.  bc[b][c] = (mean, M2) of the sample's rows in channel c.
__global__ void __launch_bounds__(GN_FIN_CH * GN_FIN_LANES)
gn_fwd_finalize_kernel(const float2 *__restrict__ partials, const int32_t *__restrict__ offsets,
                       const int32_t *__restrict__ cstart, int channels, float2 *__restrict__ bc) {
    __shared__ float s_n[GN_FIN_LANES][GN_FIN_CH], s_m[GN_FIN_LANES][GN_FIN_CH], s_q[GN_FIN_LANES][GN_FIN_CH];
    const int cl = threadIdx.x % GN_FIN_CH, pl = threadIdx.x / GN_FIN_CH;
    const int b = blockIdx.x;
    const int c = blockIdx.y * GN_FIN_CH + cl;
    const bool active = c < channels;
    const int32_t k0 = __ldg(cstart + b), k1 = __ldg(cstart + b + 1);
    const int32_t o0 = __ldg(offsets + b), o1 = __ldg(offsets + b + 1);
    float n = 0.f, m = 0.f, q = 0.f;
    if (active)
        for (int32_t k = k0 + pl; k < k1; k += GN_FIN_LANES) {
            const float2 p = partials[(int64_t)k * channels + c];
            const int32_t left = o1 - o0 - (k - k0) * GP_CHUNK;
            chan_merge(n, m, q, (float)(left < GP_CHUNK ? left : GP_CHUNK), p.x, p.y);
        }
    s_n[pl][cl] = n;
    s_m[pl][cl] = m;
    s_q[pl][cl] = q;
    for (int s = GN_FIN_LANES / 2; s >= 1; s >>= 1) {
        __syncthreads();
        if (pl < s) {
            chan_merge(n, m, q, s_n[pl + s][cl], s_m[pl + s][cl], s_q[pl + s][cl]);
            s_n[pl][cl] = n;
            s_m[pl][cl] = m;
            s_q[pl][cl] = q;
        }
    }
    if (pl == 0 && active) bc[(int64_t)b * channels + c] = make_float2(m, q);
}

// one thread per (b, g): the Cg channels of the group merged in ascending c
__global__ void __launch_bounds__(GN_THREADS)
gn_fwd_group_kernel(const float2 *__restrict__ bc, const int32_t *__restrict__ offsets, int batch_size, int channels,
                    int groups, float eps, float *__restrict__ mean_out, float *__restrict__ invstd_out) {
    const int64_t i = blockIdx.x * (int64_t)GN_THREADS + threadIdx.x;
    if (i >= (int64_t)batch_size * groups) return;
    const int b = (int)(i / groups), g = (int)(i - (int64_t)b * groups);
    const int cg = channels / groups;
    const int32_t cnt = __ldg(offsets + b + 1) - __ldg(offsets + b);
    const float2 *p = bc + (int64_t)b * channels + (int64_t)g * cg;
    float sum = 0.f;
    for (int c = 0; c < cg; ++c) sum += p[c].x;
    const float mean = __fdiv_rn(sum, (float)cg);
    const float nb = (float)cnt;
    float m2 = 0.f;
    for (int c = 0; c < cg; ++c) {
        const float d = p[c].x - mean;
        m2 += fmaf(nb * d, d, p[c].y);
    }
    const int64_t n = (int64_t)cnt * cg;
    const float var = n > 0 ? __fdiv_rn(m2, (float)n) : 0.f;
    mean_out[i] = n > 0 ? mean : 0.f;
    invstd_out[i] = __frsqrt_rn(var + eps);
}

template <typename P> __device__ __forceinline__ float gn_param(const P *p, int c, float dflt) {
    return p ? to_float(__ldg(p + c)) : dflt;
}

// Modulation of sample b: z = fmaf(h, 1 + scale[b][c], shift[b][c]), a missing operand 0; 1 + scale[b][c] is also
// the factor of gamma_c in the backward.  gn_mod_row gives the sample's row of scale or shift (NULL stays NULL).
__device__ __forceinline__ const float *gn_mod_row(const float *p, int b, int channels) {
    return p ? p + (int64_t)b * channels : nullptr;
}
__device__ __forceinline__ float gn_scale1(const float *scale_row, int c) {
    return scale_row ? 1.f + __ldg(scale_row + c) : 1.f;
}
__device__ __forceinline__ float gn_shift(const float *shift_row, int c) {
    return shift_row ? __ldg(shift_row + c) : 0.f;
}

// y = act(z); relu keeps NaN, as torch's does
__device__ __forceinline__ float gn_act(int act, float z) {
    if (act == SPX_GN_ACT_RELU) return z <= 0.f ? 0.f : z;
    if (act == SPX_GN_ACT_SILU) return z / (1.f + expf(-z));
    return z;
}

// dz = dy act'(z): relu' = (z > 0), as threshold_backward; silu' = sigma(z) (1 + z (1 - sigma(z)))
__device__ __forceinline__ float gn_act_grad(int act, float z, float dy) {
    if (act == SPX_GN_ACT_RELU) return z > 0.f ? dy : 0.f;
    if (act == SPX_GN_ACT_SILU) {
        const float s = 1.f / (1.f + expf(-z));
        return dy * (s * fmaf(z, 1.f - s, 1.f));
    }
    return dy;
}

// y = act(z) with h = (x - mean) * (gamma * invstd) + beta and z = h without scale and shift (so the unmodulated
// call keeps h's bits, -0 included), else fmaf(h, 1 + scale, shift).  The backward recomputes z with the same
// expressions.
template <typename T, typename P, int W, bool A>
__global__ void __launch_bounds__(GN_THREADS)
gn_fwd_apply_kernel(const T *__restrict__ x, T *__restrict__ y, const int32_t *__restrict__ coords, int64_t rows,
                    int row_ints, int batch_size, int channels, int vecs, int tpr, int groups,
                    const int32_t *__restrict__ num_valid, const P *__restrict__ weight, const P *__restrict__ bias,
                    const float *__restrict__ mean, const float *__restrict__ invstd,
                    const float *__restrict__ scale, const float *__restrict__ shift, int act) {
    const int lanes = GN_THREADS / tpr;
    const int64_t r = blockIdx.x * (int64_t)lanes + threadIdx.x / tpr;
    const int v = blockIdx.y * tpr + (threadIdx.x % tpr);
    if (r >= rows || v >= vecs) return;
    const int b = gn_row_sample(coords, r, row_ints, batch_size, valid_rows(num_valid, rows));
    const int cg = channels / groups;
    float f[W];
    if (b >= 0) {
        row_load<T, W, A>(x + r * channels + (int64_t)v * W, f);
        const bool mod = scale || shift;
        const float *srow = gn_mod_row(scale, b, channels), *trow = gn_mod_row(shift, b, channels);
#pragma unroll
        for (int j = 0; j < W; ++j) {
            const int c = v * W + j;
            const int64_t bg = (int64_t)b * groups + c / cg;
            const float a = gn_param(weight, c, 1.f) * __ldg(invstd + bg);
            f[j] = fmaf(f[j] - __ldg(mean + bg), a, gn_param(bias, c, 0.f));
            if (mod) f[j] = fmaf(f[j], gn_scale1(srow, c), gn_shift(trow, c));
            f[j] = gn_act(act, f[j]);
        }
    } else {
#pragma unroll
        for (int j = 0; j < W; ++j) f[j] = 0.f;
    }
    row_store<T, W, A>(y + r * channels + (int64_t)v * W, f);
}

// ---------------------------------------------------------------- backward
// The sums are over dz = dy act'(z); z is recomputed from x as the forward computes it.  ACT = (act != NONE): the
// recomputation doubles the registers of the vector instances, so the plain backward does not carry it.
template <typename T, typename P, int W, bool A, bool ACT>
__global__ void __launch_bounds__(GN_THREADS)
gn_bwd_reduce_kernel(const T *__restrict__ x, const T *__restrict__ dy, const int32_t *__restrict__ order,
                     const int32_t *__restrict__ offsets, const int32_t *__restrict__ cstart, int batch_size,
                     int channels, int vecs, int tpr, int groups, const float *__restrict__ mean_bg,
                     const float *__restrict__ invstd_bg, const P *__restrict__ weight, const P *__restrict__ bias,
                     const float *__restrict__ scale, const float *__restrict__ shift, int act,
                     float2 *__restrict__ partials) {
    __shared__ float s_a[GN_THREADS * W], s_b[GN_THREADS * W];
    int b;
    int32_t p0, end;
    if (!sample_chunk(offsets, cstart, batch_size, b, p0, end)) return;
    const int lanes = GN_THREADS / tpr;
    const RowThread t = row_thread(vecs, tpr);
    float sdy[W], sdyx[W];
#pragma unroll
    for (int j = 0; j < W; ++j) sdy[j] = sdyx[j] = 0.f;
    if (t.active) {
        const int cg = channels / groups;
        float mean[W], invstd[W];
#pragma unroll
        for (int j = 0; j < W; ++j) {
            const int64_t bg = (int64_t)b * groups + (t.v * W + j) / cg;
            mean[j] = __ldg(mean_bg + bg);
            invstd[j] = __ldg(invstd_bg + bg);
        }
        // z = fmaf(fmaf(x - mean, a, beta), s1, sh) as in the forward; a chunk is one sample's, so these are constants
        const bool mod = scale || shift;
        const float *srow = gn_mod_row(scale, b, channels), *trow = gn_mod_row(shift, b, channels);
        float a[W], beta[W], s1[W], sh[W];
#pragma unroll
        for (int j = 0; j < W; ++j) {
            const int c = t.v * W + j;
            a[j] = ACT ? gn_param(weight, c, 1.f) * invstd[j] : 0.f;
            beta[j] = ACT ? gn_param(bias, c, 0.f) : 0.f;
            s1[j] = ACT ? gn_scale1(srow, c) : 1.f;
            sh[j] = ACT ? gn_shift(trow, c) : 0.f;
        }
        const int64_t off = (int64_t)t.v * W;
        auto fold = [&](const float (&fx)[W], const float (&fd)[W]) {
#pragma unroll
            for (int j = 0; j < W; ++j) {
                const float xc = fx[j] - mean[j];
                float d = fd[j];
                if (ACT) {
                    float z = fmaf(xc, a[j], beta[j]);
                    if (mod) z = fmaf(z, s1[j], sh[j]);
                    d = gn_act_grad(act, z, d);
                }
                sdy[j] += d;
                sdyx[j] = fmaf(d, xc * invstd[j], sdyx[j]);
            }
        };
        int32_t p = p0 + t.lane;
        for (; p + lanes < end; p += 2 * lanes) {          // two rows of x and dy in flight
            float fx[2][W], fd[2][W];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int64_t o = (int64_t)__ldg(order + p + u * lanes) * channels + off;
                row_load<T, W, A>(x + o, fx[u]);
                row_load<T, W, A>(dy + o, fd[u]);
            }
#pragma unroll
            for (int u = 0; u < 2; ++u) fold(fx[u], fd[u]);
        }
        for (; p < end; p += lanes) {
            const int64_t o = (int64_t)__ldg(order + p) * channels + off;
            float fx[W], fd[W];
            row_load<T, W, A>(x + o, fx);
            row_load<T, W, A>(dy + o, fd);
            fold(fx, fd);
        }
    }
    pair_sum_lane_tree<W>(s_a, s_b, lanes, tpr, sdy, sdyx);
    if (t.lane == 0 && t.active) {
        float2 *dst = partials + (int64_t)blockIdx.x * channels + (int64_t)t.v * W;
#pragma unroll
        for (int j = 0; j < W; ++j) dst[j] = make_float2(sdy[j], sdyx[j]);
    }
}

// grid (B, ceil(C / GN_FIN_CH)): bc[b][c] = (sum dy, sum dy * xhat) of the sample's chunks, merged in chunk order
__global__ void __launch_bounds__(GN_FIN_CH * GN_FIN_LANES)
gn_bwd_finalize_kernel(const float2 *__restrict__ partials, const int32_t *__restrict__ cstart, int channels,
                       float2 *__restrict__ bc) {
    __shared__ float s_a[GN_FIN_LANES][GN_FIN_CH], s_b[GN_FIN_LANES][GN_FIN_CH];
    const int cl = threadIdx.x % GN_FIN_CH, pl = threadIdx.x / GN_FIN_CH;
    const int b = blockIdx.x;
    const int c = blockIdx.y * GN_FIN_CH + cl;
    const bool active = c < channels;
    const int32_t k0 = __ldg(cstart + b), k1 = __ldg(cstart + b + 1);
    float a = 0.f, s2 = 0.f;
    if (active)
        for (int32_t k = k0 + pl; k < k1; k += GN_FIN_LANES) {
            const float2 p = partials[(int64_t)k * channels + c];
            a += p.x;
            s2 += p.y;
        }
    s_a[pl][cl] = a;
    s_b[pl][cl] = s2;
    for (int s = GN_FIN_LANES / 2; s >= 1; s >>= 1) {
        __syncthreads();
        if (pl < s) {
            s_a[pl][cl] = a = a + s_a[pl + s][cl];
            s_b[pl][cl] = s2 = s2 + s_b[pl + s][cl];
        }
    }
    if (pl == 0 && active) bc[(int64_t)b * channels + c] = make_float2(a, s2);
}

// threads [0, C): dbias[c] / dweight[c] over ascending b, and dshift[b][c] / dscale[b][c]; threads [C, C + B G):
// coef[b][g] = (S1 / n, S2 / n) with S1, S2 over ascending c of the group.  With a scale, (1 + scale[b][c]) weighs
// the sums of sample b: without one the factor is 1 and fmaf(1, p, a) == a + p.
template <typename P>
__global__ void __launch_bounds__(GN_THREADS)
gn_bwd_coef_kernel(const float2 *__restrict__ bc, const int32_t *__restrict__ offsets, int batch_size, int channels,
                   int groups, const P *__restrict__ weight, const P *__restrict__ bias,
                   const float *__restrict__ scale, P *__restrict__ dweight, P *__restrict__ dbias,
                   float *__restrict__ dscale, float *__restrict__ dshift, float2 *__restrict__ coef) {
    const int64_t i = blockIdx.x * (int64_t)GN_THREADS + threadIdx.x;
    if (i < channels) {
        float a = 0.f, s2 = 0.f;
        const float gamma = gn_param(weight, (int)i, 1.f), beta = gn_param(bias, (int)i, 0.f);
        for (int b = 0; b < batch_size; ++b) {
            const int64_t k = (int64_t)b * channels + i;
            const float2 p = bc[k];
            const float s = gn_scale1(gn_mod_row(scale, b, channels), (int)i);
            a = fmaf(s, p.x, a);
            s2 = fmaf(s, p.y, s2);
            if (dshift) dshift[k] = p.x;
            if (dscale) dscale[k] = fmaf(gamma, p.y, beta * p.x);
        }
        if (dbias) dbias[i] = from_float<P>(a);
        if (dweight) dweight[i] = from_float<P>(s2);
        return;
    }
    const int64_t j = i - channels;
    if (j >= (int64_t)batch_size * groups) return;
    const int b = (int)(j / groups), g = (int)(j - (int64_t)b * groups);
    const int cg = channels / groups;
    const int c0 = g * cg;
    const float2 *p = bc + (int64_t)b * channels + c0;
    const float *srow = gn_mod_row(scale, b, channels);
    float s1 = 0.f, s2 = 0.f;
    for (int c = 0; c < cg; ++c) {
        const float gamma = gn_param(weight, c0 + c, 1.f) * gn_scale1(srow, c0 + c);
        s1 = fmaf(gamma, p[c].x, s1);
        s2 = fmaf(gamma, p[c].y, s2);
    }
    const int64_t n = (int64_t)(__ldg(offsets + b + 1) - __ldg(offsets + b)) * cg;
    coef[j] = n > 0 ? make_float2(__fdiv_rn(s1, (float)n), __fdiv_rn(s2, (float)n)) : make_float2(0.f, 0.f);
}

template <typename T, typename P, int W, bool A, bool ACT>
__global__ void __launch_bounds__(GN_THREADS)
gn_bwd_apply_kernel(const T *__restrict__ x, const T *__restrict__ dy, T *__restrict__ dx,
                    const int32_t *__restrict__ coords, int64_t rows, int row_ints, int batch_size, int channels,
                    int vecs, int tpr, int groups, const int32_t *__restrict__ num_valid, const P *__restrict__ weight,
                    const P *__restrict__ bias, const float *__restrict__ mean, const float *__restrict__ invstd,
                    const float *__restrict__ scale, const float *__restrict__ shift, int act,
                    const float2 *__restrict__ coef) {
    const int lanes = GN_THREADS / tpr;
    const int64_t r = blockIdx.x * (int64_t)lanes + threadIdx.x / tpr;
    const int v = blockIdx.y * tpr + (threadIdx.x % tpr);
    if (r >= rows || v >= vecs) return;
    const int b = gn_row_sample(coords, r, row_ints, batch_size, valid_rows(num_valid, rows));
    const int cg = channels / groups;
    float f[W];
    if (b >= 0) {
        float fx[W];
        const int64_t o = r * channels + (int64_t)v * W;
        row_load<T, W, A>(x + o, fx);
        row_load<T, W, A>(dy + o, f);
        const bool mod = scale || shift;
        const float *srow = gn_mod_row(scale, b, channels), *trow = gn_mod_row(shift, b, channels);
#pragma unroll
        for (int j = 0; j < W; ++j) {
            const int c = v * W + j;
            const int64_t bg = (int64_t)b * groups + c / cg;
            const float is = __ldg(invstd + bg);
            const float xc = fx[j] - __ldg(mean + bg);
            const float xhat = xc * is;
            const float gamma = gn_param(weight, c, 1.f);
            if (ACT) {                                         // dz from the forward's z
                float z = fmaf(xc, gamma * is, gn_param(bias, c, 0.f));
                if (mod) z = fmaf(z, gn_scale1(srow, c), gn_shift(trow, c));
                f[j] = gn_act_grad(act, z, f[j]);
            }
            const float2 k = __ldg(coef + bg);
            // the product is rounded on its own, as in S1: one row with Cg = 1 gives gamma dy - S1 / n = 0 exactly
            f[j] = is * (__fmul_rn(gamma * gn_scale1(srow, c), f[j]) - k.x - xhat * k.y);
        }
    } else {
#pragma unroll
        for (int j = 0; j < W; ++j) f[j] = 0.f;
    }
    row_store<T, W, A>(dx + r * channels + (int64_t)v * W, f);
}

// ---------------------------------------------------------------- host side
static int64_t gn_max_chunks(int64_t rows, int batch_size) {
    return (rows + GP_CHUNK - 1) / GP_CHUNK + batch_size;
}

static int gn_check(const char *who, int64_t rows, int row_ints, int batch_size, int channels, int groups, int dtype,
                    int param_dtype) {
    SPX_REQUIRE(rows >= 0 && rows < 2147483647ll, "%s: bad row count %lld", who, (long long)rows);
    SPX_REQUIRE(row_ints >= 1, "%s: coordinate rows must hold the batch index, got %d ints", who, row_ints);
    SPX_REQUIRE(batch_size >= 1 && batch_size <= GN_MAX_BATCH, "%s: batch_size must be in [1, 2^20], got %d", who,
                batch_size);
    SPX_REQUIRE(channels >= 1 && channels <= GN_MAX_CHANNELS, "%s: channels must be in [1, 65536], got %d", who,
                channels);
    SPX_REQUIRE(groups >= 1 && channels % groups == 0, "%s: num_groups %d must divide channels %d", who, groups,
                channels);
    SPX_REQUIRE(dtype == SPX_F32 || dtype == SPX_F16 || dtype == SPX_BF16,
                "%s: unsupported dtype %d (float32, float16 and bfloat16 only)", who, dtype);
    SPX_REQUIRE(param_dtype == SPX_F32 || param_dtype == dtype,
                "%s: parameter dtype %d must be float32 or the feature dtype %d", who, param_dtype, dtype);
    return 0;
}

struct GnWorkspace {
    uint32_t *keys;
    void *sort_ws;
    float2 *partials, *bc, *coef;
};

static GnWorkspace gn_carve(void *workspace, size_t bytes, int64_t rows, int batch_size, int channels) {
    WorkspaceCarver ws(workspace, bytes);
    GnWorkspace w;
    w.keys = ws.take<uint32_t>((size_t)rows);
    w.sort_ws = ws.take<char>(radix_argsort_workspace_bytes(rows));
    w.partials = ws.take<float2>((size_t)gn_max_chunks(rows, batch_size) * channels);
    w.bc = ws.take<float2>((size_t)batch_size * channels);
    w.coef = ws.take<float2>((size_t)batch_size * channels);
    return w;
}

struct GnArgs {
    const void *x, *dy;
    void *y, *dx;
    const int32_t *coords;
    int64_t rows;
    int row_ints, batch_size, channels, groups;
    const int32_t *num_valid;
    const void *weight, *bias;
    void *dweight, *dbias;
    float eps;
    const float *mean, *invstd;
    const int32_t *order, *offsets, *cstart;
    const float *scale, *shift;
    int act;
    float *dscale, *dshift;
    GnWorkspace ws;
};

// the row kernels of one pass: reduce = stats (fwd) / sums (bwd), or the apply
template <typename T, typename P, int W, bool A> static int gn_rows(const GnArgs &a, bool fwd, bool reduce,
                                                                   cudaStream_t stream) {
    const int vecs = a.channels / W;
    if (reduce) {
        const int tpr = row_tpr(vecs);
        const dim3 grid((unsigned)gn_max_chunks(a.rows, a.batch_size), (unsigned)div_up64(vecs, tpr));
        if (fwd) {
            gn_stats_kernel<T, W, A><<<grid, GN_THREADS, 0, stream>>>(
                static_cast<const T *>(a.x), a.order, a.offsets, a.cstart, a.batch_size, a.channels, vecs, tpr,
                a.ws.partials);
            SPX_CHECK_LAUNCH("gn_stats_kernel");
        } else {
            auto reduce = [&](auto kernel, const auto *weight, const auto *bias) {
                kernel<<<grid, GN_THREADS, 0, stream>>>(
                    static_cast<const T *>(a.x), static_cast<const T *>(a.dy), a.order, a.offsets, a.cstart,
                    a.batch_size, a.channels, vecs, tpr, a.groups, a.mean, a.invstd, weight, bias, a.scale, a.shift,
                    a.act, a.ws.partials);
            };
            // without an activation the reduce reads no parameter: one instance per feature type serves both
            // parameter dtypes
            if (a.act)
                reduce(gn_bwd_reduce_kernel<T, P, W, A, true>, static_cast<const P *>(a.weight),
                       static_cast<const P *>(a.bias));
            else
                reduce(gn_bwd_reduce_kernel<T, T, W, A, false>, static_cast<const T *>(nullptr),
                       static_cast<const T *>(nullptr));
            SPX_CHECK_LAUNCH("gn_bwd_reduce_kernel");
        }
        return 0;
    }
    const int tpr = row_tpr(vecs);
    const dim3 blocks((unsigned)div_up64(a.rows, GN_THREADS / tpr), (unsigned)div_up64(vecs, tpr));
    if (fwd) {
        gn_fwd_apply_kernel<T, P, W, A><<<blocks, GN_THREADS, 0, stream>>>(
            static_cast<const T *>(a.x), static_cast<T *>(a.y), a.coords, a.rows, a.row_ints, a.batch_size,
            a.channels, vecs, tpr, a.groups, a.num_valid, static_cast<const P *>(a.weight),
            static_cast<const P *>(a.bias), a.mean, a.invstd, a.scale, a.shift, a.act);
        SPX_CHECK_LAUNCH("gn_fwd_apply_kernel");
    } else {
        auto kernel = a.act ? gn_bwd_apply_kernel<T, P, W, A, true> : gn_bwd_apply_kernel<T, P, W, A, false>;
        kernel<<<blocks, GN_THREADS, 0, stream>>>(
            static_cast<const T *>(a.x), static_cast<const T *>(a.dy), static_cast<T *>(a.dx), a.coords, a.rows,
            a.row_ints, a.batch_size, a.channels, vecs, tpr, a.groups, a.num_valid, static_cast<const P *>(a.weight),
            static_cast<const P *>(a.bias), a.mean, a.invstd, a.scale, a.shift, a.act, a.ws.coef);
        SPX_CHECK_LAUNCH("gn_bwd_apply_kernel");
    }
    return 0;
}

static int gn_rows_typed(int dtype, int param_dtype, const GnArgs &a, bool fwd, bool reduce, cudaStream_t stream) {
    return dispatch_dtype(dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        constexpr int W = 16 / sizeof(T);
        // the reductions and the applies share one width: W whenever wide
        const RowWidth w = fwd ? row_width(a.channels * sizeof(T), a.x, a.y)
                               : row_width(a.channels * sizeof(T), a.x, a.dy, a.dx);
        auto rows = [&](auto p) {
            using P = typename decltype(p)::type;
            if (!w.wide) return gn_rows<T, P, 1, false>(a, fwd, reduce, stream);
            return w.aligned ? gn_rows<T, P, W, true>(a, fwd, reduce, stream)
                             : gn_rows<T, P, W, false>(a, fwd, reduce, stream);
        };
        return param_dtype == SPX_F32 ? rows(Type<float>{}) : rows(Type<T>{});
    });
}

template <typename P> static int gn_bwd_coef(const GnArgs &a, cudaStream_t stream) {
    const int64_t threads = a.channels + (int64_t)a.batch_size * a.groups;
    gn_bwd_coef_kernel<P><<<(unsigned)div_up64(threads, GN_THREADS), GN_THREADS, 0, stream>>>(
        a.ws.bc, a.offsets, a.batch_size, a.channels, a.groups, static_cast<const P *>(a.weight),
        static_cast<const P *>(a.bias), a.scale, static_cast<P *>(a.dweight), static_cast<P *>(a.dbias), a.dscale,
        a.dshift, a.ws.coef);
    SPX_CHECK_LAUNCH("gn_bwd_coef_kernel");
    return 0;
}

}  // namespace spx

using namespace spx;

extern "C" size_t spx_masked_group_norm_workspace_size(int64_t rows, int batch_size, int channels) {
    if (rows < 0 || batch_size < 1 || channels < 1) return 0;
    return align_up((size_t)rows * 4, 256) + align_up(radix_argsort_workspace_bytes(rows), 256) +
           align_up((size_t)gn_max_chunks(rows, batch_size) * channels * sizeof(float2), 256) +
           2 * align_up((size_t)batch_size * channels * sizeof(float2), 256);
}

namespace spx {

static int gn_check_desc(const char *who, const spx_masked_group_norm *d, const void *workspace,
                         size_t workspace_bytes) {
    SPX_REQUIRE(d != nullptr, "%s: descriptor is NULL", who);
    if (int rc = gn_check(who, d->rows, d->row_ints, d->batch_size, d->channels, d->groups, d->dtype, d->param_dtype))
        return rc;
    SPX_REQUIRE(d->mean && d->invstd && d->offsets && d->cstart && workspace,
                "%s: NULL pointer argument (mean, invstd, offsets, cstart, workspace)", who);
    const size_t need = spx_masked_group_norm_workspace_size(d->rows, d->batch_size, d->channels);
    SPX_REQUIRE(workspace_bytes >= need, "%s: workspace too small: need %zu, have %zu", who, need, workspace_bytes);
    return 0;
}

// m: the modulation, or NULL for none
static GnArgs gn_args(const spx_masked_group_norm *d, const spx_masked_group_norm_mod *m, void *workspace,
                      size_t workspace_bytes) {
    GnArgs a{};
    a.x = d->x;
    a.dy = d->dy;
    a.y = d->y;
    a.dx = d->dx;
    a.coords = d->coords;
    a.rows = d->rows;
    a.row_ints = d->row_ints;
    a.batch_size = d->batch_size;
    a.channels = d->channels;
    a.groups = d->groups;
    a.num_valid = d->num_valid;
    a.weight = d->weight;
    a.bias = d->bias;
    a.dweight = d->dweight;
    a.dbias = d->dbias;
    a.eps = d->eps;
    a.mean = d->mean;
    a.invstd = d->invstd;
    a.order = d->order;
    a.offsets = d->offsets;
    a.cstart = d->cstart;
    if (m) {
        a.scale = m->scale;
        a.shift = m->shift;
        a.act = m->act;
        a.dscale = m->dscale;
        a.dshift = m->dshift;
    }
    a.ws = gn_carve(workspace, workspace_bytes, d->rows, d->batch_size, d->channels);
    return a;
}

static int gn_check_mod(const char *who, const spx_masked_group_norm_mod *m) {
    SPX_REQUIRE(m != nullptr, "%s: descriptor is NULL", who);
    SPX_REQUIRE(m->act == SPX_GN_ACT_NONE || m->act == SPX_GN_ACT_RELU || m->act == SPX_GN_ACT_SILU,
                "%s: unknown activation %d (SPX_GN_ACT_NONE, _RELU or _SILU)", who, m->act);
    return 0;
}

static int gn_fwd(const char *who, const spx_masked_group_norm *d, const spx_masked_group_norm_mod *m,
                  void *workspace, size_t workspace_bytes, cudaStream_t stream) {
    if (int rc = gn_check_desc(who, d, workspace, workspace_bytes)) return rc;
    SPX_REQUIRE(d->rows == 0 || (d->x && d->y && d->coords && d->order),
                "%s: NULL pointer argument (x, y, coords, order)", who);
    SPX_REQUIRE(d->eps > 0.f, "%s: eps must be positive", who);
    const GnArgs a = gn_args(d, m, workspace, workspace_bytes);
    if (int rc = group_samples(a.coords, a.rows, a.row_ints, a.batch_size, a.num_valid, a.ws.keys, d->order,
                               a.ws.sort_ws, d->offsets, d->cstart, nullptr, stream))
        return rc;
    if (a.rows > 0)
        if (int rc = gn_rows_typed(d->dtype, d->param_dtype, a, true, true, stream)) return rc;
    gn_fwd_finalize_kernel<<<dim3((unsigned)a.batch_size, (unsigned)div_up64(a.channels, GN_FIN_CH)),
                             GN_FIN_CH * GN_FIN_LANES, 0, stream>>>(a.ws.partials, a.offsets, a.cstart, a.channels,
                                                                    a.ws.bc);
    SPX_CHECK_LAUNCH("gn_fwd_finalize_kernel");
    gn_fwd_group_kernel<<<(unsigned)div_up64((int64_t)a.batch_size * a.groups, GN_THREADS), GN_THREADS, 0, stream>>>(
        a.ws.bc, a.offsets, a.batch_size, a.channels, a.groups, a.eps, d->mean, d->invstd);
    SPX_CHECK_LAUNCH("gn_fwd_group_kernel");
    if (a.rows == 0) return 0;
    return gn_rows_typed(d->dtype, d->param_dtype, a, true, false, stream);
}

static int gn_bwd(const char *who, const spx_masked_group_norm *d, const spx_masked_group_norm_mod *m,
                  void *workspace, size_t workspace_bytes, cudaStream_t stream) {
    if (int rc = gn_check_desc(who, d, workspace, workspace_bytes)) return rc;
    SPX_REQUIRE(d->rows == 0 || (d->x && d->dy && d->dx && d->coords && d->order),
                "%s: NULL pointer argument (x, dy, dx, coords, order)", who);
    GnArgs a = gn_args(d, m, workspace, workspace_bytes);
    // bias is an operand of the backward only through z (an activation) and dscale; the plain backward never
    // reads it, whatever the field holds
    if (!m || (m->act == SPX_GN_ACT_NONE && !m->dscale)) a.bias = nullptr;
    if (a.rows > 0)
        if (int rc = gn_rows_typed(d->dtype, d->param_dtype, a, false, true, stream)) return rc;
    gn_bwd_finalize_kernel<<<dim3((unsigned)a.batch_size, (unsigned)div_up64(a.channels, GN_FIN_CH)),
                             GN_FIN_CH * GN_FIN_LANES, 0, stream>>>(a.ws.partials, a.cstart, a.channels, a.ws.bc);
    SPX_CHECK_LAUNCH("gn_bwd_finalize_kernel");
    const int rc =
        dispatch_dtype(d->param_dtype, [&](auto p) { return gn_bwd_coef<typename decltype(p)::type>(a, stream); });
    if (rc || a.rows == 0) return rc;
    return gn_rows_typed(d->dtype, d->param_dtype, a, false, false, stream);
}

}  // namespace spx

extern "C" int spx_masked_group_norm_fwd(const spx_masked_group_norm *d, void *workspace, size_t workspace_bytes,
                                         spx_stream_t stream) {
    return gn_fwd("masked_group_norm_fwd", d, nullptr, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int spx_masked_group_norm_bwd(const spx_masked_group_norm *d, void *workspace, size_t workspace_bytes,
                                         spx_stream_t stream) {
    return gn_bwd("masked_group_norm_bwd", d, nullptr, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int spx_masked_group_norm_mod_fwd(const spx_masked_group_norm_mod *m, void *workspace,
                                             size_t workspace_bytes, spx_stream_t stream) {
    const char *who = "masked_group_norm_mod_fwd";
    if (int rc = gn_check_mod(who, m)) return rc;
    return gn_fwd(who, &m->norm, m, workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int spx_masked_group_norm_mod_bwd(const spx_masked_group_norm_mod *m, void *workspace,
                                             size_t workspace_bytes, spx_stream_t stream) {
    const char *who = "masked_group_norm_mod_bwd";
    if (int rc = gn_check_mod(who, m)) return rc;
    return gn_bwd(who, &m->norm, m, workspace, workspace_bytes, (cudaStream_t)stream);
}
