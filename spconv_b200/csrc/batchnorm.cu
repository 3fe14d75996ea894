// Training-mode BatchNorm over the valid rows of a (possibly padded) feature matrix [rows, C]
// (MaskedBatchNorm1d, pytorch/modules.py).  M = *num_valid (NULL: every row); rows [M, rows) are never read
// and come out as exact zeros in y and dx.
//
// Every row reduction uses the same fixed structure, so results depend only on rows [0, M) and their
// values, never on `rows` or on the grid size (no float atomics):
//   chunk    : BN_CHUNK consecutive rows, one block per (chunk, channel slice).  Row lane l of the block
//              folds rows r0 + l, r0 + l + lanes, ... in ascending order, then the lanes merge in a fixed
//              binary tree; the chunk's partial goes to workspace [chunks][C].  Chunks at or beyond M exit.
//   finalize : lane p of 32 sums the partials p, p + 32, ... below ceil(M / BN_CHUNK) in order, then a fixed
//              tree over the 32 lanes.  Partials of empty chunks are never read, so padding is a no-op.
// Forward: stats (per-chunk Welford mean / M2, merged by Chan's rule) -> finalize (mean, biased variance,
// invstd, running-stat update) -> apply y = (x - mean) * (gamma * invstd) + beta.
// Backward: reduce (per-chunk sums of dy and dy * xhat) -> finalize (dbeta, dgamma, coefficients) ->
// apply dx = gamma * invstd * (dy - sum(dy) / M - xhat * sum(dy * xhat) / M).
// Feature rows move as 16-byte vectors when the row length and the pointers allow it, else per element.
#include "rows.cuh"

namespace spx {

constexpr int BN_THREADS = 256;
constexpr int BN_CHUNK = 512;        // rows per partial
constexpr int BN_FIN_CH = 8;         // finalize: channels per block
constexpr int BN_FIN_LANES = 32;     // finalize: partial lanes per channel

// rows of chunk k that are valid
__device__ __forceinline__ float bn_chunk_count(int64_t k, int64_t M) {
    const int64_t n = M - k * BN_CHUNK;
    return (float)(n < 0 ? 0 : (n > BN_CHUNK ? BN_CHUNK : n));
}

// ---------------------------------------------------------------- forward
template <typename T, int W, bool V>
__global__ void __launch_bounds__(BN_THREADS)
bn_stats_kernel(const T *__restrict__ x, int64_t rows, int channels, int vecs, int tpr,
                const int32_t *__restrict__ num_valid, float2 *__restrict__ partials) {
    __shared__ float s_mean[BN_THREADS * W], s_q[BN_THREADS * W], s_n[BN_THREADS];
    const int64_t M = valid_rows(num_valid, rows);
    const int64_t r0 = (int64_t)blockIdx.x * BN_CHUNK;
    if (r0 >= M) return;                                   // the whole block: nothing valid here
    const int lanes = BN_THREADS / tpr;
    const RowThread t = row_thread(vecs, tpr);
    const int64_t end = M < r0 + BN_CHUNK ? M : r0 + BN_CHUNK;
    float n = 0.f, mean[W], q[W];
#pragma unroll
    for (int j = 0; j < W; ++j) mean[j] = q[j] = 0.f;
    if (t.active) {
        const T *base = x + (int64_t)t.v * W;
        auto fold = [&](const float (&f)[W]) {             // Welford, rows in ascending order
            n += 1.f;
            const float inv = __frcp_rn(n);
#pragma unroll
            for (int j = 0; j < W; ++j) {
                const float d = f[j] - mean[j];
                mean[j] = fmaf(d, inv, mean[j]);
                q[j] = fmaf(d, f[j] - mean[j], q[j]);
            }
        };
        int64_t r = r0 + t.lane;
        for (; r + 3 * lanes < end; r += 4 * lanes) {     // four loads in flight, folded in row order
            float f[4][W];
#pragma unroll
            for (int u = 0; u < 4; ++u) row_load<T, W, V>(base + (r + (int64_t)u * lanes) * channels, f[u]);
#pragma unroll
            for (int u = 0; u < 4; ++u) fold(f[u]);
        }
        for (; r < end; r += lanes) {
            float f[W];
            row_load<T, W, V>(base + r * channels, f);
            fold(f);
        }
    }
    welford_lane_tree<W>(s_mean, s_q, s_n, lanes, tpr, n, mean, q);
    if (t.lane == 0 && t.active) {
        float2 *dst = partials + (int64_t)blockIdx.x * channels + (int64_t)t.v * W;
#pragma unroll
        for (int j = 0; j < W; ++j) dst[j] = make_float2(mean[j], q[j]);
    }
}

// Sum over the 32 partial lanes of one channel in a fixed tree; every thread of the channel gets the total.
__device__ __forceinline__ float bn_lane_sum(float v, float (*buf)[BN_FIN_CH], int pl, int cl) {
    buf[pl][cl] = v;
    for (int s = BN_FIN_LANES / 2; s >= 1; s >>= 1) {
        __syncthreads();
        if (pl < s) buf[pl][cl] += buf[pl + s][cl];
    }
    __syncthreads();
    const float total = buf[0][cl];
    __syncthreads();
    return total;
}

// Sum of the valid rows and M2 about their mean, from the chunk partials: sum = lane tree of n_k * mean_k, mean =
// sum / M, m2 = lane tree of q_k + n_k * (mean_k - mean)^2.  Every thread of the channel gets all three.
__device__ __forceinline__ void bn_fwd_sums(const float2 *__restrict__ partials, int64_t M, int channels, int c,
                                            bool active, float (*buf)[BN_FIN_CH], int pl, int cl, float &sum,
                                            float &mean, float &m2) {
    const int64_t K = (M + BN_CHUNK - 1) / BN_CHUNK;
    float s = 0.f;
    if (active)
        for (int64_t k = pl; k < K; k += BN_FIN_LANES) s = fmaf(bn_chunk_count(k, M), partials[k * channels + c].x, s);
    const float Mf = (float)M;
    sum = bn_lane_sum(s, buf, pl, cl);
    mean = M > 0 ? __fdiv_rn(sum, Mf) : 0.f;
    float q = 0.f;
    if (active)
        for (int64_t k = pl; k < K; k += BN_FIN_LANES) {
            const float2 p = partials[k * channels + c];
            const float d = p.x - mean;
            q += fmaf(bn_chunk_count(k, M) * d, d, p.y);
        }
    m2 = bn_lane_sum(q, buf, pl, cl);
}

// Channel c of a batch of M rows with this mean and M2: save_mean / save_invstd, the apply coefficients and the
// running-stat update.
template <typename P>
__device__ __forceinline__ void bn_fwd_write(int c, int channels, int64_t M, float mean, float m2,
                                             const P *__restrict__ weight, const P *__restrict__ bias,
                                             P *__restrict__ running_mean, P *__restrict__ running_var,
                                             const int64_t *__restrict__ num_batches_tracked, float momentum,
                                             int cumulative, float eps, float *__restrict__ save_mean,
                                             float *__restrict__ save_invstd, float *__restrict__ coef) {
    const float Mf = (float)M;
    const float var = M > 0 ? __fdiv_rn(m2, Mf) : 0.f;
    const float invstd = __frsqrt_rn(var + eps);
    const float gamma = weight ? to_float(weight[c]) : 1.f;
    const float beta = bias ? to_float(bias[c]) : 0.f;
    save_mean[c] = mean;
    save_invstd[c] = invstd;
    coef[c] = mean;
    coef[channels + c] = gamma * invstd;
    coef[2 * channels + c] = beta;
    if (running_mean != nullptr && M > 1) {                // one value per channel has no unbiased variance
        // divisors >= 1: the 2-ulp fast division is accurate here, and a third IEEE division would make ptxas
        // keep a value on the stack across its slow-path call
        const float f = cumulative ? __fdividef(1.f, (float)__ldg(num_batches_tracked)) : momentum;
        const float unbiased = __fdividef(m2, (float)(M - 1));
        running_mean[c] = from_float<P>((1.f - f) * to_float(running_mean[c]) + f * mean);
        running_var[c] = from_float<P>((1.f - f) * to_float(running_var[c]) + f * unbiased);
    }
}

template <typename P>
__global__ void __launch_bounds__(BN_FIN_CH * BN_FIN_LANES)
bn_fwd_finalize_kernel(const float2 *__restrict__ partials, int64_t rows, int channels,
                       const int32_t *__restrict__ num_valid, const P *__restrict__ weight, const P *__restrict__ bias,
                       P *__restrict__ running_mean, P *__restrict__ running_var,
                       const int64_t *__restrict__ num_batches_tracked, float momentum, int cumulative, float eps,
                       float *__restrict__ save_mean, float *__restrict__ save_invstd, float *__restrict__ coef) {
    __shared__ float buf[BN_FIN_LANES][BN_FIN_CH];
    const int cl = threadIdx.x % BN_FIN_CH, pl = threadIdx.x / BN_FIN_CH;
    const int c = blockIdx.x * BN_FIN_CH + cl;
    const bool active = c < channels;
    const int64_t M = valid_rows(num_valid, rows);
    float sum, mean, m2;
    bn_fwd_sums(partials, M, channels, c, active, buf, pl, cl, sum, mean, m2);
    if (pl != 0 || !active) return;
    bn_fwd_write<P>(c, channels, M, mean, m2, weight, bias, running_mean, running_var, num_batches_tracked, momentum,
                    cumulative, eps, save_mean, save_invstd, coef);
}

template <typename T, int W, bool V>
__global__ void __launch_bounds__(BN_THREADS)
bn_fwd_apply_kernel(const T *__restrict__ x, T *__restrict__ y, int64_t rows, int channels, int vecs,
                    const int32_t *__restrict__ num_valid, const float *__restrict__ coef) {
    const int64_t idx = blockIdx.x * (int64_t)BN_THREADS + threadIdx.x;
    const int64_t r = idx / vecs;
    const int v = (int)(idx - r * vecs);
    if (r >= rows) return;
    const int64_t M = valid_rows(num_valid, rows);
    float f[W];
    if (r < M) {
        row_load<T, W, V>(x + r * channels + v * W, f);
#pragma unroll
        for (int j = 0; j < W; ++j) {
            const int c = v * W + j;
            f[j] = fmaf(f[j] - __ldg(coef + c), __ldg(coef + channels + c), __ldg(coef + 2 * channels + c));
        }
    } else {
#pragma unroll
        for (int j = 0; j < W; ++j) f[j] = 0.f;
    }
    row_store<T, W, V>(y + r * channels + v * W, f);
}

// ---------------------------------------------------------------- backward
template <typename T, int W, bool V>
__global__ void __launch_bounds__(BN_THREADS)
bn_bwd_reduce_kernel(const T *__restrict__ x, const T *__restrict__ dy, int64_t rows, int channels, int vecs, int tpr,
                     const int32_t *__restrict__ num_valid, const float *__restrict__ save_mean,
                     const float *__restrict__ save_invstd, float2 *__restrict__ partials) {
    __shared__ float s_a[BN_THREADS * W], s_b[BN_THREADS * W];
    const int64_t M = valid_rows(num_valid, rows);
    const int64_t r0 = (int64_t)blockIdx.x * BN_CHUNK;
    if (r0 >= M) return;
    const int lanes = BN_THREADS / tpr;
    const RowThread t = row_thread(vecs, tpr);
    const int64_t end = M < r0 + BN_CHUNK ? M : r0 + BN_CHUNK;
    float sdy[W], sdyx[W];
#pragma unroll
    for (int j = 0; j < W; ++j) sdy[j] = sdyx[j] = 0.f;
    if (t.active) {
        float mean[W], invstd[W];
#pragma unroll
        for (int j = 0; j < W; ++j) {
            mean[j] = __ldg(save_mean + t.v * W + j);
            invstd[j] = __ldg(save_invstd + t.v * W + j);
        }
        const int64_t off = (int64_t)t.v * W;
        auto fold = [&](const float (&fx)[W], const float (&fd)[W]) {
#pragma unroll
            for (int j = 0; j < W; ++j) {
                sdy[j] += fd[j];
                sdyx[j] = fmaf(fd[j], (fx[j] - mean[j]) * invstd[j], sdyx[j]);
            }
        };
        int64_t r = r0 + t.lane;
        for (; r + lanes < end; r += 2 * lanes) {          // two rows of x and dy in flight
            float fx[2][W], fd[2][W];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int64_t o = (r + (int64_t)u * lanes) * channels + off;
                row_load<T, W, V>(x + o, fx[u]);
                row_load<T, W, V>(dy + o, fd[u]);
            }
#pragma unroll
            for (int u = 0; u < 2; ++u) fold(fx[u], fd[u]);
        }
        for (; r < end; r += lanes) {
            float fx[W], fd[W];
            row_load<T, W, V>(x + r * channels + off, fx);
            row_load<T, W, V>(dy + r * channels + off, fd);
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

// Lane trees of the backward partials: sum(dy) and sum(dy * xhat) over the valid rows.
__device__ __forceinline__ void bn_bwd_sums(const float2 *__restrict__ partials, int64_t M, int channels, int c,
                                            bool active, float (*buf)[BN_FIN_CH], int pl, int cl, float &sdy,
                                            float &sdyx) {
    const int64_t K = (M + BN_CHUNK - 1) / BN_CHUNK;
    float a = 0.f, b = 0.f;
    if (active)
        for (int64_t k = pl; k < K; k += BN_FIN_LANES) {
            const float2 p = partials[k * channels + c];
            a += p.x;
            b += p.y;
        }
    sdy = bn_lane_sum(a, buf, pl, cl);
    sdyx = bn_lane_sum(b, buf, pl, cl);
}

// the dx coefficients of channel c from the sums over a batch of M rows
template <typename P>
__device__ __forceinline__ void bn_bwd_write(int c, int channels, int64_t M, float sdy, float sdyx,
                                             const P *__restrict__ weight, const float *__restrict__ save_invstd,
                                             float *__restrict__ coef) {
    const float Mf = (float)M;
    const float gamma = weight ? to_float(weight[c]) : 1.f;
    coef[c] = gamma * save_invstd[c];
    coef[channels + c] = M > 0 ? __fdiv_rn(sdy, Mf) : 0.f;
    coef[2 * channels + c] = M > 0 ? __fdiv_rn(sdyx, Mf) : 0.f;
}

template <typename P>
__global__ void __launch_bounds__(BN_FIN_CH * BN_FIN_LANES)
bn_bwd_finalize_kernel(const float2 *__restrict__ partials, int64_t rows, int channels,
                       const int32_t *__restrict__ num_valid, const P *__restrict__ weight,
                       const float *__restrict__ save_invstd, P *__restrict__ dweight, P *__restrict__ dbias,
                       float *__restrict__ coef) {
    __shared__ float buf[BN_FIN_LANES][BN_FIN_CH];
    const int cl = threadIdx.x % BN_FIN_CH, pl = threadIdx.x / BN_FIN_CH;
    const int c = blockIdx.x * BN_FIN_CH + cl;
    const bool active = c < channels;
    const int64_t M = valid_rows(num_valid, rows);
    float sdy, sdyx;
    bn_bwd_sums(partials, M, channels, c, active, buf, pl, cl, sdy, sdyx);
    if (pl != 0 || !active) return;
    if (dbias) dbias[c] = from_float<P>(sdy);
    if (dweight) dweight[c] = from_float<P>(sdyx);
    bn_bwd_write<P>(c, channels, M, sdy, sdyx, weight, save_invstd, coef);
}

template <typename T, int W, bool V>
__global__ void __launch_bounds__(BN_THREADS)
bn_bwd_apply_kernel(const T *__restrict__ x, const T *__restrict__ dy, T *__restrict__ dx, int64_t rows, int channels,
                    int vecs, const int32_t *__restrict__ num_valid, const float *__restrict__ save_mean,
                    const float *__restrict__ save_invstd, const float *__restrict__ coef) {
    const int64_t idx = blockIdx.x * (int64_t)BN_THREADS + threadIdx.x;
    const int64_t r = idx / vecs;
    const int v = (int)(idx - r * vecs);
    if (r >= rows) return;
    const int64_t M = valid_rows(num_valid, rows);
    float f[W];
    if (r < M) {
        float fx[W];
        row_load<T, W, V>(x + r * channels + v * W, fx);
        row_load<T, W, V>(dy + r * channels + v * W, f);
#pragma unroll
        for (int j = 0; j < W; ++j) {
            const int c = v * W + j;
            const float xhat = (fx[j] - __ldg(save_mean + c)) * __ldg(save_invstd + c);
            f[j] = __ldg(coef + c) * (f[j] - __ldg(coef + channels + c) - xhat * __ldg(coef + 2 * channels + c));
        }
    } else {
#pragma unroll
        for (int j = 0; j < W; ++j) f[j] = 0.f;
    }
    row_store<T, W, V>(dx + r * channels + v * W, f);
}

// ---------------------------------------------------------------- cross-rank statistics (MaskedSyncBatchNorm1d)
// Each rank reduces its own rows with the kernels above, then a local kernel writes its vector
// [M_r, A_r[C], B_r[C]] (fp32, M_r exact below 2^24).  The vectors of all ranks are gathered in rank order, and a
// merge kernel (one thread per channel) folds them in rank order, the same on every rank:
//   forward : A_r = sum of the rank's rows, B_r = M2 about the rank's own mean A_r / M_r; M = sum of M_r in int64,
//             mean = (sum A_r) / M, M2 = sum [B_r + M_r (A_r / M_r - mean)^2].
//   backward: A_r = sum(dy), B_r = sum(dy * xhat) about the global mean / invstd; the merge sums them.  dweight /
//             dbias are the rank-local A_r / B_r, written by the local kernel.
// One rank: the merge is the finalize above operation for operation (its extra term is M_0 * 0^2 = +0), so the
// results equal MaskedBatchNorm1d bit for bit.  A count that is not a number in [0, 2^24] (a timed-out exchange
// delivers NaN) makes every statistic and coefficient NaN.
constexpr float BN_SYNC_MAX_ROWS = 16777216.f;        // 2^24: every count is an exact fp32 integer

__device__ __forceinline__ void bn_sync_write_local(float *__restrict__ local, int channels, int64_t M, int c,
                                                    bool active, int pl, float a, float b) {
    if (blockIdx.x == 0 && threadIdx.x == 0) local[0] = (float)M;
    if (pl != 0 || !active) return;
    local[1 + c] = a;
    local[1 + channels + c] = b;
}

__global__ void __launch_bounds__(BN_FIN_CH * BN_FIN_LANES)
bn_sync_fwd_local_kernel(const float2 *__restrict__ partials, int64_t rows, int channels,
                         const int32_t *__restrict__ num_valid, float *__restrict__ local) {
    __shared__ float buf[BN_FIN_LANES][BN_FIN_CH];
    const int cl = threadIdx.x % BN_FIN_CH, pl = threadIdx.x / BN_FIN_CH;
    const int c = blockIdx.x * BN_FIN_CH + cl;
    const bool active = c < channels;
    const int64_t M = valid_rows(num_valid, rows);
    float sum, mean, m2;
    bn_fwd_sums(partials, M, channels, c, active, buf, pl, cl, sum, mean, m2);
    bn_sync_write_local(local, channels, M, c, active, pl, sum, m2);
}

// rank-order total of the gathered counts; false when one is not a count
__device__ __forceinline__ bool bn_sync_count(const float *__restrict__ gathered, int world, int64_t stride,
                                              int64_t &M) {
    M = 0;
    bool ok = true;
    for (int r = 0; r < world; ++r) {
        const float n = gathered[r * stride];
        ok = ok && n >= 0.f && n <= BN_SYNC_MAX_ROWS;
        M += ok ? (int64_t)n : 0;
    }
    return ok;
}

template <typename P>
__global__ void __launch_bounds__(BN_THREADS)
bn_sync_fwd_merge_kernel(const float *__restrict__ gathered, int world, int channels, const P *__restrict__ weight,
                         const P *__restrict__ bias, P *__restrict__ running_mean, P *__restrict__ running_var,
                         const int64_t *__restrict__ num_batches_tracked, float momentum, int cumulative, float eps,
                         float *__restrict__ save_mean, float *__restrict__ save_invstd, float *__restrict__ coef) {
    const int c = blockIdx.x * BN_THREADS + threadIdx.x;
    if (c >= channels) return;
    const int64_t stride = 2 * (int64_t)channels + 1;
    int64_t M;
    if (!bn_sync_count(gathered, world, stride, M)) {
        const float nan = __int_as_float(0x7fc00000);
        save_mean[c] = save_invstd[c] = coef[c] = coef[channels + c] = coef[2 * channels + c] = nan;
        if (running_mean != nullptr) running_mean[c] = running_var[c] = from_float<P>(nan);
        return;
    }
    float sum = 0.f;
    for (int r = 0; r < world; ++r) {
        const float a = gathered[r * stride + 1 + c];
        sum = r == 0 ? a : sum + a;
    }
    const float mean = M > 0 ? __fdiv_rn(sum, (float)M) : 0.f;
    float m2 = 0.f;
    for (int r = 0; r < world; ++r) {
        const float *v = gathered + r * stride;
        const float n = v[0];
        const float d = (n > 0.f ? __fdiv_rn(v[1 + c], n) : 0.f) - mean;
        const float t = fmaf(n * d, d, v[1 + channels + c]);
        m2 = r == 0 ? t : m2 + t;
    }
    bn_fwd_write<P>(c, channels, M, mean, m2, weight, bias, running_mean, running_var, num_batches_tracked, momentum,
                    cumulative, eps, save_mean, save_invstd, coef);
}

template <typename P>
__global__ void __launch_bounds__(BN_FIN_CH * BN_FIN_LANES)
bn_sync_bwd_local_kernel(const float2 *__restrict__ partials, int64_t rows, int channels,
                         const int32_t *__restrict__ num_valid, P *__restrict__ dweight, P *__restrict__ dbias,
                         float *__restrict__ local) {
    __shared__ float buf[BN_FIN_LANES][BN_FIN_CH];
    const int cl = threadIdx.x % BN_FIN_CH, pl = threadIdx.x / BN_FIN_CH;
    const int c = blockIdx.x * BN_FIN_CH + cl;
    const bool active = c < channels;
    const int64_t M = valid_rows(num_valid, rows);
    float sdy, sdyx;
    bn_bwd_sums(partials, M, channels, c, active, buf, pl, cl, sdy, sdyx);
    if (pl == 0 && active) {
        if (dbias) dbias[c] = from_float<P>(sdy);
        if (dweight) dweight[c] = from_float<P>(sdyx);
    }
    bn_sync_write_local(local, channels, M, c, active, pl, sdy, sdyx);
}

template <typename P>
__global__ void __launch_bounds__(BN_THREADS)
bn_sync_bwd_merge_kernel(const float *__restrict__ gathered, int world, int channels, const P *__restrict__ weight,
                         const float *__restrict__ save_invstd, float *__restrict__ coef) {
    const int c = blockIdx.x * BN_THREADS + threadIdx.x;
    if (c >= channels) return;
    const int64_t stride = 2 * (int64_t)channels + 1;
    int64_t M;
    if (!bn_sync_count(gathered, world, stride, M)) {
        coef[c] = coef[channels + c] = coef[2 * channels + c] = __int_as_float(0x7fc00000);
        return;
    }
    float sdy = 0.f, sdyx = 0.f;
    for (int r = 0; r < world; ++r) {
        const float a = gathered[r * stride + 1 + c], b = gathered[r * stride + 1 + channels + c];
        sdy = r == 0 ? a : sdy + a;
        sdyx = r == 0 ? b : sdyx + b;
    }
    bn_bwd_write<P>(c, channels, M, sdy, sdyx, weight, save_invstd, coef);
}

// ---------------------------------------------------------------- host side
static int64_t bn_chunks(int64_t rows) { return (rows + BN_CHUNK - 1) / BN_CHUNK; }

static size_t bn_workspace(int64_t rows, int channels, int coefs) {
    if (rows < 0 || channels < 1) return 0;
    return align_up((size_t)bn_chunks(rows) * channels * sizeof(float2), 256) + align_up((size_t)coefs * channels * 4, 256);
}

static bool bn_float_dtype(int dt) { return dt == SPX_F32 || dt == SPX_F16 || dt == SPX_BF16; }

static int bn_check(const char *who, int64_t rows, int channels, int dtype, int param_dtype) {
    SPX_REQUIRE(rows >= 0 && rows < 2147483647ll, "%s: bad row count %lld", who, (long long)rows);
    SPX_REQUIRE(channels >= 1 && channels <= (1 << 20), "%s: channels must be in [1, 2^20], got %d", who, channels);
    SPX_REQUIRE(bn_float_dtype(dtype), "%s: unsupported dtype %d (float32, float16 and bfloat16 only)", who, dtype);
    SPX_REQUIRE(param_dtype == SPX_F32 || param_dtype == dtype,
                "%s: parameter dtype %d must be float32 or the feature dtype %d", who, param_dtype, dtype);
    return 0;
}

struct BnFwdArgs {
    const void *x;
    void *y;
    int64_t rows;
    int channels;
    const int32_t *num_valid;
    const void *weight, *bias;
    void *running_mean, *running_var;
    const int64_t *nbt;
    float momentum;
    int cumulative;
    float eps;
    float *save_mean, *save_invstd;
    float2 *partials;
    float *coef;
};

template <typename T, int W, bool V> static int bn_fwd_rows(const BnFwdArgs &a, bool stats, cudaStream_t stream) {
    const int vecs = a.channels / W;
    if (stats) {
        const int tpr = row_tpr(vecs);
        const dim3 grid((unsigned)bn_chunks(a.rows), (unsigned)div_up64(vecs, tpr));
        bn_stats_kernel<T, W, V><<<grid, BN_THREADS, 0, stream>>>(static_cast<const T *>(a.x), a.rows, a.channels, vecs,
                                                               tpr, a.num_valid, a.partials);
        SPX_CHECK_LAUNCH("bn_stats_kernel");
    } else {
        bn_fwd_apply_kernel<T, W, V><<<(unsigned)div_up64(a.rows * vecs, BN_THREADS), BN_THREADS, 0, stream>>>(
            static_cast<const T *>(a.x), static_cast<T *>(a.y), a.rows, a.channels, vecs, a.num_valid, a.coef);
        SPX_CHECK_LAUNCH("bn_fwd_apply_kernel");
    }
    return 0;
}

static int bn_fwd_rows_typed(int dtype, const BnFwdArgs &a, bool stats, cudaStream_t stream) {
    return dispatch_dtype(dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        constexpr int W = 16 / sizeof(T);
        const RowWidth w = row_width(a.channels * sizeof(T), a.x, a.y);   // a reduction: W whenever wide
        if (!w.wide) return bn_fwd_rows<T, 1, false>(a, stats, stream);
        return w.aligned ? bn_fwd_rows<T, W, true>(a, stats, stream) : bn_fwd_rows<T, W, false>(a, stats, stream);
    });
}

template <typename P> static int bn_fwd_finalize(const BnFwdArgs &a, cudaStream_t stream) {
    bn_fwd_finalize_kernel<P><<<(unsigned)div_up64(a.channels, BN_FIN_CH), BN_FIN_CH * BN_FIN_LANES, 0, stream>>>(
        a.partials, a.rows, a.channels, a.num_valid, static_cast<const P *>(a.weight), static_cast<const P *>(a.bias),
        static_cast<P *>(a.running_mean), static_cast<P *>(a.running_var), a.nbt, a.momentum, a.cumulative, a.eps,
        a.save_mean, a.save_invstd, a.coef);
    SPX_CHECK_LAUNCH("bn_fwd_finalize_kernel");
    return 0;
}

struct BnBwdArgs {
    const void *x, *dy;
    void *dx;
    int64_t rows;
    int channels;
    const int32_t *num_valid;
    const void *weight;
    const float *save_mean, *save_invstd;
    void *dweight, *dbias;
    float2 *partials;
    float *coef;
};

template <typename T, int W, bool V> static int bn_bwd_rows(const BnBwdArgs &a, bool reduce, cudaStream_t stream) {
    const int vecs = a.channels / W;
    if (reduce) {
        const int tpr = row_tpr(vecs);
        const dim3 grid((unsigned)bn_chunks(a.rows), (unsigned)div_up64(vecs, tpr));
        bn_bwd_reduce_kernel<T, W, V><<<grid, BN_THREADS, 0, stream>>>(
            static_cast<const T *>(a.x), static_cast<const T *>(a.dy), a.rows, a.channels, vecs, tpr, a.num_valid,
            a.save_mean, a.save_invstd, a.partials);
        SPX_CHECK_LAUNCH("bn_bwd_reduce_kernel");
    } else {
        bn_bwd_apply_kernel<T, W, V><<<(unsigned)div_up64(a.rows * vecs, BN_THREADS), BN_THREADS, 0, stream>>>(
            static_cast<const T *>(a.x), static_cast<const T *>(a.dy), static_cast<T *>(a.dx), a.rows, a.channels, vecs,
            a.num_valid, a.save_mean, a.save_invstd, a.coef);
        SPX_CHECK_LAUNCH("bn_bwd_apply_kernel");
    }
    return 0;
}

static int bn_bwd_rows_typed(int dtype, const BnBwdArgs &a, bool reduce, cudaStream_t stream) {
    return dispatch_dtype(dtype, [&](auto t) {
        using T = typename decltype(t)::type;
        constexpr int W = 16 / sizeof(T);
        const RowWidth w = row_width(a.channels * sizeof(T), a.x, a.dy, a.dx);   // a reduction: W whenever wide
        if (!w.wide) return bn_bwd_rows<T, 1, false>(a, reduce, stream);
        return w.aligned ? bn_bwd_rows<T, W, true>(a, reduce, stream) : bn_bwd_rows<T, W, false>(a, reduce, stream);
    });
}

template <typename P> static int bn_bwd_finalize(const BnBwdArgs &a, cudaStream_t stream) {
    bn_bwd_finalize_kernel<P><<<(unsigned)div_up64(a.channels, BN_FIN_CH), BN_FIN_CH * BN_FIN_LANES, 0, stream>>>(
        a.partials, a.rows, a.channels, a.num_valid, static_cast<const P *>(a.weight), a.save_invstd,
        static_cast<P *>(a.dweight), static_cast<P *>(a.dbias), a.coef);
    SPX_CHECK_LAUNCH("bn_bwd_finalize_kernel");
    return 0;
}

}  // namespace spx

using namespace spx;

extern "C" size_t spx_masked_bn_fwd_train_workspace_size(int64_t rows, int channels) {
    return bn_workspace(rows, channels, 3);
}

extern "C" size_t spx_masked_bn_bwd_workspace_size(int64_t rows, int channels) {
    return bn_workspace(rows, channels, 3);
}

extern "C" int spx_masked_bn_fwd_train(const void *x, void *y, int64_t rows, int channels, int dtype,
                                       const int32_t *num_valid, const void *weight, const void *bias,
                                       void *running_mean, void *running_var, const int64_t *num_batches_tracked,
                                       int param_dtype, float momentum, int cumulative, float eps, float *save_mean,
                                       float *save_invstd, void *workspace, size_t workspace_bytes,
                                       spx_stream_t stream_) {
    const char *who = "masked_bn_fwd_train";
    if (int rc = bn_check(who, rows, channels, dtype, param_dtype)) return rc;
    SPX_REQUIRE(save_mean && save_invstd && workspace, "%s: NULL pointer argument (save_mean, save_invstd, workspace)",
                who);
    SPX_REQUIRE(rows == 0 || (x && y), "%s: NULL pointer argument (x, y)", who);
    SPX_REQUIRE((running_mean == nullptr) == (running_var == nullptr),
                "%s: running_mean and running_var must both be given or both be NULL", who);
    SPX_REQUIRE(!(running_mean && cumulative && num_batches_tracked == nullptr),
                "%s: a cumulative average (momentum None) needs num_batches_tracked", who);
    SPX_REQUIRE(eps > 0.f, "%s: eps must be positive", who);
    const size_t need = spx_masked_bn_fwd_train_workspace_size(rows, channels);
    SPX_REQUIRE(workspace_bytes >= need, "%s: workspace too small: need %zu, have %zu", who, need, workspace_bytes);
    WorkspaceCarver ws(workspace, workspace_bytes);
    BnFwdArgs a{x, y, rows, channels, num_valid, weight, bias, running_mean, running_var, num_batches_tracked,
                momentum, cumulative, eps, save_mean, save_invstd, nullptr, nullptr};
    a.partials = ws.take<float2>((size_t)bn_chunks(rows) * channels);
    a.coef = ws.take<float>((size_t)3 * channels);
    cudaStream_t stream = (cudaStream_t)stream_;
    if (rows > 0)
        if (int rc = bn_fwd_rows_typed(dtype, a, true, stream)) return rc;
    const int rc =
        dispatch_dtype(param_dtype, [&](auto p) { return bn_fwd_finalize<typename decltype(p)::type>(a, stream); });
    if (rc || rows == 0) return rc;
    return bn_fwd_rows_typed(dtype, a, false, stream);
}

extern "C" int spx_masked_bn_bwd(const void *x, const void *dy, void *dx, int64_t rows, int channels, int dtype,
                                 const int32_t *num_valid, const void *weight, int param_dtype, const float *save_mean,
                                 const float *save_invstd, void *dweight, void *dbias, void *workspace,
                                 size_t workspace_bytes, spx_stream_t stream_) {
    const char *who = "masked_bn_bwd";
    if (int rc = bn_check(who, rows, channels, dtype, param_dtype)) return rc;
    SPX_REQUIRE(save_mean && save_invstd && workspace, "%s: NULL pointer argument (save_mean, save_invstd, workspace)",
                who);
    SPX_REQUIRE(rows == 0 || (x && dy && dx), "%s: NULL pointer argument (x, dy, dx)", who);
    const size_t need = spx_masked_bn_bwd_workspace_size(rows, channels);
    SPX_REQUIRE(workspace_bytes >= need, "%s: workspace too small: need %zu, have %zu", who, need, workspace_bytes);
    WorkspaceCarver ws(workspace, workspace_bytes);
    BnBwdArgs a{x, dy, dx, rows, channels, num_valid, weight, save_mean, save_invstd, dweight, dbias, nullptr, nullptr};
    a.partials = ws.take<float2>((size_t)bn_chunks(rows) * channels);
    a.coef = ws.take<float>((size_t)3 * channels);
    cudaStream_t stream = (cudaStream_t)stream_;
    if (rows > 0)
        if (int rc = bn_bwd_rows_typed(dtype, a, true, stream)) return rc;
    const int rc =
        dispatch_dtype(param_dtype, [&](auto p) { return bn_bwd_finalize<typename decltype(p)::type>(a, stream); });
    if (rc || rows == 0) return rc;
    return bn_bwd_rows_typed(dtype, a, false, stream);
}

// ---------------------------------------------------------------- cross-rank BatchNorm (MaskedSyncBatchNorm1d)
namespace spx {

static int bn_sync_check(const char *who, const spx_masked_sync_bn *d, bool merge, size_t workspace_bytes,
                         const void *workspace) {
    SPX_REQUIRE(d != nullptr, "%s: descriptor is NULL", who);
    if (int rc = bn_check(who, d->rows, d->channels, d->dtype, d->param_dtype)) return rc;
    SPX_REQUIRE(d->rows <= (1 << 24), "%s: %lld rows, at most 2^24 per rank and call", who, (long long)d->rows);
    SPX_REQUIRE(workspace != nullptr, "%s: NULL pointer argument (workspace)", who);
    const size_t need = spx_masked_sync_bn_workspace_size(d->rows, d->channels);
    SPX_REQUIRE(workspace_bytes >= need, "%s: workspace too small: need %zu, have %zu", who, need, workspace_bytes);
    if (merge) {
        SPX_REQUIRE(d->world >= 1 && d->world <= SPX_MAX_PEERS, "%s: world %d out of range (1..%d)", who, d->world,
                    SPX_MAX_PEERS);
        SPX_REQUIRE(d->gathered != nullptr, "%s: NULL pointer argument (gathered)", who);
    } else {
        SPX_REQUIRE(d->local != nullptr, "%s: NULL pointer argument (local)", who);
    }
    return 0;
}

static BnFwdArgs bn_sync_fwd_args(const spx_masked_sync_bn *d, void *workspace, size_t workspace_bytes) {
    BnFwdArgs a{d->x, d->y, d->rows, d->channels, d->num_valid, d->weight, d->bias, d->running_mean,
                d->running_var, d->num_batches_tracked, d->momentum, d->cumulative, d->eps, d->save_mean,
                d->save_invstd, nullptr, nullptr};
    WorkspaceCarver ws(workspace, workspace_bytes);
    a.partials = ws.take<float2>((size_t)bn_chunks(d->rows) * d->channels);
    a.coef = ws.take<float>((size_t)3 * d->channels);
    return a;
}

static BnBwdArgs bn_sync_bwd_args(const spx_masked_sync_bn *d, void *workspace, size_t workspace_bytes) {
    BnBwdArgs a{d->x, d->dy, d->dx, d->rows, d->channels, d->num_valid, d->weight, d->save_mean, d->save_invstd,
                d->dweight, d->dbias, nullptr, nullptr};
    WorkspaceCarver ws(workspace, workspace_bytes);
    a.partials = ws.take<float2>((size_t)bn_chunks(d->rows) * d->channels);
    a.coef = ws.take<float>((size_t)3 * d->channels);
    return a;
}

static unsigned bn_fin_blocks(int channels) { return (unsigned)div_up64(channels, BN_FIN_CH); }
static unsigned bn_merge_blocks(int channels) { return (unsigned)div_up64(channels, BN_THREADS); }

template <typename P> static int bn_sync_fwd_merge(const spx_masked_sync_bn *d, const BnFwdArgs &a, cudaStream_t stream) {
    bn_sync_fwd_merge_kernel<P><<<bn_merge_blocks(a.channels), BN_THREADS, 0, stream>>>(
        d->gathered, d->world, a.channels, static_cast<const P *>(a.weight), static_cast<const P *>(a.bias),
        static_cast<P *>(a.running_mean), static_cast<P *>(a.running_var), a.nbt, a.momentum, a.cumulative, a.eps,
        a.save_mean, a.save_invstd, a.coef);
    SPX_CHECK_LAUNCH("bn_sync_fwd_merge_kernel");
    return 0;
}

template <typename P> static int bn_sync_bwd_local(const spx_masked_sync_bn *d, const BnBwdArgs &a, cudaStream_t stream) {
    bn_sync_bwd_local_kernel<P><<<bn_fin_blocks(a.channels), BN_FIN_CH * BN_FIN_LANES, 0, stream>>>(
        a.partials, a.rows, a.channels, a.num_valid, static_cast<P *>(a.dweight), static_cast<P *>(a.dbias), d->local);
    SPX_CHECK_LAUNCH("bn_sync_bwd_local_kernel");
    return 0;
}

template <typename P> static int bn_sync_bwd_merge(const spx_masked_sync_bn *d, const BnBwdArgs &a, cudaStream_t stream) {
    bn_sync_bwd_merge_kernel<P><<<bn_merge_blocks(a.channels), BN_THREADS, 0, stream>>>(
        d->gathered, d->world, a.channels, static_cast<const P *>(a.weight), a.save_invstd, a.coef);
    SPX_CHECK_LAUNCH("bn_sync_bwd_merge_kernel");
    return 0;
}

}  // namespace spx

extern "C" size_t spx_masked_sync_bn_workspace_size(int64_t rows, int channels) {
    return bn_workspace(rows, channels, 3);
}

extern "C" int spx_masked_sync_bn_fwd_local(const spx_masked_sync_bn *d, void *workspace, size_t workspace_bytes,
                                            spx_stream_t stream_) {
    const char *who = "masked_sync_bn_fwd_local";
    if (int rc = bn_sync_check(who, d, false, workspace_bytes, workspace)) return rc;
    SPX_REQUIRE(d->rows == 0 || d->x, "%s: NULL pointer argument (x)", who);
    const BnFwdArgs a = bn_sync_fwd_args(d, workspace, workspace_bytes);
    cudaStream_t stream = (cudaStream_t)stream_;
    if (d->rows > 0)
        if (int rc = bn_fwd_rows_typed(d->dtype, a, true, stream)) return rc;
    bn_sync_fwd_local_kernel<<<bn_fin_blocks(a.channels), BN_FIN_CH * BN_FIN_LANES, 0, stream>>>(
        a.partials, a.rows, a.channels, a.num_valid, d->local);
    SPX_CHECK_LAUNCH("bn_sync_fwd_local_kernel");
    return 0;
}

extern "C" int spx_masked_sync_bn_fwd_merge(const spx_masked_sync_bn *d, void *workspace, size_t workspace_bytes,
                                            spx_stream_t stream_) {
    const char *who = "masked_sync_bn_fwd_merge";
    if (int rc = bn_sync_check(who, d, true, workspace_bytes, workspace)) return rc;
    SPX_REQUIRE(d->save_mean && d->save_invstd, "%s: NULL pointer argument (save_mean, save_invstd)", who);
    SPX_REQUIRE(d->rows == 0 || (d->x && d->y), "%s: NULL pointer argument (x, y)", who);
    SPX_REQUIRE((d->running_mean == nullptr) == (d->running_var == nullptr),
                "%s: running_mean and running_var must both be given or both be NULL", who);
    SPX_REQUIRE(!(d->running_mean && d->cumulative && d->num_batches_tracked == nullptr),
                "%s: a cumulative average (momentum None) needs num_batches_tracked", who);
    SPX_REQUIRE(d->eps > 0.f, "%s: eps must be positive", who);
    const BnFwdArgs a = bn_sync_fwd_args(d, workspace, workspace_bytes);
    cudaStream_t stream = (cudaStream_t)stream_;
    const int rc = dispatch_dtype(d->param_dtype,
                                  [&](auto p) { return bn_sync_fwd_merge<typename decltype(p)::type>(d, a, stream); });
    if (rc || d->rows == 0) return rc;
    return bn_fwd_rows_typed(d->dtype, a, false, stream);
}

extern "C" int spx_masked_sync_bn_bwd_local(const spx_masked_sync_bn *d, void *workspace, size_t workspace_bytes,
                                            spx_stream_t stream_) {
    const char *who = "masked_sync_bn_bwd_local";
    if (int rc = bn_sync_check(who, d, false, workspace_bytes, workspace)) return rc;
    SPX_REQUIRE(d->save_mean && d->save_invstd, "%s: NULL pointer argument (save_mean, save_invstd)", who);
    SPX_REQUIRE(d->rows == 0 || (d->x && d->dy), "%s: NULL pointer argument (x, dy)", who);
    const BnBwdArgs a = bn_sync_bwd_args(d, workspace, workspace_bytes);
    cudaStream_t stream = (cudaStream_t)stream_;
    if (d->rows > 0)
        if (int rc = bn_bwd_rows_typed(d->dtype, a, true, stream)) return rc;
    return dispatch_dtype(d->param_dtype,
                          [&](auto p) { return bn_sync_bwd_local<typename decltype(p)::type>(d, a, stream); });
}

extern "C" int spx_masked_sync_bn_bwd_merge(const spx_masked_sync_bn *d, void *workspace, size_t workspace_bytes,
                                            spx_stream_t stream_) {
    const char *who = "masked_sync_bn_bwd_merge";
    if (int rc = bn_sync_check(who, d, true, workspace_bytes, workspace)) return rc;
    SPX_REQUIRE(d->save_mean && d->save_invstd, "%s: NULL pointer argument (save_mean, save_invstd)", who);
    SPX_REQUIRE(d->rows == 0 || (d->x && d->dy && d->dx), "%s: NULL pointer argument (x, dy, dx)", who);
    const BnBwdArgs a = bn_sync_bwd_args(d, workspace, workspace_bytes);
    cudaStream_t stream = (cudaStream_t)stream_;
    const int rc = dispatch_dtype(d->param_dtype,
                                  [&](auto p) { return bn_sync_bwd_merge<typename decltype(p)::type>(d, a, stream); });
    if (rc || d->rows == 0) return rc;
    return bn_bwd_rows_typed(d->dtype, a, false, stream);
}
