// Stable LSD radix argsort of the 32-bit neighbour masks (one mask word, kv <= 32).
//
// Reference: thrust::sort_by_key on the masks with an iota payload
// (spconv/csrc/sparse/all.py:935-1000).  For the rulebook sizes of this path (1e5..1e6 keys) a
// library radix sort is launch/latency-bound: CUB's onesweep pays a launch-bound pass per 8 bits
// plus histogram/scan kernels.  This version uses 9-bit
// digits (3 passes for the 27-bit masks of a 3x3x3 kernel instead of 4) and two small kernels per
// pass:
//   hist    : (first pass only) per-block digit histogram -> counts[digit][block]
//   scan    : one block per digit: exclusive prefix over blocks + digit totals; also clears the
//             histogram buffer of the NEXT pass
//   scatter : ranks its keys stably with warp match_any, scatters them, and accumulates the next
//             pass's per-block histogram keyed by the destination block (destination positions are
//             known here, so no later pass re-reads keys to count): merged per block in shared
//             memory, then one global atomic per distinct (digit, block) cell.
// The first pass reads the masks with an implicit iota payload, the last pass writes the sorted
// masks back in place (thrust semantics) and the argsort.  Also the host helpers of segments.cuh.
#include "segments.cuh"
#include <cub/cub.cuh>

namespace spx {

constexpr int RS_BITS = 9;
constexpr int RS_BINS = 1 << RS_BITS;
constexpr int RS_THREADS = 256;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_ITEMS = 4;                        // keys per thread
constexpr int RS_TILE = RS_THREADS * RS_ITEMS;     // keys per block
constexpr int RS_AGG_BITS = 11;
constexpr int RS_AGG_SLOTS = 1 << RS_AGG_BITS;     // shared-memory merge table, 2x the keys of a block
constexpr int RS_TILE_SHIFT = 10;
static_assert((1 << RS_TILE_SHIFT) == RS_TILE, "tile shift");

// One launch serves up to two independent sorts (blockIdx.y picks the job): a regular conv sorts its
// forward masks (M outputs) and its backward masks (N inputs) -- at rulebook sizes every kernel here is
// latency-bound, so two jobs in one launch cost about as much as one.
struct RsJob {
    const uint32_t *kin; const int32_t *vin;
    int64_t n; int nblk;
    int *counts; int *totals;
    uint32_t *kout; int32_t *vout;
    int *counts_next;
};
struct RsJobs { RsJob j[2]; };

__global__ void __launch_bounds__(RS_THREADS)
rs_hist_kernel(const RsJobs jobs, int shift) {
    const RsJob &J = jobs.j[blockIdx.y];
    if ((int)blockIdx.x >= J.nblk) return;
    const uint32_t *__restrict__ keys = J.kin;
    const int64_t n = J.n;
    const int nblk = J.nblk;
    int *__restrict__ counts = J.counts;
    __shared__ int hist[RS_BINS];
    for (int i = threadIdx.x; i < RS_BINS; i += RS_THREADS) hist[i] = 0;
    __syncthreads();
    const int64_t base = (int64_t)blockIdx.x * RS_TILE;
#pragma unroll
    for (int j = 0; j < RS_ITEMS; ++j) {
        const int64_t i = base + j * RS_THREADS + threadIdx.x;
        if (i < n) atomicAdd(&hist[(keys[i] >> shift) & (RS_BINS - 1)], 1);
    }
    __syncthreads();
    // digit-major [digit][block]: each scan block walks one contiguous row
    for (int d = threadIdx.x; d < RS_BINS; d += RS_THREADS) counts[(int64_t)d * nblk + blockIdx.x] = hist[d];
}

// counts[d][b] -> exclusive prefix over b, totals[d] = sum_b; zeroes row d of the next pass's buffer
__global__ void __launch_bounds__(RS_THREADS)
rs_scan_kernel(const RsJobs jobs) {
    const RsJob &J = jobs.j[blockIdx.y];
    int *__restrict__ counts = J.counts;
    const int nblk = J.nblk;
    int *__restrict__ totals = J.totals;
    int *__restrict__ clear_next = J.counts_next;
    if (nblk == 0) return;
    const int d = blockIdx.x;
    if (clear_next)
        for (int b = threadIdx.x; b < nblk; b += RS_THREADS) clear_next[(int64_t)d * nblk + b] = 0;
    __shared__ int warp_sums[RS_WARPS];
    __shared__ int carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int b0 = 0; b0 < nblk; b0 += RS_THREADS) {
        const int b = b0 + threadIdx.x;
        const int v = b < nblk ? counts[(int64_t)d * nblk + b] : 0;
        int incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) warp_sums[warp] = incl;
        __syncthreads();
        int wbase = 0;
        for (int w = 0; w < warp; ++w) wbase += warp_sums[w];
        const int carry = carry_s;
        if (b < nblk) counts[(int64_t)d * nblk + b] = carry + wbase + incl - v;
        __syncthreads();
        if (threadIdx.x == RS_THREADS - 1) carry_s = carry + wbase + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) totals[d] = carry_s;
}

// counts hold block prefixes (rs_scan_kernel); counts_next (may be null) receives the next pass's histogram
template <bool IOTA_IN>
__global__ void __launch_bounds__(RS_THREADS)
rs_scatter_kernel(const RsJobs jobs, int shift) {
    const RsJob &J = jobs.j[blockIdx.y];
    if ((int)blockIdx.x >= J.nblk) return;
    const uint32_t *__restrict__ keys_in = J.kin;
    const int32_t *__restrict__ vals_in = J.vin;
    const int64_t n = J.n;
    const int nblk = J.nblk;
    const int *__restrict__ counts = J.counts;
    const int *__restrict__ totals = J.totals;
    uint32_t *__restrict__ keys_out = J.kout;
    int32_t *__restrict__ vals_out = J.vout;
    int *__restrict__ counts_next = J.counts_next;
    __shared__ int digit_base[RS_BINS];             // global position of this block's first key of each digit
    __shared__ int warp_cnt[RS_WARPS][RS_BINS];     // running per-warp digit counts -> warp bases
    __shared__ int scan_tmp[RS_WARPS];
    __shared__ int agg_cell[RS_AGG_SLOTS], agg_cnt[RS_AGG_SLOTS];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int blk = blockIdx.x;
    for (int i = tid; i < RS_AGG_SLOTS; i += RS_THREADS) { agg_cell[i] = -1; agg_cnt[i] = 0; }

    // ---- (1) per-digit: total over all blocks and the part before this block
    int my_total[RS_BINS / RS_THREADS], my_before[RS_BINS / RS_THREADS];
#pragma unroll
    for (int q = 0; q < RS_BINS / RS_THREADS; ++q) {
        const int d = q * RS_THREADS + tid;
        my_total[q] = __ldg(totals + d);
        my_before[q] = __ldg(counts + (int64_t)d * nblk + blk);
    }
    for (int i = tid; i < RS_WARPS * RS_BINS; i += RS_THREADS) (&warp_cnt[0][0])[i] = 0;
    // exclusive scan of the 512 digit totals (digit d = q*256 + tid; q-major order keeps d ascending)
    int run = 0;
#pragma unroll
    for (int q = 0; q < RS_BINS / RS_THREADS; ++q) {
        int v = my_total[q], incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) scan_tmp[warp] = incl;
        __syncthreads();
        int wbase = 0, all = 0;
        for (int w = 0; w < RS_WARPS; ++w) { if (w < warp) wbase += scan_tmp[w]; all += scan_tmp[w]; }
        digit_base[q * RS_THREADS + tid] = run + wbase + incl - v + my_before[q];
        run += all;
        __syncthreads();
    }

    // ---- (2) stable rank inside the block: warp w owns keys [w*128, w*128+128) of the tile, 4 rounds of 32
    const int64_t tile_base = (int64_t)blk * RS_TILE + warp * (32 * RS_ITEMS);
    uint32_t key[RS_ITEMS];
    int32_t val[RS_ITEMS];
    int rank[RS_ITEMS];
#pragma unroll
    for (int r = 0; r < RS_ITEMS; ++r) {
        const int64_t i = tile_base + r * 32 + lane;
        const bool ok = i < n;
        key[r] = ok ? keys_in[i] : 0xffffffffu;
        val[r] = ok ? (IOTA_IN ? (int32_t)i : vals_in[i]) : -1;
        const int d = ok ? (int)((key[r] >> shift) & (RS_BINS - 1)) : RS_BINS;   // RS_BINS = "no key"
        const unsigned peers = __match_any_sync(0xffffffffu, d);
        const int leader = __ffs(peers) - 1;
        int old = 0;
        if (ok && lane == leader) { old = warp_cnt[warp][d]; warp_cnt[warp][d] = old + __popc(peers); }
        old = __shfl_sync(0xffffffffu, old, leader);
        rank[r] = old + __popc(peers & ((1u << lane) - 1u));
        __syncwarp();
    }
    __syncthreads();
    // ---- (3) warp bases: exclusive scan over warps per digit (in place)
    for (int d = tid; d < RS_BINS; d += RS_THREADS) {
        int acc = 0;
#pragma unroll
        for (int w = 0; w < RS_WARPS; ++w) { const int c = warp_cnt[w][d]; warp_cnt[w][d] = acc; acc += c; }
    }
    __syncthreads();
    // ---- (4) scatter (+ next pass's histogram, keyed by the destination block).  The cells
    //      (next digit, destination block) hit by one block are few when either digit is skewed
    //      (3x3x3 masks: the dz = +-1 planes are mostly empty), and all blocks would hammer the
    //      same handful of global counters; they are first merged in a small shared-memory
    //      open-addressing table and flushed with one global atomic per distinct cell.
#pragma unroll
    for (int r = 0; r < RS_ITEMS; ++r) {
        const int64_t i = tile_base + r * 32 + lane;
        if (i < n) {
            const int d = (int)((key[r] >> shift) & (RS_BINS - 1));
            const int pos = digit_base[d] + warp_cnt[warp][d] + rank[r];
            keys_out[pos] = key[r];
            vals_out[pos] = val[r];
            if (counts_next) {
                const int dn = (int)((key[r] >> (shift + RS_BITS)) & (RS_BINS - 1));
                const int cell = dn * nblk + (pos >> RS_TILE_SHIFT);
                uint32_t slot = ((uint32_t)cell * 2654435761u) >> (32 - RS_AGG_BITS);
                while (true) {
                    const int prev = atomicCAS(&agg_cell[slot], -1, cell);
                    if (prev == -1 || prev == cell) { atomicAdd(&agg_cnt[slot], 1); break; }
                    slot = (slot + 1) & (RS_AGG_SLOTS - 1);        // <= 1024 cells in 2048 slots: terminates
                }
            }
        }
    }
    if (counts_next) {
        __syncthreads();
        for (int s2 = tid; s2 < RS_AGG_SLOTS; s2 += RS_THREADS)
            if (agg_cell[s2] >= 0) atomicAdd(counts_next + agg_cell[s2], agg_cnt[s2]);
    }
}

size_t radix_argsort_workspace_bytes(int64_t n) {
    const int64_t nblk = div_up64(n > 0 ? n : 1, RS_TILE);
    // the layout of rs_carve: keys / values double buffers, 2 count matrices, digit totals
    return 4 * align_up((size_t)n * 4, 256) + 2 * align_up((size_t)RS_BINS * nblk * 4, 256) +
           align_up(RS_BINS * 4, 256) + 1024;
}

namespace {
struct RsPlan {
    uint32_t *keys_a, *keys_b; int32_t *vals_a, *vals_b;
    int *counts_ab[2]; int *totals;
    int nblk;
};
int rs_carve(int64_t n, void *workspace, size_t bytes, RsPlan &p) {
    WorkspaceCarver ws(workspace, bytes);
    p.keys_a = ws.take<uint32_t>(n); p.vals_a = ws.take<int32_t>(n);
    p.keys_b = ws.take<uint32_t>(n); p.vals_b = ws.take<int32_t>(n);
    p.nblk = (int)div_up64(n, RS_TILE);
    p.counts_ab[0] = ws.take<int>((size_t)RS_BINS * p.nblk);
    p.counts_ab[1] = ws.take<int>((size_t)RS_BINS * p.nblk);
    p.totals = ws.take<int>(RS_BINS);
    SPX_REQUIRE(ws.ok(), "argsort workspace too small: need %zu, have %zu", ws.off, bytes);
    return 0;
}
}  // namespace

// Two-kernel-per-pass LSD sort of one or two independent key arrays with the same key width (n1 == 0: one job).
int radix_argsort_pair(uint32_t *mask0, int32_t *argsort0, int64_t n0, uint32_t *mask1, int32_t *argsort1, int64_t n1,
                       int key_bits, void *ws0, size_t ws0_bytes, void *ws1, size_t ws1_bytes, cudaStream_t stream) {
    if (n0 == 0 && n1 == 0) return 0;
    if (n0 == 0) return radix_argsort_pair(mask1, argsort1, n1, nullptr, nullptr, 0, key_bits, ws1, ws1_bytes, nullptr, 0, stream);
    if (key_bits < 1) key_bits = 1;
    if (key_bits > 32) key_bits = 32;
    const int passes = (key_bits + RS_BITS - 1) / RS_BITS;
    const int njobs = n1 > 0 ? 2 : 1;
    RsPlan pl[2];
    uint32_t *masks[2] = {mask0, mask1};
    int32_t *argsorts[2] = {argsort0, argsort1};
    const int64_t ns[2] = {n0, n1};
    if (int rc = rs_carve(n0, ws0, ws0_bytes, pl[0])) return rc;
    if (njobs == 2) if (int rc = rs_carve(n1, ws1, ws1_bytes, pl[1])) return rc;
    RsJobs jobs;
    memset(&jobs, 0, sizeof(jobs));
    int max_nblk = 0;
    for (int q = 0; q < njobs; ++q) {
        jobs.j[q].kin = masks[q]; jobs.j[q].vin = nullptr; jobs.j[q].n = ns[q]; jobs.j[q].nblk = pl[q].nblk;
        jobs.j[q].totals = pl[q].totals;
        if (pl[q].nblk > max_nblk) max_nblk = pl[q].nblk;
    }
    const dim3 grid_tiles(max_nblk, njobs), grid_scan(RS_BINS, njobs);
    for (int q = 0; q < njobs; ++q) jobs.j[q].counts = pl[q].counts_ab[0];
    rs_hist_kernel<<<grid_tiles, RS_THREADS, 0, stream>>>(jobs, 0);
    SPX_CHECK_LAUNCH("rs_hist_kernel");
    for (int pass = 0; pass < passes; ++pass) {
        const bool last = pass == passes - 1;
        for (int q = 0; q < njobs; ++q) {
            RsJob &J = jobs.j[q];
            J.kout = (pass & 1) ? pl[q].keys_b : pl[q].keys_a;
            J.vout = (pass & 1) ? pl[q].vals_b : pl[q].vals_a;
            if (last && pass > 0) { J.kout = masks[q]; J.vout = argsorts[q]; }   // never aliases kin (kin is a scratch buffer)
            J.counts = pl[q].counts_ab[pass & 1];
            J.counts_next = last ? nullptr : pl[q].counts_ab[(pass + 1) & 1];
        }
        rs_scan_kernel<<<grid_scan, RS_THREADS, 0, stream>>>(jobs);
        SPX_CHECK_LAUNCH("rs_scan_kernel");
        if (pass == 0) rs_scatter_kernel<true><<<grid_tiles, RS_THREADS, 0, stream>>>(jobs, pass * RS_BITS);
        else rs_scatter_kernel<false><<<grid_tiles, RS_THREADS, 0, stream>>>(jobs, pass * RS_BITS);
        SPX_CHECK_LAUNCH("rs_scatter_kernel");
        for (int q = 0; q < njobs; ++q) { jobs.j[q].kin = jobs.j[q].kout; jobs.j[q].vin = jobs.j[q].vout; }
    }
    if (passes == 1) {   // single pass wrote to scratch: copy back
        for (int q = 0; q < njobs; ++q) {
            SPX_CHECK_CUDA(cudaMemcpyAsync(masks[q], pl[q].keys_a, (size_t)ns[q] * 4, cudaMemcpyDeviceToDevice, stream));
            SPX_CHECK_CUDA(cudaMemcpyAsync(argsorts[q], pl[q].vals_a, (size_t)ns[q] * 4, cudaMemcpyDeviceToDevice, stream));
        }
    }
    return 0;
}

int sort_by_key(uint32_t *keys, int64_t n, int64_t max_key, int32_t *order, void *sort_ws, size_t sort_ws_bytes,
                cudaStream_t stream) {
    return radix_argsort_pair(keys, order, n, nullptr, nullptr, 0, sort_key_bits(max_key), sort_ws, sort_ws_bytes,
                              nullptr, 0, stream);
}

__global__ void segment_offsets_kernel(const uint32_t *__restrict__ keys, int64_t n, int64_t m,
                                       int32_t *__restrict__ offsets) {
    const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (k > m) return;
    offsets[k] = (int32_t)first_at_least(keys, n, k);
}

int segment_offsets(const uint32_t *sorted_keys, int64_t n, int64_t m, int32_t *offsets, cudaStream_t stream) {
    segment_offsets_kernel<<<(unsigned)div_up64(m + 1, 256), 256, 0, stream>>>(sorted_keys, n, m, offsets);
    SPX_CHECK_LAUNCH("segment_offsets_kernel");
    return 0;
}

size_t cub_sort_pairs_temp_bytes(int64_t n) {
    // The size query goes through the CUDA runtime: a stale error left by an earlier failed call (e.g. a
    // refused stream capture) would make it return early with bytes = 0, and the workspace computed here
    // would then be smaller than what the same query yields a moment later.  Clear the state first and
    // never return less than a bound that covers CUB's double buffers + histograms.
    cudaGetLastError();
    size_t bytes = 0;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr,
                                                    (const uint32_t *)nullptr, (uint32_t *)nullptr, (int)n);
    const size_t floor_bytes = (size_t)(n > 0 ? n : 1) * 16 + (1u << 20);
    if (e != cudaSuccess) { cudaGetLastError(); return floor_bytes; }
    return bytes > floor_bytes ? bytes : floor_bytes;
}

}  // namespace spx
