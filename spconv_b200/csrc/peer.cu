// Weight-gradient exchange between data-parallel ranks over NVLink peer memory.
//
// The only tensor that crosses GPUs on this path is dW (SURVEY 8e; the reference itself has no
// distributed code).  dW is small (27*C*K values: 0.4 MB fp32 at C = K = 64), so the exchange is
// latency-bound and a library all-reduce costs more in launches and protocol than in bytes.  Two kernels:
//
//   push    (peer_push_kernel = the kernel that reduces the split-K partials of tc_wgrad_kernel, or reads
//           an existing gradient): every CTA sums its 128-value slice in fp32 and writes it straight into
//           this rank's exchange buffer [slot][element] -- the reduction's output IS the send buffer, no
//           staging copy, nothing else on the critical path of the weight gradient.
//   finish  (peer_finish_kernel, a few small CTAs): publishes -- one system-scope fence, then the epoch is
//           stored into every rank's flag word for this source (world tiny release stores over NVLink);
//           waits until every source's flag shows this epoch (acquire loads on its OWN flags); pulls the
//           world's slices with TMA bulk copies through the peer mapping (its own locally) and sums them in
//           rank order -- the same order on every rank, so all replicas get bit-identical gradients;
//           scales, rounds once, writes dW, advances the epoch in device memory (CUDA-graph capturable: no
//           host argument changes between replays).
//
// The caller runs finish behind the input-gradient kernel of the same layer (on the forked stream of the
// captured backward), off the critical path.  Variants tried on the way here, all correct, at N = 2 on an earlier
// GPU generation (not re-measured on H100): (1) push + wait + sum in ONE kernel, every CTA storing into every
// rank's buffer; (2) the same split into push / finish, where one system-scope fence per CTA slowed the
// weight-gradient region; (3) local writes, the last CTA of the reduction publishing, receivers pulling (LDG or TMA
// bulk copies, 16 or 64 CTAs, gpu- or system-scope fence, normal or high-priority stream), none of these knobs
// mattering; (4) a world-of-one group (no NVLink at all) paying the same as the real exchange over the single-GPU
// graph: the cost is the shape of the captured backward (every dependent kernel behind forward -> weight gradient
// costs launch + queueing time when the next cloud's rulebook kernels share the GPU), not the wire.  Under graph
// replay the NCCL hook stayed ahead at N = 2; through the eager module API this path won (one native call per
// layer instead of a collective launch).  bench.py therefore defaults to the NCCL hook for the graph-replayed
// headline and keeps this path selectable (--allreduce fused).
//
// Gather mode (spx_peer_allgather, MaskedSyncBatchNorm1d's statistics): the same push and the same finish with
// GATHER set, which copies every rank's slice to dst[r] as 32-bit words instead of summing them.  Publish, wait,
// timeout and the epoch advance are the one code path of the sum, so the slot protocol below covers both.
//
// No grid-wide barrier, no host involvement.  Neither kernel waits for a peer before it has published, so ranks
// cannot deadlock each other; a peer that never shows up trips the group's timeout in finish (error word +
// NaN result) instead of hanging the GPU.  Two slots alternate by epoch: rank r overwrites slot e&1 in its
// push of epoch e+2, which is stream-ordered after its finish of e+1, which needed every peer's flag of e+1,
// which that peer stored in its own finish of e+1, i.e. after its finish of e -- so nobody is still reading
// r's slot e&1.  Hence the contract: on each rank push and finish of one group alternate in stream order (one
// exchange in flight), same sequence on all ranks.  tests/test_peer_protocol_cpu.py explores every interleaving of this
// state machine for 2-4 ranks (and shows that one slot, or a publish before the data, is caught).
#include "common.cuh"
#include "gemm.cuh"
#include "peer.cuh"

namespace spx {

// ---- exchange buffer layout (bytes from the base of each rank's buffer)
//   [0, 64)      local state: epoch, finished CTAs of the running finish, one unused word, error
//   [256, 320)   flags, one per source rank: last epoch (+1) that source has published (written by the peers)
//   [4096, ...)  data [2 slots][capacity] fp32: this rank's own slices
constexpr size_t PEER_FLAGS = 256, PEER_DATA = 4096;

struct PeerState { unsigned epoch, finished, done, error; };

__device__ __forceinline__ void st_release_sys(unsigned *addr, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned *addr) {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(addr) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

struct PeerPtrs { char *buf[SPX_MAX_PEERS]; };

constexpr int PX_THREADS = 256, PX_WARPS = PX_THREADS / 32;

// One CTA per 128 values (32 lanes x float4; the tail item may be partial).  partial != nullptr: the
// slice is the sum of [chunks] split-K partials (eight warps split the chunks); otherwise it is read
// from `src` (T).
template <typename T>
__global__ void __launch_bounds__(PX_THREADS)
peer_push_kernel(const float *__restrict__ partial, int64_t stride, int chunks, const T *__restrict__ src, int64_t total,
                 PeerPtrs peers, int rank, int64_t capacity) {
    __shared__ float4 acc_s[PX_WARPS][32];
    __shared__ unsigned s_epoch;
    PeerState *st = reinterpret_cast<PeerState *>(peers.buf[rank]);
    if (threadIdx.x == 0) s_epoch = st->epoch;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t i = ((int64_t)blockIdx.x * 32 + lane) * 4;
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
    if (partial) {
        if (i < total) {                                   // total % 4 == 0 on this path (channels % 16 == 0)
            const int per = (chunks + PX_WARPS - 1) / PX_WARPS;
            const int c0 = warp * per, c1 = min(chunks, c0 + per);
#pragma unroll 4
            for (int c = c0; c < c1; ++c) {
                const float4 v = __ldg(reinterpret_cast<const float4 *>(partial + (int64_t)c * stride + i));
                s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
            }
        }
        acc_s[warp][lane] = s;
    }
    __syncthreads();
    if (warp != 0) return;
    const unsigned epoch = s_epoch;
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    if (partial) {
        t = acc_s[0][lane];
#pragma unroll
        for (int w = 1; w < PX_WARPS; ++w) {
            const float4 v = acc_s[w][lane];
            t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
        }
    } else if (i < total) {
        t.x = to_float<T>(src[i]);
        if (i + 1 < total) t.y = to_float<T>(src[i + 1]);
        if (i + 2 < total) t.z = to_float<T>(src[i + 2]);
        if (i + 3 < total) t.w = to_float<T>(src[i + 3]);
    }
    if (i < total)                                         // the padded tail of the last float4 carries zeros
        *reinterpret_cast<float4 *>(reinterpret_cast<float *>(peers.buf[rank] + PEER_DATA) + (int64_t)(epoch & 1u) * capacity + i) = t;
}

// Receive side.  It runs BESIDE the persistent input-gradient kernel (whose CTAs own most of every SM's register
// file) and may have to wait for a slower rank, so its footprint must be tiny: a handful of CTAs, and the pulls are
// TMA bulk copies (cp.async.bulk global -> shared over the peer mapping, mbarrier completion) issued by one thread --
// bytes in flight without registers.  A first version (one thread per float4, ~100 CTAs x 26 k registers, spinning
// on the flags) kept the input-gradient CTAs off its SMs for as long as the slowest rank was late, which cost
// measurable time per pipelined config-2 step at N = 2.
constexpr int FIN_CHUNK_BYTES = 8192;              // per source rank per step: world x 8 KB in flight per CTA
constexpr int FIN_MAX_CTAS = 64;               // 0.44 MB per peer = 54 chunks: one round trip for the whole tensor

// GATHER: dst is [world][total] 32-bit words (T = uint32_t), rank r's slice copied unchanged to dst[r]; scale unused.
template <typename T, bool GATHER>
__global__ void __launch_bounds__(PX_THREADS)
peer_finish_kernel(T *__restrict__ dst, int64_t total, PeerPtrs peers, int world, int rank, int64_t capacity, float scale,
                   unsigned long long timeout_ns) {
    extern __shared__ __align__(128) uint8_t fin_smem[];      // [world][FIN_CHUNK_BYTES] + mbarrier
    __shared__ __align__(8) uint64_t bar;
    __shared__ unsigned s_epoch;
    __shared__ int s_bad;
    char *mine = peers.buf[rank];
    PeerState *st = reinterpret_cast<PeerState *>(mine);
    if (threadIdx.x == 0) { s_epoch = st->epoch; s_bad = 0; mbar_init(&bar, 1); mbar_fence_init(); }
    __syncthreads();
    const unsigned epoch = s_epoch, target = epoch + 1u;
    if (blockIdx.x == 0 && threadIdx.x < world) {
        // This rank's slices were written by an EARLIER kernel of this stream (the weight-gradient reduction): they
        // are complete and visible on this GPU.  One system-scope fence, then the epoch goes to every rank's flag
        // word.  (Publishing from the reduction kernel itself -- last CTA out -- put a per-CTA fence + counter and
        // the NVLink store acknowledgement on the critical path: +8 us on the weight gradient.)
        __threadfence_system();
        st_release_sys(reinterpret_cast<unsigned *>(peers.buf[threadIdx.x] + PEER_FLAGS) + rank, target);
    }
    if (threadIdx.x < world) {
        const unsigned *flag = reinterpret_cast<const unsigned *>(mine + PEER_FLAGS) + threadIdx.x;
        const unsigned long long t0 = globaltimer_ns();
        unsigned spins = 0;
        while ((int)(ld_acquire_sys(flag) - target) < 0) {
            __nanosleep(200);
            if ((++spins & 255u) == 0 && globaltimer_ns() - t0 > timeout_ns) { s_bad = 1; break; }
        }
    }
    __syncthreads();
    const bool bad = s_bad != 0;
    if (bad && threadIdx.x == 0) st->error = 1u;
    const int64_t slot_off = (int64_t)(epoch & 1u) * capacity;
    const int64_t padded = (total + 3) / 4 * 4;                       // floats every publisher wrote
    const int64_t chunk_floats = FIN_CHUNK_BYTES / 4;
    const int64_t nchunks = (padded + chunk_floats - 1) / chunk_floats;
    const float nan = __int_as_float(0x7fc00000);
    uint32_t phase = 0;
    for (int64_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
        const int64_t f0 = c * chunk_floats;
        const int nfl = (int)((padded - f0) < chunk_floats ? (padded - f0) : chunk_floats);
        if (threadIdx.x == 0) {
            asm volatile("fence.proxy.async;" ::: "memory");          // flags acquired / smem consumed in the generic proxy
            mbar_arrive_expect_tx(&bar, (uint32_t)(world * nfl * 4));
            for (int r = 0; r < world; ++r)
                bulk_copy_g2s(smem_u32(fin_smem + (size_t)r * FIN_CHUNK_BYTES),
                              reinterpret_cast<const float *>(peers.buf[r] + PEER_DATA) + slot_off + f0, (uint32_t)(nfl * 4), &bar);
        }
        mbar_wait(&bar, phase);
        phase ^= 1u;
        if constexpr (GATHER) {
            for (int j = threadIdx.x * 4; j < nfl; j += PX_THREADS * 4) {
                const int64_t i = f0 + j;
                for (int r = 0; r < world; ++r) {                      // word copies: the bits every rank sent
                    uint4 w = *reinterpret_cast<const uint4 *>(fin_smem + (size_t)r * FIN_CHUNK_BYTES + (size_t)j * 4);
                    if (bad) w = make_uint4(0x7fc00000u, 0x7fc00000u, 0x7fc00000u, 0x7fc00000u);
                    T *d = dst + (int64_t)r * total + i;
                    d[0] = w.x;
                    if (i + 1 < total) d[1] = w.y;
                    if (i + 2 < total) d[2] = w.z;
                    if (i + 3 < total) d[3] = w.w;
                }
            }
        } else {
            for (int j = threadIdx.x * 4; j < nfl; j += PX_THREADS * 4) {
                float4 t = *reinterpret_cast<const float4 *>(fin_smem + (size_t)j * 4);
                for (int r = 1; r < world; ++r) {                      // rank order: identical bits on every rank
                    const float4 v = *reinterpret_cast<const float4 *>(fin_smem + (size_t)r * FIN_CHUNK_BYTES + (size_t)j * 4);
                    t.x += v.x; t.y += v.y; t.z += v.z; t.w += v.w;
                }
                if (bad) t = make_float4(nan, nan, nan, nan);
                const int64_t i = f0 + j;
                dst[i] = from_float<T>(t.x * scale);
                if (i + 1 < total) dst[i + 1] = from_float<T>(t.y * scale);
                if (i + 2 < total) dst[i + 2] = from_float<T>(t.z * scale);
                if (i + 3 < total) dst[i + 3] = from_float<T>(t.w * scale);
            }
        }
        __syncthreads();                                               // the chunk is consumed before it is overwritten
    }
    // ---- the last CTA out advances the epoch (publish / finish of one group alternate in stream order)
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(&st->finished, 1u) == gridDim.x - 1) {
            st->finished = 0;
            st->epoch = epoch + 1;
            __threadfence();
        }
    }
}

static int check_group(const spx_peer_group *pg, int64_t total, const char *who) {
    SPX_REQUIRE(pg != nullptr, "%s: peer group is NULL", who);
    SPX_REQUIRE(pg->world >= 1 && pg->world <= SPX_MAX_PEERS && pg->rank >= 0 && pg->rank < pg->world,
                "%s: bad peer group (world %d, rank %d)", who, pg->world, pg->rank);
    SPX_REQUIRE(total >= 0 && (uint64_t)(total + 3) / 4 * 16 <= pg->capacity_bytes,
                "%s: %lld fp32 values exceed the exchange capacity of %llu bytes", who, (long long)total,
                (unsigned long long)pg->capacity_bytes);
    for (int r = 0; r < pg->world; ++r) SPX_REQUIRE(pg->buffers[r] != nullptr, "%s: buffer of rank %d is NULL", who, r);
    return 0;
}

static PeerPtrs peer_ptrs(const spx_peer_group *pg) {
    PeerPtrs pp;
    memset(&pp, 0, sizeof(pp));
    for (int r = 0; r < pg->world; ++r) pp.buf[r] = (char *)pg->buffers[r];
    return pp;
}
static unsigned push_ctas(int64_t total) { return (unsigned)div_up64(total, 128); }

int peer_push(const float *partial, int64_t stride, int chunks, const void *src, int64_t total, int dtype,
              const spx_peer_group *pg, cudaStream_t stream) {
    if (int rc = check_group(pg, total, "peer push")) return rc;
    if (total == 0) return 0;
    SPX_REQUIRE(!partial || total % 4 == 0, "peer push: partial sums need a multiple of 4 values");
    const PeerPtrs pp = peer_ptrs(pg);
    const int64_t cap = (int64_t)(pg->capacity_bytes / 4);
    const unsigned grid = push_ctas(total);
#define PX_LAUNCH(T) peer_push_kernel<T><<<grid, PX_THREADS, 0, stream>>>(partial, stride, chunks, (const T *)src, total, pp, pg->rank, cap)
    if (dtype == SPX_F16) PX_LAUNCH(__half);
    else if (dtype == SPX_BF16) PX_LAUNCH(__nv_bfloat16);
    else if (dtype == SPX_F32) PX_LAUNCH(float);
    else { set_error("peer push: dtype %d not supported", dtype); return 2; }
#undef PX_LAUNCH
    SPX_CHECK_LAUNCH("peer_push_kernel");
    return 0;
}

// gather: dst [world][total] 32-bit words; dtype and scale are ignored
static int peer_finish_any(void *dst, int64_t total, int dtype, const spx_peer_group *pg, float scale, bool gather,
                           cudaStream_t stream) {
    if (int rc = check_group(pg, total, gather ? "peer allgather" : "peer finish")) return rc;
    if (total == 0) return 0;
    const PeerPtrs pp = peer_ptrs(pg);
    const int64_t cap = (int64_t)(pg->capacity_bytes / 4);
    const int64_t nchunks = div_up64((total + 3) / 4 * 16, FIN_CHUNK_BYTES);
    int64_t max_ctas = FIN_MAX_CTAS;
    if (pg->colocated > 1 && max_ctas > FIN_MAX_CTAS / pg->colocated) max_ctas = FIN_MAX_CTAS / pg->colocated > 0 ? FIN_MAX_CTAS / pg->colocated : 1;
    const unsigned grid = (unsigned)(nchunks < max_ctas ? nchunks : max_ctas);
    const size_t smem = (size_t)pg->world * FIN_CHUNK_BYTES;
    const unsigned long long timeout_ns = (unsigned long long)(pg->timeout_ms > 0 ? pg->timeout_ms : 20000) * 1000000ull;
#define PX_LAUNCH(T, G)                                                                                               \
    do {                                                                                                              \
        auto fn = peer_finish_kernel<T, G>;                                                                            \
        if (smem > 48 * 1024 && !func_configured((const void *)fn, current_device()))                                 \
            SPX_CHECK_CUDA(cudaFuncSetAttribute((const void *)fn, cudaFuncAttributeMaxDynamicSharedMemorySize,       \
                                                SPX_MAX_PEERS * FIN_CHUNK_BYTES));                                    \
        fn<<<grid, PX_THREADS, smem, stream>>>((T *)dst, total, pp, pg->world, pg->rank, cap, scale, timeout_ns);     \
    } while (0)
    if (gather) PX_LAUNCH(uint32_t, true);
    else if (dtype == SPX_F16) PX_LAUNCH(__half, false);
    else if (dtype == SPX_BF16) PX_LAUNCH(__nv_bfloat16, false);
    else if (dtype == SPX_F32) PX_LAUNCH(float, false);
    else { set_error("peer finish: dtype %d not supported", dtype); return 2; }
#undef PX_LAUNCH
    SPX_CHECK_LAUNCH("peer_finish_kernel");
    return 0;
}

int peer_finish(void *dst, int64_t total, int dtype, const spx_peer_group *pg, float scale, cudaStream_t stream) {
    return peer_finish_any(dst, total, dtype, pg, scale, false, stream);
}

}  // namespace spx

using namespace spx;

extern "C" size_t spx_peer_buffer_bytes(size_t capacity_bytes, int world) {
    if (world < 1 || world > SPX_MAX_PEERS) return 0;
    return PEER_DATA + 2 * align_up(capacity_bytes, 16);
}

extern "C" int spx_peer_buffer_create(size_t capacity_bytes, int world, void **buffer, unsigned char handle[64]) {
    SPX_REQUIRE(buffer && handle, "peer_buffer_create: NULL output");
    SPX_REQUIRE(world >= 1 && world <= SPX_MAX_PEERS, "peer_buffer_create: world %d out of range (1..%d)", world, SPX_MAX_PEERS);
    SPX_REQUIRE(capacity_bytes % 16 == 0 && capacity_bytes > 0, "peer_buffer_create: capacity must be a positive multiple of 16");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    void *p = nullptr;
    const size_t bytes = spx_peer_buffer_bytes(capacity_bytes, world);
    SPX_CHECK_CUDA(cudaMalloc(&p, bytes));
    SPX_CHECK_CUDA(cudaMemset(p, 0, bytes));
    cudaIpcMemHandle_t h;
    cudaError_t e = cudaIpcGetMemHandle(&h, p);
    if (e != cudaSuccess) {
        cudaGetLastError();
        cudaFree(p);
        set_error("cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
        return 1;
    }
    memcpy(handle, &h, 64);
    *buffer = p;
    return 0;
}

extern "C" int spx_peer_buffer_open(const unsigned char handle[64], void **mapped) {
    SPX_REQUIRE(handle && mapped, "peer_buffer_open: NULL argument");
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    SPX_CHECK_CUDA(cudaIpcOpenMemHandle(mapped, h, cudaIpcMemLazyEnablePeerAccess));
    return 0;
}

extern "C" int spx_peer_buffer_close(void *mapped) {
    if (mapped) SPX_CHECK_CUDA(cudaIpcCloseMemHandle(mapped));
    return 0;
}

extern "C" int spx_peer_buffer_destroy(void *buffer) {
    if (buffer) SPX_CHECK_CUDA(cudaFree(buffer));
    return 0;
}

extern "C" int spx_peer_error(const spx_peer_group *pg, int *error) {
    SPX_REQUIRE(pg && error, "peer_error: NULL argument");
    PeerState st;
    SPX_CHECK_CUDA(cudaMemcpy(&st, pg->buffers[pg->rank], sizeof(st), cudaMemcpyDeviceToHost));
    *error = (int)st.error;
    return 0;
}

extern "C" int spx_peer_push(const spx_peer_group *pg, const void *data, int64_t count, int dtype, spx_stream_t stream) {
    SPX_REQUIRE(data != nullptr || count == 0, "peer_push: data is NULL");
    return peer_push(nullptr, 0, 0, data, count, dtype, pg, (cudaStream_t)stream);
}

extern "C" int spx_peer_finish(const spx_peer_group *pg, void *out, int64_t count, int dtype, float scale,
                               spx_stream_t stream) {
    SPX_REQUIRE(out != nullptr || count == 0, "peer_finish: out is NULL");
    return peer_finish(out, count, dtype, pg, scale, (cudaStream_t)stream);
}

extern "C" int spx_peer_allreduce(const spx_peer_group *pg, void *data, int64_t count, int dtype, float scale,
                                  spx_stream_t stream) {
    if (int rc = spx_peer_push(pg, data, count, dtype, stream)) return rc;
    return spx_peer_finish(pg, data, count, dtype, scale, stream);
}

extern "C" int spx_peer_allgather(const spx_peer_group *pg, const uint32_t *src, int64_t count, uint32_t *dst,
                                  spx_stream_t stream) {
    SPX_REQUIRE(count == 0 || (src != nullptr && dst != nullptr), "peer_allgather: NULL src or dst");
    if (int rc = check_group(pg, count, "peer allgather")) return rc;
    // the fp32 push reads and stores each word without arithmetic, so the bits arrive unchanged
    if (int rc = peer_push(nullptr, 0, 0, src, count, SPX_F32, pg, (cudaStream_t)stream)) return rc;
    return peer_finish_any(dst, count, SPX_F32, pg, 1.f, true, (cudaStream_t)stream);
}
