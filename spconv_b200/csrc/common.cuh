// Shared host/device helpers for the sm_90a kernels behind include/spconv_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <stdarg.h>
#include <type_traits>

#include "../../include/spconv_b200.h"

namespace spx {

// ---------------------------------------------------------------- error plumbing
void set_error(const char *fmt, ...);
void count_launch(int n = 1);
void set_family(int f);
int sm_count();          // SMs of the current device (cached)
int current_device();    // cudaGetDevice (0 on failure)

// Process-wide switches.  SPX_FORCE_SIMT / SPX_FORCE_TC are read from the
// environment ONCE, when the library is loaded; spx_debug_configure() can change them and set the
// two tf32 switches, which send the fp32 input / weight gradient to the FMA kernels.
struct RuntimeCfg {
    int force_simt = 0, force_tc = 0;
    bool tf32_dgrad_fma = false;   // debug bit 256
    bool tf32_wgrad_fma = false;   // debug bit 4096
};
RuntimeCfg &runtime_cfg();

// cudaFuncSetAttribute is per DEVICE: remember which (function, device) pairs were configured
bool func_configured(const void *fn, int dev);   // returns the previous state and marks it

// A failed runtime call also leaves its error pending on the thread; it is consumed here so that
// the next SPX_CHECK_LAUNCH does not report it again (e.g. after a refused stream capture).
#define SPX_CHECK_CUDA(expr)                                                              \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess) {                                                          \
            (void)cudaGetLastError();                                                     \
            spx::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),        \
                           __FILE__, __LINE__);                                           \
            return 1;                                                                     \
        }                                                                                 \
    } while (0)

#define SPX_CHECK_LAUNCH(name)                                                            \
    do {                                                                                  \
        cudaError_t _e = cudaGetLastError();                                              \
        if (_e != cudaSuccess) {                                                          \
            spx::set_error("launch of %s failed: %s (%s:%d)", name,                       \
                           cudaGetErrorString(_e), __FILE__, __LINE__);                   \
            return 1;                                                                     \
        }                                                                                 \
        spx::count_launch();                                                              \
    } while (0)

#define SPX_REQUIRE(cond, ...)                                                            \
    do {                                                                                  \
        if (!(cond)) {                                                                    \
            spx::set_error(__VA_ARGS__);                                                  \
            return 2;                                                                     \
        }                                                                                 \
    } while (0)

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static inline int64_t div_up64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// 16-byte vector accesses (cp.async, uint4 / float4 / int4 loads and stores, tensor maps) fault on an address
// that is not a multiple of 16.  Every caller pointer a kernel reads or writes that way is checked with this
// before that kernel is chosen; NULL passes.
static inline bool aligned16(const void *p) { return ((uintptr_t)p & 15u) == 0; }

// for kernels without an element-wise path: refuse the call, naming the argument
#define SPX_REQUIRE_ALIGNED16(ptr, who)                                                   \
    SPX_REQUIRE(spx::aligned16(ptr), "%s: %s must be 16-byte aligned (got %p)", who, #ptr, \
                (const void *)(ptr))

// carve a caller-provided workspace
struct WorkspaceCarver {
    char *base;
    size_t off = 0, cap;
    WorkspaceCarver(void *p, size_t bytes) : base((char *)p), cap(bytes) {}
    template <typename T> T *take(size_t n) {
        off = align_up(off, 256);
        T *r = (T *)(base + off);
        off += n * sizeof(T);
        return r;
    }
    bool ok() const { return off <= cap; }
};

__host__ __device__ static inline int dtype_bytes(int dt) {
    switch (dt) {
        case SPX_F32: return 4;
        case SPX_F16: return 2;
        case SPX_BF16: return 2;
        case SPX_I8: return 1;
        case SPX_E4M3: return 1;
    }
    return 0;
}

// ---------------------------------------------------------------- device helpers
#ifdef __CUDACC__

template <typename T> __device__ __forceinline__ float to_float(T v);
template <> __device__ __forceinline__ float to_float<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_float<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_float<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_float<int8_t>(int8_t v) { return (float)v; }

template <typename T> __device__ __forceinline__ T from_float(float v);
template <> __device__ __forceinline__ float from_float<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_float<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_float<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

__device__ __forceinline__ float apply_act(float v, int act, float alpha) {
    // InferenceOps activations: spconv/csrc/sparse/inference.py:26-146
    switch (act) {
        case SPX_ACT_RELU: return v > 0.f ? v : 0.f;
        case SPX_ACT_SIGMOID: return 1.f / (1.f + __expf(-v));
        case SPX_ACT_LEAKY_RELU: return v >= 0.f ? v : v * alpha;
        default: return v;
    }
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}

// ---- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
// Spin on try_wait (which itself suspends in hardware for a while).  A protocol bug must become
// an error, not a hung GPU: after ~2 s of waiting the kernel traps (cudaErrorLaunchFailure).
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 0x3FFFu) == 0u && clock64() - t0 > 4000000000ll) {
            printf("spconv_b200: mbarrier wait timed out (block %d thread %d bar 0x%x parity %u)\n",
                   (int)blockIdx.x, (int)threadIdx.x, smem_u32(bar), parity);
            __trap();
        }
    }
}
// mbar_wait without the printf, for kernels that keep a wgmma group in flight across a wait: a
// function call anywhere in such a kernel (ptxas does not tell the warp roles' paths apart) makes
// ptxas serialise all its wgmma.  The timeout still traps.
__device__ __forceinline__ void mbar_wait_silent(uint64_t *bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 0x3FFFu) == 0u && clock64() - t0 > 4000000000ll) __trap();
    }
}
// arrive (no pending-count increment) once all prior cp.async of this thread have landed
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint64_t *bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// ---- cp.async 16 B with zero fill (src_bytes = 0 -> writes 16 zero bytes, reads nothing)
__device__ __forceinline__ void cp_async_16(uint32_t dst_smem, const void *src, uint32_t src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// generic-proxy writes -> visible to the async proxy (wgmma / TMA reads of smem)
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---- TMA (tiled 2D load, mbarrier completion)
__device__ __forceinline__ void tma_load_2d(uint32_t dst_smem, const void *tmap, uint64_t *bar,
                                            int32_t c0, int32_t c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cta.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst_smem), "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
// 1-D bulk async copy global -> shared (UBLKCP), completion counted in bytes on an mbarrier
__device__ __forceinline__ void bulk_copy_g2s(uint32_t dst_smem, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const void *tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(tmap) : "memory");
}

// ---- wgmma (Hopper warpgroup MMA; the instruction wrappers are in wgmma.cuh)
enum MmaKind { KIND_F16 = 0, KIND_TF32 = 1, KIND_I8 = 2, KIND_E4M3 = 3 };

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMA
template <typename T, int R> __device__ __forceinline__ void fence_regs(T (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) {
        if constexpr (sizeof(T) == 4 && std::is_floating_point<T>::value) asm volatile("" : "+f"(d[i])::"memory");
        else asm volatile("" : "+r"(d[i])::"memory");
    }
}

// Constant (address-independent) part of a wgmma shared-memory matrix descriptor; OR it with
// ((smem_addr >> 4) & 0x3FFF).  Byte quantities, 16-byte granular; swizzle_bytes in {32, 64, 128}
// (layout type 3, 2, 1).  K-major operands: SBO = one 8-row swizzle atom, LBO unused.  MN-major:
// LBO = distance between swizzle-wide column blocks, SBO = 8 K rows.
__host__ __device__ __forceinline__ uint64_t gmma_desc_hi(uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t swizzle_bytes) {
    const uint64_t layout = swizzle_bytes == 128 ? 1ull : (swizzle_bytes == 64 ? 2ull : 3ull);
    return ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32) | (layout << 62);
}

// byte offset inside a swizzled tile whose rows are `swizzle_bytes` long and whose base is
// 1024-byte aligned: XOR the 16-byte chunk index with the row index (Swizzle<B,4,3>).
__device__ __forceinline__ uint32_t swizzle_offset(uint32_t off, uint32_t swizzle_bytes) {
    uint32_t bits = swizzle_bytes == 128 ? 7u : (swizzle_bytes == 64 ? 3u : 1u);
    return off ^ (((off >> 7) & bits) << 4);
}

#endif  // __CUDACC__

}  // namespace spx
