// Library core: thread-local error string, process-wide launch counter, device check, elementwise epilogue.
#include "common.cuh"
#include <atomic>
#include <mutex>
#include <stdlib.h>

namespace spx {

static thread_local char g_err[1024] = "";
static std::atomic<int64_t> g_launches{0};   // process-wide: a prefetch thread's launches count too
static thread_local int g_family = 0;

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
void set_family(int f) { g_family = f; }

int current_device() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    return dev;
}

static RuntimeCfg make_cfg_from_env() {
    RuntimeCfg c;
    const char *e = getenv("SPX_FORCE_SIMT");
    c.force_simt = e && e[0] == '1';
    e = getenv("SPX_FORCE_TC");
    c.force_tc = e && e[0] == '1';
    return c;
}
RuntimeCfg &runtime_cfg() {
    static RuntimeCfg cfg = make_cfg_from_env();
    return cfg;
}

bool func_configured(const void *fn, int dev) {
    // tiny open table: at most a few dozen kernel instances need the opt-in
    struct Entry { const void *fn; unsigned long long devs; };
    static Entry tab[128];
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    const unsigned long long bit = 1ull << (dev & 63);
    for (auto &e : tab) {
        if (e.fn == fn) { const bool seen = e.devs & bit; e.devs |= bit; return seen; }
        if (e.fn == nullptr) { e.fn = fn; e.devs = bit; return false; }
    }
    return false;   // table full: configure again (idempotent)
}

int sm_count() {
    static thread_local int cached_dev = -1, cached = 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (dev != cached_dev) {
        cudaDeviceProp p;
        if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return 132;
        cached = p.multiProcessorCount;
        cached_dev = dev;
    }
    return cached;
}

// x[r, j] = act(x[r, j] + bias[j])  -- InferenceOps.bias_add_act_inplace, inference.py:166-252
template <typename T>
__global__ void bias_act_kernel(T *__restrict__ x, const T *__restrict__ bias, int64_t total, int cols, int act,
                                float alpha) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < total; i += stride) {
        float v = to_float(x[i]);
        if (bias) v += to_float(bias[i % cols]);
        x[i] = from_float<T>(apply_act(v, act, alpha));
    }
}

}  // namespace spx

using namespace spx;

extern "C" const char *spx_last_error(void) { return g_err; }
extern "C" int spx_version(void) { return 100; }
extern "C" int spx_last_kernel_family(void) { return g_family; }
extern "C" int64_t spx_launch_count(int reset) {
    return reset ? g_launches.exchange(0, std::memory_order_relaxed) : g_launches.load(std::memory_order_relaxed);
}

extern "C" int spx_debug_configure(int force_family, int tc_ctas, int debug_bits, void *trace_buf, size_t trace_bytes) {
    RuntimeCfg &c = runtime_cfg();
    SPX_REQUIRE(force_family >= -1 && force_family <= 2, "debug_configure: force_family must be -1 (keep), 0 (auto), 1 (SIMT) or 2 (tensor cores)");
    SPX_REQUIRE((debug_bits & ~(256 | 4096)) == 0,
                "debug_configure: debug_bits %d not supported; accepted bits are 256 (tf32 input gradient on "
                "the FMA kernel) and 4096 (tf32 weight gradient on the FMA kernel)", debug_bits);
    SPX_REQUIRE(trace_buf == nullptr, "debug_configure: the trace buffer is not supported; pass NULL");
    (void)tc_ctas;
    (void)trace_bytes;
    if (force_family >= 0) { c.force_simt = force_family == 1; c.force_tc = force_family == 2; }
    c.tf32_dgrad_fma = (debug_bits & 256) != 0;
    c.tf32_wgrad_fma = (debug_bits & 4096) != 0;
    return 0;
}

extern "C" int spx_device_check(int dev, int *sm_count_out, int *cc_major, int *cc_minor) {
    cudaDeviceProp p;
    SPX_CHECK_CUDA(cudaGetDeviceProperties(&p, dev));
    if (sm_count_out) *sm_count_out = p.multiProcessorCount;
    if (cc_major) *cc_major = p.major;
    if (cc_minor) *cc_minor = p.minor;
    SPX_REQUIRE(p.major == 9 && p.minor == 0, "spconv_b200 is built for sm_90a only; device %d is sm_%d%d", dev, p.major, p.minor);
    return 0;
}

extern "C" int spx_bias_act_inplace(void *x, const void *bias, int64_t rows, int cols, int dtype, int act,
                                    float act_alpha, spx_stream_t stream_) {
    if (rows == 0 || cols == 0) return 0;
    SPX_REQUIRE(x != nullptr, "x is NULL");
    cudaStream_t stream = (cudaStream_t)stream_;
    int64_t total = rows * cols;
    unsigned nblk = (unsigned)(div_up64(total, 256) < 132 * 16 ? div_up64(total, 256) : 132 * 16);
    switch (dtype) {
        case SPX_F32: bias_act_kernel<float><<<nblk, 256, 0, stream>>>((float *)x, (const float *)bias, total, cols, act, act_alpha); break;
        case SPX_F16: bias_act_kernel<__half><<<nblk, 256, 0, stream>>>((__half *)x, (const __half *)bias, total, cols, act, act_alpha); break;
        case SPX_BF16: bias_act_kernel<__nv_bfloat16><<<nblk, 256, 0, stream>>>((__nv_bfloat16 *)x, (const __nv_bfloat16 *)bias, total, cols, act, act_alpha); break;
        default: SPX_REQUIRE(false, "bias_act: unsupported dtype %d", dtype);
    }
    SPX_CHECK_LAUNCH("bias_act_kernel");
    return 0;
}
