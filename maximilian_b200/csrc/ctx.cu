// Context, error reporting, kernels' shared-memory limits and the envelope-setter helpers of libmaxib200.so.
#include <math.h>

#include <map>
#include <mutex>

#include "common.cuh"

namespace mxb {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int smem_limit_at_least(const void* kern, size_t bytes, const char* what) {
    static std::mutex mu;
    static std::map<std::pair<int, const void*>, size_t> limit;       // (device, kernel) -> the limit this process set
    int dev = 0;
    MXB_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lk(mu);                                   // held across the set: two raises cannot land out of order
    size_t& cur = limit[{dev, kern}];
    if (bytes <= cur) return MXB_OK;
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e != cudaSuccess) {
        set_error("%s: dynamic shared memory limit %zu B: %s", what, bytes, cudaGetErrorString(e));
        return MXB_ERR_CUDA;
    }
    cur = bytes;
    return MXB_OK;
}
}  // namespace mxb

extern "C" {

const char* mxb_last_error(void) { return mxb::g_err; }
int32_t mxb_version(void) { return MXB_VERSION; }

int32_t mxb_ctx_create(int32_t device, int32_t sample_rate, mxb_ctx** out) {
    MXB_REQUIRE(out != nullptr, MXB_ERR_INVALID, "mxb_ctx_create: ctx is NULL");
    *out = nullptr;
    MXB_REQUIRE(sample_rate > 0, MXB_ERR_INVALID, "mxb_ctx_create: sample_rate %d", sample_rate);
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        // no CPU fallback: the product path is CUDA only
        mxb::set_error("mxb_ctx_create: no CUDA device (%s)", e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
        return MXB_ERR_CUDA;
    }
    MXB_REQUIRE(device >= 0 && device < n, MXB_ERR_INVALID, "mxb_ctx_create: device %d of %d", device, n);
    cudaDeviceProp prop;
    MXB_CUDA(cudaGetDeviceProperties(&prop, device));
    // arch-specific sm_90a code loads on compute capability 9.0 and nothing else
    MXB_REQUIRE(prop.major == 9 && prop.minor == 0, MXB_ERR_UNSUPPORTED, "mxb_ctx_create: device %d is sm_%d%d; this library is built for sm_90a only",
                device, prop.major, prop.minor);
    mxb::DeviceGuard g(device);
    MXB_REQUIRE(g.ok, MXB_ERR_CUDA, "mxb_ctx_create: cudaSetDevice(%d) failed", device);
    MXB_CUDA(cudaFree(0));
    int smem_optin = 0;
    MXB_CUDA(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    mxb_ctx* c = new mxb_ctx();
    c->device = device;
    c->sample_rate = sample_rate;
    c->sm_count = prop.multiProcessorCount;
    c->cc_major = prop.major;
    c->cc_minor = prop.minor;
    c->smem_optin = smem_optin;
    c->sine_before = 0.0;
    *out = c;
    return MXB_OK;
}

int32_t mxb_ctx_destroy(mxb_ctx* ctx) {
    if (!ctx) return MXB_OK;
    mxb::DeviceGuard g(ctx->device);
    delete ctx;
    return MXB_OK;
}

int32_t mxb_ctx_sample_rate(const mxb_ctx* ctx) { return ctx ? ctx->sample_rate : MXB_ERR_INVALID; }

int32_t mxb_ctx_synchronize(mxb_ctx* ctx) {
    MXB_REQUIRE(ctx, MXB_ERR_INVALID, "mxb_ctx_synchronize: NULL ctx");
    mxb::DeviceGuard g(ctx->device);
    MXB_CUDA(cudaDeviceSynchronize());
    return MXB_OK;
}

int32_t mxb_host_alloc(mxb_ctx* ctx, uint64_t bytes, void** ptr) {
    MXB_REQUIRE(ctx && ptr, MXB_ERR_INVALID, "mxb_host_alloc: NULL argument");
    mxb::DeviceGuard g(ctx->device);
    cudaError_t e = cudaHostAlloc(ptr, bytes ? bytes : 1, cudaHostAllocDefault);
    if (e != cudaSuccess) { mxb::set_error("cudaHostAlloc(%llu): %s", (unsigned long long)bytes, cudaGetErrorString(e)); return MXB_ERR_ALLOC; }
    return MXB_OK;
}

int32_t mxb_host_free(mxb_ctx* ctx, void* ptr) {
    MXB_REQUIRE(ctx, MXB_ERR_INVALID, "mxb_host_free: NULL ctx");
    if (ptr) MXB_CUDA(cudaFreeHost(ptr));
    return MXB_OK;
}

// maxiEnv::setAttack / setAttackMS / setDecay / setRelease, src/maximilian.cpp:1469-1486.
// sampleRate is a size_t in the reference and converts to double inside the product.
int32_t mxb_env_coeffs(int32_t kind, const double* ms, int64_t n, int32_t sample_rate, double* coeff) {
    MXB_REQUIRE(ms && coeff && n >= 0 && sample_rate > 0 && kind >= 0 && kind <= 2, MXB_ERR_INVALID, "mxb_env_coeffs: bad argument");
    const double sr = (double)(size_t)sample_rate;
    for (int64_t i = 0; i < n; ++i) {
        switch (kind) {
            case 0: coeff[i] = 1 - pow(0.01, 1.0 / (ms[i] * sr * 0.001)); break;
            case 1: coeff[i] = 1.0 / (ms[i] / 1000.0 * sr); break;
            default: coeff[i] = pow(0.01, 1.0 / (ms[i] * sr * 0.001)); break;
        }
    }
    return MXB_OK;
}

}  // extern "C"
