// Internal definitions shared by the translation units of libmaxib200.so (not installed).
#pragma once

#ifdef __CUDACC_RTC__
// Compiled at run time (NVRTC, patch_fuse.cu): only the device-side definitions of the headers are wanted; the host half of
// this file is skipped and maxib200.h arrives as an embedded header.
#include "maxib200.h"
#else
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <string.h>
#include <stdlib.h>
#include <memory>
#include <utility>
#include <vector>

#include "../../include/maxib200.h"

#include <nvtx3/nvToolsExt.h>      // header-only; ranges show up in nsys / ncu --nvtx timelines, cost nothing without a profiler

namespace mxb {

void set_error(const char* fmt, ...);

// Makes the current device's dynamic shared-memory limit of `kern` at least `bytes` before a launch that asks for `bytes`. The limit
// belongs to the kernel, shared by every handle and host thread, so it is only ever raised: a launch on another thread that needs
// less cannot lower it between this thread's check and its launch. Every launch with dynamic shared memory goes through here.
int smem_limit_at_least(const void* kern, size_t bytes, const char* what);

#define MXB_CUDA(expr)                                                                         \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            mxb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return MXB_ERR_CUDA;                                                               \
        }                                                                                      \
    } while (0)

#define MXB_REQUIRE(cond, code, ...)        \
    do {                                    \
        if (!(cond)) {                      \
            mxb::set_error(__VA_ARGS__);    \
            return (code);                  \
        }                                   \
    } while (0)

struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
};

struct DeviceGuard {
    int prev = -1;
    bool ok = true;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) { ok = false; return; }
        if (prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
        if (prev == dev) prev = -1;
    }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// One device allocation (plain cudaMalloc), freed when the buffer is destroyed. Empty until alloc / grow / upload.
template <class T>
class DevBuf {
public:
    DevBuf() = default;
    DevBuf(DevBuf&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
    DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); return *this; }
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { if (p_) cudaFree(p_); }

    // max(n, 1) elements, zero-filled unless `zero` is false; replaces any earlier allocation
    int alloc(size_t n, bool zero = true) {
        release();
        void* q = nullptr;
        cudaError_t e = cudaMalloc(&q, sizeof(T) * (n ? n : 1));
        if (e != cudaSuccess) { set_error("cudaMalloc(%zu bytes): %s", sizeof(T) * n, cudaGetErrorString(e)); return MXB_ERR_ALLOC; }
        if (zero) {
            e = cudaMemset(q, 0, sizeof(T) * (n ? n : 1));
            if (e != cudaSuccess) { set_error("cudaMemset: %s", cudaGetErrorString(e)); cudaFree(q); return MXB_ERR_CUDA; }
        }
        p_ = (T*)q; n_ = n;
        return MXB_OK;
    }
    // Grows a staging buffer to at least `n` elements (contents not kept). Work queued on `s` may still read the old
    // buffer, so `s` is synchronised before it is freed.
    int grow(size_t n, cudaStream_t s) {
        if (n <= n_) return MXB_OK;
        MXB_CUDA(cudaStreamSynchronize(s));
        return alloc(n, false);
    }
    int upload(const std::vector<T>& v) {
        const int rc = alloc(v.size(), false);
        if (rc != MXB_OK) return rc;
        MXB_CUDA(cudaMemcpy(p_, v.data(), sizeof(T) * v.size(), cudaMemcpyHostToDevice));
        return MXB_OK;
    }
    T* get() const { return p_; }
    size_t size() const { return n_; }

private:
    void release() { if (p_) cudaFree(p_); p_ = nullptr; n_ = 0; }
    T* p_ = nullptr;
    size_t n_ = 0;       // elements asked for
};

// MXB_MEM_HOST data reaches a kernel through a staging buffer of the handle. stage_in: with `host` set, copies `n`
// elements of `src` into `buf` on `s` and points `*dev` at the copy; otherwise (or for a NULL `src`) `*dev` is `src`.
template <class T>
int stage_in(bool host, const T* src, size_t n, DevBuf<T>& buf, cudaStream_t s, const T** dev) {
    *dev = src;
    if (!host || !src) return MXB_OK;
    const int rc = buf.grow(n, s);
    if (rc != MXB_OK) return rc;
    MXB_CUDA(cudaMemcpyAsync(buf.get(), src, sizeof(T) * n, cudaMemcpyHostToDevice, s));
    *dev = buf.get();
    return MXB_OK;
}
// stage_out: with `host` set, points `*dev` at `buf` grown to `n` elements (the caller copies the results back to
// `dst`); otherwise (or for a NULL `dst`) `*dev` is `dst`.
template <class T>
int stage_out(bool host, T* dst, size_t n, DevBuf<T>& buf, cudaStream_t s, T** dev) {
    *dev = dst;
    if (!host || !dst) return MXB_OK;
    const int rc = buf.grow(n, s);
    if (rc != MXB_OK) return rc;
    *dev = buf.get();
    return MXB_OK;
}

}  // namespace mxb

struct mxb_ctx {
    int device;
    int sample_rate;
    int sm_count;
    int cc_major, cc_minor;
    int smem_optin;          // cudaDevAttrMaxSharedMemoryPerBlockOptin: the most shared memory one CTA may opt in to
    mxb::DevBuf<double> d_sine;      // sineBuffer[514] ++ transition[1001] of the reference (mxb_ctx_set_tables), or empty
    double sine_before;
};
#endif  // __CUDACC_RTC__
