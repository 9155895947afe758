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
#include <vector>

#include "../../include/maxib200.h"

#include <nvtx3/nvToolsExt.h>      // header-only; ranges show up in nsys / ncu --nvtx timelines, cost nothing without a profiler

namespace mxb {

void set_error(const char* fmt, ...);

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

template <class T>
inline int dev_alloc(T** p, size_t n, bool zero = true) {
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, sizeof(T) * (n ? n : 1));
    if (e != cudaSuccess) { set_error("cudaMalloc(%zu bytes): %s", sizeof(T) * n, cudaGetErrorString(e)); return MXB_ERR_ALLOC; }
    if (zero) {
        e = cudaMemset(q, 0, sizeof(T) * (n ? n : 1));
        if (e != cudaSuccess) { set_error("cudaMemset: %s", cudaGetErrorString(e)); cudaFree(q); return MXB_ERR_CUDA; }
    }
    *p = (T*)q;
    return MXB_OK;
}

// Grows a staging buffer to at least `need` elements (contents not kept). Work queued on `s` may still read the old
// buffer, so `s` is synchronised before it is freed.
template <class T>
inline int ensure(T** p, size_t* len, size_t need, cudaStream_t s) {
    if (need <= *len) return MXB_OK;
    MXB_CUDA(cudaStreamSynchronize(s));
    cudaFree(*p); *p = nullptr; *len = 0;
    const int rc = dev_alloc(p, need, false);
    if (rc == MXB_OK) *len = need;
    return rc;
}

}  // namespace mxb

struct mxb_ctx {
    int device;
    int sample_rate;
    int sm_count;
    int cc_major, cc_minor;
    int smem_optin;          // cudaDevAttrMaxSharedMemoryPerBlockOptin: the most shared memory one CTA may opt in to
    double* d_sine;          // sineBuffer[514] ++ transition[1001] of the reference (mxb_ctx_set_tables), or NULL
    double sine_before;
};
#endif  // __CUDACC_RTC__
