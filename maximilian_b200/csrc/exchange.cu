// The mix bus (see exchange.cuh): the kernels that reduce the per-warp mix partials of a bank or a voice patch, and
// mxb_exchange, symmetric peer-memory buffers for the all-reduce of the bus between GPUs.
//
// Protocol (per call, sequence number s, slot = s & 1; every rank owns flags[world] + payload[2 slots][world][n], all
// peer-mapped with CUDA IPC). PUSH model -- nothing is ever read over NVLink, nobody polls remote memory:
//   1. every rank stores each locally reduced bus value into payload[slot][its rank] of EVERY rank's buffer (posted
//      peer stores, issued by the reducing warps as they finish), then -- once all of its CTAs are done -- publishes
//      flags[its rank] = s + 1 in every rank's buffer (release, system scope)
//   2. every rank waits on its OWN flags (local polling, acquire, system scope) until all of them reach s + 1 and adds
//      the world buses, all in local HBM, IN RANK ORDER -- every rank computes the same sum, bit for bit, every run
//   3. slot reuse at call s + 2 is safe: a rank finishes call s + 1 only after every peer's flag reached s + 2, i.e.
//      after every peer had launched call s + 1 and therefore finished reading slot(s) (stream order on the peer)
// One kernel does the local reduction and the exchange (mix_reduce_exchange_kernel); nothing here calls NCCL.
#include <new>

#include "exchange.cuh"

using namespace mxb;

namespace mxb {

constexpr int kExchMaxWorld = 16;
constexpr int kExchFlagBytes = 128;          // one flag per source rank, each alone in its line

// Every rank owns one buffer: flags[kExchMaxWorld] (128 B apart), then payload[2 slots][world][max_doubles].
// flags[r] / payload[slot][r] are WRITTEN BY RANK r (pushed over NVLink) and read only by the owner, locally.
struct ExchDev {                              // passed to the kernel by value
    double* dst_payload[kExchMaxWorld];       // [r]: payload[slot][my rank] inside rank r's buffer (own entry = local)
    unsigned long long* dst_flag[kExchMaxWorld];   // [r]: flags[my rank] inside rank r's buffer
    const double* src_payload;                // my buffer: payload[slot][0]
    const unsigned long long* src_flags;      // my buffer: flags[0]
    int rank, world, stride;                  // stride = max_doubles (doubles between two source ranks' payloads)
    unsigned long long seq1;                  // value the flags reach when this call's payload is published
    unsigned int* ticket;                     // last-CTA election
    unsigned int* status;                     // bit r set: rank r's flag did not arrive within timeout_ns (sticky)
    unsigned long long timeout_ns;            // bound of the flag wait
};

}  // namespace mxb

struct mxb_exchange {
    mxb_ctx* ctx;
    int rank, world, max_doubles;
    size_t flags_bytes, slot_bytes;           // slot = world * max_doubles doubles, 128-byte multiple
    mxb::DevBuf<unsigned char> local;         // flags + 2 slots; a plain cudaMalloc allocation, exportable with cudaIpcGetMemHandle
    unsigned char* peers[mxb::kExchMaxWorld]; // cudaIpcOpenMemHandle'd (own entry = local)
    bool connected;
    unsigned long long seq;                   // calls so far
    mxb::DevBuf<unsigned int> ticket;
    mxb::DevBuf<unsigned int> status;         // device word, see ExchDev::status
    unsigned long long timeout_ns;            // default 5 s; MXB_EXCHANGE_TIMEOUT_MS overrides

    ~mxb_exchange() {
        for (int r = 0; r < world; ++r)
            if (r != rank && peers[r]) cudaIpcCloseMemHandle(peers[r]);
    }
};

namespace {

constexpr int kMixReduceThreads = 128;

// Sum of one (frame, channel) row of per-warp partials by one CTA: every thread adds a strided subset in ascending
// order (two interleaved chains), a fixed xor tree per warp, then the four warp sums in a fixed order -- the
// summation order never changes between runs. Returned to every thread of warp 0; other warps get 0.
__device__ __forceinline__ double mix_row_sum(const double* __restrict__ p, const int W, double* sm) {
    double s0 = 0.0, s1 = 0.0;
    int w = threadIdx.x;
    for (; w + kMixReduceThreads < W; w += 2 * kMixReduceThreads) { s0 += p[w]; s1 += p[w + kMixReduceThreads]; }
    if (w < W) s0 += p[w];
    double s = s0 + s1;
#pragma unroll
    for (int m = 16; m >= 1; m >>= 1) s += __shfl_xor_sync(0xffffffffu, s, m);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
    __syncthreads();
    return threadIdx.x < 32 ? (sm[0] + sm[1]) + (sm[2] + sm[3]) : 0.0;
}

__global__ void __launch_bounds__(kMixReduceThreads) mix_reduce_kernel(const double* __restrict__ partials, double* __restrict__ mix, int rows, int W) {
    __shared__ double sm[kMixReduceThreads / 32];
    const int row = blockIdx.x;                       // one CTA per row: rows CTAs keep enough loads in flight for HBM
    const double s = mix_row_sum(partials + (size_t)row * (size_t)W, W, sm);
    if (threadIdx.x == 0) mix[row] = s;
}

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// K3 + K6 in one kernel: every row sum of the local reduction (as mix_reduce_kernel) is PUSHED into this rank's lane
// of every rank's exchange buffer over NVLink (posted stores); the last CTA to finish publishes the flags, waits on
// its own (local) flags for every peer and adds the world buses in rank order (protocol: top of this file).
__global__ void __launch_bounds__(kMixReduceThreads) mix_reduce_exchange_kernel(const double* __restrict__ partials, double* __restrict__ mix, int rows, int W, const ExchDev x) {
    __shared__ double sm[kMixReduceThreads / 32];
    const int row = blockIdx.x;
    const double s = mix_row_sum(partials + (size_t)row * (size_t)W, W, sm);
    if (threadIdx.x < x.world) x.dst_payload[threadIdx.x][row] = s;      // thread r -> rank r's buffer
    __shared__ bool last;
    __threadfence_system();                           // this CTA's peer stores are ordered before its ticket
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(x.ticket, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!last) return;
    if (threadIdx.x < x.world) {
        __threadfence_system();                       // cumulative: the other CTAs' stores were ordered before their tickets
        st_release_sys(x.dst_flag[threadIdx.x], x.seq1);
        // bounded wait: a peer that died (or never launched this block) costs timeout_ns, not a hung box; the bus is then
        // incomplete and bit `rank` of *status says whose part is missing (mxb_exchange_status / mix_bus_status report it)
        const unsigned long long t0 = globaltimer_ns();
        unsigned spins = 0;
        while (ld_acquire_sys(x.src_flags + (size_t)threadIdx.x * (kExchFlagBytes / sizeof(unsigned long long))) < x.seq1) {
            if ((++spins & 1023u) == 0 && globaltimer_ns() - t0 > x.timeout_ns) { atomicOr(x.status, 1u << threadIdx.x); break; }
        }
    }
    if (threadIdx.x == 0) *x.ticket = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < rows; i += blockDim.x) {
        double s = 0.0;
        for (int r = 0; r < x.world; ++r)             // rank order on every rank: identical bits everywhere, every run
            s += __ldcg(x.src_payload + (size_t)r * (size_t)x.stride + i);
        mix[i] = s;
    }
}

// fills the device descriptor for the next call and advances the sequence
ExchDev exchange_next(mxb_exchange* ex) {
    ExchDev d;
    memset(&d, 0, sizeof(d));
    const size_t slot_off = ex->flags_bytes + (size_t)(ex->seq & 1) * ex->slot_bytes;
    d.rank = ex->rank; d.world = ex->world; d.stride = ex->max_doubles; d.seq1 = ex->seq + 1; d.ticket = ex->ticket.get(); d.status = ex->status.get(); d.timeout_ns = ex->timeout_ns;
    for (int r = 0; r < ex->world; ++r) {
        d.dst_flag[r] = (unsigned long long*)(ex->peers[r] + (size_t)ex->rank * kExchFlagBytes);
        d.dst_payload[r] = (double*)(ex->peers[r] + slot_off) + (size_t)ex->rank * (size_t)ex->max_doubles;
    }
    d.src_flags = (const unsigned long long*)ex->local.get();
    d.src_payload = (const double*)(ex->local.get() + slot_off);
    ex->seq += 1;
    return d;
}

}  // namespace

namespace mxb {

int mix_bus_attach(const mxb_exchange* ex, int device, const char* who) {
    if (ex) MXB_REQUIRE(ex->ctx->device == device, MXB_ERR_INVALID, "%s: the exchange lives on device %d, the caller on device %d", who, ex->ctx->device, device);
    return MXB_OK;
}

int mix_bus_admit(const mxb_exchange* ex, int n_frames, const char* who) {
    if (!ex) return MXB_OK;
    MXB_REQUIRE(ex->connected, MXB_ERR_STATE, "%s: the attached exchange is not connected to its peers", who);
    MXB_REQUIRE(n_frames * 2 <= ex->max_doubles, MXB_ERR_INVALID, "%s: exchange holds %d values, the bus needs %d", who, ex->max_doubles, n_frames * 2);
    return MXB_OK;
}

int mix_bus_reduce(mxb_exchange* ex, const double* partials, int W, int n_frames, double* mix, cudaStream_t s) {
    const int rows = n_frames * 2;      // one CTA per (frame, channel) row
    if (ex) mix_reduce_exchange_kernel<<<rows, kMixReduceThreads, 0, s>>>(partials, mix, rows, W, exchange_next(ex));
    else mix_reduce_kernel<<<rows, kMixReduceThreads, 0, s>>>(partials, mix, rows, W);
    MXB_CUDA(cudaGetLastError());
    return MXB_OK;
}

int mix_bus_status(mxb_exchange* ex, const char* who) {
    if (!ex) return MXB_OK;
    int32_t m = 0;
    const int rc = mxb_exchange_status(ex, &m);
    if (rc != MXB_OK) return rc;
    MXB_REQUIRE(m == 0, MXB_ERR_STATE, "%s: mix exchange timed out waiting for rank mask 0x%x (bus incomplete)", who, (unsigned)m);
    return MXB_OK;
}

}  // namespace mxb

extern "C" {

int32_t mxb_exchange_create(mxb_ctx* ctx, int32_t rank, int32_t world, int32_t max_doubles, mxb_exchange** out) {
    MXB_REQUIRE(ctx && out, MXB_ERR_INVALID, "mxb_exchange_create: NULL argument");
    *out = nullptr;
    MXB_REQUIRE(world >= 1 && world <= kExchMaxWorld && rank >= 0 && rank < world, MXB_ERR_INVALID, "mxb_exchange_create: rank %d of %d", rank, world);
    MXB_REQUIRE(max_doubles > 0, MXB_ERR_INVALID, "mxb_exchange_create: max_doubles %d", max_doubles);
    DeviceGuard g(ctx->device);
    std::unique_ptr<mxb_exchange> ex(new (std::nothrow) mxb_exchange());
    MXB_REQUIRE(ex, MXB_ERR_ALLOC, "mxb_exchange_create: out of host memory");
    ex->ctx = ctx; ex->rank = rank; ex->world = world; ex->max_doubles = max_doubles;
    ex->flags_bytes = (size_t)kExchMaxWorld * kExchFlagBytes;
    ex->slot_bytes = (sizeof(double) * (size_t)max_doubles * (size_t)world + 127) & ~(size_t)127;
    int rc = ex->local.alloc(ex->flags_bytes + 2 * ex->slot_bytes);      // zero-filled, like ticket and status
    if (rc == MXB_OK) rc = ex->ticket.alloc(1);
    if (rc == MXB_OK) rc = ex->status.alloc(1);
    if (rc != MXB_OK) return rc;
    {   // a dead peer must not hang the others: the flag wait is bounded (the kernel then reports through `status`)
        const char* t = getenv("MXB_EXCHANGE_TIMEOUT_MS");
        const double ms = t ? atof(t) : 5000.0;
        ex->timeout_ns = (unsigned long long)((ms > 0.0 ? ms : 5000.0) * 1e6);
    }
    ex->peers[rank] = ex->local.get();
    ex->connected = (world == 1);
    *out = ex.release();
    return MXB_OK;
}

int32_t mxb_exchange_local_handle(mxb_exchange* ex, void* handle, int32_t handle_bytes) {
    MXB_REQUIRE(ex && handle, MXB_ERR_INVALID, "mxb_exchange_local_handle: NULL argument");
    MXB_REQUIRE(handle_bytes >= (int32_t)sizeof(cudaIpcMemHandle_t), MXB_ERR_INVALID, "mxb_exchange_local_handle: need %zu bytes", sizeof(cudaIpcMemHandle_t));
    DeviceGuard g(ex->ctx->device);
    cudaIpcMemHandle_t h;
    MXB_CUDA(cudaIpcGetMemHandle(&h, ex->local.get()));
    memcpy(handle, &h, sizeof(h));
    return MXB_OK;
}

int32_t mxb_exchange_connect(mxb_exchange* ex, const void* all_handles) {
    MXB_REQUIRE(ex && all_handles, MXB_ERR_INVALID, "mxb_exchange_connect: NULL argument");
    DeviceGuard g(ex->ctx->device);
    const unsigned char* hs = (const unsigned char*)all_handles;
    for (int r = 0; r < ex->world; ++r) {
        if (r == ex->rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, hs + (size_t)r * sizeof(h), sizeof(h));
        void* p = nullptr;
        MXB_CUDA(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
        ex->peers[r] = (unsigned char*)p;
    }
    ex->connected = true;
    return MXB_OK;
}

int32_t mxb_exchange_status(mxb_exchange* ex, int32_t* timed_out_ranks) {
    MXB_REQUIRE(ex && timed_out_ranks, MXB_ERR_INVALID, "mxb_exchange_status: NULL argument");
    DeviceGuard g(ex->ctx->device);
    unsigned int m = 0;
    MXB_CUDA(cudaMemcpy(&m, ex->status.get(), sizeof(m), cudaMemcpyDeviceToHost));      // synchronises with the kernels that may set it
    *timed_out_ranks = (int32_t)m;
    return MXB_OK;
}

int32_t mxb_exchange_destroy(mxb_exchange* ex) {
    if (!ex) return MXB_OK;
    DeviceGuard g(ex->ctx->device);
    cudaDeviceSynchronize();
    delete ex;
    return MXB_OK;
}

}  // extern "C"
