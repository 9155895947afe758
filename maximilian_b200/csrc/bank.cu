// Voice bank host side: handles, parameter upload, coefficient design (the reference's formulas, run once
// per parameter change on the host with the same libm the reference uses), launches.
#include <math.h>
#include <algorithm>

#include <new>
#include <thread>
#include <type_traits>

#include "bank_kernels.cuh"
#include "delay_kernels.cuh"
#include "exchange.cuh"
#include "filter_design.cuh"

using namespace mxb;

struct mxb_bank {
    mxb_ctx* ctx;
    mxb_bank_desc desc;
    int V;
    bool set_mask[MXB_P_COUNT];
    std::vector<double> hp[MXB_P_COUNT];     // host copies of the parameter arrays (coefficient design input)
    double* dp[MXB_P_COUNT];                 // device copies: the buffer the next block reads (== dp_buf[id][dp_cur[id]])
    // Block-rate control data uploaded with mxb_bank_set_param_async from host memory is double-buffered: the copy of block
    // k+1's values runs on a private copy stream into the buffer block k is NOT reading, so it overlaps block k's kernel.
    DevBuf<double> dp_buf[MXB_P_COUNT][2];   // [1] allocated on first asynchronous host upload
    int dp_cur[MXB_P_COUNT];
    bool dp_pending[MXB_P_COUNT];            // an upload into dp_buf[id][1 - cur] is in flight: the next block flips to it
    cudaEvent_t ev_up[MXB_P_COUNT];          // upload finished (copy stream)
    cudaEvent_t ev_read[MXB_P_COUNT][2];     // last kernel that read dp_buf[id][k] finished (process stream)
    bool ev_read_set[MXB_P_COUNT][2];
    cudaStream_t up_stream;
    DevBuf<double> osc_out;
    DevBuf<double> f0, f1, f2, cf[5];
    DevBuf<double> env_amp, env_output;
    DevBuf<long long> env_holdcount, env_hold;
    DevBuf<int> env_flags;
    DevBuf<int> trig_on, trig_off;           // staging for MXB_MEM_HOST gates
    DevBuf<int> dl_phase, dl_size, dl_pos;
    DevBuf<double> ring;                     // [V][delay_taps]
    DevBuf<double> partials;
    DevBuf<double> mix_dev;                  // [max_frames][2]
    DevBuf<unsigned char> out_stage;         // staging for MXB_MEM_HOST out (bytes: fp64 or fp32)
    DevBuf<double> fm_stage;                 // staging for host-resident per-sample frequencies
    DevBuf<double> cm_stage;                 // ... and cutoffs
    DevBuf<double> ds_stage;                 // ... and delay sizes
    DevBuf<unsigned char> tv_stage;          // ... and per-sample triggers
    int64_t launches;
    mxb_exchange* ex;                        // peer-memory mix exchange (multi-GPU), or NULL

    ~mxb_bank() {
        for (int i = 0; i < MXB_P_COUNT; ++i) {
            if (ev_up[i]) cudaEventDestroy(ev_up[i]);
            for (auto e : ev_read[i]) if (e) cudaEventDestroy(e);
        }
        if (up_stream) cudaStreamDestroy(up_stream);
    }
};

namespace {

// coefficient design, once per parameter change, on the host with the libm the reference calls (filter_design.cuh holds the
// reference's formulas, shared with the per-sample device design of patch stages)
void design_lores(const mxb_bank* b, std::vector<double>* cf, const int v_lo, const int v_hi) {
    const double sr = (double)(size_t)b->ctx->sample_rate;
    for (int v = v_lo; v < v_hi; ++v) design_lores_one(b->hp[MXB_P_CUTOFF][v], b->hp[MXB_P_RESONANCE][v], sr, cf[0][v], cf[1][v]);
}
void design_svf(const mxb_bank* b, std::vector<double>* cf, const int v_lo, const int v_hi) {
    const double sr = (double)(size_t)b->ctx->sample_rate;
    for (int v = v_lo; v < v_hi; ++v) {
        double c[5];
        design_svf_one(b->hp[MXB_P_CUTOFF][v], b->hp[MXB_P_RESONANCE][v], sr, c);
        for (int i = 0; i < 5; ++i) cf[i][v] = c[i];
    }
}
void design_biquad(const mxb_bank* b, std::vector<double>* cf, const int v_lo, const int v_hi) {
    const double sr = (double)(size_t)b->ctx->sample_rate;
    for (int v = v_lo; v < v_hi; ++v) {
        double c[5];
        design_biquad_one(b->desc.biquad_type, b->hp[MXB_P_CUTOFF][v], b->hp[MXB_P_RESONANCE][v], b->hp[MXB_P_GAIN][v], sr, c);
        for (int i = 0; i < 5; ++i) cf[i][v] = c[i];
    }
}

int redesign(mxb_bank* b) {
    const int fk = b->desc.filt_kind;
    if (fk == MXB_FILT_NONE) return MXB_OK;
    if ((fk == MXB_FILT_LORES || fk == MXB_FILT_HIRES) && !(b->set_mask[MXB_P_CUTOFF] && b->set_mask[MXB_P_RESONANCE])) return MXB_OK;
    if (fk == MXB_FILT_BIQUAD && !(b->set_mask[MXB_P_CUTOFF] && b->set_mask[MXB_P_RESONANCE])) return MXB_OK;   // untouched maxiBiquad: all-zero coefficients
    std::vector<double> cf[5];
    for (auto& c : cf) c.assign((size_t)b->V, 0.0);
    // the design runs on the host with the libm the reference calls (bit-identical coefficients); a large bank is split
    // over host threads (voices are independent), so that one cutoff change on 1 Mi voices costs a block, not dozens
    auto part = [&](int lo, int hi) {
        if (fk == MXB_FILT_LORES || fk == MXB_FILT_HIRES) design_lores(b, cf, lo, hi);
        else if (fk == MXB_FILT_SVF) design_svf(b, cf, lo, hi);
        else design_biquad(b, cf, lo, hi);
    };
    const unsigned hw = std::thread::hardware_concurrency();
    const int nt = b->V < 32768 ? 1 : (int)std::min<unsigned>(hw ? hw : 1u, 32u);
    if (nt <= 1) part(0, b->V);
    else {
        std::vector<std::thread> ts;
        for (int i = 0; i < nt; ++i) ts.emplace_back(part, (int)((long long)b->V * i / nt), (int)((long long)b->V * (i + 1) / nt));
        for (auto& t : ts) t.join();
    }
    for (int i = 0; i < 5; ++i) MXB_CUDA(cudaMemcpy(b->cf[i].get(), cf[i].data(), sizeof(double) * (size_t)b->V, cudaMemcpyHostToDevice));
    return MXB_OK;
}

// ring slots [0, n) of one voice <-> a linear array (set != 0: linear -> ring)
__global__ void ring_linear_kernel(double* __restrict__ ring, size_t V, size_t voice, double* __restrict__ lin, int n, int set) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    if (set) ring[dl_slot(V, voice, r)] = lin[r]; else lin[r] = ring[dl_slot(V, voice, r)];
}

// the fp64 state array of a state id (MXB_S_*), or NULL for the integer ones and unknown ids
double* f64_state(mxb_bank* b, int32_t id) {
    switch (id) {
        case MXB_S_FILT_0: return b->f0.get();
        case MXB_S_FILT_1: return b->f1.get();
        case MXB_S_FILT_2: return b->f2.get();
        case MXB_S_ENV_AMPLITUDE: return b->env_amp.get();
        case MXB_S_ENV_OUTPUT: return b->env_output.get();
        case MXB_S_OSC_OUTPUT: return b->osc_out.get();
        default: return nullptr;
    }
}

int upload_fill(double* dst, size_t n, double value) {
    std::vector<double> h(n, value);
    MXB_CUDA(cudaMemcpy(dst, h.data(), sizeof(double) * n, cudaMemcpyHostToDevice));
    return MXB_OK;
}

// Calls launch(std::integral_constant<int, filt_t>()) for a filter family FILT_T_*: the one place that maps a family to the
// instantiations built for it (launch_bank_filt, launch_delay_filt; build.py builds one object per family)
template <class L>
int with_filt(const int filt_t, L&& launch) {
    switch (filt_t) {
        case FILT_T_NONE:   return launch(std::integral_constant<int, FILT_T_NONE>());
        case FILT_T_LORES:  return launch(std::integral_constant<int, FILT_T_LORES>());
        case FILT_T_HIRES:  return launch(std::integral_constant<int, FILT_T_HIRES>());
        case FILT_T_SVF:    return launch(std::integral_constant<int, FILT_T_SVF>());
        case FILT_T_SVF_LP: return launch(std::integral_constant<int, FILT_T_SVF_LP>());
        case FILT_T_BIQUAD: return launch(std::integral_constant<int, FILT_T_BIQUAD>());
        default: break;
    }
    set_error("bank: filter family %d", filt_t);
    return MXB_ERR_UNSUPPORTED;
}

}  // namespace

extern "C" {

int32_t mxb_bank_create(mxb_ctx* ctx, const mxb_bank_desc* d, mxb_bank** out) {
    MXB_REQUIRE(ctx && d && out, MXB_ERR_INVALID, "mxb_bank_create: NULL argument");
    *out = nullptr;
    MXB_REQUIRE(d->voices > 0, MXB_ERR_INVALID, "mxb_bank_create: voices %d", d->voices);
    MXB_REQUIRE(d->osc_kind >= MXB_OSC_SINEWAVE && d->osc_kind <= MXB_OSC_PHASORBETWEEN, MXB_ERR_INVALID, "mxb_bank_create: osc_kind %d", d->osc_kind);
    MXB_REQUIRE(d->filt_kind >= MXB_FILT_NONE && d->filt_kind <= MXB_FILT_BIQUAD, MXB_ERR_INVALID, "mxb_bank_create: filt_kind %d", d->filt_kind);
    MXB_REQUIRE(d->biquad_type >= MXB_BQ_LOWPASS && d->biquad_type <= MXB_BQ_HIGHSHELF, MXB_ERR_INVALID, "mxb_bank_create: biquad_type %d", d->biquad_type);
    MXB_REQUIRE(d->env_kind == MXB_ENV_NONE || d->env_kind == MXB_ENV_ADSR || d->env_kind == MXB_ENV_AR, MXB_ERR_INVALID, "mxb_bank_create: env_kind %d", d->env_kind);
    MXB_REQUIRE(d->delay_mode == MXB_DELAY_DL || d->delay_mode == MXB_DELAY_FROM_POSITION, MXB_ERR_INVALID, "mxb_bank_create: delay_mode %d", d->delay_mode);
    MXB_REQUIRE(d->delay_taps >= 0, MXB_ERR_INVALID, "mxb_bank_create: delay_taps %d", d->delay_taps);
    MXB_REQUIRE(d->max_frames > 0, MXB_ERR_INVALID, "mxb_bank_create: max_frames %d", d->max_frames);
    DeviceGuard g(ctx->device);
    MXB_REQUIRE(g.ok, MXB_ERR_CUDA, "mxb_bank_create: cudaSetDevice failed");
    std::unique_ptr<mxb_bank> b(new (std::nothrow) mxb_bank());
    MXB_REQUIRE(b, MXB_ERR_ALLOC, "mxb_bank_create: out of host memory");
    b->ctx = ctx; b->desc = *d; b->V = d->voices;           // every other member is value-initialised: zero / NULL
    const size_t V = (size_t)d->voices;
    int rc = MXB_OK;
    static const double defaults[MXB_P_COUNT] = {0, 0, 0.5, 1000.0, 1.0, 0, 0, 0, 0, 0, 1.0, 1.0, 0, 0.5, 0, 0, 1.0};
    for (int i = 0; i < MXB_P_COUNT && rc == MXB_OK; ++i) {
        rc = b->dp_buf[i][0].alloc(V);
        b->dp[i] = b->dp_buf[i][0].get();
        b->hp[i].assign(V, defaults[i]);
        if (rc == MXB_OK && defaults[i] != 0.0) rc = upload_fill(b->dp[i], V, defaults[i]);
    }
    if (rc == MXB_OK) rc = b->osc_out.alloc(V);
    if (rc == MXB_OK) rc = b->f0.alloc(V);
    if (rc == MXB_OK) rc = b->f1.alloc(V);
    if (rc == MXB_OK) rc = b->f2.alloc(V);
    for (int i = 0; i < 5 && rc == MXB_OK; ++i) rc = b->cf[i].alloc(V);
    if (rc == MXB_OK) rc = b->env_amp.alloc(V);
    if (rc == MXB_OK) rc = b->env_output.alloc(V);
    if (rc == MXB_OK) rc = b->env_holdcount.alloc(V);
    if (rc == MXB_OK) rc = b->env_flags.alloc(V);
    if (rc == MXB_OK) rc = b->env_hold.upload(std::vector<long long>(V, 1));      // maxiEnv::holdtime = 1, src/maximilian.h:913
    if (rc == MXB_OK) rc = b->trig_on.alloc(V);
    if (rc == MXB_OK) rc = b->trig_off.alloc(V);
    if (rc == MXB_OK) rc = b->mix_dev.alloc((size_t)d->max_frames * 2);
    if (rc == MXB_OK && d->delay_taps > 0) {
        rc = b->dl_phase.alloc(V);
        if (rc == MXB_OK) rc = b->dl_pos.alloc(V);
        if (rc == MXB_OK) rc = b->dl_size.upload(std::vector<int>(V, 1));
        if (rc == MXB_OK) rc = b->ring.alloc(dl_ring_doubles(V, d->delay_taps));   // zeroed: maxiDelayline ctor memset, src/maximilian.cpp:415-417
    }
    if (rc == MXB_OK && d->filt_kind == MXB_FILT_SVF) {          // maxiSVF ctor: setParams(1000, 1), src/maximilian.h:1284
        b->set_mask[MXB_P_CUTOFF] = b->set_mask[MXB_P_RESONANCE] = true;
        rc = redesign(b.get());
        b->set_mask[MXB_P_CUTOFF] = b->set_mask[MXB_P_RESONANCE] = false;
    }
    if (rc != MXB_OK) return rc;
    *out = b.release();
    return MXB_OK;
}

int32_t mxb_bank_destroy(mxb_bank* b) {
    if (!b) return MXB_OK;
    DeviceGuard g(b->ctx->device);
    cudaDeviceSynchronize();
    delete b;
    return MXB_OK;
}

int32_t mxb_bank_voices(const mxb_bank* b) { return b ? b->V : MXB_ERR_INVALID; }

int32_t mxb_bank_set_exchange(mxb_bank* b, mxb_exchange* ex) {
    MXB_REQUIRE(b, MXB_ERR_INVALID, "mxb_bank_set_exchange: NULL bank");
    const int rc = mix_bus_attach(ex, b->ctx->device, "mxb_bank_set_exchange");
    if (rc != MXB_OK) return rc;
    b->ex = ex;
    return MXB_OK;
}
int64_t mxb_bank_launch_count(const mxb_bank* b) { return b ? b->launches : 0; }

int32_t mxb_bank_set_param(mxb_bank* b, int32_t id, const double* values, int32_t mem) {
    MXB_REQUIRE(b && values, MXB_ERR_INVALID, "mxb_bank_set_param: NULL argument");
    MXB_REQUIRE(id >= 0 && id < MXB_P_COUNT, MXB_ERR_INVALID, "mxb_bank_set_param: unknown id %d", id);
    MXB_REQUIRE(mem == MXB_MEM_HOST || mem == MXB_MEM_DEVICE, MXB_ERR_INVALID, "mxb_bank_set_param: mem %d", mem);
    DeviceGuard g(b->ctx->device);
    const size_t V = (size_t)b->V, bytes = sizeof(double) * V;
    // Parameters change between blocks. The copies below run on the legacy default stream: they are ordered after every
    // block already enqueued on it or on any other blocking stream; a caller driving the bank from a NON-blocking stream
    // synchronises that stream first. An asynchronous upload still in flight for this id is superseded.
    if (b->dp_pending[id]) { MXB_CUDA(cudaEventSynchronize(b->ev_up[id])); b->dp_pending[id] = false; }
    if (mem == MXB_MEM_HOST) {
        memcpy(b->hp[id].data(), values, bytes);
        MXB_CUDA(cudaMemcpy(b->dp[id], values, bytes, cudaMemcpyHostToDevice));
    } else {
        MXB_CUDA(cudaMemcpy(b->dp[id], values, bytes, cudaMemcpyDeviceToDevice));
        MXB_CUDA(cudaMemcpy(b->hp[id].data(), values, bytes, cudaMemcpyDeviceToHost));
    }
    b->set_mask[id] = true;
    if (id == MXB_P_CUTOFF || id == MXB_P_RESONANCE || id == MXB_P_GAIN) {
        int rc = redesign(b);
        if (rc != MXB_OK) return rc;
    } else if (id == MXB_P_ENV_HOLDTIME) {
        std::vector<long long> h(V);
        for (size_t v = 0; v < V; ++v) {
            // the kernels count holdcount/holdtime in 32-bit registers (holdcount never passes holdtime)
            MXB_REQUIRE(fabs(b->hp[id][v]) < 2147483648.0, MXB_ERR_INVALID, "mxb_bank_set_param: holdtime %.0f of voice %zu does not fit 32 bits", b->hp[id][v], v);
            h[v] = (long long)b->hp[id][v];
        }
        MXB_CUDA(cudaMemcpy(b->env_hold.get(), h.data(), sizeof(long long) * V, cudaMemcpyHostToDevice));
    } else if (id == MXB_P_DELAY_POSITION && b->dl_pos.get()) {
        std::vector<int> h(V);
        for (size_t v = 0; v < V; ++v) {
            const double s = b->hp[id][v];
            MXB_REQUIRE(fabs(s) < 2147483648.0, MXB_ERR_INVALID, "mxb_bank_set_param: delay position %.0f of voice %zu does not fit an int", s, v);
            h[v] = (int)s;
        }
        MXB_CUDA(cudaMemcpy(b->dl_pos.get(), h.data(), sizeof(int) * V, cudaMemcpyHostToDevice));
    } else if (id == MXB_P_DELAY_SIZE && b->dl_size.get()) {
        std::vector<int> h(V);
        for (size_t v = 0; v < V; ++v) {
            const double s = b->hp[id][v];
            // the reference takes any int (size <= 0 pins the index to slot 0); NaN / out-of-int values have no int conversion
            MXB_REQUIRE(s == s && s > -2147483649.0 && s <= (double)b->desc.delay_taps, MXB_ERR_INVALID,
                        "mxb_bank_set_param: delay size %g of voice %zu is not an int <= delay_taps %d", s, v, b->desc.delay_taps);
            h[v] = (int)s;
        }
        MXB_CUDA(cudaMemcpy(b->dl_size.get(), h.data(), sizeof(int) * V, cudaMemcpyHostToDevice));
    }
    return MXB_OK;
}

int32_t mxb_bank_set_param_async(mxb_bank* b, int32_t id, const double* values, int32_t mem, void* stream_) {
    MXB_REQUIRE(b && values, MXB_ERR_INVALID, "mxb_bank_set_param_async: NULL argument");
    MXB_REQUIRE(id >= 0 && id < MXB_P_COUNT, MXB_ERR_INVALID, "mxb_bank_set_param_async: unknown id %d", id);
    MXB_REQUIRE(mem == MXB_MEM_HOST || mem == MXB_MEM_DEVICE, MXB_ERR_INVALID, "mxb_bank_set_param_async: mem %d", mem);
    const bool needs_host_pass = id == MXB_P_CUTOFF || id == MXB_P_RESONANCE || id == MXB_P_GAIN ||
                                 id == MXB_P_ENV_HOLDTIME || id == MXB_P_DELAY_SIZE || id == MXB_P_DELAY_POSITION;
    if (needs_host_pass) return mxb_bank_set_param(b, id, values, mem);      // coefficient design / integer conversion on the host
    DeviceGuard g(b->ctx->device);
    const size_t bytes = sizeof(double) * (size_t)b->V;
    if (mem == MXB_MEM_DEVICE) {
        // the source was produced on `stream`: one stream-ordered device copy into the buffer the next block reads. A host
        // upload still pending for this id is older and is dropped, so that the next block does not switch to its values: its
        // copy lands in the other buffer, which nothing reads before the next host upload, queued after it on the copy stream.
        b->dp_pending[id] = false;
        MXB_CUDA(cudaMemcpyAsync(b->dp[id], values, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream_));
        b->set_mask[id] = true;
        return MXB_OK;
    }
    // Host source: the upload goes to the buffer the running / enqueued blocks do NOT read, on the bank's own copy stream,
    // so it overlaps them; the next mxb_bank_process waits for it (event) and switches over. The copy waits for the event
    // recorded when the blocks last switched away from that buffer, i.e. for the end of every block that read it.
    if (!b->up_stream) MXB_CUDA(cudaStreamCreateWithFlags(&b->up_stream, cudaStreamNonBlocking));
    if (!b->ev_up[id]) MXB_CUDA(cudaEventCreateWithFlags(&b->ev_up[id], cudaEventDisableTiming));
    const int tgt = 1 - b->dp_cur[id];
    if (!b->dp_buf[id][tgt].get()) { int rc = b->dp_buf[id][tgt].alloc((size_t)b->V, false); if (rc != MXB_OK) return rc; }
    if (b->ev_read_set[id][tgt]) MXB_CUDA(cudaStreamWaitEvent(b->up_stream, b->ev_read[id][tgt], 0));
    MXB_CUDA(cudaMemcpyAsync(b->dp_buf[id][tgt].get(), values, bytes, cudaMemcpyHostToDevice, b->up_stream));
    MXB_CUDA(cudaEventRecord(b->ev_up[id], b->up_stream));
    b->dp_pending[id] = true;
    b->set_mask[id] = true;
    return MXB_OK;
}

int32_t mxb_bank_get_state(mxb_bank* b, int32_t id, double* values, int32_t mem) {
    MXB_REQUIRE(b && values, MXB_ERR_INVALID, "mxb_bank_get_state: NULL argument");
    MXB_REQUIRE(mem == MXB_MEM_HOST || mem == MXB_MEM_DEVICE, MXB_ERR_INVALID, "mxb_bank_get_state: mem %d", mem);
    DeviceGuard g(b->ctx->device);
    MXB_CUDA(cudaDeviceSynchronize());
    const size_t V = (size_t)b->V;
    const cudaMemcpyKind kind = mem == MXB_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    const double* src = id >= 0 && id < MXB_P_COUNT ? b->dp[id] : f64_state(b, id);
    if (src) { MXB_CUDA(cudaMemcpy(values, src, sizeof(double) * V, kind)); return MXB_OK; }
    // integer state, returned as doubles
    std::vector<double> h(V, 0.0);
    if (id == MXB_S_ENV_HOLDCOUNT) {
        std::vector<long long> t(V);
        MXB_CUDA(cudaMemcpy(t.data(), b->env_holdcount.get(), sizeof(long long) * V, cudaMemcpyDeviceToHost));
        for (size_t v = 0; v < V; ++v) h[v] = (double)t[v];
    } else if (id == MXB_S_ENV_FLAGS || id == MXB_S_DELAY_PHASE) {
        const int* s = id == MXB_S_ENV_FLAGS ? b->env_flags.get() : b->dl_phase.get();
        if (s) {
            std::vector<int> t(V);
            MXB_CUDA(cudaMemcpy(t.data(), s, sizeof(int) * V, cudaMemcpyDeviceToHost));
            for (size_t v = 0; v < V; ++v) h[v] = (double)t[v];
        }
    } else {
        set_error("mxb_bank_get_state: unknown id %d", id);
        return MXB_ERR_INVALID;
    }
    MXB_CUDA(cudaMemcpy(values, h.data(), sizeof(double) * V, mem == MXB_MEM_HOST ? cudaMemcpyHostToHost : cudaMemcpyHostToDevice));
    return MXB_OK;
}

int32_t mxb_bank_get_ring(mxb_bank* b, int32_t voice, double* dst, int32_t n, int32_t mem) {
    MXB_REQUIRE(b && dst, MXB_ERR_INVALID, "mxb_bank_get_ring: NULL argument");
    MXB_REQUIRE(b->ring.get(), MXB_ERR_STATE, "mxb_bank_get_ring: bank has no delay line");
    MXB_REQUIRE(voice >= 0 && voice < b->V && n >= 0 && n <= b->desc.delay_taps, MXB_ERR_INVALID, "mxb_bank_get_ring: voice %d n %d", voice, n);
    MXB_REQUIRE(mem == MXB_MEM_HOST || mem == MXB_MEM_DEVICE, MXB_ERR_INVALID, "mxb_bank_get_ring: mem %d", mem);
    if (n == 0) return MXB_OK;
    DeviceGuard g(b->ctx->device);
    // the ring is chunk-interleaved and swizzled (delay_kernels.cuh): one small kernel walks the voice's slots
    DevBuf<double> tmp;
    double* d_lin = dst;
    if (mem == MXB_MEM_HOST) { int rc = tmp.alloc((size_t)n, false); if (rc != MXB_OK) return rc; d_lin = tmp.get(); }
    ring_linear_kernel<<<(n + 255) / 256, 256>>>(b->ring.get(), (size_t)b->V, (size_t)voice, d_lin, n, 0);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && mem == MXB_MEM_HOST) e = cudaMemcpy(dst, d_lin, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost);
    else if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { set_error("mxb_bank_get_ring: %s", cudaGetErrorString(e)); return MXB_ERR_CUDA; }
    return MXB_OK;
}

int32_t mxb_bank_set_ring(mxb_bank* b, int32_t voice, const double* src, int32_t n, int32_t mem) {
    MXB_REQUIRE(b && src, MXB_ERR_INVALID, "mxb_bank_set_ring: NULL argument");
    MXB_REQUIRE(b->ring.get(), MXB_ERR_STATE, "mxb_bank_set_ring: bank has no delay line");
    MXB_REQUIRE(voice >= 0 && voice < b->V && n >= 0 && n <= b->desc.delay_taps, MXB_ERR_INVALID, "mxb_bank_set_ring: voice %d n %d", voice, n);
    MXB_REQUIRE(mem == MXB_MEM_HOST || mem == MXB_MEM_DEVICE, MXB_ERR_INVALID, "mxb_bank_set_ring: mem %d", mem);
    if (n == 0) return MXB_OK;
    DeviceGuard g(b->ctx->device);
    DevBuf<double> tmp;
    double* d_lin = const_cast<double*>(src);
    if (mem == MXB_MEM_HOST) {
        int rc = tmp.alloc((size_t)n, false); if (rc != MXB_OK) return rc;
        d_lin = tmp.get();
        cudaError_t e0 = cudaMemcpy(d_lin, src, sizeof(double) * (size_t)n, cudaMemcpyHostToDevice);
        if (e0 != cudaSuccess) { set_error("mxb_bank_set_ring: %s", cudaGetErrorString(e0)); return MXB_ERR_CUDA; }
    }
    ring_linear_kernel<<<(n + 255) / 256, 256>>>(b->ring.get(), (size_t)b->V, (size_t)voice, d_lin, n, 1);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { set_error("mxb_bank_set_ring: %s", cudaGetErrorString(e)); return MXB_ERR_CUDA; }
    return MXB_OK;
}

int32_t mxb_bank_set_state(mxb_bank* b, int32_t id, const double* values, int32_t mem) {
    MXB_REQUIRE(b && values, MXB_ERR_INVALID, "mxb_bank_set_state: NULL argument");
    MXB_REQUIRE(mem == MXB_MEM_HOST || mem == MXB_MEM_DEVICE, MXB_ERR_INVALID, "mxb_bank_set_state: mem %d", mem);
    DeviceGuard g(b->ctx->device);
    MXB_CUDA(cudaDeviceSynchronize());
    const size_t V = (size_t)b->V;
    double* dst = f64_state(b, id);
    if (dst) {
        MXB_CUDA(cudaMemcpy(dst, values, sizeof(double) * V, mem == MXB_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice));
        return MXB_OK;
    }
    MXB_REQUIRE(id == MXB_S_ENV_HOLDCOUNT || id == MXB_S_ENV_FLAGS || id == MXB_S_DELAY_PHASE, MXB_ERR_INVALID,
                "mxb_bank_set_state: unknown id %d (parameters go through mxb_bank_set_param)", id);
    std::vector<double> h(V);                     // integer state arrives as doubles, like mxb_bank_get_state returns it
    MXB_CUDA(cudaMemcpy(h.data(), values, sizeof(double) * V, mem == MXB_MEM_HOST ? cudaMemcpyHostToHost : cudaMemcpyDeviceToHost));
    if (id == MXB_S_ENV_HOLDCOUNT) {
        std::vector<long long> t(V);
        for (size_t v = 0; v < V; ++v) {
            MXB_REQUIRE(fabs(h[v]) < 2147483648.0, MXB_ERR_INVALID, "mxb_bank_set_state: holdcount[%zu] = %g", v, h[v]);
            t[v] = (long long)h[v];
        }
        MXB_CUDA(cudaMemcpy(b->env_holdcount.get(), t.data(), sizeof(long long) * V, cudaMemcpyHostToDevice));
    } else {
        int* d = id == MXB_S_ENV_FLAGS ? b->env_flags.get() : b->dl_phase.get();
        MXB_REQUIRE(d, MXB_ERR_STATE, "mxb_bank_set_state: bank has no delay line");
        std::vector<int> t(V);
        for (size_t v = 0; v < V; ++v) {
            MXB_REQUIRE(fabs(h[v]) < 2147483648.0, MXB_ERR_INVALID, "mxb_bank_set_state: value[%zu] = %g", v, h[v]);
            // a negative ring index is an out-of-bounds access in the reference (memory[phase]); refused here
            if (id == MXB_S_DELAY_PHASE) MXB_REQUIRE(h[v] >= 0.0, MXB_ERR_INVALID, "mxb_bank_set_state: delay phase[%zu] = %g is negative", v, h[v]);
            t[v] = (int)h[v];
            if (id == MXB_S_ENV_FLAGS) t[v] &= 31;
        }
        MXB_CUDA(cudaMemcpy(d, t.data(), sizeof(int) * V, cudaMemcpyHostToDevice));
    }
    return MXB_OK;
}

// Deep copy: parameters, designed coefficients, every state array and the delay rings -- what copying an array of the
// reference's objects (they hold their state by value, src/maximilian.h:266-281) does. The copy lives on the same context.
int32_t mxb_bank_clone(mxb_bank* src, mxb_bank** out) {
    MXB_REQUIRE(src && out, MXB_ERR_INVALID, "mxb_bank_clone: NULL argument");
    *out = nullptr;
    mxb_bank* b = nullptr;
    int rc = mxb_bank_create(src->ctx, &src->desc, &b);
    if (rc != MXB_OK) return rc;
    DeviceGuard g(src->ctx->device);
    cudaError_t e = cudaDeviceSynchronize();
    // whole buffers; the two banks have the same description, so the same buffers of the same sizes
    auto cp = [&](auto& d, const auto& s) {
        if (e == cudaSuccess && d.get() && s.get()) e = cudaMemcpy(d.get(), s.get(), sizeof(*s.get()) * s.size(), cudaMemcpyDeviceToDevice);
    };
    for (int i = 0; i < MXB_P_COUNT; ++i) {     // the current parameter buffers (an upload still in flight on the source is not part of its state yet)
        b->hp[i] = src->hp[i]; b->set_mask[i] = src->set_mask[i];
        cp(b->dp_buf[i][0], src->dp_buf[i][src->dp_cur[i]]);
    }
    cp(b->osc_out, src->osc_out);
    cp(b->f0, src->f0); cp(b->f1, src->f1); cp(b->f2, src->f2);
    for (int i = 0; i < 5; ++i) cp(b->cf[i], src->cf[i]);
    cp(b->env_amp, src->env_amp); cp(b->env_output, src->env_output);
    cp(b->env_holdcount, src->env_holdcount); cp(b->env_hold, src->env_hold); cp(b->env_flags, src->env_flags);
    cp(b->dl_phase, src->dl_phase); cp(b->dl_size, src->dl_size); cp(b->dl_pos, src->dl_pos);
    cp(b->ring, src->ring);
    if (e != cudaSuccess) { set_error("mxb_bank_clone: %s", cudaGetErrorString(e)); mxb_bank_destroy(b); return MXB_ERR_CUDA; }
    *out = b;
    return MXB_OK;
}

int32_t mxb_bank_process(mxb_bank* b, int32_t n_frames, const int32_t* trig_on, const int32_t* trig_off,
                         void* out, int32_t out_dtype, double* mix, int32_t mem, void* stream_) {
    return mxb_bank_process_fm(b, n_frames, nullptr, trig_on, trig_off, out, out_dtype, mix, mem, stream_);
}

int32_t mxb_bank_process_fm(mxb_bank* b, int32_t n_frames, const double* freq_tv, const int32_t* trig_on, const int32_t* trig_off,
                            void* out, int32_t out_dtype, double* mix, int32_t mem, void* stream_) {
    mxb_modulation m; m.freq_tv = freq_tv; m.cutoff_tv = nullptr; m.delay_size_tv = nullptr; m.trig_tv = nullptr;
    return mxb_bank_process_mod(b, n_frames, &m, trig_on, trig_off, out, out_dtype, mix, mem, stream_);
}

int32_t mxb_bank_process_mod(mxb_bank* b, int32_t n_frames, const mxb_modulation* mod, const int32_t* trig_on, const int32_t* trig_off,
                             void* out, int32_t out_dtype, double* mix, int32_t mem, void* stream_) {
    NvtxRange nvtx_("mxb_bank_process_mod");
    MXB_REQUIRE(b, MXB_ERR_INVALID, "mxb_bank_process: NULL bank");
    const double* freq_tv = mod ? mod->freq_tv : nullptr;
    const double* cutoff_tv = mod ? mod->cutoff_tv : nullptr;
    const double* dsize_tv = mod ? mod->delay_size_tv : nullptr;
    const uint8_t* trig_tv = mod ? mod->trig_tv : nullptr;
    if (trig_tv) {
        MXB_REQUIRE(b->desc.env_kind != MXB_ENV_NONE, MXB_ERR_INVALID, "mxb_bank_process_mod: trig_tv on a bank without an envelope stage");
        MXB_REQUIRE(!trig_on && !trig_off, MXB_ERR_INVALID, "mxb_bank_process_mod: trig_tv replaces trig_on / trig_off (pass NULL for both)");
    }
    MXB_REQUIRE(n_frames >= 0 && n_frames <= b->desc.max_frames, MXB_ERR_INVALID, "mxb_bank_process: n_frames %d (max_frames %d)", n_frames, b->desc.max_frames);
    const bool async_host = (mem & MXB_MEM_ASYNC) != 0;   // host buffers, but return as soon as everything is enqueued
    mem &= ~MXB_MEM_ASYNC;
    MXB_REQUIRE(mem == MXB_MEM_HOST || mem == MXB_MEM_DEVICE || mem == MXB_MEM_SPLIT, MXB_ERR_INVALID, "mxb_bank_process: mem %d", mem);
    const bool host_ctl = mem != MXB_MEM_DEVICE;      // gates and mix in host memory
    const bool host_out = mem == MXB_MEM_HOST;        // out in host memory
    MXB_REQUIRE(out_dtype == MXB_F64 || out_dtype == MXB_F32, MXB_ERR_INVALID, "mxb_bank_process: out_dtype %d", out_dtype);
    MXB_REQUIRE((trig_on == nullptr) == (trig_off == nullptr), MXB_ERR_INVALID, "mxb_bank_process: trig_on/trig_off must both be given or both NULL");
    MXB_REQUIRE(out || mix, MXB_ERR_INVALID, "mxb_bank_process: neither out nor mix requested");
    const int fk = b->desc.filt_kind;
    if (fk == MXB_FILT_LORES || fk == MXB_FILT_HIRES)
        MXB_REQUIRE(b->set_mask[MXB_P_CUTOFF] && b->set_mask[MXB_P_RESONANCE], MXB_ERR_STATE,
                    "mxb_bank_process: lores/hires need MXB_P_CUTOFF and MXB_P_RESONANCE (they are call arguments in the reference)");
    if (mix) {     // before any kernel runs: a refused call must leave phase / filter / envelope / ring state untouched
        const int rc = mix_bus_admit(b->ex, n_frames, "mxb_bank_process");
        if (rc != MXB_OK) return rc;
    }
    if (n_frames == 0) return MXB_OK;
    DeviceGuard g(b->ctx->device);
    cudaStream_t s = (cudaStream_t)stream_;
    const size_t V = (size_t)b->V;
    const size_t esz = out_dtype == MXB_F32 ? 4 : 8;

    if (cutoff_tv)
        MXB_REQUIRE(fk == MXB_FILT_LORES || fk == MXB_FILT_HIRES || fk == MXB_FILT_SVF, MXB_ERR_UNSUPPORTED,
                    "mxb_bank_process_mod: per-sample cutoff is built for lores / hires / maxiSVF");
    if (dsize_tv)
        MXB_REQUIRE(b->desc.delay_taps > 0, MXB_ERR_UNSUPPORTED, "mxb_bank_process_mod: delay_size_tv on a bank without a delay line");
    // per-sample parameters are control data: they live where the gates live
    const size_t nv = (size_t)n_frames * V;
    const double *d_fm, *d_cm, *d_ds;
    const unsigned char* d_tv;
    const int *d_on, *d_off;
    unsigned char* d_out;
    double* d_mix;
    int rc = stage_in(host_ctl, freq_tv, nv, b->fm_stage, s, &d_fm);
    if (rc == MXB_OK) rc = stage_in(host_ctl, cutoff_tv, nv, b->cm_stage, s, &d_cm);
    if (rc == MXB_OK) rc = stage_in(host_ctl, dsize_tv, nv, b->ds_stage, s, &d_ds);
    if (rc == MXB_OK) rc = stage_in(host_ctl, trig_tv, nv, b->tv_stage, s, &d_tv);
    if (rc == MXB_OK) rc = stage_in(host_ctl, trig_on, V, b->trig_on, s, &d_on);
    if (rc == MXB_OK) rc = stage_in(host_ctl, trig_off, V, b->trig_off, s, &d_off);
    if (rc == MXB_OK) rc = stage_out(host_out, (unsigned char*)out, nv * esz, b->out_stage, s, &d_out);
    if (rc == MXB_OK) rc = stage_out(host_ctl, mix, (size_t)n_frames * 2, b->mix_dev, s, &d_mix);
    if (rc != MXB_OK) return rc;

    const int per_cta = kBankBlock * kBankVPT;
    const int grid = (int)((V + per_cta - 1) / per_cta);
    // warps that own at least one voice (warps past the end of the bank exit without writing partials)
    const int W = b->desc.delay_taps > 0 ? delay_bank_warps(b->V) : (int)((V + 32 * kBankVPT - 1) / (32 * kBankVPT));
    if (mix) {
        rc = b->partials.grow((size_t)b->desc.max_frames * 2 * (size_t)W, s);
        if (rc != MXB_OK) return rc;
    }

    for (int id = 0; id < MXB_P_COUNT; ++id) {
        if (!b->dp_pending[id]) continue;                 // an asynchronous host upload for this block: wait for it on the stream, switch over
        // every block that reads the old buffer is enqueued on `s` before this point: the event marks their end, and the next
        // upload into the old buffer waits for it
        const int old = b->dp_cur[id];
        if (!b->ev_read[id][old]) MXB_CUDA(cudaEventCreateWithFlags(&b->ev_read[id][old], cudaEventDisableTiming));
        MXB_CUDA(cudaEventRecord(b->ev_read[id][old], s));
        b->ev_read_set[id][old] = true;
        MXB_CUDA(cudaStreamWaitEvent(s, b->ev_up[id], 0));
        b->dp_cur[id] ^= 1; b->dp[id] = b->dp_buf[id][b->dp_cur[id]].get(); b->dp_pending[id] = false;
    }
    BankArgs a;
    memset(&a, 0, sizeof(a));
    a.V = b->V; a.n_frames = n_frames; a.osc_kind = b->desc.osc_kind;
    a.out_f32 = out_dtype == MXB_F32;
    a.vec_ok = (V % kBankVPT == 0) && d_out && (((uintptr_t)d_out) % (esz * kBankVPT) == 0);
    a.W = W;
    a.sr = (double)(size_t)b->ctx->sample_rate;
    for (int i = 0; i < 4; ++i) a.svf_mix[i] = b->desc.svf_mix[i];
    a.freq_tv = d_fm; a.cutoff_tv = d_cm; a.res = b->dp[MXB_P_RESONANCE];
    a.freq = b->dp[MXB_P_FREQ]; a.duty = b->dp[MXB_P_DUTY]; a.pstart = b->dp[MXB_P_PHASOR_START]; a.pend = b->dp[MXB_P_PHASOR_END]; a.phase = b->dp[MXB_P_PHASE]; a.osc_out = b->osc_out.get();
    a.f0 = b->f0.get(); a.f1 = b->f1.get(); a.f2 = b->f2.get();
    for (int i = 0; i < 5; ++i) a.cf[i] = b->cf[i].get();
    a.env_att = b->dp[MXB_P_ENV_ATTACK]; a.env_dec = b->dp[MXB_P_ENV_DECAY];
    a.env_sus = b->dp[MXB_P_ENV_SUSTAIN]; a.env_rel = b->dp[MXB_P_ENV_RELEASE];
    a.env_hold = b->env_hold.get(); a.env_amp = b->env_amp.get(); a.env_output = b->env_output.get();
    a.env_holdcount = b->env_holdcount.get(); a.env_flags = b->env_flags.get();
    a.trig_on = d_on; a.trig_off = d_off; a.trig_tv = d_tv;
    a.out = d_out; a.pan = b->dp[MXB_P_PAN]; a.partials = b->partials.get();

    int osc_t = OSC_T_GENERIC;
    if (b->desc.osc_kind == MXB_OSC_SINEWAVE) osc_t = OSC_T_SINE;
    else if (b->desc.osc_kind == MXB_OSC_PHASOR) osc_t = OSC_T_PHASOR;
    else if (b->desc.osc_kind == MXB_OSC_SAW) osc_t = OSC_T_SAW;
    const int env = b->desc.env_kind != MXB_ENV_NONE ? 1 : 0;
    a.env_ar = b->desc.env_kind == MXB_ENV_AR ? 1 : 0;
    // the filter family of the instantiations: the SVF with mix (1, 0, 0, 0) runs the low-pass-only one
    int filt_t = FILT_T_NONE;
    switch (fk) {
        case MXB_FILT_LORES:  filt_t = FILT_T_LORES; break;
        case MXB_FILT_HIRES:  filt_t = FILT_T_HIRES; break;
        case MXB_FILT_SVF:    filt_t = b->desc.svf_mix[0] == 1.0 && b->desc.svf_mix[1] == 0.0 && b->desc.svf_mix[2] == 0.0 &&
                                       b->desc.svf_mix[3] == 0.0 ? FILT_T_SVF_LP : FILT_T_SVF; break;
        case MXB_FILT_BIQUAD: filt_t = FILT_T_BIQUAD; break;
        default: break;
    }

    if (b->desc.delay_taps > 0) {
        DelayArgs da;
        da.phase = b->dl_phase.get(); da.size = b->dl_size.get(); da.feedback = b->dp[MXB_P_DELAY_FEEDBACK];
        da.ring = b->ring.get(); da.taps = b->desc.delay_taps;
        da.from_position = b->desc.delay_mode == MXB_DELAY_FROM_POSITION ? 1 : 0; da.position = b->dl_pos.get();
        da.size_tv = d_ds;
        const int saw = a.osc_kind == MXB_OSC_SAW;
        const int outmode = !out ? 0 : (a.out_f32 ? 2 : 1);      // DL_OUT_NONE / F64 / F32
        const bool modk = a.freq_tv || a.cutoff_tv;               // per-sample frequency / cutoff: the modulated instantiations
        rc = with_filt(filt_t, [&](auto f) {
            constexpr int F = decltype(f)::value;
            return modk ? launch_delay_filt<F, true>(a, da, saw, env, outmode, mix != nullptr, s)
                        : launch_delay_filt<F, false>(a, da, saw, env, outmode, mix != nullptr, s);
        });
    } else {
        const size_t smem = mix ? sizeof(double) * (kBankBlock / 32) * 2 * kMixTT * 33 : 0;
        rc = with_filt(filt_t, [&](auto f) {
            return launch_bank_filt<decltype(f)::value>(a, osc_t, env, out != nullptr, mix != nullptr, grid, smem, s);
        });
    }
    if (rc != MXB_OK) return rc;
    b->launches += 1;
    if (mix) {
        rc = mix_bus_reduce(b->ex, b->partials.get(), W, n_frames, d_mix, s);
        if (rc != MXB_OK) return rc;
        b->launches += 1;
    }
    if (host_ctl) {
        if (out && host_out) MXB_CUDA(cudaMemcpyAsync(out, d_out, (size_t)n_frames * V * esz, cudaMemcpyDeviceToHost, s));
        if (mix) MXB_CUDA(cudaMemcpyAsync(mix, d_mix, sizeof(double) * (size_t)n_frames * 2, cudaMemcpyDeviceToHost, s));
        if (async_host) return MXB_OK;            // results are valid once `stream` (or the context) has been synchronised
        MXB_CUDA(cudaStreamSynchronize(s));
        if (mix) return mix_bus_status(b->ex, "mxb_bank_process");      // the call is synchronous in this mode: a timed-out exchange is an error of THIS call
    }
    return MXB_OK;
}

// The block-dispatch shim: what routing() does for a reference patch (cpp/commandline/player.cpp:25-44) -- fill the audio
// driver's interleaved RTAUDIO_FLOAT64 buffer [n_frames][channels] with the next block: the bank's stereo bus goes to channels
// 0 and 1 (a mono device gets the left bus), further channels are silent.
int32_t mxb_play_block(mxb_bank* b, double* interleaved_out, int32_t n_frames, int32_t channels) {
    MXB_REQUIRE(b && interleaved_out, MXB_ERR_INVALID, "mxb_play_block: NULL argument");
    MXB_REQUIRE(channels >= 1 && n_frames >= 0, MXB_ERR_INVALID, "mxb_play_block: channels %d n_frames %d", channels, n_frames);
    if (channels == 2) return mxb_bank_process(b, n_frames, nullptr, nullptr, nullptr, MXB_F64, interleaved_out, MXB_MEM_HOST, nullptr);
    std::vector<double> bus((size_t)n_frames * 2);
    int rc = mxb_bank_process(b, n_frames, nullptr, nullptr, nullptr, MXB_F64, bus.data(), MXB_MEM_HOST, nullptr);
    if (rc != MXB_OK) return rc;
    for (int t = 0; t < n_frames; ++t)
        for (int c = 0; c < channels; ++c) interleaved_out[(size_t)t * channels + c] = c < 2 ? bus[(size_t)t * 2 + c] : 0.0;
    return MXB_OK;
}

}  // extern "C"
