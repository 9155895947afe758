// K2: oscillator -> [envelope] -> [filter] -> maxiDelayline::dl -> out / stereo mix.   (kernel template; delay_k.cu instantiates it,
// once per filter family and MODK)
//
// maxiDelayline::dl (src/maximilian.cpp:420-429) reads ring[phase] and writes it back every sample:
// 8 B read + 8 B write of ring traffic per voice-sample on top of the 8 B output -- the one genuinely
// HBM-bound stage of the path. A thread walking its own ring straight out of global memory would issue
// one 8-byte load per sample with 32 different lines per warp request; instead each WARP stages the next
// T = 16 ring slots of each of its 32 voices through shared memory, double-buffered:
//
//   prefetch k+1: uniform schedule: ONE bulk copy (cp.async.bulk.shared.global, SASS UBLKCP) of the warp's 4 KB run, completion
//                 on an mbarrier, in flight while window k is computed; generic schedule: 16 cp.async requests, two voices
//                 each (warp-private tiles, no __syncthreads anywhere)
//   compute k:    lane = voice; 16 steps of the chain, ring slot j of the window read and updated in smem
//                 (rows of 16 doubles, slot j at position j ^ (lane % 16) -- the swizzle of the HBM layout, so the uniform
//                 schedule's bulk image and the generic schedule's per-slot staging look the same: conflict-free for 64-bit accesses)
//   write-back:   uniform: one bulk copy smem -> HBM (cp.async.bulk.global.shared, bulk group); generic: per-slot stores
//
// Why 16 slots: 32-slot windows double-buffered leave few warps per SM, issue-starved; single-buffered they leave too few
// bytes in flight; 16-slot windows give both: more resident warps AND a prefetch in flight for every warp all the time.
//
// Two schedules share the per-step code:
//   * uniform: every voice of the warp has the same ring size (a multiple of 16) and the same, chunk-aligned
//     index -- voices started together, the common case. With the chunk-interleaved ring layout
//     (delay_kernels.cuh) the warp's 32 windows are ONE contiguous 4 KB run: address arithmetic collapses to
//     pointer increments and DRAM sees pure streaming.
//   * generic: any per-voice size / phase (ragged banks, rings that shrank between blocks): each window is
//     located per voice (wrap at `size`, chunk crossing), still 128 B per voice. Voices whose ring is
//     shorter than two windows (32 slots), and dlFromPosition, take the literal per-sample path against global memory.
//
// The ring index `phase` is an int and follows the reference statement for statement --
// `if (phase >= size) phase = 0` BEFORE the access -- so index sequences are bit-exact.
#pragma once
#include "delay_kernels.cuh"

namespace mxb {

constexpr int kDlT = kDlChunk;                    // steps per staged window
constexpr int kDlRow = kDlT;                      // tile row stride in doubles: unpadded, slot j of row i at position j ^ (i % 16)
constexpr int kStageDoubles = 32 * kDlRow;        // one staged window tile per warp (4 KB: the image one bulk copy moves)
// CTA shape of K2. Without a mix tile a warp needs 8 KB of staging: 4 warps per CTA, 24 warps per SM. Left alone,
// ptxas gives the block-constant kernels 96 registers on sm_90a, which leaves 20 warps per SM; the launch bound holds them to 80
// (a few bytes of spill) for the 24, which runs ~3 % faster on an H100. With the mix tile (8-row tile: 12.1 KB per warp with the
// two window stages) shared memory allows 4 CTAs of 4 warps per SM.
template <bool MIX> struct DelayShape {
    static constexpr int kThreads = 128;
    static constexpr int kMinCtas = (MIX ? 16 : 24) * 32 / kThreads;     // resident CTAs per SM the registers must allow
};
constexpr int kDlStages = 2;                      // staged windows per warp: window k + 1 is requested while window k is computed
constexpr int kDlVoicesPerReq = 32 / kDlT;        // voices covered by one cooperative request (2)
// Rows (steps) of the per-warp mix tile of K2. The tile costs shared memory the window stages compete for: with 16 rows a 4-warp CTA
// needs 65 KB (3 CTAs = 12 warps per SM), with 8 rows 48.5 KB (4 CTAs = 16 warps per SM) at twice the row-sum instructions -- K2 has
// the fp64 slots for them, unlike K1. The 8-row tile was the faster of the two for out + mix.
constexpr int kDlMixRows = 8;
constexpr int kMixDoubles = 2 * kDlMixRows * 33;
constexpr int kFastMinSize = 2 * kDlT;
constexpr unsigned kFull = 0xffffffffu;
enum { DL_OUT_NONE = 0, DL_OUT_F64 = 1, DL_OUT_F32 = 2 };
static_assert(kDlT % kDlMixRows == 0, "a staged window is a whole number of mix tiles");

__device__ __forceinline__ void cp_async8(double* smem_dst, const double* gsrc) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait1() { asm volatile("cp.async.wait_group 1;\n" ::: "memory"); }

// ---- bulk asynchronous copies (the TMA engine, 1-D form) with mbarrier completion ----
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* b, int count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* b, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* b, unsigned parity) {
    asm volatile("{\n.reg .pred p;\nMXB_WAIT_%=:\nmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n@p bra MXB_DONE_%=;\nbra MXB_WAIT_%=;\nMXB_DONE_%=:\n}"
                 ::"r"(smem_u32(b)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, unsigned bytes, unsigned long long* b) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, unsigned bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }   // sources read: smem reusable
__device__ __forceinline__ void bulk_wait_but7() { asm volatile("cp.async.bulk.wait_group 7;" ::: "memory"); }         // all but the latest 7 groups performed
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }           // writes performed
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

struct DlVoice {
    double phase, oout, inc, duty, pend, fb, gl, gr, res;
    FiltRegs fr;
    EnvRegs er;
    int ph, size, pos;
    bool live, fast;
};

// one window (<= 16 steps) of one voice against its staged row (ALLFAST) or, for short rings, against global memory
// ESTEADY: every voice of the warp spends this whole window in one of the two steady states of maxiEnv::adsr (see
// dl_window); `relmode` tells which one this lane is in.
// MODW: the block carries a per-sample oscillator frequency (a.freq_tv) and / or filter cutoff (a.cutoff_tv): the reference takes both
// by argument on every call (FM: maximilian_examples/5.FM1/main.cpp:29), so the increment / the filter design are redone each sample,
// in the order the patch evaluates them (oscillator, envelope, design, filter). Its own instantiation of the window body;
// modulated blocks run their own instantiation of the KERNEL (MODK; objects delay_km_*.o), so the block-constant kernels are compiled exactly
// as before (with both bodies in one kernel the headline instantiation was slower).
template <int OSC, int FILT, int ENV, bool ALLFAST, int OUTMODE, bool MIX, bool ESTEADY, bool MODW = false>
__device__ __forceinline__ void dl_stage(DlVoice& s, double* row, const int tn, const int t0, const BankArgs& a, const DelayArgs& d,
                                         const size_t V, const size_t v, const int lane, const int gwarp, double* mixtile,
                                         const bool relmode, const int swz) {
    double* out64 = (double*)a.out + (size_t)t0 * V + v;
    float* out32 = (float*)a.out + (size_t)t0 * V + v;
    for (int jb = 0; jb < tn; jb += kDlMixRows) {         // one mix tile
    const int jn = min(kDlMixRows, tn - jb);
#pragma unroll 4
    for (int jj = 0; jj < jn; ++jj) {
        const int j = jb + jj;
        const int t = t0 + j;
        if (MODW && a.freq_tv) {
            const bool pb = OSC == OSC_T_GENERIC && a.osc_kind == MXB_OSC_PHASORBETWEEN;
            if (s.live && t + kFmPrefetch < a.n_frames)          // look-ahead on the stream, as in K1
                asm volatile("prefetch.global.L2 [%0];" ::"l"(a.freq_tv + (size_t)(t + kFmPrefetch) * V + v));
            const double fq = s.live ? a.freq_tv[(size_t)t * V + v] : 1.0;
            s.inc = pb ? ((s.pend - s.duty) / (a.sr / fq)) : osc_increment(a.sr, fq);
        }
        double x = osc_tick<OSC>(s.phase, s.oout, s.inc, s.duty, a.osc_kind, s.pend);
        if (ENV && ESTEADY) {
            // what env_tick() reduces to in the steady states -- same operands, same roundings
            if (relmode) { if (s.er.amp > 0.) { s.er.amp *= s.er.rel; s.er.output = x * s.er.amp; } }
            else s.er.output = x * s.er.amp;
            x = s.er.output;
        } else if (ENV) {
            const bool trig = a.trig_tv ? (s.live && a.trig_tv[(size_t)t * V + v] == 1) : (t >= s.er.on && t < s.er.off);
            x = a.env_ar ? env_ar_tick(s.er, x, trig) : env_tick(s.er, x, trig);
        }
        if constexpr (MODW && (FILT == FILT_T_LORES || FILT == FILT_T_HIRES || FILT == FILT_T_SVF || FILT == FILT_T_SVF_LP)) {
            if (a.cutoff_tv) filt_design<FILT>(s.fr, s.live ? a.cutoff_tv[(size_t)t * V + v] : 1000.0, s.res, a.sr);
        }
        x = filt_tick<FILT>(s.fr, x, a.svf_mix);
        // maxiDelayline::dl, src/maximilian.cpp:420-429
        double y = 0.0;
        if (ALLFAST ? s.live : s.fast) {          // lanes past the end of the bank contribute an exact 0
            const double m = row[j ^ swz];             // swz = lane % 16: the swizzle of the staged image (and of the HBM layout)
            row[j ^ swz] = (m * s.fb) + (x * s.fb) * 0.5;
            y = m;
        } else if (!ALLFAST && s.live) {
            // `size` is an argument of every call in the reference: with size_tv a new one each sample (double -> int)
            const int sz = d.size_tv ? (int)d.size_tv[(size_t)t * V + v] : s.size;
            if (s.ph >= sz) s.ph = 0;
            const int idx = min(max(s.ph, 0), d.taps - 1);     // size <= taps: enforced for the parameter, the caller's contract for size_tv
            double* slot = d.ring + dl_slot(V, v, idx);
            const double m = *slot;
            if (d.from_position) {
                // maxiDelayline::dlFromPosition, src/maximilian.cpp:431-439: the output comes from `position`, the
                // write has chandiv (== 1) where dl() has 0.5
                int pos = s.pos;
                if (pos >= sz) pos = 0;
                y = d.ring[dl_slot(V, v, min(max(pos, 0), d.taps - 1))];
                *slot = (m * s.fb) + (x * s.fb) * 1.0;
            } else {
                *slot = (m * s.fb) + (x * s.fb) * 0.5;
                y = m;
            }
            s.ph += 1;
        }
        if (OUTMODE == DL_OUT_F64) { if (s.live) __stcs(out64, y); out64 += V; }
        if (OUTMODE == DL_OUT_F32) { if (s.live) __stcs(out32, (float)y); out32 += V; }
        if (MIX) {
            mixtile[(0 * kDlMixRows + jj) * 33 + lane] = y * s.gl;
            mixtile[(1 * kDlMixRows + jj) * 33 + lane] = y * s.gr;
        }
    }
    if (MIX) {
        __syncwarp();
        const int ch = lane / kDlMixRows, rw = lane % kDlMixRows;
        if (ch < 2 && rw < jn) {
            const double* r = mixtile + (ch * kDlMixRows + rw) * 33;
            double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;       // fixed order: deterministic
#pragma unroll
            for (int q = 0; q < 32; q += 4) { s0 += r[q]; s1 += r[q + 1]; s2 += r[q + 2]; s3 += r[q + 3]; }
            a.partials[((size_t)(t0 + jb + rw) * 2 + ch) * (size_t)a.W + (size_t)gwarp] = (s0 + s1) + (s2 + s3);
        }
        __syncwarp();
    }
    }
}

// One window of the warp. An ADSR envelope spends most of its life in two states in which maxiEnv::adsr
// (src/maximilian.cpp:1415-1466) does nothing but multiply:
//   release: no trigger, flags == {release}: `if (amplitude > 0) { amplitude *= release; output = input*amplitude; }`
//   sustain: trigger held, flags == {hold}, holdcount >= holdtime: `output = input*amplitude`
// (every other statement of the function is a no-op there: the first four tests fail on the flags, `holdphase = false;
// releasephase = true` re-assigns what is already set). When the gate does not change inside the window and every
// voice of the warp is in one of the two, the window runs those statements alone; otherwise the full state machine.
template <int OSC, int FILT, int ENV, bool ALLFAST, int OUTMODE, bool MIX, bool MODK>
__device__ __forceinline__ void dl_window(DlVoice& s, double* row, const int tn, const int t0, const BankArgs& a, const DelayArgs& d,
                                          const size_t V, const size_t v, const int lane, const int gwarp, double* mixtile, const int swz) {
    if (MODK) {
        dl_stage<OSC, FILT, ENV, ALLFAST, OUTMODE, MIX, false, true>(s, row, tn, t0, a, d, V, v, lane, gwarp, mixtile, false, swz);
        return;
    }
    if (ENV) {
        const EnvRegs& e = s.er;
        const bool notrig = e.off <= t0 || e.on >= t0 + tn || e.on >= e.off;
        const bool alltrig = e.on <= t0 && e.off >= t0 + tn;
        const bool relmode = e.st == ENV_R && notrig;
        const bool susmode = e.st == ENV_H && e.holdcount >= e.holdtime && alltrig;
        if (!a.env_ar && !a.trig_tv && __all_sync(kFull, relmode || susmode || !s.live)) {
            dl_stage<OSC, FILT, ENV, ALLFAST, OUTMODE, MIX, true>(s, row, tn, t0, a, d, V, v, lane, gwarp, mixtile, relmode, swz);
            return;
        }
    }
    dl_stage<OSC, FILT, ENV, ALLFAST, OUTMODE, MIX, false>(s, row, tn, t0, a, d, V, v, lane, gwarp, mixtile, false, swz);
}

template <int OSC, int FILT, int ENV, int OUTMODE, bool MIX, bool MODK = false>
__global__ void __launch_bounds__(DelayShape<MIX>::kThreads, DelayShape<MIX>::kMinCtas) delay_bank_kernel(const BankArgs a, const DelayArgs d) {
    const int lane = threadIdx.x & 31;
    const int gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long v0 = (long long)gwarp * 32;
    if (v0 >= a.V) return;
    const long long v = v0 + lane;
    const size_t V = (size_t)a.V;

    extern __shared__ __align__(128) double smem[];
    __shared__ unsigned long long s_bar[DelayShape<MIX>::kThreads / 32][kDlStages];     // one mbarrier per warp and stage (bulk loads)
    constexpr int per_warp = kDlStages * kStageDoubles + (MIX ? kMixDoubles : 0);      // a multiple of 16 doubles: stages stay 128-byte aligned
    static_assert((kStageDoubles * 8) % 128 == 0 && (per_warp * 8) % 128 == 0, "bulk copies need aligned stages");
    double* wsm = smem + (size_t)(threadIdx.x >> 5) * per_warp;
    double* mixtile = wsm + kDlStages * kStageDoubles;

    // ---- per-voice state (lane = voice) ----
    DlVoice s;
    s.live = v < a.V;
    const long long vv = s.live ? v : 0;
    osc_load<OSC>(a, vv, s.phase, s.oout, s.inc, s.duty, s.pend);
    filt_load<FILT>(a, vv, s.fr);
    s.res = (MODK && a.cutoff_tv) ? a.res[vv] : 0.0;
    env_load<ENV>(a, vv, s.er);
    s.gl = s.gr = 0.0;
    if (MIX) stereo_gains(a.pan[vv], s.live, s.gl, s.gr);
    s.ph = d.phase[vv];
    s.size = d.size[vv];
    s.fb = d.feedback[vv];
    s.pos = d.from_position ? d.position[vv] : 0;
    s.fast = s.live && s.size >= kFastMinSize && !d.from_position && !d.size_tv;      // dlFromPosition, per-sample size: literal path
    // ring index of the first access of the next window: the reference tests `phase >= size` before it reads
    int base = (s.ph >= s.size) ? 0 : s.ph;

    const int nstages = (a.n_frames + kDlT - 1) / kDlT;
    const int size0 = __shfl_sync(kFull, s.size, 0), base0 = __shfl_sync(kFull, base, 0);     // lane 0 is always live
    const bool uniform = __all_sync(kFull, !s.live || (s.fast && s.size == size0 && base == base0)) &&
                         (size0 & (kDlT - 1)) == 0 && (base0 & (kDlT - 1)) == 0;
    const int nlive = __popc(__ballot_sync(kFull, s.live));
    const int sl = lane & (kDlT - 1), hv = lane >> kDlShift;        // slot within a window / which voice of a request

    if (uniform) {
        // ---------------- all windows of the warp form one contiguous run of nlive * 128 B: one bulk copy each way ----------------
        const int nchunks = size0 >> kDlShift;
        int chunk = base0 >> kDlShift;
        const unsigned bytes = (unsigned)nlive * (kDlChunk * 8u);
        unsigned long long* bar = s_bar[threadIdx.x >> 5];
        double* run = d.ring + (size_t)v0 * kDlChunk;                      // chunk c of this warp's voices starts at run + c * V * 16
        if (lane == 0) {
#pragma unroll
            for (int i = 0; i < kDlStages; ++i) mbar_init(&bar[i], 1);
        }
        fence_proxy_async();                                                // the initialised barriers become visible to the copy engine
        __syncwarp();
        // Window k lives in stage k % 2 and is requested one window early. The chunk a request reads must not be the target of a
        // write-back still under way: the write-back of window k - j hits the chunk of window k + 1 when 1 + j is a multiple of
        // nchunks, first at j = nchunks - 1. A ring of at least 9 chunks only needs the write-backs older than the latest seven
        // performed (cp.async.bulk.wait_group 7: they were issued seven windows ago, the wait is free); a shorter ring waits for all
        // of them.
        const bool tight = nchunks < 9;
        auto chunk_of = [&](int kk) { return (int)(((long long)(base0 >> kDlShift) + kk) % nchunks); };
        if (lane == 0 && nstages > 0) {
            mbar_expect_tx(&bar[0], bytes);
            bulk_g2s(wsm, run + (size_t)chunk_of(0) * V * kDlChunk, bytes, &bar[0]);
        }
        const int swz = dl_swz((size_t)lane);
        int sidx = 0, nidx = 1;                                             // stage of window k / of window k + 1
        unsigned par = 0;                                                   // parity of stage sidx's barrier: flips every kDlStages windows
        int nchunk = chunk_of(1);
        for (int k = 0; k < nstages; ++k) {
            double* buf = wsm + sidx * kStageDoubles;
            const int t0 = k * kDlT;
            const int tn = min(kDlT, a.n_frames - t0);
            if (k + 1 < nstages && lane == 0) {
                // stage nidx last held window k - 1, source of a write-back: wait until the engine has READ it
                if (tight) bulk_wait_all(); else { bulk_wait_read0(); bulk_wait_but7(); }
                mbar_expect_tx(&bar[nidx], bytes);
                bulk_g2s(wsm + nidx * kStageDoubles, run + (size_t)nchunk * V * kDlChunk, bytes, &bar[nidx]);
            }
            mbar_wait(&bar[sidx], par);                                     // window k has landed
            dl_window<OSC, FILT, ENV, true, OUTMODE, MIX, MODK>(s, buf + lane * kDlChunk, tn, t0, a, d, V, (size_t)vv, lane, gwarp, mixtile, swz);
            fence_proxy_async();                                            // this lane's updates of the window, ordered before the engine reads them
            __syncwarp();
            if (lane == 0) { bulk_s2g(run + (size_t)chunk * V * kDlChunk, buf, bytes); bulk_commit(); }
            if (++chunk >= nchunks) chunk = 0;
            if (++nchunk >= nchunks) nchunk = 0;
            if (++sidx == kDlStages) { sidx = 0; par ^= 1u; }
            if (++nidx == kDlStages) nidx = 0;
        }
        if (lane == 0) bulk_wait_all();
        // phase += 1 after the last access: the window of the last stage started at slot 16*last_chunk
        if (s.live) {
            int last_chunk = (base0 >> kDlShift) + (nstages - 1);
            last_chunk %= nchunks;
            const int tn_last = a.n_frames - (nstages - 1) * kDlT;
            s.ph = last_chunk * kDlT + tn_last;
        }
    } else {
        // ---------------- generic: per-voice size and phase ----------------
        auto issue_loads = [&](double* buf, int wbase) {
#pragma unroll 4
            for (int q = 0; q < 32 / kDlVoicesPerReq; ++q) {
                const int i = kDlVoicesPerReq * q + hv;                    // the voice this lane serves in request q
                const int f_i = __shfl_sync(kFull, (int)s.fast, i);
                const int b_i = __shfl_sync(kFull, wbase, i);
                const int s_i = __shfl_sync(kFull, s.size, i);
                if (!f_i) continue;
                int r = b_i + sl;
                if (r >= s_i) r -= s_i;
                cp_async8(buf + i * kDlRow + (sl ^ dl_swz((size_t)i)), d.ring + dl_slot(V, (size_t)(v0 + i), r));
            }
        };
        issue_loads(wsm, base);
        cp_async_commit();
        for (int k = 0; k < nstages; ++k) {
            double* buf = wsm + (k & 1) * kStageDoubles;
            const int t0 = k * kDlT;
            const int tn = min(kDlT, a.n_frames - t0);
            int next_base = base + kDlT;
            if (s.fast && next_base >= s.size) next_base -= s.size;
            if (k + 1 < nstages) issue_loads(wsm + ((k + 1) & 1) * kStageDoubles, next_base);
            cp_async_commit();
            cp_async_wait1();
            __syncwarp();
            dl_window<OSC, FILT, ENV, false, OUTMODE, MIX, MODK>(s, buf + lane * kDlRow, tn, t0, a, d, V, (size_t)vv, lane, gwarp, mixtile, dl_swz((size_t)lane));
            __syncwarp();
#pragma unroll 4
            for (int q = 0; q < 32 / kDlVoicesPerReq; ++q) {
                const int i = kDlVoicesPerReq * q + hv;
                const int f_i = __shfl_sync(kFull, (int)s.fast, i);
                const int b_i = __shfl_sync(kFull, base, i);
                const int s_i = __shfl_sync(kFull, s.size, i);
                if (f_i && sl < tn) {
                    int r = b_i + sl;
                    if (r >= s_i) r -= s_i;
                    d.ring[dl_slot(V, (size_t)(v0 + i), r)] = buf[i * kDlRow + (sl ^ dl_swz((size_t)i))];
                }
            }
            __syncwarp();
            if (s.fast) {
                int last = base + tn - 1;
                if (last >= s.size) last -= s.size;
                s.ph = last + 1;                     // phase += 1 after the last access of the window
                base = (tn == kDlT) ? next_base : ((s.ph >= s.size) ? 0 : s.ph);
            }
        }
    }

    if (s.live) {
        voice_store<FILT, ENV>(a, v, s.phase, s.oout, s.fr, s.er);
        d.phase[v] = s.ph;
    }
}

template <int OSC, int FILT, int ENV, int OUTMODE, bool MIX, bool MODK>
inline int launch_delay_one(const BankArgs& a, const DelayArgs& d, cudaStream_t s) {
    constexpr int threads = DelayShape<MIX>::kThreads;
    constexpr size_t smem = sizeof(double) * (threads / 32) * (kDlStages * kStageDoubles + (MIX ? kMixDoubles : 0));
    const int grid = (a.V + threads - 1) / threads;
    auto kern = delay_bank_kernel<OSC, FILT, ENV, OUTMODE, MIX, MODK>;
    const int rc = smem_limit_at_least((const void*)kern, smem, "delay_bank_kernel");
    if (rc != MXB_OK) return rc;
    kern<<<grid, threads, smem, s>>>(a, d);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("delay_bank_kernel launch: %s", cudaGetErrorString(e)); return MXB_ERR_CUDA; }
    return MXB_OK;
}

}  // namespace mxb
