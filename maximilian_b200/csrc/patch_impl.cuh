// Voice patches: what the interpreting kernel (patch.cu) and the kernels generated per patch (patch_fuse.cu, compiled at
// run time with NVRTC) share -- the argument block, the stage bodies, each stage's state layout and the conversions of its
// operands. Each body is the reference method restated (same
// statements, same order; compiled without multiply-add contraction), taking its stage kind as a plain int: the interpreter
// passes it at run time (warp-uniform), a generated kernel passes a literal and the branches fold away.
//
// This header is also handed to NVRTC as text (build.py embeds it into the library): it must stay free of host-only
// constructs outside `#ifndef __CUDACC_RTC__`.
#pragma once
#include "bank_kernels.cuh"
#include "filter_design.cuh"

namespace mxb {

constexpr int kPatchThreads = 128;
constexpr int kMaxStages = 64, kMaxParams = 32, kMaxConsts = 64, kMaxInputs = 8, kMaxRegs = 16, kMaxEg = 16;
constexpr int kMaxEgShapes = 4;          // maxiEnvGen shapes of one patch (9.Envelopes2 plays three); their segment tables are kernel arguments

struct EgStage { double startlevel, endlevel, gradient, curve; long long length; int hold; int pad; };

// one call's events of an MXB_IN_EVENTS stream, on the device (mxb_events)
struct EvStream { const int* first; const int* frame; const double* value; };

struct PatchArgs {
    int V, n_frames, n_stages, n_params, n_state, W, taps;
    double sr;
    const mxb_stage* stages;         // device, n_stages                                (interpreter only)
    const int* state_base;           // device, n_stages: first state slot of each stage (interpreter only)
    const int* ring_of;              // device, n_stages: ring index of a delay-like stage, else -1 (interpreter only)
    const double* consts;            // device, kMaxConsts                              (interpreter only: generated kernels hold them as literals)
    const double* params;            // [n_params][V]
    double* state;                   // [n_state][V]
    const void* inputs[kMaxInputs];  // [n_frames][V] each: doubles, bytes or packed bits (in_kind[k] = MXB_IN_*)
    unsigned char in_kind[kMaxInputs];
    double* out;                     // [n_frames][V] or NULL
    double* partials;                // [n_frames][2][W] or NULL
    double* rings;                   // [n_rings][taps][V]
    const double* sine;              // sineBuffer[514], src/maximilian.cpp:63
    const double* transition;        // transition[1001], src/maximilian.cpp:67-200
    double sine_before;              // what sinebuf4 reads at sineBuffer[-1] on its wrap sample (out of bounds in the reference)
    int eg_n[kMaxEgShapes], eg_loop[kMaxEgShapes], eg_retrigger[kMaxEgShapes];      // shape k: an ENVGEN stage of kind k plays it
    EgStage eg[kMaxEgShapes][kMaxEg];
    int n_ev;                        // events streams (MXB_IN_EVENTS), numbered in input order
    unsigned char ev_of[kMaxInputs]; // input stream k -> its events stream number (events streams only)
    EvStream ev[kMaxInputs];         // events stream e of this call
    double* held;                    // [n_ev][V]: each events stream's held value, carried from call to call
};
static_assert(sizeof(PatchArgs) <= 4096, "PatchArgs must fit the 4 KB kernel parameter block");

// table oscillators, src/maximilian.cpp:237-274, 342-359
__device__ __forceinline__ double osc_table_tick(const int kind, double& phase, double& output, const double frequency, const double sr,
                                                 const double* __restrict__ sine, const double* __restrict__ transition, const double sine_before) {
    if (kind == MXB_OSC_SINEBUF4) {          // :237-264
        phase += 512. / (sr / (frequency));
        if (phase >= 511) phase -= 512;
        const double remainder = phase - floor(phase);
        double a, b, c, d;
        const long long ip = (long long)phase;
        if (phase == 0) { a = sine[512]; b = sine[ip]; c = sine[ip + 1]; d = sine[ip + 2]; }
        else { a = ip - 1 < 0 ? sine_before : sine[ip - 1]; b = sine[ip]; c = sine[ip + 1]; d = sine[ip + 2]; }
        const double a1 = 0.5 * (c - a);
        const double a2 = a - 2.5 * b + 2.0 * c - 0.5 * d;
        const double a3 = 0.5 * (d - a) + 1.5 * (b - c);
        output = ((a3 * remainder + a2) * remainder + a1) * remainder + b;
    } else if (kind == MXB_OSC_SINEBUF) {    // :266-274 (chandiv == 1)
        phase += 512. / (sr / (frequency * 1.0));
        if (phase >= 511) phase -= 512;
        const double remainder = phase - floor(phase);
        const long long ip = (long long)phase;
        output = (1 - remainder) * sine[1 + ip] + remainder * sine[2 + ip];
    } else {                                 // sawn, :342-359
        if (phase >= 0.5) phase -= 1.0;
        phase += osc_increment(sr, frequency);
        double temp = (8820.22 / frequency) * phase;
        if (temp < -0.5) temp = -0.5;
        if (temp > 0.5) temp = 0.5;
        temp *= 1000.0;
        temp += 500.0;
        const double remainder = temp - floor(temp);
        const long long it = (long long)temp;
        // transition[1 + it] with it == 1000 is one past the table in the reference, multiplied by remainder == 0
        const double t1 = it + 1 <= 1000 ? transition[it + 1] : 0.0;
        output = ((1.0 - remainder) * transition[it] + remainder * t1) - phase;
    }
    return output;
}

// maxiOsc::* as a patch stage: the phase oscillators of bank_kernels.cuh or the table oscillators above
__device__ __forceinline__ double stage_osc(const int kind, double& phase, double& oout, const double f, const double d0, const double d1, const double sr,
                                            const double* __restrict__ sine, const double* __restrict__ transition, const double sine_before) {
    if (kind >= MXB_OSC_SINEBUF) return osc_table_tick(kind, phase, oout, f, sr, sine, transition, sine_before);
    const double inc = kind == MXB_OSC_PHASORBETWEEN ? ((d1 - d0) / (sr / (f))) : osc_increment(sr, f);
    return osc_tick<OSC_T_GENERIC>(phase, oout, inc, d0, kind, d1);
}

// maxiEnv::adsr / ar as a patch stage (env_tick / env_ar_tick of bank_kernels.cuh): holdtime and holdcount are 64-bit like the
// reference's `long` (src/maximilian.h:915-916), because a patch reads holdtime from any operand -- a holdtime of 2^32 + 3 holds for
// 2^32 + 3 samples, not 3. The bank's EnvRegs keeps 32-bit ints (mxb_bank_set_param refuses |holdtime| >= 2^31).
struct PatchEnvRegs {
    double amp, output, att, dec, sus, rel;
    long long holdcount, holdtime;
    int st;                    // ENV_* bits
    int on, off;
};

// maxiTrigger::onZX, src/maximilian.h:564-585
__device__ __forceinline__ double on_zx(double& previousValue, double& firstTrigger, const double input) {
    double isZX = 0.0;
    if ((previousValue <= 0.0 || firstTrigger != 0.0) && input > 0) isZX = 1.0;
    previousValue = input;
    firstTrigger = 0.0;
    return isZX;
}

// maxiEnvGen::play, src/maximilian.h:2276-2357. state (WAITING 0, TRIGGERED 1, HOLDING 2); currentlevel is the level of the current
// segment (every other segment's are 0); the three maxiTrigger detectors as (previousValue, firstTrigger) pairs.
struct EgRegs {
    double envval, currentlevel, tp, tf, hp, hf, rp, rf;
    long long counter;
    int phase, state;
    bool nxc;
};
__device__ __forceinline__ double envgen_tick(EgRegs& g, const double trigger, const EgStage* __restrict__ eg, const int eg_n, const int eg_loop, const int eg_retrigger) {
    bool run = true;
    if (g.state == 0) {
        if (on_zx(g.tp, g.tf, trigger) != 0.0) { if (eg_n > 0) { g.state = 1; g.nxc = false; } else run = false; }
        else run = false;
    }
    if (run && g.state == 1) {
        const EgStage& cs = eg[g.phase < eg_n ? g.phase : 0];
        if (on_zx(g.hp, g.hf, -trigger) != 0.0) g.nxc = true;
        if (cs.hold) g.state = 2;
        else {
            double val = pow(g.currentlevel, cs.curve);
            val = (1.0 < val) ? 1.0 : val;                                     // maxiMap::linlin, src/maximilian.h:801-805: std::min, then
            val = (val < 0.0) ? 0.0 : val;                                     // std::max -- a NaN passes both, as it does there
            g.envval = ((val - 0.0) / (1.0 - 0.0) * (cs.endlevel - cs.startlevel)) + cs.startlevel;
            g.counter++;
            if (g.counter == cs.length) { g.counter = 0; g.currentlevel = 0; g.phase++; }
            else g.currentlevel += cs.gradient;
            if (eg_retrigger) { if (on_zx(g.rp, g.rf, trigger) != 0.0) { g.nxc = false; g.counter = 0; g.currentlevel = 0; g.phase = 0; g.state = 1; } }
            run = false;
        }
    }
    if (run && g.state == 2) {
        if (on_zx(g.hp, g.hf, -trigger) != 0.0) g.nxc = true;
        if (g.nxc) { g.state = 1; g.phase++; }
        if (eg_retrigger) { if (on_zx(g.rp, g.rf, trigger) != 0.0) { g.nxc = false; g.counter = 0; g.currentlevel = 0; g.phase = 0; g.state = 1; } }
    }
    if (g.phase == eg_n) { g.counter = 0; g.currentlevel = 0; g.phase = 0; g.state = 1; if (!eg_loop) g.state = 0; }
    return g.envval;
}

// maxiFilter::lopass / hipass / bandpass with their one or two words of history, src/maximilian.cpp:442-453, 487-500
__device__ __forceinline__ double onepole_tick(const int kind, double& z0, const double in, const double c) {
    const double y = kind == MXB_FILT_LOPASS ? z0 + c * (in - z0) : in - (z0 + c * (in - z0));
    z0 = y;
    return y;
}
__device__ __forceinline__ double bandpass_tick(double& z0, double& z1, const double in, const double c0, const double c1, const double c2) {
    const double y = c0 * in + c1 * z0 + c2 * z1;
    z1 = z0;
    z0 = y;
    return y;
}

// maxiDCBlocker::play, src/maximilian.h:1261-1266
__device__ __forceinline__ double dcblock_tick(double& xm1, double& ym1, const double in, const double R) {
    ym1 = in - xm1 + R * ym1;
    xm1 = in;
    return ym1;
}

// maxiNonlinearity, src/maximilian.h:1076-1137
__device__ __forceinline__ double nonlin_eval(const int kind, double x, const double p1, const double p2) {
    switch (kind) {
        case MXB_NL_ATANDIST: x = (1.0 / atan(p1)) * atan(x * p1); break;
        case MXB_NL_FASTATANDIST: x = (1.0 / (p1 / (1.0 + 0.28 * (p1 * p1)))) * ((x * p1) / (1.0 + 0.28 * ((x * p1) * (x * p1)))); break;
        case MXB_NL_SOFTCLIP: if (x >= 1) x = 1; else if (x <= -1) x = -1; else x = (2 / 3.0) * (x - pow(x, 3.0) / 3.0); break;
        case MXB_NL_HARDCLIP: x = x >= 1 ? 1 : (x <= -1 ? -1 : x); break;
        case MXB_NL_ASYMCLIP: if (x >= 1) x = 1; else if (x <= -1) x = -1; else if (x < 0) x = -(pow(-x, p1)); else x = pow(x, p2); break;
        default: x = (x / (1.0 + 0.28 * (x * x))); break;       // fastatan
    }
    return x;
}

// maxiDelayline::dl / dlFromPosition (src/maximilian.cpp:420-452) on this voice's ring: slot r at ring[r * V] (time-major across
// voices, so that a warp's 32 rings are read and written 256 contiguous bytes at a time). `ph` is the int ring index.
__device__ __forceinline__ double delay_tick(const bool from_position, double* __restrict__ ring, const size_t V, const int taps, const bool live, int& ph,
                                             const double in, const int size, const double fb, const int position) {
    if (ph >= size) ph = 0;
    const int idx = min(max(ph, 0), taps - 1);
    double outv = 0.0;
    if (live) {
        const double m = ring[(size_t)idx * V];
        if (from_position) {                                                   // :431-439
            int pos = position;
            if (pos >= size) pos = 0;
            outv = ring[(size_t)min(max(pos, 0), taps - 1) * V];
            ring[(size_t)idx * V] = (m * fb) + (in * fb) * 1.0;
        } else {
            outv = m;
            ring[(size_t)idx * V] = (m * fb) + (in * fb) * 0.5;
        }
    }
    ph += 1;
    return outv;
}
// maxiFlanger::flange, src/maximilian.h:1167-1175: lfo.triangle(speed), size = delay + lfo*depth*delay + 1 (-> int), dl, normalise
__device__ __forceinline__ double flanger_tick(double* __restrict__ ring, const size_t V, const int taps, const bool live, int& ph, double& lph, double& lout,
                                               const double in, const unsigned int delay, const double fb, const double speed, const double depth, const double sr) {
    const double lfoVal = osc_tick<OSC_T_GENERIC>(lph, lout, osc_increment(sr, speed), 0.0, MXB_OSC_TRIANGLE, 0.0);
    const int size = (int)(delay + (lfoVal * depth * delay) + 1);
    double outv = delay_tick(false, ring, V, taps, live, ph, in, size, fb, 0);
    const double normalise = (1 - fabs(outv));
    outv *= normalise;
    return (outv + in) / 2.0;
}

// maxiChorus::chorus, src/maximilian.h:1200-1212, from the noise value on: lfoVal = lopass.lores(noise, speed, 1.0) * 2.0 (the design is
// the caller's: it is block-constant when `speed` is), two delay lines swept by it, normalise, average
__device__ __forceinline__ double chorus_tick(double* __restrict__ ringA, double* __restrict__ ringB, const size_t V, const int taps, const bool live, int& ph1, int& ph2,
                                              FiltRegs& lp, const double in, const unsigned int delay, const double fb, const double depth, const double noise) {
    const double lfoVal = filt_tick<FILT_T_LORES>(lp, noise, nullptr) * 2.0;
    double output1 = delay_tick(false, ringA, V, taps, live, ph1, in, (int)(delay + (lfoVal * depth * delay) + 1), fb, 0);
    double output2 = delay_tick(false, ringB, V, taps, live, ph2, in, (int)((delay + (lfoVal * depth * delay * 1.02) + 1) * 0.98), fb * 0.99, 0);
    output1 *= (1.0 - fabs(output1));
    output2 *= (1.0 - fabs(output2));
    return (output1 + output2 + in) / 3.0;
}

// maxiMix::stereo (src/maximilian.cpp:503-509) of one voice, accumulated into the bus sums of this sample
__device__ __forceinline__ void mix_stereo_acc(double& ml, double& mr, const double in, double x) {
    if (x > 1) x = 1;
    if (x < 0) x = 0;
    ml += in * sqrt(1.0 - x);
    mr += in * sqrt(x);
}

// The warp's two bus sums of one sample in five exchange steps instead of ten: in the first step the lower half-warp keeps the left
// sums and hands its right sums to the upper half (and the other way round), then each half reduces ONE value. Fixed tree, so the
// result is the same from run to run and in both ways a patch runs; lanes 0 and 16 end up with the left / right sum.
__device__ __forceinline__ void mix_warp_store(double ml, double mr, const int lane, double* __restrict__ partials, const size_t t, const size_t W, const size_t gwarp) {
    const bool up = (lane & 16) != 0;
    double v = (up ? mr : ml) + __shfl_xor_sync(0xffffffffu, up ? ml : mr, 16);
#pragma unroll
    for (int m = 8; m >= 1; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    if ((lane & 15) == 0) partials[(t * 2 + (up ? 1 : 0)) * W + gwarp] = v;
}

// ---- the state layout: which of a stage's state words holds which member (maxib200.h documents the order with the ops) ----
// One function per stateful op moves its registers in (LOAD) or out of its words over an accessor, anything with `double& operator[](int)
// const` (by value): the interpreter's Lane over shared memory, or a generated kernel's StateColumn, where `sb` is a literal.
// one thread's registers, parameters or state in the interpreter's shared memory: slot-major, thread-minor
struct Lane {
    double* base; int stride;
    __device__ __forceinline__ double& operator[](int slot) const { return base[slot * stride]; }
};
// voice v's words of a.state (read from the argument block at each use: a kernel then compiles as if it indexed a.state itself)
struct StateColumn {
    const PatchArgs& a; size_t V; long long v;
    __device__ __forceinline__ double& operator[](int k) const { return a.state[(size_t)k * V + (size_t)v]; }
};
template <bool LOAD, class T> __device__ __forceinline__ void word(double& w, T& m) { if (LOAD) m = (T)w; else w = (double)m; }     // one word, one member
template <bool LOAD> __device__ __forceinline__ void word(double& w, bool& m) { if (LOAD) m = w != 0.0; else w = m ? 1.0 : 0.0; }
// OSC: phase, output
struct OscRegs { double phase, output; };
template <bool LOAD, class A> __device__ __forceinline__ void osc_state(const A s, const int sb, OscRegs& o) { word<LOAD>(s[sb], o.phase); word<LOAD>(s[sb + 1], o.output); }
// ENV_ADSR / ENV_AR: amp, output, holdcount, the ENV_* flags (E: PatchEnvRegs, or EnvRegs for a constant 32-bit holdtime)
template <bool LOAD, class A, class E> __device__ __forceinline__ void env_state(const A s, const int sb, E& e) {
    word<LOAD>(s[sb], e.amp); word<LOAD>(s[sb + 1], e.output); word<LOAD>(s[sb + 2], e.holdcount);
    if (LOAD) env_unpack(e, (int)s[sb + 3]); else s[sb + 3] = (double)env_pack(e);
}
// ENVGEN: 0 envval, 1 phase, 2 state, 3 nxcHappened, 4 counter, 5 currentlevel, 6/7 trigDetector, 8/9 holdDetector,
// 10/11 retriggerDetector (previousValue, firstTrigger)
template <bool LOAD, class A> __device__ __forceinline__ void envgen_state(const A s, const int sb, EgRegs& q) {
    word<LOAD>(s[sb], q.envval); word<LOAD>(s[sb + 1], q.phase); word<LOAD>(s[sb + 2], q.state); word<LOAD>(s[sb + 3], q.nxc); word<LOAD>(s[sb + 4], q.counter);
    word<LOAD>(s[sb + 5], q.currentlevel); word<LOAD>(s[sb + 6], q.tp); word<LOAD>(s[sb + 7], q.tf); word<LOAD>(s[sb + 8], q.hp); word<LOAD>(s[sb + 9], q.hf);
    word<LOAD>(s[sb + 10], q.rp); word<LOAD>(s[sb + 11], q.rf);
}
// filters: the first N words of FiltRegs' history. FILTER lores / hires, BIQUAD: s0, s1; FILTER lopass / hipass: s0; FILTER bandpass:
// its two outputs; SVF: s0, s1, s2; DCBLOCK: xm1, ym1
template <int N, bool LOAD, class A> __device__ __forceinline__ void filt_state(const A s, const int sb, FiltRegs& f) {
    word<LOAD>(s[sb], f.s0);
    if (N > 1) word<LOAD>(s[sb + 1], f.s1);
    if (N > 2) word<LOAD>(s[sb + 2], f.s2);
}
// DELAY: the ring index. FLANGER: the same, then its triangle LFO's OSC words at sb + 1 (its maxiDelayline and maxiOsc)
template <bool LOAD, class A> __device__ __forceinline__ void delay_state(const A s, const int sb, int& ph) { word<LOAD>(s[sb], ph); }
// CHORUS: the two ring indices, then the lores LFO's s0, s1
template <bool LOAD, class A> __device__ __forceinline__ void chorus_state(const A s, const int sb, int& ph1, int& ph2, FiltRegs& lp) {
    word<LOAD>(s[sb], ph1); word<LOAD>(s[sb + 1], ph2); filt_state<2, LOAD>(s, sb + 2, lp);
}

// ---- operands as the reference's methods take them (every operand arrives as a double) ----
__device__ __forceinline__ bool trigger_arg(const double x) { return (int)x == 1; }                  // maxiEnv's `int trigger`
__device__ __forceinline__ int int_arg(const double x) { return (int)x; }                            // a delay line's size or position
__device__ __forceinline__ unsigned int uint_arg(const double x) { return (unsigned int)x; }         // maxiFlanger / maxiChorus delay
// maxiEnv's `long holdtime`, in the width of the register type E
template <class E> __device__ __forceinline__ decltype(E::holdtime) env_holdtime(const double x) { return (decltype(E::holdtime))(long long)x; }

// number of state words of a stage, by op: OSC 2, ENV_ADSR / ENV_AR 4, ENVGEN 12, FILTER 2, SVF 3, BIQUAD 2, DCBLOCK 2, DELAY 1, FLANGER 3, CHORUS 4
__host__ __device__ inline int patch_state_slots(const int op) {
    constexpr int slots[MXB_OP_CHORUS + 1] = {0, 2, 4, 4, 12, 2, 3, 2, 2, 0, 1, 3, 0, 0, 0, 0, 0, 0, 4};
    return op >= 0 && op <= MXB_OP_CHORUS ? slots[op] : 0;
}
// initial value of a state word: 0, but for maxiEnvGen's maxiTrigger detectors (previousValue = 1, firstTrigger = 1, src/maximilian.h:583-584)
__host__ __device__ inline double patch_state_init(const int op, const int slot) { return op == MXB_OP_ENVGEN && slot >= 6 ? 1.0 : 0.0; }
// delay lines (rings of delay_taps slots) a stage owns
__host__ __device__ inline int patch_stage_rings(const int op) { return op == MXB_OP_CHORUS ? 2 : (op == MXB_OP_DELAY || op == MXB_OP_FLANGER) ? 1 : 0; }

// sample t of input stream k for voice v
__device__ __forceinline__ double patch_input(const PatchArgs& a, const int k, const size_t t, const size_t v, const size_t V) {
    if (a.in_kind[k] == MXB_IN_BITS) return (double)((((const unsigned*)a.inputs[k])[t * ((V + 31) >> 5) + (v >> 5)] >> (v & 31)) & 1u);   // one word per warp
    return a.in_kind[k] == MXB_IN_U8 ? (double)((const unsigned char*)a.inputs[k])[t * V + v] : ((const double*)a.inputs[k])[t * V + v];
}
// bytes of one block of an input stream
__host__ __device__ inline size_t patch_input_bytes(const int kind, const size_t n_frames, const size_t V) {
    return kind == MXB_IN_BITS ? n_frames * ((V + 31) >> 5) * 4 : n_frames * V * (kind == MXB_IN_U8 ? 1 : 8);
}

// An events stream (MXB_IN_EVENTS) of voice v, shared by both kernels. The caller keeps the held value, the cursor into the voice's
// events and the frame of the event at the cursor (kEvNever: none left), so that a sample with nothing due costs one compare. T: the
// interpreter keeps cursor and frame as doubles in shared memory, a generated kernel as ints in registers.
constexpr int kEvNever = 0x7fffffff;
template <class T> __device__ __forceinline__ void ev_start(const EvStream& e, const size_t v, const bool live, T& cur, T& next) {
    cur = 0; next = (T)kEvNever;
    if (!live) return;
    const int c = e.first[v], end = e.first[v + 1];
    cur = (T)c;
    if (c < end) next = (T)e.frame[c];
}
// before the stages of frame t read the stream: apply, in list order, every event due by t. Event i takes effect at max(its frame, the
// frame event i-1 took effect at), so the reads stay inside [first[v], first[v+1]) whatever order the list is in.
template <class T> __device__ __forceinline__ void ev_advance(const EvStream& e, const size_t v, const int t, double& held, T& cur, T& next) {
    if (next > (T)t) return;
    const int end = e.first[v + 1];
    do {
        const int c = (int)cur;
        held = e.value[c];
        cur = (T)(c + 1);
        next = c + 1 < end ? (T)e.frame[c + 1] : (T)kEvNever;
    } while (next <= (T)t);
}

}  // namespace mxb

#ifndef __CUDACC_RTC__
#include <string>
// host side of a patch, shared by patch.cu (C ABI, interpreter launch) and patch_fuse.cu (code generator, NVRTC, module loading)
struct mxb_fused;      // a compiled patch: the loaded module and its kernel (patch_fuse.cu)
struct mxb_patch {
    mxb_ctx* ctx;
    int V, n_stages, n_params, n_consts, n_inputs, max_frames, taps, n_state, n_rings;
    std::vector<mxb_stage> stages;
    std::vector<int> state_base, ring_of;
    std::vector<double> consts;
    mxb::DevBuf<mxb_stage> d_stages; mxb::DevBuf<int> d_state_base, d_ring_of; mxb::DevBuf<double> d_consts;
    mxb::DevBuf<double> params, state, rings;
    mxb::DevBuf<unsigned char> in_stage[mxb::kMaxInputs];      // staging for MXB_MEM_HOST input streams (bytes)
    int in_type[mxb::kMaxInputs];
    int n_ev;                                                  // MXB_IN_EVENTS streams; ev_of[k]: the number of input k among them
    unsigned char ev_of[mxb::kMaxInputs];
    mxb::DevBuf<double> held;                                  // [n_ev][V]
    mxb::DevBuf<int> ev_first[mxb::kMaxInputs], ev_frame[mxb::kMaxInputs];     // staging for MXB_MEM_HOST events, by events stream
    mxb::DevBuf<double> ev_value[mxb::kMaxInputs];
    mxb::DevBuf<double> out_stage, partials, mix_dev;
    int n_shapes;          // maxiEnvGen shapes; ENVGEN stage kinds index them
    int eg_n[mxb::kMaxEgShapes], eg_loop[mxb::kMaxEgShapes], eg_retrigger[mxb::kMaxEgShapes];
    mxb::EgStage eg[mxb::kMaxEgShapes][mxb::kMaxEg];
    int64_t launches;
    int mode;              // MXB_PATCH_INTERPRET | MXB_PATCH_FUSED
    mxb_fused* fused;      // compiled on the first fused launch; owned by the module cache, which outlives the patch
    mxb_exchange* ex;      // peer-memory mix exchange (multi-GPU), or NULL
};

namespace mxb {
// CUDA source of the kernel that runs exactly this stage list (no device needed)
std::string patch_generate_source(const mxb_stage* stages, int n_stages, int n_params, const double* consts, int n_consts, int n_inputs, const int* input_types);
// NVRTC: source -> sm_90a cubin (no device needed); MXB_OK or an error code with the compiler log in the error string
int patch_compile(const std::string& src, std::vector<char>& cubin);
int patch_fused_load(mxb_patch* p);                                   // generate + compile + load, once
int patch_fused_launch(mxb_patch* p, const PatchArgs& a, int grid, cudaStream_t s);
}  // namespace mxb
#endif
