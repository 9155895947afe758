/*
 * maxib200.h -- C ABI of libmaxib200.so: Maximilian's per-sample DSP hot path as batched
 * many-voice block kernels for NVIDIA H100 (sm_90a).
 *
 * The reference has no plugin/FFI boundary: its interface is the C++ class surface
 *   maxiOsc / maxiFilter / maxiSVF / maxiBiquad / maxiEnv / maxiDelayline / maxiMix
 *   (src/maximilian.h:169-419, 888-932, 1281-1486) and maxiFFT / maxiIFFT / maxiMFCC
 *   (src/libs/maxiFFT.h:46-156, src/libs/maxiMFCC.h:40-211),
 * called once per sample from the audio callback routing() (cpp/commandline/player.cpp:25-44).
 * This header is that surface restated for V voices x n frames per call: plain pointers and
 * sizes, opaque handles, an int32 status on every entry point, no exceptions, no exit().
 * include/maximilian_b200.hpp wraps it in C++ classes with the reference's names.
 *
 * Conventions
 *   - every function returns MXB_OK (0) or a negative MXB_ERR_*; mxb_last_error() gives the text
 *     (thread-local). Nothing here ever falls back to a CPU implementation: without a CUDA device
 *     mxb_ctx_create fails with MXB_ERR_CUDA.
 *   - `mem` says where ALL data pointers of that call live: MXB_MEM_HOST (the call copies in, runs,
 *     copies out and returns when the results are in host memory) or MXB_MEM_DEVICE (asynchronous on
 *     `stream`, a cudaStream_t passed as void*; NULL = the legacy default stream).
 *   - one handle is driven from one thread/stream at a time (like the reference objects, which are
 *     owned by the audio thread); different handles are independent, also when they are called from
 *     different host threads at the same time. Host-memory calls on the NULL stream of one context
 *     still run one after another on the device.
 *   - sample values are fp64 for the oscillator/filter/envelope/delay/mix path (the reference's
 *     `double`), fp32 for the FFT path (the reference's `float`), fp64 for MFCCs.
 */
#ifndef MAXIB200_H
#define MAXIB200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MXB_VERSION 100

/* status codes */
enum {
    MXB_OK = 0,
    MXB_ERR_INVALID = -1,      /* bad argument (NULL handle, size out of range, unknown id) */
    MXB_ERR_CUDA = -2,         /* CUDA runtime error, or no CUDA device */
    MXB_ERR_ALLOC = -3,        /* out of host or device memory */
    MXB_ERR_UNSUPPORTED = -4,  /* a combination this build has no kernel for */
    MXB_ERR_STATE = -5         /* call out of order (e.g. parameter never set) */
};

/* MXB_MEM_SPLIT (mxb_bank_process only): control data (gates) and the mix bus in host memory, `out`
 * in device memory -- the voice signals stay on the GPU for the next stage, the host gets the mix. */
enum { MXB_MEM_HOST = 0, MXB_MEM_DEVICE = 1, MXB_MEM_SPLIT = 2,
       /* flag, OR-ed into MXB_MEM_HOST / MXB_MEM_SPLIT of mxb_bank_process*: do not wait. The call returns once the copies and
        * kernels are enqueued on `stream`; host buffers must be page-locked (mxb_host_alloc) and are valid after the stream or
        * the context (mxb_ctx_synchronize) has been synchronised. A block loop then never stalls the host: block k+1's control
        * data goes up (mxb_bank_set_param_async, double-buffered on the bank's copy stream) while block k computes and block
        * k-1's mix comes down. */
       MXB_MEM_ASYNC = 0x100 };
enum { MXB_F64 = 0, MXB_F32 = 1 };

/* oscillator kinds: maxiOsc methods, src/maximilian.cpp */
enum {
    MXB_OSC_SINEWAVE = 0,  /* :228-235 */
    MXB_OSC_COSWAVE = 1,   /* :276-283 */
    MXB_OSC_PHASOR = 2,    /* :285-291 */
    MXB_OSC_SAW = 3,       /* :333-340 */
    MXB_OSC_SQUARE = 4,    /* :293-300 */
    MXB_OSC_PULSE = 5,     /* :302-311 */
    MXB_OSC_IMPULSE = 6,   /* :312-319 */
    MXB_OSC_TRIANGLE = 7,  /* :362-373 */
    MXB_OSC_PHASORBETWEEN = 8  /* :321-330, phasorBetween(frequency, startphase, endphase) */
    /* 9..11: the table oscillators, patch stages only (MXB_OSC_SINEBUF ...) */
};
/* filter kinds */
enum {
    MXB_FILT_NONE = 0,
    MXB_FILT_LORES = 1,    /* maxiFilter::lores  src/maximilian.cpp:455-468 */
    MXB_FILT_HIRES = 2,    /* maxiFilter::hires  src/maximilian.cpp:471-484 */
    MXB_FILT_SVF = 3,      /* maxiSVF::play      src/maximilian.h:1305-1319 */
    MXB_FILT_BIQUAD = 4    /* maxiBiquad::play   src/maximilian.h:1360-1367 */
};
/* maxiBiquad::filterTypes, src/maximilian.h:1348-1357 */
enum { MXB_BQ_LOWPASS = 0, MXB_BQ_HIGHPASS, MXB_BQ_BANDPASS, MXB_BQ_NOTCH, MXB_BQ_PEAK, MXB_BQ_LOWSHELF, MXB_BQ_HIGHSHELF };
enum {
    MXB_ENV_NONE = 0,
    MXB_ENV_ADSR = 1,   /* maxiEnv::adsr(input, trigger) src/maximilian.cpp:1415-1466; the overload with explicit
                           attack/decay/sustain/release/holdtime arguments (:1362-1413) is the same computation on
                           its arguments, i.e. on the per-voice arrays below */
    MXB_ENV_AR = 2      /* maxiEnv::ar(input, attack, release, holdtime, trigger) src/maximilian.cpp:1319-1358 */
};
/* delay_mode of mxb_bank_desc */
enum {
    MXB_DELAY_DL = 0,            /* maxiDelayline::dl              src/maximilian.cpp:420-429 */
    MXB_DELAY_FROM_POSITION = 1  /* maxiDelayline::dlFromPosition  src/maximilian.cpp:431-439 */
};

/* per-voice parameter / state arrays: double[voices] */
enum {
    MXB_P_FREQ = 0,           /* frequency argument of the maxiOsc method, Hz */
    MXB_P_PHASE = 1,          /* maxiOsc::phaseReset (src/maximilian.cpp:222-226); readable as state */
    MXB_P_DUTY = 2,           /* maxiOsc::pulse duty */
    MXB_P_CUTOFF = 3,         /* lores/hires cutoff1 | maxiSVF::setCutoff | maxiBiquad::set cutoff */
    MXB_P_RESONANCE = 4,      /* lores/hires resonance | maxiSVF::setResonance | maxiBiquad::set Q */
    MXB_P_GAIN = 5,           /* maxiBiquad::set peakGain */
    MXB_P_ENV_ATTACK = 6,     /* maxiEnv::attack  (public member; see mxb_env_coeffs for the setters) */
    MXB_P_ENV_DECAY = 7,      /* maxiEnv::decay */
    MXB_P_ENV_SUSTAIN = 8,    /* maxiEnv::sustain */
    MXB_P_ENV_RELEASE = 9,    /* maxiEnv::release */
    MXB_P_ENV_HOLDTIME = 10,  /* maxiEnv::holdtime (integral value; default 1, src/maximilian.h:913) */
    MXB_P_DELAY_SIZE = 11,    /* maxiDelayline::dl size argument (integral value) */
    MXB_P_DELAY_FEEDBACK = 12,/* maxiDelayline::dl feedback argument */
    MXB_P_PAN = 13,           /* maxiMix::stereo x (src/maximilian.cpp:503-509) */
    MXB_P_DELAY_POSITION = 14,/* maxiDelayline::dlFromPosition position argument (integral value) */
    MXB_P_PHASOR_START = 15,  /* maxiOsc::phasorBetween startphase */
    MXB_P_PHASOR_END = 16,    /* maxiOsc::phasorBetween endphase (default 1) */
    MXB_P_COUNT = 17,
    /* state (mxb_bank_get_state / mxb_bank_set_state) */
    MXB_S_FILT_0 = 32,        /* lores/hires x | svf v0z | biquad v[1] */
    MXB_S_FILT_1 = 33,        /* lores/hires y | svf v1  | biquad v[2] */
    MXB_S_FILT_2 = 34,        /* svf v2 */
    MXB_S_ENV_AMPLITUDE = 35,
    MXB_S_ENV_OUTPUT = 36,
    MXB_S_ENV_HOLDCOUNT = 37,
    MXB_S_ENV_FLAGS = 38,     /* attackphase | decayphase<<1 | sustainphase<<2 | holdphase<<3 | releasephase<<4 */
    MXB_S_DELAY_PHASE = 39,   /* maxiDelayline::phase (the ring index, an int in the reference) */
    MXB_S_OSC_OUTPUT = 40     /* maxiOsc::output (square / pulse / triangle hold their last value in it) */
};

typedef struct mxb_ctx mxb_ctx;
typedef struct mxb_bank mxb_bank;
typedef struct mxb_stft mxb_stft;
typedef struct mxb_mfcc mxb_mfcc;
typedef struct mxb_istft mxb_istft;

const char* mxb_last_error(void);
int32_t mxb_version(void);

/* ------------------------------------------------------------------------------------------------
 * Context = one CUDA device + the sample rate. Replaces the process-global maxiSettings::setup()
 * (src/maximilian.h:117-163); the rate is captured here instead of being re-read on every sample
 * (src/maximilian.cpp:232,460). */
int32_t mxb_ctx_create(int32_t device, int32_t sample_rate, mxb_ctx** ctx);
int32_t mxb_ctx_destroy(mxb_ctx* ctx);
int32_t mxb_ctx_sample_rate(const mxb_ctx* ctx);
int32_t mxb_ctx_synchronize(mxb_ctx* ctx);
/* page-locked host memory for MXB_MEM_HOST buffers (cudaHostAlloc); pageable memory works too, slower */
int32_t mxb_host_alloc(mxb_ctx* ctx, uint64_t bytes, void** ptr);
int32_t mxb_host_free(mxb_ctx* ctx, void* ptr);

/* ------------------------------------------------------------------------------------------------
 * Voice bank: `voices` independent voices, each the chain
 *     x = maxiOsc::<osc_kind>(freq)  ->  [maxiEnv::adsr(x, trigger)]  ->  [filter]  ->
 *         [maxiDelayline::dl(x, size, feedback)]  ->  out[t][v] = x,  mix[t][0..1] += maxiMix::stereo(x, pan)
 * i.e. the body of a reference play() that loops over an array of voices
 * (cpp/commandline/maximilian_examples/15.polysynth/main.cpp:54-70), for n frames per call.
 * All state (phase, filter memory, envelope flags, delay ring and its int index) lives on the device
 * between calls, exactly as it lives in the reference objects between play() calls. */
typedef struct {
    int32_t voices;
    int32_t osc_kind;        /* MXB_OSC_* */
    int32_t filt_kind;       /* MXB_FILT_* */
    int32_t biquad_type;     /* MXB_BQ_*   (filt_kind == MXB_FILT_BIQUAD) */
    int32_t env_kind;        /* MXB_ENV_* */
    int32_t delay_taps;      /* 0 = no delay line; else ring slots per voice (reference: 705600 fixed, src/maximilian.h:273) */
    int32_t max_frames;      /* largest n_frames a process call will use (maxiSettings::bufferSize) */
    int32_t delay_mode;      /* MXB_DELAY_* (delay_taps > 0) */
    double  svf_mix[4];      /* lpmix, bpmix, hpmix, notchmix arguments of maxiSVF::play */
} mxb_bank_desc;

int32_t mxb_bank_create(mxb_ctx* ctx, const mxb_bank_desc* desc, mxb_bank** bank);
int32_t mxb_bank_destroy(mxb_bank* bank);
int32_t mxb_bank_voices(const mxb_bank* bank);
/* values: double[voices]. Ordered like a cudaMemcpy on the legacy default stream (after every block enqueued on blocking
 * streams; no device-wide synchronisation). Filter coefficients are designed here, once per change (host threads share
 * a large bank), with the
 * reference's own formulas (lores/hires src/maximilian.cpp:457-462, maxiSVF::setParams
 * src/maximilian.h:1322-1334, maxiBiquad::set src/maximilian.h:1375-1479): block-constant
 * parameters hoist out of the per-sample loop exactly. */
int32_t mxb_bank_set_param(mxb_bank* bank, int32_t id, const double* values, int32_t mem);
/* Asynchronous variant for block-rate control data (a new frequency / pan / feedback array every block); takes effect
 * with the NEXT mxb_bank_process call. From host memory (page-locked; unchanged until that block has started) the copy
 * runs on the bank's own copy stream into the second of two device buffers, overlapping the blocks already enqueued;
 * the next block waits for it on its stream and switches buffers. From device memory it is one copy on `stream`.
 * Of several calls for the same id before one mxb_bank_process, synchronous (mxb_bank_set_param) or asynchronous, from host or
 * device memory, the later call wins: that block and the ones after it read the values of the last call.
 * Parameters that need a host pass (cutoff / resonance / gain: coefficient design; holdtime / delay size: integer
 * conversion) fall back to mxb_bank_set_param. The reference passes these values by argument on every sample. */
int32_t mxb_bank_set_param_async(mxb_bank* bank, int32_t id, const double* values, int32_t mem, void* stream);
int32_t mxb_bank_get_state(mxb_bank* bank, int32_t id, double* values, int32_t mem);
/* ring slots [0, n) of voice v (debug / checkpoint) */
int32_t mxb_bank_get_ring(mxb_bank* bank, int32_t voice, double* dst, int32_t n, int32_t mem);
/* The reference's objects hold their state by value (src/maximilian.h:266-281, 888-932): a patch checkpoints or forks a
 * voice by copying the object and restores it by assigning members. The counterparts: mxb_bank_set_state writes one
 * MXB_S_* array (integral ones arrive as doubles, as mxb_bank_get_state returns them), mxb_bank_set_ring one voice's
 * ring slots, mxb_bank_clone makes a deep copy of the whole bank (parameters, coefficients, state, rings). */
int32_t mxb_bank_set_state(mxb_bank* bank, int32_t id, const double* values, int32_t mem);
int32_t mxb_bank_set_ring(mxb_bank* bank, int32_t voice, const double* src, int32_t n, int32_t mem);
int32_t mxb_bank_clone(mxb_bank* bank, mxb_bank** copy);
/* One block. trigger_v(t) = 1 for trig_on[v] <= t < trig_off[v] (t counts frames inside this call),
 * both NULL = trigger 0. out: [n_frames][voices] of out_dtype, or NULL. mix: double [n_frames][2]
 * (overwritten), or NULL; voices are summed in a fixed order, so results are run-to-run identical. */
int32_t mxb_bank_process(mxb_bank* bank, int32_t n_frames,
                         const int32_t* trig_on, const int32_t* trig_off,
                         void* out, int32_t out_dtype, double* mix,
                         int32_t mem, void* stream);
/* The same block with a per-sample oscillator frequency freq_tv[t][v] (n_frames x voices doubles, in the memory the
 * gates live in; NULL = the block-constant MXB_P_FREQ). The reference takes the frequency by argument on every
 * sample, so a patch may modulate it at audio rate -- FM: osc.sinewave(440 + lfo.sinewave(1)*100),
 * cpp/commandline/maximilian_examples/5.FM1/main.cpp:29. Costs one 8-byte read per voice-sample. Works on every bank
 * chain, oscillator -> [envelope] -> [filter] -> [delay line] -> out / mix (with a delay stage the staged-window kernel runs a
 * modulated instantiation of its window body). */
int32_t mxb_bank_process_fm(mxb_bank* bank, int32_t n_frames, const double* freq_tv,
                            const int32_t* trig_on, const int32_t* trig_off,
                            void* out, int32_t out_dtype, double* mix,
                            int32_t mem, void* stream);
/* ... and with a per-sample filter cutoff cutoff_tv[t][v] as well (either pointer may be NULL). maxiFilter::lores/hires
 * take the cutoff as an argument of every call (src/maximilian.cpp:455,471) and a maxiSVF patch calls setCutoff() before
 * play() on every sample (src/maximilian.h:1287-1290): a swept filter. The coefficient design (cos/sqrt/pow, tan) then
 * runs per sample on the device -- libdevice instead of glibc, so results agree to rounding of those functions (asserted
 * at 1e-9 relative) instead of bit for bit. The modulation lasts for this call; MXB_P_CUTOFF is in force again afterwards.
 * maxiBiquad (whose set() is a design routine, not a per-sample argument): MXB_ERR_UNSUPPORTED (a voice patch covers it). Chains with
 * a delay stage take freq_tv / cutoff_tv like the others.
 * delay_size_tv[t][v] (integral values, 1 .. delay_taps): the `size` argument of maxiDelayline::dl / dlFromPosition, which a
 * flanger or chorus changes on every call (maxiFlanger::flange, src/maximilian.h:1144-1180). Works on any chain with a
 * delay stage, also together with freq_tv / cutoff_tv; the ring is then addressed slot by slot in HBM (the staged-window
 * schedule needs a size that holds for a block), indices exactly as the reference computes them. */
typedef struct {
    const double* freq_tv;        /* [n_frames][voices] or NULL */
    const double* cutoff_tv;      /* [n_frames][voices] or NULL */
    const double* delay_size_tv;  /* [n_frames][voices] or NULL */
    const uint8_t* trig_tv;       /* [n_frames][voices] bytes or NULL: maxiEnv::trigger for EVERY sample (1 = note on), in place of the
                                     trig_on / trig_off interval -- the trigger is a public int a patch writes at any sample
                                     (src/maximilian.h:913, maximilian_examples/10.Filters/main.cpp:27-36): several notes per block */
} mxb_modulation;
int32_t mxb_bank_process_mod(mxb_bank* bank, int32_t n_frames, const mxb_modulation* mod,
                             const int32_t* trig_on, const int32_t* trig_off,
                             void* out, int32_t out_dtype, double* mix,
                             int32_t mem, void* stream);
/* Block-dispatch shim, the counterpart of routing() in cpp/commandline/player.cpp:25-44 (RtAudio callback): fills the driver's
 * interleaved RTAUDIO_FLOAT64 buffer interleaved_out[n_frames][channels] (host memory) with the next block of the bank's
 * stereo bus (channels 0 / 1; further channels silent; one channel: the left bus). Synchronous, trigger 0. */
int32_t mxb_play_block(mxb_bank* bank, double* interleaved_out, int32_t n_frames, int32_t channels);
/* kernels launched by this library on behalf of `bank` since creation (for bench.py's gpu_launches) */
int64_t mxb_bank_launch_count(const mxb_bank* bank);

/* ------------------------------------------------------------------------------------------------
 * Voice patch: a per-voice signal GRAPH, run sample by sample for `voices` voices -- the body of any reference play()
 * written with the classes of this path. The bank above is hard-wired to osc -> env -> filter -> delay -> mix (the chains
 * BASELINE.json measures, at the HBM roofline); a patch expresses what real patches do and the bank cannot: two
 * oscillators summed into one filter, an LFO added to a frequency or a cutoff, the envelope multiplying the FILTER OUTPUT
 * (cpp/commandline/maximilian_examples/15.polysynth/main.cpp:54-70), a trigger that changes on any sample
 * (10.Filters/main.cpp:27-36), and the rest of the family: table oscillators, one-pole filters, maxiDCBlocker,
 * maxiNonlinearity, maxiEnvGen, maxiFlanger, maxiChorus. State lives on the device between calls like a bank's. A patch runs in one
 * of two ways (mxb_patch_set_mode), with identical state layout and results:
 *   MXB_PATCH_FUSED (default)  the library writes the CUDA source of ONE kernel for exactly this stage list -- stage state and
 *                              parameters in registers, constants as literals, coefficient designs whose arguments do not
 *                              change within a block hoisted out of the sample loop -- compiles it for sm_90a with NVRTC on
 *                              first use (about a second, once per distinct program: compiled kernels are kept in the process and, as cubin
 *                              files, under $MXB_PATCH_CACHE | $XDG_CACHE_HOME/maxib200 | ~/.cache/maxib200; MXB_PATCH_CACHE=0: no files) and
 *                              launches it like the built-in kernels;
 *   MXB_PATCH_INTERPRET        one interpreting kernel walks the stage list (warp-uniform dispatch: every voice runs the same
 *                              program), registers / parameters / state in shared memory. No run-time compiler needed.
 * Neither is a CPU path; a fused patch on a box without libnvrtc.so.12 fails with MXB_ERR_UNSUPPORTED and says so.
 *
 * A stage computes dst = op(src...) on 16 per-voice registers that read 0 until written within the sample. Operands: */
#define MXB_STAGE_SRCS 8
#define MXB_NONE (-1)
#define MXB_REG(i)   (i)             /* register i, 0..15 */
#define MXB_PARAM(j) (0x100 + (j))   /* per-voice parameter array j (mxb_patch_set_param), 0..31 */
#define MXB_CONST(k) (0x200 + (k))   /* scalar k of mxb_patch_desc.consts, 0..63 */
#define MXB_INPUT(m) (0x300 + (m))   /* per-sample input stream m of mxb_patch_process: [n_frames][voices] doubles (or bytes, input_types), 0..7 */
#define MXB_IN_F64 0                 /* input stream element types (mxb_patch_desc.input_types) */
#define MXB_IN_U8 1                  /* unsigned bytes, read as (double)byte: triggers and gates (maxiEnv::trigger is an int) at 1 B / voice-sample */
#define MXB_IN_BITS 2                /* one bit per voice-sample, read as 0.0 / 1.0: uint32 words [n_frames][(voices + 31) / 32], voice v = bit v % 32 of word v / 32 */
#define MXB_IN_EVENTS 3              /* control events: per-voice values set at any frame and held (mxb_events); costs 16 B per event, not per voice-sample */
/* An events stream: inputs[m] of mxb_patch_process points to one of these, in host memory; the three arrays live where `mem` says.
 * Voice v's events are first[v] .. first[v+1]-1 (first[voices] is the count); a voice with first[v+1] <= first[v] has none.
 * The stream reads the voice's HELD value. Its events apply in list order: event i takes effect at frame max(frame[i], the frame
 * at which event i-1 took effect), before the stages of that sample read the stream. So for a sorted list the stream is the value
 * of the last event with frame <= t (several on one frame: the last wins); a negative frame takes effect at frame 0; events at
 * frames >= n_frames (and every later one of that voice) are dropped. The held value carries over to the next call; it starts at
 * 0.0 (mxb_patch_get_held / set_held). A NULL descriptor or array, or with MXB_MEM_HOST a negative first[0] or a decreasing
 * `first`, is MXB_ERR_INVALID. */
typedef struct {
    const int32_t* first;    /* [voices + 1] */
    const int32_t* frame;    /* [first[voices]]: frame within this call of each event */
    const double* value;     /* [first[voices]] */
} mxb_events;
/* oscillator kinds of MXB_OP_OSC beyond MXB_OSC_*: the table oscillators (tables: mxb_ctx_set_tables) */
enum { MXB_OSC_SINEBUF = 9 /* maxiOsc::sinebuf src/maximilian.cpp:266-274 */, MXB_OSC_SINEBUF4 = 10 /* :237-264 */, MXB_OSC_SAWN = 11 /* :342-359 */ };
/* filter kinds of MXB_OP_FILTER beyond MXB_FILT_LORES / HIRES */
enum { MXB_FILT_LOPASS = 5 /* maxiFilter::lopass src/maximilian.cpp:442-446 */, MXB_FILT_HIPASS = 6 /* :449-453 */, MXB_FILT_BANDPASS = 7 /* :487-500 */ };
/* maxiNonlinearity (src/maximilian.h:1046-1137) */
enum { MXB_NL_ATANDIST = 0, MXB_NL_FASTATANDIST, MXB_NL_SOFTCLIP, MXB_NL_HARDCLIP, MXB_NL_ASYMCLIP, MXB_NL_FASTATAN };
#define MXB_ENVGEN_HOLD (-46692.0)   /* maxiEnvGen::HOLD, src/maximilian.h:2271 */
enum {
    MXB_OP_OSC = 1,      /* kind MXB_OSC_*: src0 frequency, src1 duty | startphase, src2 endphase.              state: phase, output */
    MXB_OP_ENV_ADSR,     /* maxiEnv::adsr(input, attack, decay, sustain, release, holdtime, trigger) src/maximilian.cpp:1362-1413:
                            src0 input, src1 trigger ((int)value == 1), src2..6 attack decay sustain release holdtime. state: amplitude, output, holdcount, flags */
    MXB_OP_ENV_AR,       /* maxiEnv::ar :1319-1358: src0 input, src1 trigger, src2 attack, src3 release, src4 holdtime */
    MXB_OP_ENVGEN,       /* maxiEnvGen::play(trigger) src/maximilian.h:2276-2357: src0 trigger. kind = index of the stage's envelope shape
                            (mxb_patch_create2; mxb_patch_create: 0, the shape in mxb_patch_desc.eg_*) */
    MXB_OP_FILTER,       /* kind MXB_FILT_LORES | HIRES | LOPASS | HIPASS | BANDPASS: src0 input, src1 cutoff, src2 resonance */
    MXB_OP_SVF,          /* maxiSVF setCutoff + setResonance + play src/maximilian.h:1287-1334: src0 input, src1 cutoff, src2 resonance, src3..6 lp bp hp notch mix */
    MXB_OP_BIQUAD,       /* kind MXB_BQ_*: maxiBiquad::set + play src/maximilian.h:1360-1479: src0 input, src1 cutoff, src2 Q, src3 peakGain */
    MXB_OP_DCBLOCK,      /* maxiDCBlocker::play src/maximilian.h:1255-1267: src0 input, src1 R.                  state: xm1, ym1 */
    MXB_OP_NONLIN,       /* kind MXB_NL_*: src0 input, src1 shape | a, src2 b */
    MXB_OP_DELAY,        /* kind MXB_DELAY_*: maxiDelayline::dl / dlFromPosition: src0 input, src1 size, src2 feedback, src3 position. state: phase */
    MXB_OP_FLANGER,      /* maxiFlanger::flange src/maximilian.h:1144-1180: src0 input, src1 delay, src2 feedback, src3 speed, src4 depth. state: dl phase, lfo phase, lfo output */
    MXB_OP_ADD, MXB_OP_SUB, MXB_OP_MUL, MXB_OP_DIV,   /* src0 (+ - * /) src1: the arithmetic a play() does between the calls */
    MXB_OP_MIX_STEREO,   /* maxiMix::stereo(src0, two, src1 = pan) summed into the bus (src/maximilian.cpp:503-509) */
    MXB_OP_OUT,          /* out[t][voice] = src0 */
    MXB_OP_CHORUS        /* maxiChorus::chorus src/maximilian.h:1180-1212: src0 input, src1 delay, src2 feedback, src3 speed, src4 depth, src5 noise -- the
                            value maxiOsc::noise() returns for this sample (libc rand() scaled to [-1, 1], src/maximilian.cpp:214-220): the caller
                            owns the random stream, the stage is everything after it (lores(noise, speed, 1) * 2 sweeping two delay lines).
                            state: dl phase, dl2 phase, lopass x, lopass y; two rings (mxb_patch_get_ring returns them back to back) */
};
/* Operand domain: the inputs on which the reference itself is defined. Outside it the reference reads out of bounds or converts out of
 * range, and no result is promised:
 *   - a double -> int conversion out of range or of a NaN: a trigger, holdtime, delay size or position, flanger / chorus delay
 *     (holdtime and the hold count are 64-bit like the reference's `long`: integral holdtimes up to 2^53 behave as there);
 *   - the table oscillators (MXB_OSC_SINEBUF, SINEBUF4, SAWN) at a negative frequency or one above the sample rate, and SAWN at 0 Hz;
 *   - a delay index at or beyond the ring: a size or position above delay_taps, or a negative position.
 * Everything else -- frequencies of 0, -0, below 0, above Nyquist; duties outside [0, 1]; cutoffs, resonances and gains at and past the
 * reference's clamps; infinities, NaNs and subnormals in any operand that is not converted to an integer -- is computed as the reference does. */
typedef struct { int32_t op, kind, dst, reserved; int32_t src[MXB_STAGE_SRCS]; } mxb_stage;
typedef struct {
    int32_t voices, n_stages, n_params, n_consts, n_inputs, max_frames;
    int32_t delay_taps;           /* ring slots per voice of every DELAY / FLANGER stage and of each of a CHORUS stage's two lines */
    int32_t eg_stages, eg_loop, eg_retrigger;     /* maxiEnvGen::setup(levels, times, curves, looping, allowRetrigger): eg_stages + 1 levels.
                                                     The one shape of mxb_patch_create; empty (eg_stages 0) for mxb_patch_create2 */
    const mxb_stage* stages;
    const double* consts;
    const double *eg_levels, *eg_times /* ms or MXB_ENVGEN_HOLD */, *eg_curves;
    const int32_t* input_types;   /* n_inputs x MXB_IN_*, or NULL: every stream is doubles */
} mxb_patch_desc;
typedef struct mxb_patch mxb_patch;
/* One maxiEnvGen shape: the arguments of maxiEnvGen::setup(levels, times, curves, looping, allowRetrigger), src/maximilian.h:2371-2402.
 * stages + 1 levels, stages times (ms or MXB_ENVGEN_HOLD; at most one HOLD, as setup() requires) and stages curves. stages == 0 is a
 * maxiEnvGen whose setup() was never called: it never triggers and plays 0. */
typedef struct { int32_t stages, loop, retrigger; const double *levels, *times, *curves; } mxb_envgen_shape;
/* The reference's lookup tables sineBuffer[514] and transition[1001] (src/maximilian.cpp:63, 67-200) are DATA of the
 * reference: an integration passes its own arrays (they have external linkage there). sine_before: the double that
 * maxiOsc::sinebuf4 reads at sineBuffer[-1] on the one sample per cycle where its phase has just wrapped into [-1, 0)
 * (an out-of-bounds read in the reference, src/maximilian.cpp:251); pass (&sineBuffer[0])[-1] for bit parity with a given
 * build, or sineBuffer[511] for the periodic extension the author intended. */
int32_t mxb_ctx_set_tables(mxb_ctx* ctx, const double* sine514, const double* transition1001, double sine_before);
/* mxb_patch_create: every MXB_OP_ENVGEN stage (kind 0) plays the one shape in desc->eg_*.
 * mxb_patch_create2: one shape per maxiEnvGen object of the patch (an amp envelope and a filter envelope, ...): an ENVGEN stage plays
 * shapes[kind], kind < n_shapes (0 .. 4). Stages may share a shape; each keeps its own state. desc->eg_stages must be 0. */
int32_t mxb_patch_create(mxb_ctx* ctx, const mxb_patch_desc* desc, mxb_patch** patch);
int32_t mxb_patch_create2(mxb_ctx* ctx, const mxb_patch_desc* desc, int32_t n_shapes, const mxb_envgen_shape* shapes, mxb_patch** patch);
int32_t mxb_patch_destroy(mxb_patch* patch);
int32_t mxb_patch_set_param(mxb_patch* patch, int32_t j, const double* values, int32_t mem);
/* state slot `slot` of stage `stage` (the order given with the ops above; integral members arrive / return as doubles) */
int32_t mxb_patch_set_state(mxb_patch* patch, int32_t stage, int32_t slot, const double* values, int32_t mem);
int32_t mxb_patch_get_state(mxb_patch* patch, int32_t stage, int32_t slot, double* values, int32_t mem);
int32_t mxb_patch_get_ring(mxb_patch* patch, int32_t stage, int32_t voice, double* dst, int32_t n, int32_t mem);
/* the held values [voices] of events stream m (MXB_IN_EVENTS): to start a voice at a given value, or to checkpoint a patch. Any other stream is MXB_ERR_INVALID. */
int32_t mxb_patch_get_held(mxb_patch* patch, int32_t m, double* values, int32_t mem);
int32_t mxb_patch_set_held(mxb_patch* patch, int32_t m, const double* values, int32_t mem);
/* inputs: n_inputs pointers to [n_frames][voices] of each stream's element type (MXB_IN_BITS: [n_frames][(voices + 31) / 32] words; MXB_IN_EVENTS: an mxb_events); out: [n_frames][voices] or NULL; mix: [n_frames][2] or NULL */
int32_t mxb_patch_process(mxb_patch* patch, int32_t n_frames, const void* const* inputs, double* out, double* mix, int32_t mem, void* stream);
int64_t mxb_patch_launch_count(const mxb_patch* patch);
#define MXB_PATCH_INTERPRET 0
#define MXB_PATCH_FUSED 1
/* FUSED compiles at once (so that a patch the compiler rejects fails here and not in the audio loop). Patches start FUSED unless
 * the environment says MXB_PATCH_MODE=interpret. */
int32_t mxb_patch_set_mode(mxb_patch* patch, int32_t mode);
int32_t mxb_patch_get_mode(const mxb_patch* patch);
/* The CUDA source the library generates for a descriptor (voices / max_frames / eg_* are not looked at: envelope shapes travel as kernel
 * arguments, so one program serves every set of shapes; ENVGEN kinds 0 .. 3), NUL-terminated into buf[cap]
 * (may be NULL / 0); *needed = its size with the terminator. compile != 0 also runs it through NVRTC for sm_90a. Needs no device. */
int32_t mxb_patch_codegen(const mxb_patch_desc* desc, char* buf, int64_t cap, int64_t* needed, int32_t compile);

/* ------------------------------------------------------------------------------------------------
 * Multi-GPU mix-down: one process per GPU, voices sharded, every rank ends each block with the SAME stereo bus
 * = sum over all ranks, in rank order (bit-identical on every rank and from run to run). The exchange is a
 * symmetric peer-mapped buffer (CUDA IPC over NVLink/NVSwitch); the reduction of the per-warp partials and the
 * exchange with the peers run in ONE kernel (no NCCL call on the data path). Setup: every rank creates an
 * exchange, publishes mxb_exchange_local_handle() to the others (any side channel: torch.distributed,
 * MPI, a pipe), calls mxb_exchange_connect() with all handles in rank order, and attaches it to its bank;
 * mxb_bank_process then delivers the all-reduced bus in `mix`. All ranks must process the same blocks in the
 * same order. The reference has no counterpart: it is single-threaded (SURVEY.md 2.4). */
typedef struct mxb_exchange mxb_exchange;
#define MXB_EXCHANGE_HANDLE_BYTES 64
int32_t mxb_exchange_create(mxb_ctx* ctx, int32_t rank, int32_t world, int32_t max_doubles, mxb_exchange** ex);
int32_t mxb_exchange_local_handle(mxb_exchange* ex, void* handle, int32_t handle_bytes);
int32_t mxb_exchange_connect(mxb_exchange* ex, const void* all_handles /* world x MXB_EXCHANGE_HANDLE_BYTES, rank order */);
/* The kernel's wait for the peers' flags is bounded (5 s; environment MXB_EXCHANGE_TIMEOUT_MS at creation): a rank that
 * died or never launched its block must not hang the others. *timed_out_ranks receives a bit mask of the ranks whose
 * contribution was missing from some bus so far (0 = every bus complete); synchronises the device. mxb_bank_process in
 * MXB_MEM_HOST / MXB_MEM_SPLIT mode checks it itself and returns MXB_ERR_STATE. */
int32_t mxb_exchange_status(mxb_exchange* ex, int32_t* timed_out_ranks);
int32_t mxb_exchange_destroy(mxb_exchange* ex);
int32_t mxb_bank_set_exchange(mxb_bank* bank, mxb_exchange* ex /* NULL detaches */);
/* ... and a voice patch's bus likewise (banks and patches share one mix-reduce kernel with the exchange fused in): a sharded polysynth ends every block
 * with the global stereo bus on every rank. One exchange serves one bank or patch at a time (its sequence numbers count the blocks). */
int32_t mxb_patch_set_exchange(mxb_patch* patch, mxb_exchange* ex /* NULL detaches */);

/* the reference's envelope setters, vectorised: kind 0 = setAttack (1 - pow(0.01, 1/(ms*sr*0.001))),
 * 1 = setAttackMS (1/(ms/1000*sr)), 2 = setDecay == setRelease (pow(0.01, 1/(ms*sr*0.001))).
 * src/maximilian.cpp:1469-1486. Host arrays. */
int32_t mxb_env_coeffs(int32_t kind, const double* ms, int64_t n, int32_t sample_rate, double* coeff);

/* ------------------------------------------------------------------------------------------------
 * Streaming STFT over `channels` independent channels = one maxiFFT::setup(fft_size, hop_size, fft_size)
 * + process(x, WITH_POLAR_CONVERSION) per channel (src/libs/maxiFFT.cpp:45-91). The transform replays
 * the reference's float arithmetic (recurrence twiddles, conjugate sign, DC/Nyquist packed in bin 0,
 * bin N/4 left untangled: src/libs/fft.cpp:118-282), so real/imag/magnitude are bit-identical.
 * Sample (c, t) of the input is in[c*stride_c + t*stride_t] (planar: stride_c = n, stride_t = 1;
 * time-major like a bank's out: stride_c = 1, stride_t = channels).
 * Frame f of channel c is written at ((c*max_frames) + f)*bins of mags/phases/re/im (each optional)
 * and at ((c*max_frames) + f)*num_coeffs of coeffs when an mfcc handle is given (fused: the spectrum
 * never leaves the chip unless asked for). *n_frames receives the frames fired per channel.
 * Input contract: samples are finite with |x| < 2^48. Then |X_k| <= fft_size * max|x| (1024 * max|x| < 2^58
 * for the 1024-point kernel, < 2^59 at 2048), the power |X_k|^2 < 2^118 stays below FLT_MAX (~2^128) and no
 * magnitude overflows. The fused 1024-point MFCC
 * (K4s) relies on it: it does not look for non-finite magnitudes. The other sizes, and mxb_mfcc_process on
 * caller-supplied magnitudes, follow the reference there too: a NaN anywhere in a frame, or an inf at a bin
 * where a band has zero weight, makes that band 0 (the reference's band is NaN, and its > 1e-6 gate fails). */
int32_t mxb_stft_create(mxb_ctx* ctx, int32_t channels, int32_t fft_size, int32_t hop_size, mxb_stft** st);
int32_t mxb_stft_destroy(mxb_stft* st);
int32_t mxb_stft_process(mxb_stft* st, const float* in, int64_t stride_c, int64_t stride_t, int32_t n_samples,
                         int32_t max_frames, float* mags, float* phases, float* re, float* im,
                         mxb_mfcc* mfcc, double* coeffs, int32_t* n_frames, int32_t mem, void* stream);
int64_t mxb_stft_launch_count(const mxb_stft* st);

/* The same call with the per-frame spectral features of maxiFFT fused in as further optional outputs
 * (SURVEY.md 8f-3): mags_db = getMagnitudesDB()/magsToDB (src/libs/maxiFFT.cpp:101-111, fft.cpp:526-534) laid out like
 * mags; flatness / centroid = spectralFlatness() / spectralCentroid() (src/libs/maxiFFT.cpp:113-132), one float per
 * frame at c*max_frames + f. The reference sums 512 floats in bin order; here each lane sums every 32nd bin and a
 * shuffle tree combines the lanes: equal to float reassociation (asserted at 1e-4 relative). */
typedef struct {
    float *mags, *phases, *re, *im;      /* as in mxb_stft_process */
    float *mags_db, *flatness, *centroid;
    double* coeffs;                      /* with `mfcc` */
} mxb_stft_outputs;
int32_t mxb_stft_process2(mxb_stft* st, const float* in, int64_t stride_c, int64_t stride_t, int32_t n_samples,
                          int32_t max_frames, const mxb_stft_outputs* out, mxb_mfcc* mfcc,
                          int32_t* n_frames, int32_t mem, void* stream);

/* maxiFFTOctaveAnalyzer (src/libs/maxiFFT.h:162-205, maxiFFT.cpp:201-300) and maxiBark (src/libs/maxiBark.h:36-126, SURVEY.md 8f-3)
 * as further epilogues of the transform, computed per frame from the magnitudes while they are in shared memory.
 * mxb_octave = setup(samplingRate, nBandsInTheFFT, nAveragesPerOctave) for every channel of one mxb_stft: the bin -> band map and the
 * per-channel averages / peaks / peakHoldTimes (state carried from frame to frame and call to call, zero at creation; the reference
 * leaves them uninitialised). mxb_octave_config sets the public members peakHoldTime, peakDecayRate, linearEQIntercept, linearEQSlope.
 * octave_averages / octave_peaks: float [channels][max_frames][mxb_octave_n_averages()] after each frame's calculate().
 * bark != 0: maxiBarkScaleAnalyser::setup(sample rate of the context, fft_size); bark_specific / bark_relative: double
 * [channels][max_frames][24] (specificLoudness / relativeLoudness of the magnitudes), bark_total: double [channels][max_frames].
 * pow(sum, 0.23) is libdevice's: 1e-12 relative. Fused into the 1024-point kernel only (other sizes: MXB_ERR_UNSUPPORTED); on any
 * spectrum, at any size, mxb_octave_process / mxb_bark_process below compute the same values from magnitudes in memory. */
typedef struct mxb_octave mxb_octave;
int32_t mxb_octave_create(mxb_ctx* ctx, int32_t channels, float sampling_rate, int32_t n_bands, int32_t n_per_octave, mxb_octave** o);
int32_t mxb_octave_destroy(mxb_octave* o);
int32_t mxb_octave_n_averages(const mxb_octave* o);
int32_t mxb_octave_config(mxb_octave* o, int32_t peak_hold_time, float peak_decay_rate, float eq_intercept, float eq_slope);
typedef struct {
    mxb_octave* octave; float *octave_averages, *octave_peaks;
    int32_t bark; double *bark_specific, *bark_relative, *bark_total;
} mxb_stft_post;
int32_t mxb_stft_process3(mxb_stft* st, const float* in, int64_t stride_c, int64_t stride_t, int32_t n_samples,
                          int32_t max_frames, const mxb_stft_outputs* out, const mxb_stft_post* post, mxb_mfcc* mfcc,
                          int32_t* n_frames, int32_t mem, void* stream);
/* Channels that advance independently, as separate maxiFFT objects do: channel c takes n_samples[c] >= 0 samples (host array [channels]),
 * read at in[c*stride_c + t*stride_t], and fires frames_c = pos_c + n_samples[c] >= fft_size ? (pos_c + n_samples[c] - fft_size) / hop + 1
 * : 0 frames, written to rows [c][0 .. frames_c) of the outputs of mxb_stft_process3 (same layouts, epilogues, MFCC and bars; the octave
 * and Bark analysers at 1024 points only). n_frames: host array [channels], frames_c. In MXB_MEM_HOST mode rows frames_c .. of a channel
 * up to the most frames any channel fired are overwritten with unspecified values. A negative count, frames_c > max_frames or more than
 * 2^31 - 1 frames in all: MXB_ERR_INVALID, and the handle is unchanged.
 * The handle keeps each channel's pos (maxiFFT::pos; mxb_stft_get_pos: host array [channels]). While they are all equal -- always, on a
 * handle never driven ragged -- mxb_stft_process / 2 / 3 work as before; once they differ those calls return MXB_ERR_STATE. */
int32_t mxb_stft_process_ragged(mxb_stft* st, const float* in, int64_t stride_c, int64_t stride_t, const int32_t* n_samples,
                                int32_t max_frames, const mxb_stft_outputs* out, const mxb_stft_post* post, mxb_mfcc* mfcc,
                                int32_t* n_frames, int32_t mem, void* stream);
int32_t mxb_stft_get_pos(mxb_stft* st, int32_t* pos);
/* maxiFFTOctaveAnalyzer::calculate(fftData) (src/libs/maxiFFT.cpp:261-300) on caller-supplied spectra, for every channel of o.
 * mags: float, frame f of channel c at ((c*max_frames)+f)*n_bands (the layout mxb_stft_process writes), frames 0..frames-1 analysed in
 * order. averages / peaks (each optional): float at ((c*max_frames)+f)*n_averages. The state is the handle's own: averages, peaks and
 * hold counters, the same state the fused 1024-point epilogue carries. So one handle may alternate between the two paths.
 * Spectra may hold NaN, inf or negative values: they flow through the float sums and the >= peak test as in the reference.
 * frames == 0 does nothing; frames < 0 or > max_frames: MXB_ERR_INVALID. */
int32_t mxb_octave_process(mxb_octave* o, const float* mags, int32_t frames, int32_t max_frames,
                           float* averages, float* peaks, int32_t mem, void* stream);
/* maxiBarkScaleAnalyser::setup(sR, bS) + specificLoudness / relativeLoudness / totalLoudness (src/libs/maxiBark.h:36-113).
 * buffer_size: 2 .. 4096 (the reference's barkScale[2048]); sample_rate: > 0, with (buffer_size/2 - 1) * sample_rate < 2^32 (the
 * reference's bin-to-Hz conversion is unsigned int arithmetic). The band limits do not depend on the context's sample rate. */
typedef struct mxb_bark mxb_bark;
int32_t mxb_bark_create(mxb_ctx* ctx, int32_t sample_rate, int32_t buffer_size, mxb_bark** b);
int32_t mxb_bark_destroy(mxb_bark* b);
/* spectrum: float [n][buffer_size/2]; specific / relative: double [n][24]; total: double [n] (each optional). n == 0 does nothing.
 * NaN, inf and negative bins follow the reference through the band sum, pow and the > max scan (relative = specific / max). */
int32_t mxb_bark_process(mxb_bark* b, const float* spectrum, int64_t n, double* specific, double* relative, double* total,
                         int32_t mem, void* stream);

/* maxiMFCC::setup(numBins, numFilters, numCoeffs, minFreq, maxFreq) + mfcc() (src/libs/maxiMFCC.h:56-111,
 * src/libs/maxiMFCC.cpp:48-66). mags: float [n][num_bins]; coeffs: double [n][num_coeffs];
 * melbands (optional): double [n][num_filters] after the log stage. */
int32_t mxb_mfcc_create(mxb_ctx* ctx, int32_t num_bins, int32_t num_filters, int32_t num_coeffs,
                        double min_freq, double max_freq, mxb_mfcc** m);
int32_t mxb_mfcc_destroy(mxb_mfcc* m);
int32_t mxb_mfcc_process(mxb_mfcc* m, const float* mags, int64_t n, double* coeffs, double* melbands,
                         int32_t mem, void* stream);

/* maxiIFFT::setup + process(mags, phases, SPECTRUM) per channel (src/libs/maxiFFT.cpp:141-192).
 * fft_size: a power of two in [64, 2048]; hop_size: 1 .. fft_size (it need not divide fft_size). Anything else: MXB_ERR_INVALID.
 * mags/phases: frame f of channel c at (c*frames + f)*bins; out: planar float [channels][frames*hop]. */
int32_t mxb_istft_create(mxb_ctx* ctx, int32_t channels, int32_t fft_size, int32_t hop_size, mxb_istft** st);
int32_t mxb_istft_destroy(mxb_istft* st);
int32_t mxb_istft_process(mxb_istft* st, const float* mags, const float* phases, int32_t frames, float* out,
                          int32_t mem, void* stream);
/* Channels that advance independently: channel c resynthesises frames[c] frames (host array [channels], 0 .. max_frames), read at
 * (c*max_frames + f)*bins of mags / phases, into out[c*max_frames*hop .. + frames[c]*hop). A channel with no frame keeps its overlap-add
 * buffer. In MXB_MEM_HOST mode out samples past frames[c]*hop of a row, up to the most frames any channel has, are overwritten with
 * unspecified values. A count outside 0 .. max_frames: MXB_ERR_INVALID, and the handle is unchanged. */
int32_t mxb_istft_process_ragged(mxb_istft* st, const float* mags, const float* phases, const int32_t* frames, int32_t max_frames,
                                 float* out, int32_t mem, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MAXIB200_H */
