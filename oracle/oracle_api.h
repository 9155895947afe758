/*
 * oracle_api.h -- TEST INFRASTRUCTURE ONLY (never linked into the product).
 *
 * One C interface, exported twice under the same symbol names:
 *   oracle/_ref/libmaxiref.so   the UNMODIFIED reference classes, compiled from
 *                               /root/reference/src by oracle/Makefile, driven
 *                               by oracle/ref_shim.cpp ("kind: reference");
 *   oracle/libmaxioracle.so     oracle/maxi_oracle.c, a plain-C restatement of
 *                               the same algorithms ("kind: port"), pinned
 *                               bit-for-bit against the first.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load either library.
 *
 * A "bank" is V independent voices, each one reference object per stage:
 *     x = maxiOsc::<osc>(freq_v)                    src/maximilian.cpp:228-373
 *     x = maxiEnv::adsr(x, trigger_v(t))            src/maximilian.cpp:1415-1466
 *     x = maxiFilter::lores|hires / maxiSVF::play / maxiBiquad::play
 *                                                   src/maximilian.cpp:455-484, src/maximilian.h:1305-1367
 *     x = maxiDelayline::dl(x, size_v, feedback_v)  src/maximilian.cpp:420-429
 *     out[t][v] = x ; mix[t][0..1] += maxiMix::stereo(x, pan_v)   src/maximilian.cpp:503-509
 * called once per sample t, voices in ascending order inside each frame,
 * exactly like a reference play() looping over an array of voices
 * (cpp/commandline/maximilian_examples/15.polysynth/main.cpp:54-70).
 */
#ifndef MAXI_ORACLE_API_H
#define MAXI_ORACLE_API_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* stage selectors (values shared with include/maxib200.h) */
enum { MXO_OSC_SINEWAVE = 0, MXO_OSC_COSWAVE = 1, MXO_OSC_PHASOR = 2, MXO_OSC_SAW = 3,
       MXO_OSC_SQUARE = 4, MXO_OSC_PULSE = 5, MXO_OSC_IMPULSE = 6, MXO_OSC_TRIANGLE = 7,
       MXO_OSC_PHASORBETWEEN = 8 };   /* maxiOsc::phasorBetween(frequency, startphase, endphase), src/maximilian.cpp:321-330 */
enum { MXO_FILT_NONE = 0, MXO_FILT_LORES = 1, MXO_FILT_HIRES = 2, MXO_FILT_SVF = 3, MXO_FILT_BIQUAD = 4 };
enum { MXO_ENV_NONE = 0, MXO_ENV_ADSR = 1 /* maxiEnv::adsr(input, trigger) */,
       MXO_ENV_AR = 2 /* maxiEnv::ar(input, attack, release, holdtime, trigger), src/maximilian.cpp:1319-1358 */ };
/* chain.delay_on: 0 none, 1 maxiDelayline::dl, 2 maxiDelayline::dlFromPosition (src/maximilian.cpp:431-439) */

/* per-voice parameter / state arrays (double[V]) */
enum {
    MXO_P_FREQ = 0,       /* oscillator frequency, Hz */
    MXO_P_PHASE = 1,      /* oscillator phase (maxiOsc::phaseReset); also a state */
    MXO_P_DUTY = 2,       /* pulse duty */
    MXO_P_CUTOFF = 3,     /* lores/hires cutoff1, SVF cutoff, biquad cutoff */
    MXO_P_RESONANCE = 4,  /* lores/hires resonance, SVF resonance, biquad Q */
    MXO_P_GAIN = 5,       /* biquad peakGain */
    MXO_P_ENV_ATTACK = 6, /* maxiEnv::attack (raw coefficient) */
    MXO_P_ENV_DECAY = 7,
    MXO_P_ENV_SUSTAIN = 8,
    MXO_P_ENV_RELEASE = 9,
    MXO_P_ENV_HOLDTIME = 10, /* maxiEnv::holdtime, integral value */
    MXO_P_DELAY_SIZE = 11,   /* dl() size argument, integral value */
    MXO_P_DELAY_FEEDBACK = 12,
    MXO_P_PAN = 13,          /* maxiMix::stereo x */
    MXO_P_DELAY_POSITION = 14, /* dlFromPosition position argument, integral value */
    MXO_P_PHASOR_START = 15,   /* phasorBetween startphase */
    MXO_P_PHASOR_END = 16,     /* phasorBetween endphase */
    MXO_P_COUNT = 17,
    /* read-only state ids for mxo_bank_get */
    MXO_S_FILT_0 = 32,    /* lores/hires x | svf v0z | biquad v[1] */
    MXO_S_FILT_1 = 33,    /* lores/hires y | svf v1  | biquad v[2] */
    MXO_S_FILT_2 = 34,    /* svf v2 */
    MXO_S_ENV_AMPLITUDE = 35,
    MXO_S_ENV_OUTPUT = 36,
    MXO_S_ENV_HOLDCOUNT = 37,
    MXO_S_ENV_FLAGS = 38, /* attack | decay<<1 | sustain<<2 | hold<<3 | release<<4 */
    MXO_S_DELAY_PHASE = 39,
    MXO_S_OSC_OUTPUT = 40  /* maxiOsc::output (assigned by every method but impulse) */
};

typedef struct {
    int32_t sample_rate;   /* maxiSettings::sampleRate */
    int32_t osc_kind;
    int32_t filt_kind;
    int32_t biquad_type;   /* maxiBiquad::filterTypes, src/maximilian.h:1348-1357 */
    int32_t env_kind;
    int32_t delay_on;
    int32_t delay_capacity; /* ring slots per voice for the port (reference: 705600 fixed) */
    int32_t reserved;
    double  svf_mix[4];    /* lpmix, bpmix, hpmix, notchmix of maxiSVF::play */
} mxo_chain;

void*   mxo_bank_create(const mxo_chain* chain, int32_t voices);
void    mxo_bank_destroy(void* bank);
int32_t mxo_bank_set(void* bank, int32_t id, const double* values);
int32_t mxo_bank_get(void* bank, int32_t id, double* values);
/* trigger_v(t) = 1 for trig_on[v] <= t < trig_off[v] (t = frame index inside this call), else 0;
 * NULL pointers mean trigger 0 throughout. out: [nframes][V] or NULL; mix: [nframes][2] or NULL
 * (mix is overwritten, not accumulated across calls). first/count restrict the call to a voice
 * sub-range (used to thread the CPU baseline); pass 0, V for everything. */
int32_t mxo_bank_process(void* bank, int32_t nframes, const int32_t* trig_on, const int32_t* trig_off,
                         double* out, double* mix, int32_t first, int32_t count);
/* the same with a per-sample oscillator frequency freq_tv[t][v] (NULL = the MXO_P_FREQ array): frequency modulation,
 * cpp/commandline/maximilian_examples/5.FM1/main.cpp:29 */
int32_t mxo_bank_process_fm(void* bank, int32_t nframes, const double* freq_tv, const int32_t* trig_on, const int32_t* trig_off,
                            double* out, double* mix, int32_t first, int32_t count);
/* ... and a per-sample filter cutoff cutoff_tv[t][v] (NULL = the MXO_P_CUTOFF array): lores/hires take the cutoff as an
 * argument of every call (src/maximilian.cpp:455,471); for maxiSVF the patch calls setCutoff() before play() on every
 * sample (src/maximilian.h:1287-1290, tests/svftest in the reference). The modulation lasts for this call: afterwards
 * the MXO_P_CUTOFF values are in force again. Not available for maxiBiquad (returns -3).
 * delay_size_tv[t][v] (integral values): the `size` argument of maxiDelayline::dl / dlFromPosition, which a flanger or
 * chorus changes on every call (src/maximilian.cpp:420,431; maxiFlanger::flange, src/maximilian.h:1144-1180). */
int32_t mxo_bank_process_mod(void* bank, int32_t nframes, const double* freq_tv, const double* cutoff_tv, const double* delay_size_tv,
                             const int32_t* trig_on, const int32_t* trig_off, double* out, double* mix, int32_t first, int32_t count);
/* ... and with maxiEnv::trigger given for every sample: trig_tv[t][v] bytes (NULL = the trig_on / trig_off interval) */
int32_t mxo_bank_process_mod2(void* bank, int32_t nframes, const double* freq_tv, const double* cutoff_tv, const double* delay_size_tv,
                              const uint8_t* trig_tv, const int32_t* trig_on, const int32_t* trig_off, double* out, double* mix, int32_t first, int32_t count);
/* copies ring slots [0, n) of voice v */
int32_t mxo_bank_get_ring(void* bank, int32_t v, double* dst, int32_t n);

/* parameter helpers = the reference setters */
double  mxo_env_attack_coeff(double attackMS, int32_t sample_rate);   /* maxiEnv::setAttack   src/maximilian.cpp:1478-1480 */
double  mxo_env_attack_ms_coeff(double attackMS, int32_t sample_rate);/* maxiEnv::setAttackMS src/maximilian.cpp:1484-1486 */
double  mxo_env_decay_coeff(double ms, int32_t sample_rate);          /* setDecay / setRelease src/maximilian.cpp:1469-1476 */

/* streaming STFT: C channels, each a maxiFFT::setup(fftSize, hopSize, fftSize), WITH_POLAR_CONVERSION.
 * in: planar [C][n]. Frame f of channel c lands at index (c*max_frames + f)*bins in mags/phases/re/im
 * (any of them may be NULL). Returns the number of frames fired per channel, or <0. */
void*   mxo_stft_create(int32_t channels, int32_t fft_size, int32_t hop_size);
void    mxo_stft_destroy(void* st);
int32_t mxo_stft_process(void* st, const float* in, int32_t n, int32_t max_frames,
                         float* mags, float* phases, float* re, float* im);
int32_t mxo_stft_window(void* st, float* window);   /* fft_size floats */

/* Per-frame spectral features of maxiFFT computed from magnitudes[n_frames][bins] (bins = fft_size/2):
 * db[n_frames][bins] = maxiFFT::magsToDB / fft::convToDB (src/libs/maxiFFT.cpp:101-111, src/libs/fft.cpp:526-534),
 * flatness[n_frames] = maxiFFT::spectralFlatness (:113-123), centroid[n_frames] = maxiFFT::spectralCentroid (:125-132)
 * with maxiSettings::sampleRate = sample_rate. Any output may be NULL. */
int32_t mxo_spectral_features(const float* mags, int32_t n_frames, int32_t fft_size, int32_t sample_rate,
                              float* db, float* flatness, float* centroid);

/* maxiMFCC::setup(numBins, numFilters, numCoeffs, minFreq, maxFreq) with maxiSettings::sampleRate = sample_rate.
 * mags: [n][numBins] floats; coeffs: [n][numCoeffs]; melbands (optional): [n][numFilters] after the log stage. */
void*   mxo_mfcc_create(int32_t num_bins, int32_t num_filters, int32_t num_coeffs,
                        double min_freq, double max_freq, int32_t sample_rate);
void    mxo_mfcc_destroy(void* m);
int32_t mxo_mfcc_process(void* m, const float* mags, int32_t n, double* coeffs, double* melbands);

/* maxiIFFT (SPECTRUM mode), C channels. mags/phases: frame f of channel c at (c*frames + f)*bins;
 * out: planar [C][frames*hop]. */
void*   mxo_istft_create(int32_t channels, int32_t fft_size, int32_t hop_size);
void    mxo_istft_destroy(void* st);
int32_t mxo_istft_process(void* st, const float* mags, const float* phases, int32_t frames, float* out);

/* ---- voice patches: the stage lists of include/maxib200.h (mxb_stage / mxb_patch_desc), same codes, run on the CPU ---- */
enum { MXO_OSC_SINEBUF = 9, MXO_OSC_SINEBUF4 = 10, MXO_OSC_SAWN = 11 };                 /* src/maximilian.cpp:266-274, 237-264, 342-359 */
enum { MXO_FILT_LOPASS = 5, MXO_FILT_HIPASS = 6, MXO_FILT_BANDPASS = 7 };                /* src/maximilian.cpp:442-453, 487-500 */
enum { MXO_NL_ATANDIST = 0, MXO_NL_FASTATANDIST, MXO_NL_SOFTCLIP, MXO_NL_HARDCLIP, MXO_NL_ASYMCLIP, MXO_NL_FASTATAN };   /* src/maximilian.h:1046-1137 */
#define MXO_ENVGEN_HOLD (-46692.0)                                                       /* maxiEnvGen::HOLD, src/maximilian.h:2271 */
enum { MXO_OP_OSC = 1, MXO_OP_ENV_ADSR, MXO_OP_ENV_AR, MXO_OP_ENVGEN, MXO_OP_FILTER, MXO_OP_SVF, MXO_OP_BIQUAD, MXO_OP_DCBLOCK, MXO_OP_NONLIN,
       MXO_OP_DELAY, MXO_OP_FLANGER, MXO_OP_ADD, MXO_OP_SUB, MXO_OP_MUL, MXO_OP_DIV, MXO_OP_MIX_STEREO, MXO_OP_OUT,
       MXO_OP_CHORUS /* maxiChorus::chorus, src/maximilian.h:1200-1212: src5 = the value maxiOsc::noise() returns this sample */ };
typedef struct { int32_t op, kind, dst, reserved; int32_t src[8]; } mxo_stage;      /* operands: 0..15 register, 0x100+j parameter, 0x200+k constant, 0x300+m input, -1 none */
/* one maxiEnvGen shape, the arguments of maxiEnvGen::setup (src/maximilian.h:2371-2402), as mxb_envgen_shape: levels[stages + 1],
 * times[stages], curves[stages]. A shape of no segments is a maxiEnvGen whose setup() was never called (levels[0] only). */
typedef struct {
    int32_t stages, loop, retrigger;
    const double *levels, *times, *curves;
} mxo_envgen_shape;
enum { MXO_MAX_EG_SHAPES = 4, MXO_MAX_EG_SEGMENTS = 16 };                                  /* the library's limits */
/* An ENVGEN stage plays shapes[kind]; mxo_patch_create returns NULL for a kind outside [0, n_shapes) or a shape list past the limits.
 * Both libraries copy what they need at create time: the arrays may be freed afterwards. */
typedef struct {
    int32_t voices, n_stages, n_params, n_consts, n_inputs, sample_rate;
    int32_t delay_taps;
    int32_t n_shapes;
    const mxo_stage* stages;
    const double* consts;
    const mxo_envgen_shape* shapes;
} mxo_patch_desc;
/* the shape checks of mxo_patch_create, shared by both libraries */
static inline int mxo_patch_shapes_ok(const mxo_patch_desc* d) {
    if (d->n_shapes < 0 || d->n_shapes > MXO_MAX_EG_SHAPES || (d->n_shapes > 0 && !d->shapes)) return 0;
    for (int k = 0; k < d->n_shapes; ++k) {
        const mxo_envgen_shape* s = &d->shapes[k];
        if (s->stages < 0 || s->stages > MXO_MAX_EG_SEGMENTS || !s->levels || (s->stages > 0 && (!s->times || !s->curves))) return 0;
    }
    for (int i = 0; i < d->n_stages; ++i)
        if (d->stages[i].op == MXO_OP_ENVGEN && (d->stages[i].kind < 0 || d->stages[i].kind >= d->n_shapes)) return 0;
    return 1;
}
/* sineBuffer[514] / transition[1001] of the reference (src/maximilian.cpp:63, 67-200) and the double before sineBuffer[0] that
 * sinebuf4 reads on its wrap sample. The compiled reference returns its own; the port is handed them (mxo_set_tables). */
int32_t mxo_set_tables(const double* sine514, const double* transition1001, double sine_before);
int32_t mxo_get_tables(double* sine514, double* transition1001, double* sine_before);
void*   mxo_patch_create(const mxo_patch_desc* desc);
void    mxo_patch_destroy(void* patch);
int32_t mxo_patch_set_param(void* patch, int32_t j, const double* values);
int32_t mxo_patch_set_state(void* patch, int32_t stage, int32_t slot, const double* values);
int32_t mxo_patch_get_state(void* patch, int32_t stage, int32_t slot, double* values);
int32_t mxo_patch_get_ring(void* patch, int32_t stage, int32_t voice, double* dst, int32_t n);
int32_t mxo_patch_process(void* patch, int32_t nframes, const double* const* inputs, double* out, double* mix);
/* maxiChorus draws its modulator from libc rand() through maxiOsc::noise() (src/maximilian.cpp:214-220). mxo_noise_fill: srand(seed), then n
 * values exactly as noise() produces them (both libraries: the same libc); mxo_srand: re-seed before the compiled reference runs a patch
 * with ONE chorus stage and no other noise source, so that it draws the sequence mxo_noise_fill returned, in (frame, voice) order. */
void    mxo_noise_fill(uint32_t seed, int64_t n, double* out);
void    mxo_srand(uint32_t seed);

/* maxiFFTOctaveAnalyzer (src/libs/maxiFFT.h:162-205, maxiFFT.cpp:201-300), one analyser per channel, fed magnitude frames:
 * mags[C][frames][n_bands] -> averages / peaks [C][frames][nAverages] (the values after each calculate()). averages[], peaks[]
 * and peakHoldTimes[] start at zero (the reference leaves them uninitialised). config: the public members peakHoldTime,
 * peakDecayRate, linearEQIntercept, linearEQSlope. */
void*   mxo_octave_create(int32_t channels, float sampling_rate, int32_t n_bands, int32_t n_per_octave);
void    mxo_octave_destroy(void* o);
int32_t mxo_octave_n_averages(void* o);
int32_t mxo_octave_config(void* o, int32_t peak_hold_time, float peak_decay_rate, float eq_intercept, float eq_slope);
int32_t mxo_octave_process(void* o, const float* mags, int32_t frames, float* averages, float* peaks);
/* maxiBarkScaleAnalyser::setup(sample_rate, buffer_size) + specificLoudness / relativeLoudness / totalLoudness
 * (src/libs/maxiBark.h:36-126) on spectrum[n_frames][buffer_size/2]: specific, relative [n_frames][24], total [n_frames] */
int32_t mxo_bark(const float* spectrum, int32_t n_frames, int32_t sample_rate, int32_t buffer_size, double* specific, double* relative, double* total);

/* "reference" or "port" */
const char* mxo_kind(void);

#ifdef __cplusplus
}
#endif
#endif
